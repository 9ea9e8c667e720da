"""Speculative decoding on the device against the plain device loops.

    python scripts/bench_speculative.py [--reps 3] [--steps 128] [--drafts 1,2,4,8]

LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU with a Q6_K output.weight (as bench_generate.py), a 16-token
prompt (1 + (i * 7919 mod 31999)).  Prints the GPU's name and power limit, read in the same call, then:
  1. the device time of one checking pass, b200_session_forward_steps with 2, 3, 5, 9 and 16 rows at positions around
     256 and 500, next to one decode-graph replay (b200_session_forward_device, one row) at the same positions: CUDA
     events on the slice's stream, median of alternating runs;
  2. tok/s of b200_generate_speculative against b200_generate_greedy and b200_generate_sample (T 0.7, rp 1.1) for each
     n_draft, with three drafts and the measured acceptance (accepted / drafted) beside each rate:
       same       the target loaded a second time (acceptance 1 at the full draft cost),
       skip2      the first 2 layers of the same synthetic 7B plus its extra layers, as separate handles,
       unrelated  a synthetic OpenLLaMA-3B (acceptance near 0: the overhead floor).
     The ids of every speculative run are checked against the plain loop's before timing.  Rates are medians of
     alternating runs, host clock around calls that end in a device synchronise.
  3. the rate each draft and n_draft would give as a function of acceptance a, from measured costs only: the draft part D
     of an iteration (the arm's measured iteration time minus the checking pass c(k + 1) of section 1) and c(k + 1); an
     iteration emits E(a) = (1 - a^(k+1)) / (1 - a) ids (a proposal is kept only if all before it were) and costs D + c,
     and the acceptance from which that beats one plain decode step per id.
Synthetic weights say nothing about the acceptance of real models; the acceptance column is that of these weights.
Ends with one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributedllm_b200 import capi, ggjt  # noqa: E402
import bench  # noqa: E402


def gpu_card() -> dict:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit": out[1], "max_sm_clock": out[2]}


PROMPT = [1 + (i * 7919) % 31999 for i in range(16)]


def pass_costs(sl, rows_list, positions, reps):
    """ms of device time per call: {(pos, rows): ms}, rows 1 = the decode graph."""
    E = sl.n_embd
    x = np.random.default_rng(0).standard_normal((16, E), dtype=np.float32)
    import torch
    buf = torch.from_numpy(x).cuda()
    out = {}
    for pos in positions:
        sl.session_clear(0)                  # rows below pos valid, so every call can rewind to pos
        sl.session_forward(0, np.random.default_rng(1).standard_normal((pos, E), dtype=np.float32))
        times = {r: [] for r in [1] + rows_list}
        for rep in range(reps + 1):
            order = [1] + rows_list if rep % 2 == 0 else list(reversed([1] + rows_list))
            for r in order:
                sl.session_rewind(0, pos)
                sl.sync()
                torch.cuda.synchronize()
                sl.mark(0)
                for _ in range(5):
                    sl.session_rewind(0, pos)
                    if r == 1:
                        capi.check(capi.lib().b200_session_forward_device(sl.handle, 0, capi.C.c_void_p(buf.data_ptr()), 1,
                                                                          capi.C.c_void_p(sl.dev_out), 0))
                    else:
                        capi.check(capi.lib().b200_session_forward_steps_device(
                            sl.handle, 0, capi.C.c_void_p(buf.data_ptr()), r, capi.C.c_void_p(sl.dev_out), 0))
                sl.mark(1)
                sl.sync()
                if rep > 0:
                    times[r].append(sl.mark_elapsed_ms() / 5)
        for r, v in times.items():
            out[(pos, r)] = statistics.median(v)
    return out


def timed(fn, reps_out, key):
    t0 = time.perf_counter()
    r = fn()
    dt = time.perf_counter() - t0
    reps_out.setdefault(key, []).append(dt)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--drafts", default="1,2,4,8")
    ap.add_argument("--pass-reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_speculative.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    n_ctx = 600
    ks = [int(k) for k in args.drafts.split(",") if k]
    assert 16 + args.steps - 1 + max(ks) <= n_ctx
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx)
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
        dextra = capi.Extra(extra_path, 0)
        sh3 = ggjt.SHAPES["3b"]
        p3, e3 = os.path.join(d, "u3b.bin"), os.path.join(d, "u3b_extra.bin")
        ggjt.write_fast_q4_slice(p3, sh3, 0, sh3.n_layer - 1, seed=11)
        ggjt.write_fast_q4_extra(e3, sh3, seed=11)
        drafts = {"same": ([capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx)], dextra),
                  "skip2": ([capi.Slice(bench.slice_file("7b", 0, 1), 0, n_ctx)], capi.Extra(extra_path, 0)),
                  "unrelated": ([capi.Slice(p3, 0, n_ctx)], capi.Extra(e3, 0))}

    # 1. cost of one checking pass
    rows_list = [2, 3, 5, 9, 16]
    costs = pass_costs(sl, rows_list, [256, 500 - 16], args.pass_reps)
    for pos in (256, 484):
        one = costs[(pos, 1)]
        print("position %d: decode graph %.3f ms; " % (pos, one) +
              ", ".join("%d rows %.3f ms (%.2fx)" % (r, costs[(pos, r)], costs[(pos, r)] / one) for r in rows_list), flush=True)

    # 2. tok/s
    def clear_all():
        sl.session_clear(-1)
        for dsl, _ in drafts.values():
            for s in dsl:
                s.session_clear(-1)

    seed = 1234
    plain = {"greedy": lambda: capi.generate_greedy([sl], extra, [0], [PROMPT], args.steps)[:, 0],
             "sample": lambda: capi.generate_sample([sl], extra, [0], [PROMPT], args.steps, 0.7, 1.1, [seed])[:, 0]}
    ref = {}
    for mode, fn in plain.items():
        clear_all()
        ref[mode] = fn()

    def spec(mode, name, k):
        dsl, de = drafts[name]
        kw = {} if mode == "greedy" else {"temperature": 0.7, "repeat_penalty": 1.1, "seed": seed}
        return capi.generate_speculative([sl], extra, 0, dsl, de, 0, PROMPT, args.steps, k, **kw)

    arms = {}
    for mode in ("greedy", "sample"):
        arms[(mode, "plain", 0)] = plain[mode]
        for name in drafts:
            for k in ks:
                arms[(mode, name, k)] = (lambda m=mode, n=name, kk=k: spec(m, n, kk))
    same = True
    stats = {}
    for key, fn in arms.items():                         # warm-up and the ids check
        clear_all()
        r = fn()
        if key[1] != "plain":
            ids, st = r
            ok = ids.tolist() == ref[key[0]].tolist()
            same &= ok
            stats[key] = st
            if not ok:
                print("ids DIFFER", key, flush=True)
    times = {}
    keys = list(arms)
    for rep in range(args.reps):
        for key in (keys if rep % 2 == 0 else list(reversed(keys))):
            clear_all()
            sl.sync()
            timed(arms[key], times, key)
            sl.sync()
    results = []
    for mode in ("greedy", "sample"):
        base = args.steps / statistics.median(times[(mode, "plain", 0)])
        print("%s: plain device loop %.1f tok/s" % (mode, base), flush=True)
        results.append({"mode": mode, "draft": "plain", "n_draft": 0, "tok_s": base})
        for name in drafts:
            for k in ks:
                key = (mode, name, k)
                rate = args.steps / statistics.median(times[key])
                st = stats[key]
                acc = st["accepted"] / st["drafted"] if st["drafted"] else 0.0
                print("%s  draft %-9s n_draft %2d: %7.1f tok/s (%.2fx plain)  acceptance %.3f  passes %d"
                      % (mode, name, k, rate, rate / base, acc, st["passes"]), flush=True)
                results.append({"mode": mode, "draft": name, "n_draft": k, "tok_s": rate, "over_plain": rate / base,
                                "acceptance": acc, **st})

    # 3. rate as a function of acceptance, from measured costs only.  Per draft and n_draft: the iteration time is the
    # greedy arm's median call time over its passes (step 0's share included), and the draft part D is that minus the
    # checking pass c(k + 1) measured in section 1 (so D carries the k proposals with the draft's two-row first pass, the
    # lm_heads, the picks, k_spec_accept and any launch gap).  rate(a) = E(a) / (D + c), E(a) = (1 - a^(k+1)) / (1 - a).
    model = {}
    step_ms = costs[(256, 1)]
    plain_rate = args.steps / statistics.median(times[("greedy", "plain", 0)])
    for name in drafts:
        model[name] = {}
        for k in ks:
            c = costs[(256, k + 1)]
            it = 1e3 * statistics.median(times[("greedy", name, k)]) / stats[("greedy", name, k)]["passes"]
            D = it - c
            rates = {str(a): 1e3 * ((1 - a ** (k + 1)) / (1 - a) if a < 1 else k + 1) / (D + c)
                     for a in (0.0, 0.25, 0.5, 0.75, 0.9, 1.0)}
            even = next((a / 100 for a in range(0, 101) if 1e3 * ((1 - (a / 100) ** (k + 1)) / (1 - a / 100) if a < 100
                                                                else k + 1) / (D + c) >= plain_rate), None)
            model[name][k] = {"iteration_ms": it, "draft_part_ms": D, "check_ms": c, "tok_s_by_acceptance": rates,
                              "break_even_acceptance": even}
            print("draft %-9s n_draft %d: iteration %.3f ms = draft part %.3f + checking pass %.3f; modelled tok/s by "
                  "acceptance %s; beats the plain greedy loop (%.1f tok/s) from acceptance %s"
                  % (name, k, it, D, c, ", ".join("%s: %.0f" % kv for kv in rates.items()), plain_rate,
                     "%.2f" % even if even is not None else "never"), flush=True)
    print("plain decode step at 256 (graph replay, kernels only): %.3f ms = %.1f tok/s upper bound" % (step_ms, 1e3 / step_ms))
    for dsl, de in drafts.values():
        for s in dsl:
            s.close()
        de.close()
    extra.close()
    sl.close()
    print(json.dumps({"bench": "generate_speculative", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "prompt_tokens": 16, "steps": args.steps, "reps": args.reps, "gpu": card, "ids_identical": same,
                      "pass_ms": {"%d@%d" % (r, p): v for (p, r), v in costs.items()}, "results": results,
                      "modelled_tok_s": model}))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
