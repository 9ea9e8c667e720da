"""Top-k / top-p truncation in the device sampler: what the truncation stage costs.

    python scripts/bench_truncation.py [--reps 5] [--steps 256] [--batches 1,8] [--rows 1,8,64]

bench_generate.py's model: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU, with a Q6_K output.weight,
a 16-token prompt and --steps generated tokens for each of B sessions, T 0.7, rp 1.1.
  - Draw kernel: device time of b200_extra_sample (k_sample_rows) on --rows rows of 32000 logits, from torch.profiler in
    a window of its own (copies excluded), for: off, top_k 40, top_p 0.95, and top_k 40 + top_p 0.95.
  - Generation rate: one b200_generate_sample call per repetition, tokens/s over all sessions, off against
    top_k 40 + top_p 0.95, the two arms alternated; medians of --reps, timed with a host clock around work that ends in a
    device synchronise.
  - Id check: the truncated run's ids against the host loop with client.Sampler(top_k=40, top_p=0.95) under the
    ambiguity rule (tests/trunc_ref.py): a session is compared up to its first ambiguous draw.
Prints the GPU's name and power limit, one line per measurement, then one JSON line.  Exits non-zero on a disagreement.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from distributedllm_b200 import capi, ggjt  # noqa: E402
from distributedllm_b200.client import Sampler  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card, prompts_for  # noqa: E402
import sample_ref  # noqa: E402
import trunc_ref  # noqa: E402

T, RP, K, P = 0.7, 1.1, 40, 0.95
SETTINGS = {"off": (0, 0.0), "k40": (K, 0.0), "p0.95": (0, P), "k40+p0.95": (K, P)}


def host_loop(sl, extra, prompts, n_steps, seeds):
    """The client's loop with the twin: -> (ids [n_steps][B], per session the draws before its first ambiguous one)."""
    B = len(prompts)
    samplers = [Sampler(T, RP, rng=np.random.Generator(np.random.Philox(key=s)), top_k=K, top_p=P) for s in seeds]
    ids = np.zeros((n_steps, B), np.int32)
    safe = [n_steps] * B

    def pick(step, logits):
        for k in range(B):
            if safe[k] == n_steps:
                _, amb, _ = trunc_ref.sample(logits[k], T, RP, samplers[k].previous_ids, sample_ref.uniform(seeds[k], step), K, P)
                if amb:
                    safe[k] = step
            ids[step, k] = samplers[k](logits[k])

    sessions = list(range(B))
    x = sl.mixed_forward(sessions, [len(p) for p in prompts], extra.embed([t for p in prompts for t in p]))
    pick(0, extra.logits(x[np.cumsum([len(p) for p in prompts]) - 1]))
    for step in range(1, n_steps):
        x = sl.batch_forward(sessions, extra.embed(ids[step - 1])) if B > 1 else sl.session_forward(0, extra.embed(ids[step - 1]))
        pick(step, extra.logits(x))
    return ids, safe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--rows", default="1,8,64")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_truncation.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    batches = [int(b) for b in args.batches.split(",") if b]
    n_ctx = 512
    assert 16 + args.steps - 1 <= n_ctx
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx, n_sessions=max(batches + [1]))
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    ok, results = True, []
    for B in batches:
        prompts = prompts_for(B)
        seeds = [1000 + 7 * k for k in range(B)]
        sl.session_clear(-1)
        host_ids, safe = host_loop(sl, extra, prompts, args.steps, seeds)
        arms = {name: (lambda kp=kp: capi.generate_sample([sl], extra, list(range(B)), prompts, args.steps, T, RP, seeds,
                                                          top_k=kp[0], top_p=kp[1]))
                for name, kp in (("off", SETTINGS["off"]), ("k40+p0.95", SETTINGS["k40+p0.95"]))}
        times = {a: [] for a in arms}
        outs = {a: [] for a in arms}
        for rep in range(1 + args.reps):                     # repetition 0 warms up every shape
            for name in (list(arms) if rep % 2 == 0 else list(arms)[::-1]):
                sl.session_clear(-1)
                sl.sync()
                t0 = time.perf_counter()
                out = arms[name]()
                sl.sync()
                dt = time.perf_counter() - t0
                outs[name].append(out)
                if rep > 0:
                    times[name].append(B * args.steps / dt)
        dev = outs["k40+p0.95"][0]
        disagree = sum(int((host_ids[:safe[k], k] != dev[:safe[k], k]).sum()) for k in range(B))
        ambiguous = sum(1 for s in safe if s < args.steps)
        repeatable = all((o == outs[a][0]).all() for a in outs for o in outs[a])
        ok &= disagree == 0 and repeatable
        med = {a: statistics.median(v) for a, v in times.items()}
        print("B=%d  off %.1f tok/s (%.1f..%.1f)  k40+p0.95 %.1f tok/s (%.1f..%.1f)  ratio %.3f  vs host twin: %d ids "
              "differ outside the ambiguity rule, %d sessions hit an ambiguous draw; device ids %s across repetitions"
              % (B, med["off"], min(times["off"]), max(times["off"]), med["k40+p0.95"], min(times["k40+p0.95"]),
                 max(times["k40+p0.95"]), med["k40+p0.95"] / med["off"], disagree, ambiguous,
                 "identical" if repeatable else "DIFFER"), flush=True)
        results.append({"batch": B, "off_tok_s": med["off"], "truncated_tok_s": med["k40+p0.95"],
                        "off_range": [min(times["off"]), max(times["off"])],
                        "truncated_range": [min(times["k40+p0.95"]), max(times["k40+p0.95"])],
                        "ids_differ_outside_ambiguity": disagree, "ambiguous_sessions": ambiguous,
                        "device_repeatable": repeatable})
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    kern_ms = {}
    for n in [int(r) for r in args.rows.split(",") if r]:
        x = (rng.standard_normal((n, sh.n_vocab)) * 3).astype(np.float32)
        seeds = list(range(1, n + 1))
        hist = [rng.integers(0, sh.n_vocab, 64).tolist() for _ in range(n)]
        for name, (k, p) in SETTINGS.items():
            for _ in range(3):
                extra.sample(x, T, RP, seeds, 0, hist, top_k=k, top_p=p)
            calls = 20
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for c in range(calls):
                    extra.sample(x, T, RP, seeds, c, hist, top_k=k, top_p=p)
            total = 0.0
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", None)
                t = ev.cuda_time_total if t is None else t
                if t and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
                    total += t / calls / 1e3
            kern_ms["%s/%d" % (name, n)] = total
            print("k_sample_rows %-9s %2d row(s) of %d: %.4f ms per call" % (name, n, sh.n_vocab, total), flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "truncation", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "temperature": T, "repeat_penalty": RP, "top_k": K, "top_p": P, "prompt_tokens": 16,
                      "steps": args.steps, "reps": args.reps, "gpu": card, "results": results, "k_sample_rows_ms": kern_ms}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
