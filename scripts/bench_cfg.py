"""The cost of classifier-free guidance (b200_generate_cfg) in the device generation loop.

    python scripts/bench_cfg.py [--reps 5] [--steps 256] [--batches 1,8]

bench_logprobs.py's model: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU with a Q6_K output.weight, a
16-token prompt and --steps tokens per session; guided sessions get a 16-id negative prompt, scale 1.5, smooth_factor 1.
Greedy and sampled (T 0.7, rp 1.1, top_k 40, top_p 0.95), guidance off (generate_greedy / generate_sample) and on
(guidance=), alternated in one process; repetition 0 warms up and is not timed; medians of --reps, each timed end to end
with a host clock around work that ends in a device synchronise.  tok/s counts the generating sessions' ids only.
Before the timing, 8 greedy and 8 sampled guided ids of one session are checked against a host loop (session_forward on
both sessions, b200_extra_logits, client.cfg_logits, then max_element or the sampler's door).
Then bench_logprobs.py's serving mix (--requests requests, prompts 16-128, budgets 32-256, at most 8 in flight, sampled)
through one stream, unguided and with every other request guided (its guidance session beside it); each arm's ids must
repeat across repetitions.
Then k_cfg_rows alone (b200_extra_cfg on 1, 8 and 64 pairs of 32000 logits): its device time per call from
torch.profiler, copies excluded, in a profiled window of its own.
Prints the GPU's name and power limit, one line per workload, then one JSON line.  Exits non-zero on a mismatch.
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from distributedllm_b200 import capi, client, ggjt  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card, prompts_for  # noqa: E402

T, RP, TOP_K, TOP_P = 0.7, 1.1, 40, 0.95
SCALE, SF = 1.5, 1.0
CONC = 8


def mix(sl, extra, reqs, negs, guided):
    """The serving mix through one stream; request j is guided (guidance session len(reqs) + j) when guided and j is
    even.  -> (ids per request, seconds)."""
    t0 = time.perf_counter()
    ids = [[] for _ in reqs]
    nxt = 0

    def add(st, j):
        p, b, s = reqs[j]
        g = (len(reqs) + j, negs[j], SCALE, SF) if guided and j % 2 == 0 else None
        st.add(j, p, b, temperature=T, repeat_penalty=RP, seed=s, top_k=TOP_K, top_p=TOP_P, guidance=g)

    with capi.Stream([sl], extra) as st:
        while nxt < min(CONC, len(reqs)):
            add(st, nxt)
            nxt += 1
        while True:
            recs = st.read(256)
            if not recs:
                break
            for k, t in recs:
                ids[k].append(t)
                if len(ids[k]) == reqs[k][1] and nxt < len(reqs):
                    add(st, nxt)
                    nxt += 1
    return ids, time.perf_counter() - t0


def host_check(sl, extra, prompt, neg, n):
    """Guided greedy and sampled ids of session 0 (guidance session 1) against the host loop.  -> True when equal."""
    ok = True
    for sampled in (False, True):
        sl.session_clear(-1)
        g = ([1], [neg], SCALE, SF)
        if sampled:
            ids = capi.generate_sample([sl], extra, [0], [prompt], n, T, RP, [5], top_k=TOP_K, top_p=TOP_P, guidance=g)[:, 0]
        else:
            ids = capi.generate_greedy([sl], extra, [0], [prompt], n, guidance=g)[:, 0]
        sl.session_clear(-1)
        toks, gtoks = prompt, neg
        for j in range(n):
            b = extra.logits(sl.session_forward(0, extra.embed(toks))[-1:])[0]
            gl = extra.logits(sl.session_forward(1, extra.embed(gtoks))[-1:])[0]
            row = client.cfg_logits(b[None], gl[None], SCALE, SF)[0]
            if sampled:
                want = int(extra.sample(row[None], T, RP, [5], first_draw=j, history=[ids[:j].tolist()], top_k=TOP_K,
                                        top_p=TOP_P)[0])
            else:
                want = client.cfg_greedy(row)
            ok &= want == int(ids[j])
            toks = gtoks = [int(ids[j])]
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--pairs", default="1,8,64", help="k_cfg_rows pair counts to time")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_cfg.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    batches = [int(b) for b in args.batches.split(",") if b]
    n_ctx = 1024
    assert 16 + args.steps - 1 <= n_ctx
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx, n_sessions=2 * max(batches + [args.requests]))
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(11)
    negs_all = [rng.integers(1, sh.n_vocab, 16).tolist() for _ in range(max(batches))]
    ok = host_check(sl, extra, prompts_for(1)[0], negs_all[0], 8)
    print("host loop check (8 greedy + 8 sampled guided ids): %s" % ("equal" if ok else "DIFFER"), flush=True)
    results = []
    for sampled in (False, True):
        for B in batches:
            prompts, seeds, sessions = prompts_for(B), [1000 + 7 * k for k in range(B)], list(range(B))
            guidance = (list(range(B, 2 * B)), negs_all[:B], SCALE, SF)

            def arm(on):
                g = guidance if on else None
                if sampled:
                    return capi.generate_sample([sl], extra, sessions, prompts, args.steps, T, RP, seeds, top_k=TOP_K,
                                                top_p=TOP_P, guidance=g)
                return capi.generate_greedy([sl], extra, sessions, prompts, args.steps, guidance=g)

            rate = {False: [], True: []}
            ids = {}
            for rep in range(1 + args.reps):
                for on in ((False, True) if rep % 2 == 0 else (True, False)):
                    sl.session_clear(-1)
                    sl.sync()
                    t0 = time.perf_counter()
                    got = arm(on)
                    sl.sync()
                    dt = time.perf_counter() - t0
                    if rep > 0:
                        rate[on].append(B * args.steps / dt)
                    ids.setdefault(on, got)
                    ok &= bool((got == ids[on]).all())
            med = {on: statistics.median(v) for on, v in rate.items()}
            mode = "sampled" if sampled else "greedy"
            print("%s B=%d tok/s: guidance off %.1f, on %.1f (%.3fx)" % (mode, B, med[False], med[True],
                                                                        med[True] / med[False]), flush=True)
            results.append({"mode": mode, "batch": B, "tok_s_off": med[False], "tok_s_on": med[True],
                            "ratio": med[True] / med[False], "tok_s_range_off": [min(rate[False]), max(rate[False])],
                            "tok_s_range_on": [min(rate[True]), max(rate[True])]})
    rng_m = np.random.default_rng(7)
    reqs = [(rng_m.integers(1, sh.n_vocab, int(rng_m.integers(16, 129))).tolist(), int(rng_m.integers(32, 257)),
             int(rng_m.integers(0, 2 ** 63))) for _ in range(args.requests)]
    negs = [rng_m.integers(1, sh.n_vocab, 16).tolist() for _ in range(args.requests)]
    mrate = {"off": [], "half_guided": []}
    mids = {}
    useful = sum(b for _, b, _ in reqs)
    for rep in range(1 + args.reps):
        for a in (("off", "half_guided") if rep % 2 == 0 else ("half_guided", "off")):
            sl.session_clear(-1)
            sl.sync()
            got, dt = mix(sl, extra, reqs, negs, a == "half_guided")
            if rep > 0:
                mrate[a].append(useful / dt)
            mids.setdefault(a, got)
            ok &= got == mids[a]
    mm = {a: statistics.median(v) for a, v in mrate.items()}
    print("mix: %d requests, %d tokens, at most %d in flight: off %.1f tok/s, half guided %.1f tok/s (%.3fx)"
          % (args.requests, useful, CONC, mm["off"], mm["half_guided"], mm["half_guided"] / mm["off"]), flush=True)
    from torch.profiler import ProfilerActivity, profile
    kern_ms = {}
    for n in [int(r) for r in args.pairs.split(",") if r]:
        b = (rng.standard_normal((n, sh.n_vocab)) * 3).astype(np.float32)
        g = (rng.standard_normal((n, sh.n_vocab)) * 3).astype(np.float32)
        out, _ = extra.cfg(b, g, SCALE, SF)
        ok &= bool(np.array_equal(out, client.cfg_logits(b, g, SCALE, SF), equal_nan=True))
        for _ in range(3):
            extra.cfg(b, g, SCALE, SF)
        calls = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                extra.cfg(b, g, SCALE, SF)
        kern = {}
        for ev in prof.key_averages():
            v = getattr(ev, "device_time_total", None)
            v = ev.cuda_time_total if v is None else v
            if v and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
                kern[ev.key] = v / calls / 1e3
        kern_ms[n] = sum(kern.values())
        print("k_cfg_rows %2d pair(s) of %d: %.4f ms per call  [%s]"
              % (n, sh.n_vocab, kern_ms[n], ", ".join("%s %.4f" % (k.split("(")[0][:40], v) for k, v in kern.items())),
              flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "cfg", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "scale": SCALE, "smooth_factor": SF, "negative_prompt_tokens": 16, "prompt_tokens": 16,
                      "temperature": T, "repeat_penalty": RP, "top_k": TOP_K, "top_p": TOP_P, "steps": args.steps,
                      "reps": args.reps, "gpu": card, "results": results,
                      "mix": {"requests": args.requests, "tokens": useful, "tok_s": mm,
                              "tok_s_range": {a: [min(v), max(v)] for a, v in mrate.items()}},
                      "k_cfg_rows_ms": {str(k): v for k, v in kern_ms.items()}, "ids_ok": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
