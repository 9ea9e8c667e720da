"""The cost of log-probabilities (b200_generate_lp, b200_stream_add_lp) in the device generation loops.

    python scripts/bench_logprobs.py [--reps 5] [--steps 256] [--batches 1,8] [--requests 32]

bench_sample.py's model: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU with a Q6_K output.weight, a
16-token prompt and --steps tokens per session, sampled at T 0.7, rp 1.1, top_k 40, top_p 0.95.  Arms are alternated in
one process, repetition 0 warms up and is not timed, medians of --reps, each timed end to end with a host clock around
work that ends in a device synchronise:
  (a) generate_sample with logprobs off, and with n_top 0, 5 and 20, at each batch size;
  (b) bench_stream.py's serving mix (--requests requests, prompts 16-128, budgets 32-256, at most 8 in flight) through one
      stream, with logprobs off for every request, and with every other request asking for top-5.
Then k_logprob_rows alone (b200_extra_logprobs, n_top 5, on 1, 8 and 64 rows of 32000 logits): its device time per call
from torch.profiler, copies excluded, in a profiled window of its own.
Before anything is printed, the ids of every arm must equal the logprobs-off arm's.  Prints the GPU's name and power limit,
one line per workload, then one JSON line.  Exits non-zero on a mismatch.
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
from distributedllm_b200 import capi, ggjt  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card, prompts_for  # noqa: E402

T, RP, TOP_K, TOP_P = 0.7, 1.1, 40, 0.95
CONC = 8


def mix(sl, extra, reqs, lp_every):
    """bench_stream.py's mix through one stream; request j asks for top-5 when lp_every and j % lp_every == 0.
    -> (ids per request, seconds)."""
    t0 = time.perf_counter()
    ids = [[] for _ in reqs]
    nxt = 0

    def add(st, j):
        p, b, s = reqs[j]
        st.add(j, p, b, temperature=T, repeat_penalty=RP, seed=s, top_k=TOP_K, top_p=TOP_P,
               logprobs=5 if lp_every and j % lp_every == 0 else None)

    with capi.Stream([sl], extra) as st:
        while nxt < min(CONC, len(reqs)):
            add(st, nxt)
            nxt += 1
        while True:
            recs = st.read_logprobs(256) if lp_every else st.read(256)
            if not recs:
                break
            for r in recs:
                ids[r[0]].append(r[1])
                if len(ids[r[0]]) == reqs[r[0]][1] and nxt < len(reqs):
                    add(st, nxt)
                    nxt += 1
    return ids, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--rows", default="1,8,64", help="k_logprob_rows row counts to time")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_logprobs.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    batches = [int(b) for b in args.batches.split(",") if b]
    n_ctx = 1024
    rng = np.random.default_rng(7)
    reqs = [(rng.integers(1, sh.n_vocab, int(rng.integers(16, 129))).tolist(), int(rng.integers(32, 257)),
             int(rng.integers(0, 2 ** 63))) for _ in range(args.requests)]
    assert 16 + args.steps - 1 <= n_ctx
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx, n_sessions=max(batches + [args.requests, CONC]))
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    ok, results = True, []
    for B in batches:
        prompts = prompts_for(B)
        seeds = [1000 + 7 * k for k in range(B)]

        def arm(n_top):
            out = capi.generate_sample([sl], extra, list(range(B)), prompts, args.steps, T, RP, seeds, top_k=TOP_K,
                                       top_p=TOP_P, logprobs=n_top)
            return out if n_top is None else out[0]

        names = ["off", 0, 5, 20]
        rate = {a: [] for a in names}
        ids = {}
        for rep in range(1 + args.reps):
            for a in (names if rep % 2 == 0 else names[::-1]):
                sl.session_clear(-1)
                sl.sync()
                t0 = time.perf_counter()
                got = arm(None if a == "off" else a)
                sl.sync()
                dt = time.perf_counter() - t0
                if rep > 0:
                    rate[a].append(B * args.steps / dt)
                ids.setdefault(a, got)
                ok &= bool((got == ids["off" if "off" in ids else a]).all())
        med = {a: statistics.median(v) for a, v in rate.items()}
        same = all((ids[a] == ids["off"]).all() for a in names)
        ok &= same
        print("B=%d  generate_sample tok/s: off %.1f, n_top 0 %.1f (%+.2f%%), 5 %.1f (%+.2f%%), 20 %.1f (%+.2f%%); ids %s"
              % (B, med["off"], med[0], 100 * (med[0] / med["off"] - 1), med[5], 100 * (med[5] / med["off"] - 1),
                 med[20], 100 * (med[20] / med["off"] - 1), "identical" if same else "DIFFER"), flush=True)
        results.append({"batch": B, "tok_s": {str(a): med[a] for a in names},
                        "tok_s_range": {str(a): [min(rate[a]), max(rate[a])] for a in names}, "ids_identical": same})
    # (b) the serving mix
    mrate = {"off": [], "half_top5": []}
    mids = {}
    useful = sum(b for _, b, _ in reqs)
    for rep in range(1 + args.reps):
        for a in (("off", "half_top5") if rep % 2 == 0 else ("half_top5", "off")):
            sl.session_clear(-1)
            sl.sync()
            got, dt = mix(sl, extra, reqs, 2 if a == "half_top5" else 0)
            if rep > 0:
                mrate[a].append(useful / dt)
            mids.setdefault(a, got)
            ok &= got == mids[a]
    same_mix = mids["off"] == mids["half_top5"]
    ok &= same_mix
    mm = {a: statistics.median(v) for a, v in mrate.items()}
    print("mix: %d requests, %d tokens, at most %d in flight: off %.1f tok/s, half top-5 %.1f tok/s (%+.2f%%); ids %s"
          % (args.requests, useful, CONC, mm["off"], mm["half_top5"], 100 * (mm["half_top5"] / mm["off"] - 1),
             "identical" if same_mix else "DIFFER"), flush=True)
    # k_logprob_rows alone: device time from torch.profiler (copies excluded), in a profiled window of its own
    from torch.profiler import ProfilerActivity, profile
    kern_ms = {}
    for n in [int(r) for r in args.rows.split(",") if r]:
        x = (rng.standard_normal((n, sh.n_vocab)) * 3).astype(np.float32)
        t = rng.integers(0, sh.n_vocab, n).astype(np.int32)
        for _ in range(3):
            extra.logprobs(x, t, 5)
        calls = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                extra.logprobs(x, t, 5)
        kern = {}
        for ev in prof.key_averages():
            v = getattr(ev, "device_time_total", None)
            v = ev.cuda_time_total if v is None else v
            if v and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
                kern[ev.key] = v / calls / 1e3
        kern_ms[n] = sum(kern.values())
        print("k_logprob_rows %2d row(s) of %d, n_top 5: %.4f ms per call  [%s]"
              % (n, sh.n_vocab, kern_ms[n], ", ".join("%s %.4f" % (k.split("(")[0][:40], v) for k, v in kern.items())),
              flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "logprobs", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "temperature": T, "repeat_penalty": RP, "top_k": TOP_K, "top_p": TOP_P, "prompt_tokens": 16,
                      "steps": args.steps, "reps": args.reps, "gpu": card, "results": results,
                      "mix": {"requests": args.requests, "tokens": useful, "tok_s": mm,
                              "tok_s_range": {a: [min(v), max(v)] for a, v in mrate.items()}, "ids_identical": same_mix},
                      "k_logprob_rows_ms": {str(k): v for k, v in kern_ms.items()}, "ids_ok": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
