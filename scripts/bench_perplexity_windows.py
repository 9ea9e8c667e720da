"""llama.cpp's windowed perplexity on the device: windows per pass, exact and fast mode, against b200_score.

    python scripts/bench_perplexity_windows.py [--windows 64] [--reps 1]

The model is bench_perplexity.py's: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU with a Q6_K
output.weight, here loaded at n_ctx 2048 with 4 sessions, so up to 4 windows of 512 share a pass.  The input is a
synthetic id stream of --windows windows of 512 ids (n_batch 512, so one segment per window; rows 256..510 scored).
Arms, alternated in the same process, each timed with a host clock around work that ends in a device synchronise:
  w1, w2, w4   b200_perplexity_windows, exact, with 1, 2 and 4 sessions (windows per pass)
  w4 fast      the same with fast = 1 (tensor-core prefill)
  score        b200_score on the same BOS-replaced windows, 4 per call (sessions 0-3, cleared between calls): the
               project's existing scoring path, which projects and scores every row (511 per window)
Rates: evaluated tok/s counts the ids run through the model (512 per window; 511 for score), scored tok/s the rows
scored (255 per window; 511 for score).  Every arm is run once on 4 windows to warm up first.  Checks in the same run:
w1, w2 and w4 give the same bits; fast mode's running perplexity within 1e-2 relative of exact mode's.
Then, in a profiled run of its own (torch.profiler, CUDA activities), 8 windows through w4 exact and w4 fast: the device
time of k_ppl_rows against the device time of every kernel of the call.  Prints the GPU's name and power limit, one line
per arm, then one JSON line.  Exits non-zero if a check fails.
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from distributedllm_b200 import capi, ggjt  # noqa: E402
from distributedllm_b200.client import running_perplexity  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card  # noqa: E402

N_CTX, N_BATCH = 512, 512
FAST_TOL = 1e-2


def id_stream(n_windows, n_vocab):
    rng = np.random.default_rng(1234)
    return rng.integers(3, n_vocab, n_windows * N_CTX).tolist()


def score_arm(sl, extra, tokens):
    """b200_score over the windows, BOS first, 4 sessions per call."""
    out = []
    n = len(tokens) // N_CTX
    for c0 in range(0, n, 4):
        texts = [[1] + tokens[c * N_CTX + 1:(c + 1) * N_CTX] for c in range(c0, min(c0 + 4, n))]
        sl.session_clear(-1)
        out += capi.score([sl], extra, list(range(len(texts))), texts)
    sl.session_clear(-1)
    return out


def profile_share(sl, extra, tokens, fast):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        capi.perplexity_windows([sl], extra, [0, 1, 2, 3], tokens, N_CTX, N_BATCH, fast=fast)
    ppl_us = total_us = 0.0
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        dt = ev.cuda_time_total if dt is None else dt
        if ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
            continue
        total_us += dt
        if "k_ppl_rows" in ev.key:
            ppl_us += dt
    return ppl_us / 1e3, total_us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--reps", type=int, default=1)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_perplexity_windows.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, 2048, n_sessions=4)
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    tokens = id_stream(args.windows, sh.n_vocab)
    n_chunk, _, first, n_scored = capi.ppl_window_rows(len(tokens), N_CTX, N_BATCH)
    arms = {
        "w1": lambda t: capi.perplexity_windows([sl], extra, [0], t, N_CTX, N_BATCH),
        "w2": lambda t: capi.perplexity_windows([sl], extra, [0, 1], t, N_CTX, N_BATCH),
        "w4": lambda t: capi.perplexity_windows([sl], extra, [0, 1, 2, 3], t, N_CTX, N_BATCH),
        "w4 fast": lambda t: capi.perplexity_windows([sl], extra, [0, 1, 2, 3], t, N_CTX, N_BATCH, fast=True),
        "score": lambda t: score_arm(sl, extra, t),
    }
    per_window = {"w1": (N_CTX, n_scored), "w2": (N_CTX, n_scored), "w4": (N_CTX, n_scored),
                  "w4 fast": (N_CTX, n_scored), "score": (N_CTX - 1, N_CTX - 1)}
    for f in arms.values():                                 # warm every shape
        f(tokens[:4 * N_CTX])
    times = {a: [] for a in arms}
    out = {}
    names = list(arms)
    for rep in range(args.reps):
        for a in (names if rep % 2 == 0 else names[::-1]):
            sl.sync()
            t0 = time.perf_counter()
            out[a] = arms[a](tokens)
            sl.sync()
            times[a].append(time.perf_counter() - t0)
    ok = True
    same = all(np.array_equal(out[a].view(np.uint32), out["w1"].view(np.uint32)) for a in ("w2", "w4"))
    ok &= same
    exact, fast = np.asarray(running_perplexity(out["w4"])), np.asarray(running_perplexity(out["w4 fast"]))
    fast_rel = float(np.max(np.abs(fast - exact) / exact))
    ok &= bool(np.isfinite(fast).all() and fast_rel <= FAST_TOL)
    results = []
    for a in names:
        t = statistics.median(times[a])
        ev, sc = per_window[a]
        r = {"arm": a, "seconds": t, "evaluated_tok_s": n_chunk * ev / t, "scored_tok_s": n_chunk * sc / t}
        results.append(r)
        print("%-8s %7.2f s  evaluated %8.1f tok/s  scored %8.1f tok/s" % (a, t, r["evaluated_tok_s"], r["scored_tok_s"]),
              flush=True)
    print("w1 / w2 / w4 terms bit-identical: %s; final perplexity exact %.6f, fast %.6f (largest relative difference of "
          "a running value %.3g)" % (same, exact[-1], fast[-1], fast_rel), flush=True)
    share = {}
    for fast_mode in (False, True):
        ppl_ms, total_ms = profile_share(sl, extra, tokens[:8 * N_CTX], fast_mode)
        key = "fast" if fast_mode else "exact"
        share[key] = {"k_ppl_rows_ms": ppl_ms, "all_kernels_ms": total_ms, "share": ppl_ms / total_ms,
                      "k_ppl_rows_ms_per_window": ppl_ms / 8}
        print("k_ppl_rows, w4 %s, 8 windows: %.3f ms of %.1f ms of kernels (%.2f %%), %.3f ms per window"
              % (key, ppl_ms, total_ms, 100 * ppl_ms / total_ms, ppl_ms / 8), flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "perplexity_windows",
                      "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU, slice n_ctx 2048",
                      "n_ctx": N_CTX, "n_batch": N_BATCH, "windows": n_chunk, "scored_per_window": n_scored,
                      "reps": args.reps, "gpu": card, "results": results, "bit_identical_packings": same,
                      "fast_max_rel_diff": fast_rel, "k_ppl_rows": share, "ok": bool(ok)}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
