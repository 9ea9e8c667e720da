"""Perplexity through the host against scoring on the device.

    python scripts/bench_perplexity.py [--reps 5]

The model is bench_generate.py's: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU, with a Q6_K
output.weight, n_ctx 512 and 8 sessions.  Three cases: one 511-token text; 8 texts of 64 tokens (504 fed rows, one pass);
8 texts of 511 tokens (one pass each).  Two arms, alternated in the same process, each timed end to end with a host
clock around work that ends in a device synchronise:
  A  the host path, as DistributedLLM.perplexity runs it, through the C ABI: for each text b200_extra_embed of
     tokens[:-1] -> b200_session_forward -> b200_extra_logits of every row (copied to the host) -> the client's float64
     softmax and -log p in numpy
  B  one b200_score call over every text
Every session is cleared before each repetition.  Tokens/s counts scored tokens (len - 1 per text) over all texts.  A and
B must agree within |b - a| <= 1e-12 * max(1, |a|) per token (checked in the same run).  Then, in a profiled window of its
own, k_nll_rows alone (b200_extra_nll on 512 rows of 32000 logits): its device time from torch.profiler, copies
excluded.  Prints the GPU's name and power limit, one line per case, then one JSON line.  Exits non-zero if A and B
disagree.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import scipy.special

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributedllm_b200 import capi, ggjt  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card  # noqa: E402

TOL = 1e-12
CASES = (("1 x 511 tokens", 1, 511), ("8 x 64 tokens", 8, 64), ("8 x 511 tokens", 8, 511))


def texts_for(batch, length):
    return [[1 + ((i + 3 * k) * 7919) % 31999 for i in range(length)] for k in range(batch)]


def host_path(sl, extra, texts):
    """-> per text the NLL of each scored token, computed as the reference client does after get_logits."""
    out = []
    for k, toks in enumerate(texts):
        logits = extra.logits(sl.session_forward(k, extra.embed(toks[:-1])))
        n = len(toks) - 1
        pmf = scipy.special.softmax(logits.astype(np.float64), axis=1)
        out.append(-np.log(pmf[np.arange(n), toks[1:]]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_perplexity.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, 512, n_sessions=8)
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    results, ok = [], True
    for name, B, L in CASES:
        texts = texts_for(B, L)
        sessions = list(range(B))
        arms = {"A": lambda: host_path(sl, extra, texts), "B": lambda: capi.score([sl], extra, sessions, texts)}
        times = {a: [] for a in arms}
        out = {}
        for rep in range(1 + args.reps):                    # repetition 0 warms up every shape
            for arm in (("A", "B") if rep % 2 == 0 else ("B", "A")):
                sl.session_clear(-1)
                sl.sync()
                t0 = time.perf_counter()
                out[arm] = arms[arm]()
                sl.sync()
                dt = time.perf_counter() - t0
                if rep > 0:
                    times[arm].append(B * (L - 1) / dt)
        a, b = np.concatenate(out["A"]), np.concatenate(out["B"])
        worst = float(np.max(np.abs(b - a) / np.maximum(1.0, np.abs(a))))
        agree = bool(np.isfinite(a).all() and worst <= TOL)
        ok &= agree
        med = {k: statistics.median(v) for k, v in times.items()}
        print("%-15s A host path %.1f tok/s (%.1f..%.1f)  B b200_score %.1f tok/s (%.1f..%.1f)  B/A %.3f  "
              "largest relative NLL difference %.3g (%s)"
              % (name, med["A"], min(times["A"]), max(times["A"]), med["B"], min(times["B"]), max(times["B"]),
                 med["B"] / med["A"], worst, "agree" if agree else "DISAGREE"), flush=True)
        results.append({"case": name, "texts": B, "tokens_per_text": L, "host_tok_s": med["A"], "device_tok_s": med["B"],
                        "host_range": [min(times["A"]), max(times["A"])],
                        "device_range": [min(times["B"]), max(times["B"])],
                        "max_rel_nll_diff": worst, "agree": agree})
    # k_nll_rows alone: device time from torch.profiler (copies excluded), in a profiled window of its own
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((512, sh.n_vocab)) * 3).astype(np.float32)
    t = rng.integers(0, sh.n_vocab, 512)
    for _ in range(3):
        extra.nll(x, t)
    calls = 20
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            extra.nll(x, t)
    kern_ms = 0.0
    for ev in prof.key_averages():
        dt = getattr(ev, "device_time_total", None)
        dt = ev.cuda_time_total if dt is None else dt
        if "k_nll_rows" in ev.key:
            kern_ms += dt / calls / 1e3
    print("k_nll_rows: %.4f ms per 512 rows of %d logits" % (kern_ms, sh.n_vocab), flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "perplexity", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "n_ctx": 512, "reps": args.reps, "gpu": card, "results": results,
                      "k_nll_rows_ms_per_512_rows": kern_ms}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
