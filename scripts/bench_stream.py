"""Generation streams (b200_stream_*) against the closed device loop (b200_generate_sample).

    python scripts/bench_stream.py [--reps 5] [--steps 256] [--requests 32] [--concurrent 8]

bench_generate.py's model: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU with a Q6_K output.weight,
n_ctx 1024, sampling at T 0.7, rp 1.1.  Arms are alternated in the same process; repetition 0 warms up and is not timed.
  (a) one session, a 16-token prompt and --steps tokens:
      S  a capi.Stream: open, add, read the ids as they come, close
      G  one generate_sample call
      Reports the time to the first id (for G the whole call: it returns every id at once) and tok/s.
  (b) a serving mix: --requests requests drawn from a seed (prompts of 16-128 tokens, budgets of 32-256), all waiting at
      t = 0, at most --concurrent in flight:
      S  one stream; a request is added as soon as one in flight ends (one session per request, every one at n_past 0)
      B  static batches of --concurrent requests in arrival order through generate_sample, each batch running to its
         longest budget
      Reports generated tok/s (the requested tokens only) and the mean request latency (t = 0 to the request's last id).
Before anything is reported, every request's ids from S must equal G's / B's (bit for bit, as the stream guarantees).
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
from distributedllm_b200 import capi, ggjt  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card, prompts_for  # noqa: E402

T, RP = 0.7, 1.1


def single_stream(sl, extra, prompt, n, seed):
    """-> (ids, seconds to the first id, seconds in all)."""
    t0 = time.perf_counter()
    ids, first = [], None
    with capi.Stream([sl], extra) as st:
        st.add(0, prompt, n, temperature=T, repeat_penalty=RP, seed=seed)
        while True:
            pairs = st.read(256)
            if not pairs:
                break
            if first is None:
                first = time.perf_counter() - t0
            ids += [t for _, t in pairs]
    return ids, first, time.perf_counter() - t0


def single_call(sl, extra, prompt, n, seed):
    t0 = time.perf_counter()
    ids = capi.generate_sample([sl], extra, [0], [prompt], n, T, RP, [seed])[:, 0].tolist()
    dt = time.perf_counter() - t0
    return ids, dt, dt


def mix_stream(sl, extra, reqs, conc):
    """-> (ids per request, latency per request in seconds, seconds in all)."""
    t0 = time.perf_counter()
    ids = [[] for _ in reqs]
    lat = [0.0] * len(reqs)
    nxt = 0
    with capi.Stream([sl], extra) as st:
        while nxt < min(conc, len(reqs)):
            p, b, s = reqs[nxt]
            st.add(nxt, p, b, temperature=T, repeat_penalty=RP, seed=s)
            nxt += 1
        while True:
            pairs = st.read(256)
            if not pairs:
                break
            now = time.perf_counter() - t0
            for k, t in pairs:
                ids[k].append(t)
                if len(ids[k]) == reqs[k][1]:              # the request is complete: the next one takes its place
                    lat[k] = now
                    if nxt < len(reqs):
                        p, b, s = reqs[nxt]
                        st.add(nxt, p, b, temperature=T, repeat_penalty=RP, seed=s)
                        nxt += 1
    return ids, lat, time.perf_counter() - t0


def mix_batches(sl, extra, reqs, conc):
    t0 = time.perf_counter()
    ids, lat = [], []
    for b0 in range(0, len(reqs), conc):
        batch = reqs[b0:b0 + conc]
        sl.session_clear(-1)
        out = capi.generate_sample([sl], extra, list(range(len(batch))), [r[0] for r in batch], max(r[1] for r in batch),
                                   T, RP, [r[2] for r in batch])
        now = time.perf_counter() - t0
        for j, r in enumerate(batch):
            ids.append(out[:r[1], j].tolist())
            lat.append(now)
    return ids, lat, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--concurrent", type=int, default=8)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    n_ctx = 1024                 # a static batch's prompts run as one mixed pass: up to 8 x 128 rows
    rng = np.random.default_rng(args.seed)
    reqs = [(rng.integers(1, sh.n_vocab, int(rng.integers(16, 129))).tolist(), int(rng.integers(32, 257)),
             int(rng.integers(0, 2 ** 63))) for _ in range(args.requests)]
    assert all(len(p) + b - 1 <= n_ctx for p, b, _ in reqs) and 16 + args.steps - 1 <= n_ctx
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx, n_sessions=max(args.requests, args.concurrent))
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    ok = True
    # (a) one session
    prompt, seed = prompts_for(1)[0], 1000
    arms = {"S": lambda: single_stream(sl, extra, prompt, args.steps, seed),
            "G": lambda: single_call(sl, extra, prompt, args.steps, seed)}
    first = {a: [] for a in arms}
    rate = {a: [] for a in arms}
    outs = {a: [] for a in arms}
    for rep in range(1 + args.reps):
        for name in (("S", "G") if rep % 2 == 0 else ("G", "S")):
            sl.session_clear(-1)
            sl.sync()
            ids, t_first, t_all = arms[name]()
            outs[name].append(ids)
            if rep > 0:
                first[name].append(t_first * 1e3)
                rate[name].append(args.steps / t_all)
    same_a = all(o == outs["G"][0] for o in outs["S"] + outs["G"])
    ok &= same_a
    med = {a: (statistics.median(first[a]), statistics.median(rate[a])) for a in arms}
    print("(a) one session, 16-token prompt + %d tokens: stream first id %.2f ms, %.1f tok/s (%.1f..%.1f); "
          "generate_sample first id %.2f ms, %.1f tok/s (%.1f..%.1f); stream/one-shot tok/s %.3f; ids %s"
          % (args.steps, med["S"][0], med["S"][1], min(rate["S"]), max(rate["S"]), med["G"][0], med["G"][1],
             min(rate["G"]), max(rate["G"]), med["S"][1] / med["G"][1], "identical" if same_a else "DIFFER"), flush=True)
    # (b) the serving mix
    arms_b = {"S": lambda: mix_stream(sl, extra, reqs, args.concurrent),
              "B": lambda: mix_batches(sl, extra, reqs, args.concurrent)}
    useful = sum(b for _, b, _ in reqs)
    tps = {a: [] for a in arms_b}
    lat = {a: [] for a in arms_b}
    outs_b = {a: [] for a in arms_b}
    for rep in range(1 + args.reps):
        for name in (("S", "B") if rep % 2 == 0 else ("B", "S")):
            sl.session_clear(-1)
            sl.sync()
            ids, l, t_all = arms_b[name]()
            outs_b[name].append(ids)
            if rep > 0:
                tps[name].append(useful / t_all)
                lat[name].append(statistics.mean(l) * 1e3)
    same_b = all(o == outs_b["B"][0] for o in outs_b["S"] + outs_b["B"])
    ok &= same_b
    mb = {a: (statistics.median(tps[a]), statistics.median(lat[a])) for a in arms_b}
    print("(b) %d requests (prompts 16-128, budgets 32-256, %d tokens), at most %d in flight: stream %.1f tok/s "
          "(%.1f..%.1f), mean latency %.0f ms; static batches %.1f tok/s (%.1f..%.1f), mean latency %.0f ms; "
          "stream/static tok/s %.3f; ids %s"
          % (args.requests, useful, args.concurrent, mb["S"][0], min(tps["S"]), max(tps["S"]), mb["S"][1], mb["B"][0],
             min(tps["B"]), max(tps["B"]), mb["B"][1], mb["S"][0] / mb["B"][0], "identical" if same_b else "DIFFER"),
          flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "stream", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "temperature": T, "repeat_penalty": RP, "reps": args.reps, "gpu": card,
                      "single": {"steps": args.steps, "stream_first_id_ms": med["S"][0], "stream_tok_s": med["S"][1],
                                 "one_shot_first_id_ms": med["G"][0], "one_shot_tok_s": med["G"][1],
                                 "stream_tok_s_range": [min(rate["S"]), max(rate["S"])],
                                 "one_shot_tok_s_range": [min(rate["G"]), max(rate["G"])], "ids_identical": same_a},
                      "mix": {"requests": args.requests, "concurrent": args.concurrent, "tokens": useful,
                              "stream_tok_s": mb["S"][0], "stream_mean_latency_ms": mb["S"][1],
                              "static_tok_s": mb["B"][0], "static_mean_latency_ms": mb["B"][1],
                              "stream_tok_s_range": [min(tps["S"]), max(tps["S"])],
                              "static_tok_s_range": [min(tps["B"]), max(tps["B"])], "ids_identical": same_b}}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
