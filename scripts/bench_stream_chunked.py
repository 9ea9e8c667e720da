"""Generation streams with long prompts: whole-prompt segments against prompts fed in chunks (b200_stream_open_ex).

    python scripts/bench_stream_chunked.py [--reps 2] [--chunks 32,64,128,256] [--plan-only]

Model: bench.py's synthetic LLaMA-7B Q4_0 (32 layers) with a Q6_K output.weight on one GPU, n_ctx 2048, sampling at
T 0.7, rp 1.1.  Load: --decoders sessions (16-id prompts) decode --budget ids each; while they run, --requests requests
with prompts of 512-1536 ids (budget --long-budget) arrive, one after every --every ids the decoders have delivered.
Arms, alternated in one process (repetition 0 warms up and is not timed):
  C = 0    one stream with max_rows = n_ctx: a long prompt joins as one segment, and no session decodes while it runs
  C > 0    prefill_chunk C with max_rows = C + --decoders: every step carries the decode rows and at most one chunk
Reports per arm: the decoders' gaps at read (median, p99, max over every decoder), each long prompt's time to its first
id (from its add), and generated ids per second over the run.  A decoder's gap is the time between two reads that return
ids of it; the ids one read returns share its timestamp, so they make one gap, not one gap and zeros.  Before anything is printed, every request's
ids must equal the reference arrangement for its arm on the same handles (session_forward of each non-final chunk, then
generate_sample with the last chunk); the decoders' prompts fit in one chunk, so their reference is one call for all
arms.  Prints the GPU's name and power limit, one line per arm, then one JSON line.  Exits non-zero on a mismatch.
--plan-only prints the workload and each arm's chunk boundaries and exits without a GPU.
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

T, RP, N_CTX = 0.7, 1.1, 2048


def chunks(prompt, C):
    """The segments a stream with prefill_chunk C feeds: [0, C), [C, 2C), ...; C = 0: the whole prompt."""
    return [prompt[i:i + C] for i in range(0, len(prompt), C)] if C else [prompt]


def workload(args, n_vocab):
    """-> (decoders, requests): lists of (prompt, budget, seed); request j arrives after (j + 1) * every decoder ids."""
    rng = np.random.default_rng(args.seed)
    dec = [(rng.integers(1, n_vocab, 16).tolist(), args.budget, int(rng.integers(0, 2 ** 63))) for _ in range(args.decoders)]
    req = [(rng.integers(1, n_vocab, int(rng.integers(512, 1537))).tolist(), args.long_budget, int(rng.integers(0, 2 ** 63)))
           for _ in range(args.requests)]
    assert all(len(p) + b - 1 <= N_CTX for p, b, _ in dec + req)
    assert args.requests * args.every < args.decoders * args.budget, "every request must arrive while the decoders run"
    return dec, req


def run_arm(capi, sl, extra, dec, req, C, every):
    """One stream over the workload -> (ids per session, decoder gaps in ms (one per read that returned ids of the
    decoder), time to first id per request in ms, tok/s).
    Sessions 0 .. len(dec) - 1 are the decoders, then the requests."""
    nd = len(dec)
    ids = [[] for _ in dec + req]
    last = [None] * nd
    gaps, ttft, added = [], [None] * len(req), [None] * len(req)
    max_rows = C + nd if C else N_CTX
    t0 = time.perf_counter()
    with capi.Stream([sl], extra, max_rows=max_rows, prefill_chunk=C) as st:
        for k, (p, b, s) in enumerate(dec):
            st.add(k, p, b, temperature=T, repeat_penalty=RP, seed=s)
        n_dec, nxt = 0, 0
        while True:
            pairs = st.read(256)
            if not pairs:
                break
            now = time.perf_counter()
            for k, t in pairs:
                ids[k].append(t)
                if k < nd:
                    n_dec += 1
                elif ttft[k - nd] is None:
                    ttft[k - nd] = (now - added[k - nd]) * 1e3
            for k in {k for k, _ in pairs if k < nd}:        # one gap per read that delivered to the decoder
                if last[k] is not None:
                    gaps.append((now - last[k]) * 1e3)
                last[k] = now
            while nxt < len(req) and n_dec >= (nxt + 1) * every:
                p, b, s = req[nxt]
                st.add(nd + nxt, p, b, temperature=T, repeat_penalty=RP, seed=s)
                added[nxt] = time.perf_counter()
                nxt += 1
    dt = time.perf_counter() - t0
    return ids, gaps, ttft, sum(len(x) for x in ids) / dt


def reference(capi, sl, extra, dec, req, C):
    """The reference arrangement of every request for prefill_chunk C (session k + len(dec)), on sl from n_past 0."""
    out = []
    for j, (p, b, s) in enumerate(req):
        k = len(dec) + j
        parts = chunks(p, C)
        for part in parts[:-1]:
            sl.session_forward(k, extra.embed(part))
        out.append(capi.generate_sample([sl], extra, [k], [parts[-1]], b, T, RP, [s])[:, 0].tolist())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--chunks", default="32,64,128,256", help="the chunked arms' C; C = 0 always runs")
    ap.add_argument("--decoders", type=int, default=8)
    ap.add_argument("--budget", type=int, default=384, help="ids per decoding session")
    ap.add_argument("--requests", type=int, default=4)
    ap.add_argument("--long-budget", type=int, default=16, help="ids per long-prompt request")
    ap.add_argument("--every", type=int, default=512, help="decoder ids delivered between two long-prompt arrivals")
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--plan-only", action="store_true")
    args = ap.parse_args()
    arms = [0] + [int(c) for c in args.chunks.split(",") if c]
    if any(c <= 0 or c + args.decoders > N_CTX for c in arms[1:]):
        raise SystemExit("every chunk must be in [1, %d]" % (N_CTX - args.decoders))
    from distributedllm_b200 import ggjt
    sh = ggjt.SHAPES["7b"]
    dec, req = workload(args, sh.n_vocab)
    if args.plan_only:
        print("decoders: %d x (16-id prompt, %d ids); requests: %s" % (len(dec), args.budget, [(len(p), b) for p, b, _ in req]))
        for C in arms:
            segs = [[len(c) for c in chunks(p, C)] for p, _, _ in req]
            print("C %d: max_rows %d, request segments %s" % (C, C + len(dec) if C else N_CTX,
                                                              ", ".join("%d x %d + %d" % (len(g) - 1, g[0], g[-1]) if len(g) > 1
                                                                        else str(g[0]) for g in segs)))
        return 0
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_chunked.py needs a GPU")
    from distributedllm_b200 import capi
    import bench
    from bench_generate import gpu_card
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, N_CTX, n_sessions=len(dec) + len(req))
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    ok = True
    want_dec = capi.generate_sample([sl], extra, list(range(len(dec))), [p for p, _, _ in dec], args.budget, T, RP,
                                    [s for _, _, s in dec])
    want_dec = [want_dec[:, k].tolist() for k in range(len(dec))]
    want = {}
    for C in arms:
        sl.session_clear(-1)
        want[C] = want_dec + reference(capi, sl, extra, dec, req, C)
    res = {C: {"gaps": [], "ttft": [], "tok_s": []} for C in arms}
    for rep in range(1 + args.reps):
        for C in (arms if rep % 2 == 0 else arms[::-1]):
            sl.session_clear(-1)
            sl.sync()
            ids, gaps, ttft, tps = run_arm(capi, sl, extra, dec, req, C, args.every)
            same = ids == want[C]
            ok &= same
            if not same:
                print("C %d repetition %d: ids DIFFER from the reference arrangement" % (C, rep), flush=True)
            if rep > 0:
                res[C]["gaps"] += gaps
                res[C]["ttft"] += ttft
                res[C]["tok_s"].append(tps)
    if not ok:
        return 1
    summary = {}
    for C in arms:
        g = np.array(res[C]["gaps"])
        s = {"max_rows": C + len(dec) if C else N_CTX, "gap_ms_median": float(np.median(g)),
             "gap_ms_p99": float(np.percentile(g, 99)), "gap_ms_max": float(g.max()),
             "first_id_ms": [round(v, 1) for v in res[C]["ttft"]],
             "first_id_ms_median": float(statistics.median(res[C]["ttft"])),
             "tok_s": float(statistics.median(res[C]["tok_s"])), "tok_s_range": [min(res[C]["tok_s"]), max(res[C]["tok_s"])]}
        summary[str(C)] = s
        print("C %4d (max_rows %4d): decoder gap median %.1f ms, p99 %.1f ms, max %.1f ms; long prompt first id median "
              "%.0f ms (%s); %.1f tok/s (%.1f..%.1f); ids identical to the reference"
              % (C, s["max_rows"], s["gap_ms_median"], s["gap_ms_p99"], s["gap_ms_max"], s["first_id_ms_median"],
                 ", ".join("%.0f" % v for v in res[C]["ttft"]), s["tok_s"], s["tok_s_range"][0], s["tok_s_range"][1]),
              flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "stream_chunked", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "n_ctx": N_CTX, "temperature": T, "repeat_penalty": RP, "reps": args.reps, "gpu": card,
                      "decoders": len(dec), "decoder_budget": args.budget,
                      "requests": [len(p) for p, _, _ in req], "request_budget": args.long_budget,
                      "every": args.every, "arms": summary, "ids_identical": ok}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
