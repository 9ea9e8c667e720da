"""Session copy, save / restore and forking a shared prompt prefix (b200_session_copy / _save / _restore, Stream.fork).

    python scripts/bench_session_fork.py [--reps 3] [--copy-reps 20]

bench_stream.py's model: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU with a Q6_K output.weight, n_ctx
2048, so one session's cache is 1 GiB (kv_bytes_per_pos = 512 KiB).
  (a) session_copy of n_keep rows (512, 2047) from one session to n_dst others (1, 4, 8): the call's time (it
      synchronises) and GB/s over the bytes the copy needs, one read plus n_dst writes.  Beside it, torch's strided copy
      of the same rows into each destination (one copy_ per destination and plane, on tensors shaped as the cache, timed
      with CUDA events), which reads the source once per destination.
  (b) session_save and session_restore of 512 positions (256 MiB), to and from pinned and pageable host buffers.
  (c) a serving mix: a 384-id shared prefix; --requests requests with suffixes of 16-64 ids and budgets of 32-128
      (drawn from a seed, sampled at T 0.7, rp 1.1), all waiting at t = 0, at most --concurrent in flight, one stream:
      F  the prefix session is fed the prefix once (add(prefix, max_tokens=1)); each request forks it, then adds its
         suffix
      R  each request's session is fed the prefix as its own segment (add(prefix, max_tokens=1)), then its suffix
      Both compute the same rows, so every request's ids must be equal in both arms.  Reports the mean time to the
      first id and the mean latency (t = 0 to the request's first / last id) and generated tok/s.
Arms are alternated in the same process; repetition 0 warms up and is not timed.  Prints the GPU's name and power limit,
one line per workload, then one JSON line.  Exits non-zero on an id mismatch.
"""
import argparse
import ctypes as C
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
from bench_generate import gpu_card  # noqa: E402

T, RP = 0.7, 1.1
N_CTX = 2048
PREFIX = 384


def timed(fn, reps):
    """Median seconds of fn() over reps calls, after one untimed call."""
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts)


def copy_bench(sl, src, n_keep, n_dst, reps, kvb):
    """-> (session_copy ms, GB/s, torch ms, GB/s); torch's bytes counted as the same one read plus n_dst writes."""
    import torch
    dsts = [d for d in range(sl.n_sessions) if d != src][:n_dst]
    ms = timed(lambda: sl.session_copy(src, dsts, n_keep), reps) * 1e3
    i = sl.info
    planes = [torch.empty((n_dst + 1, i.n_layer, i.n_ctx, i.n_embd), dtype=torch.float16, device="cuda") for _ in range(2)]

    def torch_copy():
        for t in planes:
            for d in range(1, n_dst + 1):
                t[d, :, :n_keep].copy_(t[0, :, :n_keep])

    torch_copy()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    tms = []
    for _ in range(reps):
        ev[0].record()
        torch_copy()
        ev[1].record()
        torch.cuda.synchronize()
        tms.append(ev[0].elapsed_time(ev[1]))
    del planes
    torch.cuda.empty_cache()
    tms = statistics.median(tms)
    moved = (1 + n_dst) * n_keep * kvb
    return ms, moved / ms / 1e6, tms, moved / tms / 1e6


def state_bench(sl, session, reps):
    """-> {"pinned"|"pageable": (save ms, restore ms)} for the session's current state."""
    import torch
    lib, h = capi.lib(), sl.handle
    n = C.c_size_t()
    capi.check(lib.b200_session_state_size(h, session, C.byref(n)))
    out = {}
    for kind in ("pinned", "pageable"):
        if kind == "pinned":
            t = torch.empty(n.value, dtype=torch.uint8, pin_memory=True)
            ptr = C.c_void_p(t.data_ptr())
        else:
            t = np.empty(n.value, np.uint8)
            ptr = capi._ptr(t)
        save = timed(lambda: capi.check(lib.b200_session_save(h, session, ptr, n.value, None)), reps)
        restore = timed(lambda: capi.check(lib.b200_session_restore(h, session, ptr, n.value)), reps)
        out[kind] = (save * 1e3, restore * 1e3)
        del t
    return out, n.value


def serve(sl, extra, prefix, reqs, conc, fork):
    """One arm of (c).  -> (ids per request, first-id seconds per request, last-id seconds per request, seconds)."""
    psess = sl.n_sessions - 1
    ids = [[] for _ in reqs]
    first, last = [0.0] * len(reqs), [0.0] * len(reqs)
    phase = {}                             # request j runs on session j: "prefix" (arm R's first segment) or "gen"
    nxt = 0
    t0 = time.perf_counter()
    with capi.Stream([sl], extra) as st:
        def start():
            nonlocal nxt
            j = nxt
            nxt += 1
            if fork:
                st.fork(psess, j, len(prefix))
                st.add(j, reqs[j][0], reqs[j][1], temperature=T, repeat_penalty=RP, seed=reqs[j][2])
                phase[j] = "gen"
            else:
                st.add(j, prefix, 1)
                phase[j] = "prefix"

        if fork:
            st.add(psess, prefix, 1)
            assert len(list(st)) == 1
        while nxt < min(conc, len(reqs)):
            start()
        while True:
            pairs = st.read(256)
            if not pairs:
                break
            now = time.perf_counter() - t0
            for j, t in pairs:
                if phase[j] == "prefix":           # arm R: the prefix is in; the prefix's own id is not the request's
                    st.add(j, reqs[j][0], reqs[j][1], temperature=T, repeat_penalty=RP, seed=reqs[j][2])
                    phase[j] = "gen"
                    continue
                if not ids[j]:
                    first[j] = now
                ids[j].append(t)
                if len(ids[j]) == reqs[j][1]:
                    last[j] = now
                    if nxt < len(reqs):
                        start()
    return ids, first, last, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--copy-reps", type=int, default=20)
    ap.add_argument("--requests", type=int, default=32)
    ap.add_argument("--concurrent", type=int, default=8)
    ap.add_argument("--seed", type=int, default=11)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_session_fork.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    # sessions 0 .. requests - 1 serve one request each (every one starts at n_past 0); the last holds the prefix
    n_sess = max(args.requests, args.concurrent, 9) + 1
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, N_CTX, n_sessions=n_sess)
    kvb = sl.info.kv_bytes_per_pos
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    rng = np.random.default_rng(args.seed)
    # (a) copies from session 0 filled to 2047 positions
    x = rng.standard_normal((512, sh.n_embd), dtype=np.float32)
    for lo in range(0, 2047, 512):
        sl.session_forward(0, x[:min(512, 2047 - lo)])
    copies = []
    for n_keep in (512, 2047):
        for n_dst in (1, 4, 8):
            ms, gbs, tms, tgbs = copy_bench(sl, 0, n_keep, n_dst, args.copy_reps, kvb)
            copies.append({"n_keep": n_keep, "n_dst": n_dst, "bytes": (1 + n_dst) * n_keep * kvb, "session_copy_ms": ms,
                           "session_copy_gbs": gbs, "torch_ms": tms, "torch_gbs": tgbs})
            print("(a) session_copy n_keep %4d -> %d: %.3f ms, %.0f GB/s; torch strided copy per destination %.3f ms, "
                  "%.0f GB/s; %.2fx" % (n_keep, n_dst, ms, gbs, tms, tgbs, tms / ms), flush=True)
    # (b) save / restore of 512 positions
    sl.session_copy(0, [1], 512)
    st_times, st_bytes = state_bench(sl, 1, args.copy_reps)
    for kind, (s_ms, r_ms) in st_times.items():
        print("(b) %d positions (%.0f MiB), %s host buffer: save %.2f ms (%.1f GB/s), restore %.2f ms (%.1f GB/s)"
              % (512, st_bytes / 2 ** 20, kind, s_ms, st_bytes / s_ms / 1e6, r_ms, st_bytes / r_ms / 1e6), flush=True)
    # (c) the serving mix
    prefix = rng.integers(1, sh.n_vocab, PREFIX).tolist()
    reqs = [(rng.integers(1, sh.n_vocab, int(rng.integers(16, 65))).tolist(), int(rng.integers(32, 129)),
             int(rng.integers(0, 2 ** 63))) for _ in range(args.requests)]
    useful = sum(b for _, b, _ in reqs)
    arms = {"F": True, "R": False}
    res = {a: {"ttft": [], "lat": [], "tps": [], "ids": []} for a in arms}
    for rep in range(1 + args.reps):
        for name in (("F", "R") if rep % 2 == 0 else ("R", "F")):
            sl.session_clear(-1)
            sl.sync()
            ids, first, last, t_all = serve(sl, extra, prefix, reqs, args.concurrent, arms[name])
            res[name]["ids"].append(ids)
            if rep > 0:
                res[name]["ttft"].append(statistics.mean(first) * 1e3)
                res[name]["lat"].append(statistics.mean(last) * 1e3)
                res[name]["tps"].append(useful / t_all)
    same = all(o == res["R"]["ids"][0] for a in arms for o in res[a]["ids"])
    same &= all(len(o) == r[1] for o, r in zip(res["R"]["ids"][0], reqs))
    med = {a: {m: statistics.median(res[a][m]) for m in ("ttft", "lat", "tps")} for a in arms}
    print("(c) %d-id prefix, %d requests (suffixes 16-64, budgets 32-128, %d tokens), at most %d in flight: fork "
          "first id %.0f ms, latency %.0f ms, %.1f tok/s; recompute first id %.0f ms, latency %.0f ms, %.1f tok/s; "
          "fork/recompute tok/s %.2f; ids %s"
          % (PREFIX, args.requests, useful, args.concurrent, med["F"]["ttft"], med["F"]["lat"], med["F"]["tps"],
             med["R"]["ttft"], med["R"]["lat"], med["R"]["tps"], med["F"]["tps"] / med["R"]["tps"],
             "identical" if same else "DIFFER"), flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "session_fork", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "n_ctx": N_CTX, "kv_bytes_per_pos": kvb, "gpu": card, "copy": copies,
                      "state": {"positions": 512, "bytes": st_bytes,
                                **{k: {"save_ms": v[0], "restore_ms": v[1]} for k, v in st_times.items()}},
                      "mix": {"prefix": PREFIX, "requests": args.requests, "concurrent": args.concurrent, "tokens": useful,
                              "reps": args.reps, "temperature": T, "repeat_penalty": RP,
                              **{"fork" if a == "F" else "recompute": {"first_id_ms": med[a]["ttft"],
                                                                       "latency_ms": med[a]["lat"],
                                                                       "tok_s": med[a]["tps"],
                                                                       "tok_s_range": [min(res[a]["tps"]), max(res[a]["tps"])]}
                                 for a in arms},
                              "ids_identical": same}}))
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
