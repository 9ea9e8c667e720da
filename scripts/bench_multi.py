"""Multi-GPU measurements of BASELINE.json configs 4 and 5 (one process per GPU, launch with torch.distributed.run):

  config 5  LLaMA-13B Q4_0, N slices across N H100s, n_ctx 512, S sessions in THROUGHPUT MODE:
              serial      one session after another, each token waits for its ring result (what a bs=1 client does)
              batched     all S sessions in one batched step travelling through the slices (weights read once per slice)
              pipelined   sessions (or micro-batches of sessions) issued back to back with ring = 2 and collected later:
                          rank r works on group k while rank r+1 works on group k-1 -- every GPU busy
            per-session outputs of the pipelined modes are compared bit for bit with the serial mode; session 0 of the
            serial mode is compared with the compiled reference run over the N slice files on the host.
  config 4  LLaMA-7B F16 (no quantisation), N slices, n_ctx 2048: decode tokens/s at p ~ 1024 and the F16 weight stream.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 scripts/bench_multi.py [5] [4]
Rank 0 prints one JSON object per config.  Timing: CUDA events on every rank's slice stream, max over ranks."""
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402
from distributedllm_b200 import capi, ggjt  # noqa: E402
from distributedllm_b200.pipeline import join_pipeline, layer_ranges, torch_collectives  # noqa: E402

rank, world, local = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
DEV = torch.device("cuda", local)
PEAK, PEAK_SRC = bench.measured_peak()
lib = capi.lib()
cudart = bench._cudart()


def barrier(sl):
    sl.sync()
    dist.barrier()
    sl.sync()


def max_over_ranks(v):
    t = torch.tensor([v], dtype=torch.float64, device=DEV)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t[0])


def h2d(ptr, x):
    x = np.ascontiguousarray(x, np.float32)
    assert cudart.cudaMemcpy(C.c_void_p(ptr), C.c_void_p(x.ctypes.data), C.c_size_t(x.nbytes), 1) == 0
    assert cudart.cudaDeviceSynchronize() == 0       # pageable source: the DMA tail may outlive the call (see bench._h2d)


def d2h(ptr, shape):
    out = np.empty(shape, np.float32)
    assert cudart.cudaMemcpy(C.c_void_p(out.ctypes.data), C.c_void_p(ptr), C.c_size_t(out.nbytes), 2) == 0
    return out


def timed(sl, fn, rounds):
    barrier(sl)
    sl.mark(0)
    for _ in range(rounds):
        fn()
    sl.mark(1)
    barrier(sl)
    return max_over_ranks(sl.mark_elapsed_ms()) / rounds


def reference_chain(paths, acts, n_ctx=512):
    """The reference's multi-node data flow on the host: acts (a list of [n, E] calls) through the slice files in order."""
    from oracle import oracle
    if not oracle.have_ref():
        return None
    threads = min(16, len(os.sched_getaffinity(0)))
    for p in paths:
        sl = oracle.RefSlice(p, n_threads=threads, n_ctx=n_ctx)
        acts = [sl.forward(a) for a in acts]
        sl.close()
    return acts


def config5():
    sh = ggjt.SHAPES["13b"]
    E = sh.n_embd
    S = int(os.environ.get("CFG5_SESSIONS", "8"))
    G = int(os.environ.get("CFG5_GROUPS", "8"))                  # micro-batches of S / G sessions in the pipelined-batch mode
    PRE = int(os.environ.get("CFG5_PREFILL", "256"))
    K = int(os.environ.get("CFG5_ROUNDS", "16"))
    ranges = layer_ranges(sh.n_layer, world)
    a, b = ranges[rank]
    path = bench.slice_file("13b", a, b)
    sl = capi.Slice(path, local, 512, n_sessions=S)
    bcast, gather = torch_collectives(dist, DEV)
    transport = join_pipeline(sl, rank, world, bcast, gather) if world > 1 else "single"
    h = sl.handle
    vp = C.c_void_p

    def step_session(k, n, ring, src=None):
        if world == 1:
            capi.check(lib.b200_session_forward_device(h, k, vp(src or sl.dev_in), n, vp(sl.dev_out), 0))
        else:
            capi.check(lib.b200_pipeline_step_session(h, k, vp(src or sl.dev_in), n, ring))

    def step_batch(ids, ring, src=None):
        arr = np.ascontiguousarray(ids, np.int32)
        if world == 1:
            capi.check(lib.b200_batch_forward_device(h, vp(arr.ctypes.data), len(arr), vp(src or sl.dev_in), vp(sl.dev_out), 0))
        else:
            capi.check(lib.b200_pipeline_step_batch(h, vp(arr.ctypes.data), len(arr), vp(src or sl.dev_in), ring))

    def collect(n, dst):
        if world > 1:
            capi.check(lib.b200_pipeline_collect(h, n, vp(dst)))

    def result_ptr():
        return sl.pipeline_result if world > 1 else sl.dev_out

    def rewind_all(p):
        for k in range(S):
            sl.session_rewind(k, p)

    # ---- prefill every session (untimed)
    xp = bench.synth_inputs(PRE, E, 6)
    t0 = time.perf_counter()
    CH = int(os.environ.get("CFG5_CHUNK", "64"))
    for k in range(S):
        for i in range(0, PRE, CH):
            n = min(CH, PRE - i)
            if rank == 0:
                h2d(sl.dev_in, xp[i:i + n] + np.float32(0.001 * k))
            step_session(k, n, 0)
            sl.sync()
    barrier(sl)
    prefill_s = time.perf_counter() - t0
    xs = bench.synth_inputs(S, E, 7)
    if rank == 0:
        h2d(sl.dev_in, xs)                                          # row k of dev_in = the next token of session k
    res = torch.zeros((S, E), dtype=torch.float32, device=DEV)
    row = lambda k: sl.dev_in + 4 * E * k                           # noqa: E731
    out_row = lambda k: res.data_ptr() + 4 * E * k                  # noqa: E731
    per = S // G
    groups = [list(range(g * per, (g + 1) * per)) for g in range(G)]

    def round_serial():
        for k in range(S):
            step_session(k, 1, 1, row(k))

    def round_batched():
        step_batch(list(range(S)), 1, row(0))

    # rank 0 keeps at most LAG steps un-collected: the mailboxes buffer two messages per link, so `world` steps in flight
    # can never wedge the ring; over NCCL (rendezvous semantics) a step must be collected before the next is issued
    LAG = world if transport == "peer" else 1

    def round_pipelined():
        for i in range(S + LAG):
            if i < S:
                step_session(i, 1, 2, row(i))
            if rank == 0 and i >= LAG:
                collect(1, out_row(i - LAG))

    def round_pipelined_groups():
        for i in range(G + LAG):
            if i < G:
                step_batch(groups[i], 2, row(groups[i][0]))
            if rank == 0 and i >= LAG:
                g = groups[i - LAG]
                collect(len(g), out_row(g[0]))

    # steady state, the way a generation loop runs: session k's next token is issued as soon as ITS previous result is
    # back, so the pipeline never drains between rounds (each call = `rounds` tokens for every session / group)
    def steady(n_items, issue, gather, rounds):
        total = n_items * rounds
        win = min(LAG, n_items)
        for j in range(total + win):
            if rank == 0 and j >= win:
                gather((j - win) % n_items)
            if j < total:
                issue(j % n_items)

    def steady_sessions(rounds):
        steady(S, lambda k: step_session(k, 1, 2, row(k)), lambda k: collect(1, out_row(k)), rounds)

    def steady_groups(rounds):
        steady(G, lambda g: step_batch(groups[g], 2, row(groups[g][0])), lambda g: collect(len(groups[g]), out_row(groups[g][0])), rounds)

    # ---- parity: pipelined modes vs the serial mode, same tokens, same positions (3 rounds each, rewound in between)
    R = 3
    outs = {}
    for name, fn in (("serial", None), ("batched", round_batched), ("pipelined", round_pipelined), ("pipelined_groups", round_pipelined_groups),
                     ("steady_sessions", steady_sessions), ("steady_groups", steady_groups)):
        rewind_all(PRE)
        barrier(sl)
        rec = np.zeros((R, S, E), np.float32)
        for r_ in range(R):
            if name == "serial":
                for k in range(S):
                    step_session(k, 1, 1, row(k))
                    sl.sync()
                    if rank == 0:
                        rec[r_, k] = d2h(result_ptr(), (1, E))[0]
            elif name == "batched":
                fn()
                sl.sync()
                if rank == 0:
                    rec[r_] = d2h(result_ptr(), (S, E))
            elif name.startswith("steady"):
                if r_ == R - 1:                  # R tokens per session in ONE pipelined run; only the last round's outputs remain
                    fn(R)
                    sl.sync()
                    if rank == 0:
                        rec[r_] = res.cpu().numpy() if world > 1 else 0
            else:
                fn()
                sl.sync()
                if rank == 0:
                    rec[r_] = res.cpu().numpy() if world > 1 else 0
            barrier(sl)
        outs[name] = rec
    parity = None
    if rank == 0:
        parity = {}
        for name in ("batched", "pipelined", "pipelined_groups"):
            if world == 1 and name != "batched":
                continue
            parity[name + "_vs_serial_mismatching_floats"] = int((outs[name].view(np.uint32) != outs["serial"].view(np.uint32)).sum())
        for name in ("steady_sessions", "steady_groups"):
            if world > 1:                        # the last of R tokens per session, produced without ever draining the pipeline
                parity[name + "_vs_serial_mismatching_floats"] = int((outs[name][R - 1].view(np.uint32) != outs["serial"][R - 1].view(np.uint32)).sum())
        parity["checked_floats_per_mode"] = int(outs["serial"].size)
    # session 0's first serial step against the compiled reference over the slice files (prompt + 1 token)
    if rank == 0 and not os.environ.get("CFG5_NO_REF"):
        try:
            t1 = time.perf_counter()
            want = reference_chain([bench.slice_file("13b", x, y) for x, y in ranges],
                                   [xp[i:i + 32] for i in range(0, PRE, 32)] + [xs[0:1]])
            if want is not None:
                parity["session0_step0_vs_reference_mismatching_floats"] = int(
                    (np.ascontiguousarray(want[-1]).view(np.uint32) != outs["serial"][0, 0:1].view(np.uint32)).sum())
                parity["reference_seconds"] = round(time.perf_counter() - t1, 1)
        except Exception as ex:  # noqa: BLE001
            parity["reference_error"] = repr(ex)
    barrier(sl)

    # ---- timing
    modes = {}
    for name, fn in (("serial", round_serial), ("batched", round_batched), ("pipelined", round_pipelined),
                     ("pipelined_groups", round_pipelined_groups)):
        if world == 1 and name.startswith("pipelined"):
            continue
        rewind_all(PRE)
        for _ in range(2):
            fn()
        ms = timed(sl, fn, K)
        modes[name] = {"ms_per_round": ms, "tokens_per_s": S * 1e3 / ms}
    if world > 1:
        for name, fn in (("steady_sessions", steady_sessions), ("steady_groups", steady_groups)):
            rewind_all(PRE)
            fn(2)
            ms = timed(sl, lambda: fn(K), 1) / K
            modes[name] = {"ms_per_round": ms, "tokens_per_s": S * 1e3 / ms,
                           "note": "%d tokens per session in one pipelined run, a session's next token issued when its previous result is back" % K}
    err = lib.b200_pipeline_error(h) if world > 1 else 0
    info = sl.info
    out = None
    if rank == 0:
        w_all = sum(4 * (E * E // 32 * 18) + 3 * (E * sh.n_ff // 32 * 18) + 2 * E * 4 for _ in range(sh.n_layer))
        kv_pos = sh.n_layer * 2 * E * 2
        p_mid = PRE + 2 + K / 2
        single = peak_single = PEAK * 1e9 / (w_all + kv_pos * p_mid)
        out = {"config": "BASELINE config 5: LLaMA-13B Q4_0, %d slice(s) x %s layers on %dxH100, n_ctx 512, %d sessions (throughput mode), "
                         "decode at p~%d" % (world, "/".join(str(y - x + 1) for x, y in ranges), world, S, p_mid),
               "transport": transport, "modes": modes, "groups": G, "sessions": S, "steps_in_flight": LAG,
               "aggregate_tokens_per_s": max(m["tokens_per_s"] for m in modes.values()),
               "single_sequence_tokens_per_s": modes["serial"]["tokens_per_s"],
               "speedup_over_single_sequence": max(m["tokens_per_s"] for m in modes.values()) / modes["serial"]["tokens_per_s"],
               "bounds": {"one_gpu_bs1_tokens_per_s": single,
                          "n_gpus_pipelined_bs1_tokens_per_s": world * peak_single,
                          "note": "b * BW / (W + sum KV) per slice; BW = %.0f GB/s (%s)" % (PEAK, PEAK_SRC)},
               "parity": parity, "mailbox_timeout": bool(err), "prefill_seconds": round(prefill_s, 2),
               "this_rank_weight_bytes": int(info.weight_bytes)}
    if world > 1:
        capi.check(lib.b200_pipeline_destroy(h))
    sl.close()
    return out


def config4():
    sh = ggjt.SHAPES["7b"]
    E = sh.n_embd
    NCTX, PRE, K = 2048, int(os.environ.get("CFG4_PREFILL", "1024")), int(os.environ.get("CFG4_STEPS", "64"))
    ranges = layer_ranges(sh.n_layer, world)
    a, b = ranges[rank]

    def f16_file(x, y):
        p = os.path.join(bench.model_dir(), "7b_f16_s0_layers_%d_%d.bin" % (x, y))
        if not os.path.isfile(p):
            ggjt.write_fast_f16_slice(p + ".tmp%d" % os.getpid(), sh, x, y, 0)
            os.replace(p + ".tmp%d" % os.getpid(), p)
        return p
    path = f16_file(a, b)
    sl = capi.Slice(path, local, NCTX)
    bcast, gather = torch_collectives(dist, DEV)
    transport = join_pipeline(sl, rank, world, bcast, gather) if world > 1 else "single"
    h, vp = sl.handle, C.c_void_p

    def step(n, ring):
        if world == 1:
            sl.forward_device(sl.dev_in, n, sl.dev_out)
        else:
            capi.check(lib.b200_pipeline_step(h, vp(sl.dev_in), n, ring))
    # ---- parity on a short run against the compiled reference over the N slice files (the reference is fixed at n_ctx 512)
    parity = None
    x0, x1 = bench.synth_inputs(8, E, 8), bench.synth_inputs(3, E, 9)
    got = []
    for x in [x0] + [x1[i:i + 1] for i in range(3)]:
        if rank == 0:
            h2d(sl.dev_in, x)
        step(x.shape[0], 1)
        sl.sync()
        if rank == 0:
            got.append(d2h(sl.pipeline_result if world > 1 else sl.dev_out, x.shape))
    barrier(sl)
    if rank == 0 and not os.environ.get("CFG4_NO_REF"):
        try:
            t1 = time.perf_counter()
            want = reference_chain([f16_file(x, y) for x, y in ranges], [x0] + [x1[i:i + 1] for i in range(3)])
            if want is not None:
                bad = sum(int((np.ascontiguousarray(w).view(np.uint32) != g.view(np.uint32)).sum()) for w, g in zip(want, got))
                parity = {"mismatching_floats": bad, "checked_floats": int(sum(g.size for g in got)), "against": "reference",
                          "what": "8-token prompt + 3 decode steps through the %d F16 slice files" % world,
                          "reference_seconds": round(time.perf_counter() - t1, 1)}
        except Exception as ex:  # noqa: BLE001
            parity = {"error": repr(ex)}
    barrier(sl)
    sl.clear_context()
    barrier(sl)
    # ---- prefill to p = 1024, then timed decode
    xp = bench.synth_inputs(PRE, E, 5)
    t0 = time.perf_counter()
    for i in range(0, PRE, 128):
        n = min(128, PRE - i)
        if rank == 0:
            h2d(sl.dev_in, xp[i:i + n])
        step(n, 0)
        sl.sync()
    barrier(sl)
    prefill_s = time.perf_counter() - t0
    if rank == 0:
        h2d(sl.dev_in, xp[0:1])
    for _ in range(4):
        step(1, 1)
    ms = timed(sl, lambda: step(1, 1), K)
    # this rank's own layers, no hand-off: the F16 weight stream of one slice
    sl.rewind(PRE)
    for _ in range(3):
        sl.forward_device(sl.dev_in, 1, sl.dev_out)
    sl.sync()
    sl.mark(0)
    for _ in range(32):
        sl.forward_device(sl.dev_in, 1, sl.dev_out)
    sl.mark(1)
    sl.sync()
    own_ms = sl.mark_elapsed_ms() / 32
    info = sl.info
    own_bytes = info.weight_bytes + info.kv_bytes_per_pos * (PRE + 20)
    own_gbs = own_bytes / (own_ms * 1e-3) / 1e9
    t = torch.tensor([own_gbs], dtype=torch.float64, device=DEV)
    gl = [torch.zeros_like(t) for _ in range(world)]
    dist.all_gather(gl, t)
    err = lib.b200_pipeline_error(h) if world > 1 else 0
    out = None
    if rank == 0:
        w_all = sh.n_layer * (4 * E * E * 2 + 3 * E * sh.n_ff * 2 + 2 * E * 4)
        kv_pos = sh.n_layer * 2 * E * 2
        p_mid = PRE + 4 + K / 2
        bound = PEAK * 1e9 / (w_all + kv_pos * p_mid)
        out = {"config": "BASELINE config 4: LLaMA-7B F16 (no quantisation), %d slice(s) x %s layers on %dxH100, n_ctx 2048 batch 1, "
                         "decode at p~%d after a %d-token prefill" % (world, "/".join(str(y - x + 1) for x, y in ranges), world, p_mid, PRE),
               "transport": transport, "tokens_per_s": 1e3 / ms, "ms_per_step": ms, "us_per_layer_incl_handoff": 1e3 * ms / sh.n_layer,
               "roofline_tokens_per_s_one_gpu": bound, "frac_of_one_gpu": (1e3 / ms) / bound,
               "per_rank_slice_gbs": [round(float(x[0]), 1) for x in gl], "per_rank_slice_frac_of_peak": [round(float(x[0]) / PEAK, 3) for x in gl],
               "peak_gbs": PEAK, "prefill_tokens_per_s": PRE / prefill_s, "parity": parity, "mailbox_timeout": bool(err)}
    if world > 1:
        capi.check(lib.b200_pipeline_destroy(h))
    sl.close()
    return out


if __name__ == "__main__":
    which = [a for a in sys.argv[1:] if a in ("4", "5")] or ["5", "4"]
    for w in which:
        r = config5() if w == "5" else config4()
        if rank == 0:
            print(json.dumps(r), flush=True)
        dist.barrier()
    dist.destroy_process_group()
