"""Mixed passes (b200_mixed_forward): prompt chunks and decode tokens of several sessions in one pass.  Every session's rows
must equal, bit for bit, the C restatement fed the same chunks and the GPU's own per-session call on a second handle; the
device positions must advance by the counts, so later single-token steps (graph replays) stay exact."""
import os
import subprocess
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _port(path, wtype, n_ctx):
    """The C restatement that covers this slice's weight type."""
    if wtype in (ggjt.T_Q5_0, ggjt.T_Q5_1):
        from q5_port import Q5PortSlice
        return Q5PortSlice(path, n_ctx)
    if wtype in (ggjt.T_Q4_K, ggjt.T_Q6_K):
        from kq_port import KQPortSlice
        return KQPortSlice(path, n_ctx)
    from oracle import oracle
    return oracle.PortSlice(path, n_ctx)


def _mixed_pass(gpu, twin, refs, ids, counts, rng, n_embd, where):
    """One mixed pass on `gpu`; each session's rows against its private restatement and twin.session_forward."""
    x = rng.standard_normal((sum(counts), n_embd), dtype=np.float32)
    got = gpu.mixed_forward(ids, counts, x)
    r0 = 0
    for k, c in zip(ids, counts):
        rows = x[r0:r0 + c]
        bad_ref = int((_bits(got[r0:r0 + c]) != _bits(refs[k].forward(rows))).sum())
        bad_twin = int((_bits(got[r0:r0 + c]) != _bits(twin.session_forward(k, rows))).sum())
        assert bad_ref == 0 and bad_twin == 0, (where, k, c, bad_ref, bad_twin)
        r0 += c


def _decode_rounds(gpu, twin, refs, ids, rng, n_embd, rounds, where):
    """Interleaved single-token steps of every session (graph replays that read the device position)."""
    for r in range(rounds):
        for k in ids:
            x = rng.standard_normal((1, n_embd), dtype=np.float32)
            got = gpu.session_forward(k, x)
            assert (_bits(got) == _bits(refs[k].forward(x))).all(), (where, r, k)
            if twin is not None:
                assert (_bits(got) == _bits(twin.session_forward(k, x))).all(), (where, r, k)


def _slice_path(tmp_models, tmp_path, shape, wtype):
    if wtype == ggjt.T_Q4_K:
        path = str(tmp_path / "kq.bin")
        ggjt.write_kquant_slice(path, ggjt.SHAPES[shape], 2, 4, "q4_K_M", seed=21)
        return path
    return tmp_models(shape, wtype, 0, 1, seed=21)


@pytest.mark.parametrize("shape,wtype", [("tiny128", ggjt.T_Q4_0), ("tiny128", ggjt.T_Q8_0), ("tiny128", ggjt.T_Q4_1),
                                         ("tiny128", ggjt.T_Q5_0), ("tiny3b", ggjt.T_Q4_0), ("tiny", ggjt.T_F16),
                                         ("tinyk128", ggjt.T_Q4_K)],
                         ids=["tiny128-q4_0", "tiny128-q8_0", "tiny128-q4_1", "tiny128-q5_0", "tiny3b-q4_0", "tiny-f16",
                              "tinyk128-q4_K_M"])
def test_mixed_pass_equals_private_contexts(tmp_models, tmp_path, shape, wtype):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    path = _slice_path(tmp_models, tmp_path, shape, wtype)
    n_ctx, S = 256, 6
    gpu, twin = capi.Slice(path, 0, n_ctx, n_sessions=S), capi.Slice(path, 0, n_ctx, n_sessions=S)
    refs = {}
    rng = np.random.default_rng(7)
    try:
        for k, n in zip((0, 1, 2, 3, 5), (5, 1, 30, 12, 2)):      # every session at its own position; session 4 starts empty
            refs[k] = _port(path, wtype, n_ctx)
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            want = refs[k].forward(x)
            assert (_bits(gpu.session_forward(k, x)) == _bits(want)).all() and (_bits(twin.session_forward(k, x)) == _bits(want)).all()
        refs[4] = _port(path, wtype, n_ctx)
        plans = [([0, 1, 2, 3, 4], [1, 17, 1, 5, 40]), ([4, 2, 0, 5, 1], [1, 40, 5, 1, 17]), ([3, 5, 1], [16, 1, 33]),
                 ([2, 4, 0, 1, 3, 5], [1, 1, 9, 1, 1, 2])]
        for i, (ids, counts) in enumerate(plans):
            _mixed_pass(gpu, twin, refs, ids, counts, rng, sh.n_embd, ("pass", i))
        want_past = [gpu.session_n_past(k) for k in range(S)]
        assert want_past == [twin.session_n_past(k) for k in range(S)]
        assert want_past == [5 + 1 + 5 + 9, 1 + 17 + 17 + 33 + 1, 30 + 1 + 40 + 1, 12 + 5 + 16 + 1, 40 + 1 + 1, 2 + 1 + 1 + 2]
        _decode_rounds(gpu, twin, refs, list(range(S)), rng, sh.n_embd, 2, "decode")
    finally:
        for r in refs.values():
            r.close()
        gpu.close()
        twin.close()


@pytest.mark.parametrize("shape", ["tiny128", "tiny3b"])
def test_all_counts_one_is_the_batched_step(tmp_models, shape):
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES[shape]
    path = tmp_models(shape, ggjt.T_Q4_0, 0, 1, seed=21)
    a, b = capi.Slice(path, 0, 96, n_sessions=5), capi.Slice(path, 0, 96, n_sessions=5)
    rng = np.random.default_rng(8)
    try:
        for k, n in enumerate((4, 1, 20, 7, 11)):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            assert (_bits(a.session_forward(k, x)) == _bits(b.session_forward(k, x))).all()
        for ids in ([3, 0, 4, 1, 2], [2, 4], [1, 0, 3]):
            x = rng.standard_normal((len(ids), sh.n_embd), dtype=np.float32)
            assert (_bits(a.batch_forward(ids, x)) == _bits(b.mixed_forward(ids, [1] * len(ids), x))).all(), ids
        assert [a.session_n_past(k) for k in range(5)] == [b.session_n_past(k) for k in range(5)]
    finally:
        a.close()
        b.close()


@pytest.mark.parametrize("tiled", ["1", "0"])
def test_both_sides_of_the_staged_window(tmp_models, monkeypatch, tiled):
    """n_ctx 1024: in one pass, prompt segments ending at or below 512 (query-tiled kernel) and above it (per-query cluster
    kernel, with the segment's row length), plus single tokens below and above 512."""
    from distributedllm_b200 import capi
    monkeypatch.setenv("B200_TILED_ATTN", tiled)
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=23)
    n_ctx = 1024
    gpu, twin = capi.Slice(path, 0, n_ctx, n_sessions=5), capi.Slice(path, 0, n_ctx, n_sessions=5)
    refs = {}
    rng = np.random.default_rng(9)
    try:
        for k, n in enumerate((300, 480, 10, 600, 505)):
            refs[k] = _port(path, ggjt.T_Q4_0, n_ctx)
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            want = refs[k].forward(x)
            assert (_bits(gpu.session_forward(k, x)) == _bits(want)).all() and (_bits(twin.session_forward(k, x)) == _bits(want)).all()
        # ends: 400 (tiled), 540 (crosses 512), 11, 601, 512 (exactly at the window)
        _mixed_pass(gpu, twin, refs, [0, 1, 2, 3, 4], [100, 60, 1, 1, 7], rng, sh.n_embd, "window")
        _mixed_pass(gpu, twin, refs, [3, 2, 1, 0], [37, 50, 1, 3], rng, sh.n_embd, "window2")
        _decode_rounds(gpu, twin, refs, list(range(5)), rng, sh.n_embd, 1, "decode")
    finally:
        for r in refs.values():
            r.close()
        gpu.close()
        twin.close()


def test_fast_prefill_never_applies_to_a_mixed_pass(tmp_models, monkeypatch):
    """tiny128b is a shape the tensor-core prefill tiles.  Control: with fast mode on and min_tokens 1, a prompt chunk of one
    session alone does take it (its rows differ from the exact restatement).  A mixed pass on the same handle, whose
    columns include prompt segments as long as that chunk, stays bit-exact."""
    from distributedllm_b200 import capi
    monkeypatch.setenv("B200_FAST_PREFILL", "1")
    sh = ggjt.SHAPES["tiny128b"]
    path = tmp_models("tiny128b", ggjt.T_Q4_0, 0, 1, seed=24)
    gpu = capi.Slice(path, 0, 128, n_sessions=4)
    gpu.set_fast_prefill(True, 1)
    refs = {k: _port(path, ggjt.T_Q4_0, 128) for k in range(4)}
    rng = np.random.default_rng(10)
    try:
        x = rng.standard_normal((48, sh.n_embd), dtype=np.float32)
        control = int((_bits(gpu.session_forward(3, x)) != _bits(refs[3].forward(x))).sum())
        assert control > 0, "fast mode did not apply to a 48-token session_forward: the check below would prove nothing"
        x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
        assert (_bits(gpu.session_forward(0, x)) == _bits(refs[0].forward(x))).all()
        for ids, counts in (([0, 1, 2], [1, 48, 33]), ([2, 0, 1], [1, 64, 1]), ([1, 2], [2, 40])):
            x = rng.standard_normal((sum(counts), sh.n_embd), dtype=np.float32)
            got = gpu.mixed_forward(ids, counts, x)
            r0 = 0
            for k, c in zip(ids, counts):
                bad = int((_bits(got[r0:r0 + c]) != _bits(refs[k].forward(x[r0:r0 + c]))).sum())
                assert bad == 0, (k, c, bad)
                r0 += c
    finally:
        for r in refs.values():
            r.close()
        gpu.close()


def test_batched_step_over_more_than_32_sessions_advances_every_position(tmp_models):
    """The device position of every listed session moves, not only the first 32: single-token steps (graph replays that
    read it) of sessions listed at index >= 32 stay exact."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=25)
    gpu = capi.Slice(path, 0, 64, n_sessions=48)
    ids = [int(v) for v in np.random.default_rng(11).permutation(48)[:40]]
    refs = {k: _port(path, ggjt.T_Q4_0, 64) for k in ids}
    rng = np.random.default_rng(12)
    try:
        for step in range(2):
            x = rng.standard_normal((len(ids), sh.n_embd), dtype=np.float32)
            got = gpu.batch_forward(ids, x)
            for j, k in enumerate(ids):
                assert (_bits(got[j]) == _bits(refs[k].forward(x[j:j + 1])[0])).all(), (step, j)
        _decode_rounds(gpu, None, refs, ids[32:] + ids[:2], rng, sh.n_embd, 2, "after-batch")
        assert [gpu.session_n_past(k) for k in ids[32:]] == [4] * 8
    finally:
        for r in refs.values():
            r.close()
        gpu.close()


def test_mixed_pass_errors_change_nothing(tmp_models):
    import ctypes as C
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=26)
    gpu = capi.Slice(path, 0, 64, n_sessions=4)
    refs = {k: _port(path, ggjt.T_Q4_0, 64) for k in range(4)}
    rng = np.random.default_rng(13)
    try:
        for k, n in ((0, 3), (1, 60), (2, 1)):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            assert (_bits(gpu.session_forward(k, x)) == _bits(refs[k].forward(x))).all()
        before = [gpu.session_n_past(k) for k in range(4)]
        cases = [([0, 0], [1, 2], 1), ([0, 2], [0, 3], 1), ([0, 2, 3], [30, 20, 15], 1), ([0, 1], [2, 5], 5),
                 ([0, 4], [1, 1], 1), ([2, 3, 0, 1], [1, 1, 1, 5], 5)]
        for ids, counts, code in cases:
            with pytest.raises(capi.B200Error) as e:
                gpu.mixed_forward(ids, counts, np.zeros((sum(counts), sh.n_embd), np.float32))
            assert e.value.code == code, (ids, counts, str(e.value))
            assert [gpu.session_n_past(k) for k in range(4)] == before, (ids, counts)
        L = capi.lib()
        ids, cnt, buf = np.array([0, 2], np.int32), np.array([1, 1], np.int32), np.zeros((2, sh.n_embd), np.float32)
        p = lambda a: C.c_void_p(a.ctypes.data)
        for args in ((None, p(cnt), p(buf), p(buf)), (p(ids), None, p(buf), p(buf)), (p(ids), p(cnt), None, p(buf)),
                     (p(ids), p(cnt), p(buf), None)):
            assert L.b200_mixed_forward(gpu.handle, args[0], args[1], 2, args[2], args[3]) == 1
        assert L.b200_mixed_forward(None, p(ids), p(cnt), 2, p(buf), p(buf)) == 1
        assert L.b200_mixed_forward(gpu.handle, p(ids), p(cnt), 0, p(buf), p(buf)) == 1
        assert [gpu.session_n_past(k) for k in range(4)] == before
        # nothing was written to any cache: the sessions continue exactly
        x = rng.standard_normal((7, sh.n_embd), dtype=np.float32)
        got = gpu.mixed_forward([2, 0, 3], [1, 4, 2], x)
        for k, r0, c in ((2, 0, 1), (0, 1, 4), (3, 5, 2)):
            assert (_bits(got[r0:r0 + c]) == _bits(refs[k].forward(x[r0:r0 + c]))).all(), k
        _decode_rounds(gpu, None, refs, [0, 1, 2, 3], rng, sh.n_embd, 1, "after-errors")
    finally:
        for r in refs.values():
            r.close()
        gpu.close()


def test_one_7b_layer_mixed_pass(tmp_path):
    """One LLaMA-7B-shape layer (H = 32): seven single tokens plus a 128-token prompt segment equal the per-session calls."""
    from distributedllm_b200 import capi
    sh = ggjt.SHAPES["7b"]
    path = str(tmp_path / "l.bin")
    ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=2)
    gpu, twin = capi.Slice(path, 0, 512, n_sessions=8), capi.Slice(path, 0, 512, n_sessions=8)
    rng = np.random.default_rng(14)
    try:
        for k, n in enumerate((3, 17, 40, 1, 64, 9, 100)):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            assert (_bits(gpu.session_forward(k, x)) == _bits(twin.session_forward(k, x))).all()
        for ids, counts in (([0, 1, 2, 3, 4, 5, 6, 7], [1] * 7 + [128]), ([7, 0, 1, 2, 3, 4, 5, 6], [1] * 8),
                            ([0, 1, 2, 7, 3, 4, 5, 6], [1, 1, 1, 128, 1, 1, 1, 1])):
            x = rng.standard_normal((sum(counts), sh.n_embd), dtype=np.float32)
            got = gpu.mixed_forward(ids, counts, x)
            r0 = 0
            for k, c in zip(ids, counts):
                bad = int((_bits(got[r0:r0 + c]) != _bits(twin.session_forward(k, x[r0:r0 + c]))).sum())
                assert bad == 0, (ids, k, c, bad)
                r0 += c
        for k in range(8):
            x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
            assert (_bits(gpu.session_forward(k, x)) == _bits(twin.session_forward(k, x))).all(), k
    finally:
        gpu.close()
        twin.close()


def test_llm_module_mixed(tmp_models):
    from distributedllm_b200 import capi
    from distributedllm_b200.compute_node.slices import import_llm
    llm = import_llm()
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 1, seed=27)
    twin = capi.Slice(path, 0, 64, n_sessions=3)
    assert llm.load_slice(path, n_ctx=64, n_sessions=3) == 0
    rng = np.random.default_rng(15)
    try:
        for k, n in enumerate((4, 9, 1)):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            got = np.frombuffer(llm.propagate_forward_session(k, x), np.float32).reshape(n, -1)
            assert (_bits(got) == _bits(twin.session_forward(k, x))).all()
        for ids, counts in (([2, 0, 1], [3, 1, 5]), ([0, 1, 2], [1, 1, 1])):
            x = rng.standard_normal((sum(counts), sh.n_embd), dtype=np.float32)
            got = np.frombuffer(llm.propagate_forward_mixed(ids, counts, x), np.float32).reshape(sum(counts), -1)
            assert (_bits(got) == _bits(twin.mixed_forward(ids, counts, x))).all(), (ids, counts)
        with pytest.raises(RuntimeError):
            llm.propagate_forward_mixed([0, 0], [1, 1], np.zeros((2, sh.n_embd), np.float32))
        with pytest.raises(ValueError):
            llm.propagate_forward_mixed([0, 1], [1, 2], np.zeros((2, sh.n_embd), np.float32))
        with pytest.raises(ValueError):
            llm.propagate_forward_mixed([0, 1], [1], np.zeros((1, sh.n_embd), np.float32))
        with pytest.raises(TypeError):
            llm.propagate_forward_mixed((0, 1), [1, 1], np.zeros((2, sh.n_embd), np.float32))
    finally:
        llm.unload_slice()
        twin.close()


WORKER = r'''
import os, sys, ctypes as C
sys.path.insert(0, %(root)r)
import numpy as np, torch, torch.distributed as dist
from distributedllm_b200 import capi, ggjt
from distributedllm_b200.pipeline import layer_ranges, join_pipeline, torch_collectives
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
sh = ggjt.SHAPES["tiny128"]
d = %(tmp)r
a, b = layer_ranges(sh.n_layer, world)[rank]
p = os.path.join(d, "s_%%d_%%d.bin" %% (a, b))
ggjt.write_synth_slice(p, sh, a, b, ggjt.T_Q4_0, seed=0)
sl = capi.Slice(p, local, 64, n_sessions=4)
lib = capi.lib()
bcast, gather = torch_collectives(dist, torch.device("cuda", local))
transport = join_pipeline(sl, rank, world, bcast, gather, peer=os.environ.get("B200_PP_PEER", "1") != "0")
_rt = C.CDLL("libcudart.so.12")
def h2d(x):
    assert _rt.cudaMemcpy(C.c_void_p(sl.dev_in), C.c_void_p(x.ctypes.data), C.c_size_t(x.nbytes), 1) == 0
    _rt.cudaDeviceSynchronize()
def fetch(n):
    out = np.empty((n, sh.n_embd), np.float32)
    assert _rt.cudaMemcpy(C.c_void_p(out.ctypes.data), C.c_void_p(sl.pipeline_result), C.c_size_t(out.nbytes), 2) == 0
    _rt.cudaDeviceSynchronize()
    return out
rng = np.random.default_rng(31)
ok = True
if rank == 0:
    whole = os.path.join(d, "whole.bin"); ggjt.write_synth_slice(whole, sh, 0, sh.n_layer - 1, ggjt.T_Q4_0, seed=0)
    ref = capi.Slice(whole, local, 64, n_sessions=4)
for k, n in ((1, 3), (2, 9)):
    x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
    if rank == 0:
        h2d(x)
    capi.check(lib.b200_pipeline_step_session(sl.handle, k, C.c_void_p(sl.dev_in), n, 1))
    sl.sync()
    if rank == 0:
        ok = ok and bool((fetch(n).view(np.uint32) == ref.session_forward(k, x).view(np.uint32)).all())
for ids, counts in (([3, 1, 2], [1, 6, 1]), ([2, 0, 3, 1], [5, 1, 17, 1]), ([0, 1], [1, 1])):
    x = rng.standard_normal((sum(counts), sh.n_embd), dtype=np.float32)
    if rank == 0:
        h2d(x)
    sl.pipeline_step_mixed(ids, counts, sl.dev_in, 1)
    sl.sync()
    if rank == 0:
        got = fetch(sum(counts))
        r0 = 0
        for k, c in zip(ids, counts):
            ok = ok and bool((got[r0:r0 + c].view(np.uint32) == ref.session_forward(k, x[r0:r0 + c]).view(np.uint32)).all())
            r0 += c
# single-token pipeline steps of every session after the mixed steps (positions advanced on both ranks)
for k in range(4):
    x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
    if rank == 0:
        h2d(x)
    capi.check(lib.b200_pipeline_step_session(sl.handle, k, C.c_void_p(sl.dev_in), 1, 1))
    sl.sync()
    if rank == 0:
        ok = ok and bool((fetch(1).view(np.uint32) == ref.session_forward(k, x).view(np.uint32)).all())
ok = ok and [sl.session_n_past(k) for k in range(4)] == [1 + 1 + 1, 3 + 6 + 1 + 1 + 1, 9 + 1 + 5 + 1, 1 + 17 + 1]
dist.barrier()
capi.check(lib.b200_pipeline_destroy(sl.handle))
err = lib.b200_pipeline_error(sl.handle)
if rank == 0:
    print(("PIPELINE_OK" if ok and not err else "PIPELINE_MISMATCH") + " transport=" + transport)
dist.destroy_process_group()
'''


@pytest.mark.parametrize("peer", [1, 0], ids=["peer", "nccl"])
def test_two_gpu_pipeline_mixed_step(tmp_path, peer):
    """A mixed pass through a 2-rank pipeline equals the un-sliced model's per-session calls, on both transports."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT, "tmp": str(tmp_path)})
    env = dict(os.environ, B200_PP_PEER=str(peer), B200_PP_FOLD="1")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(29611 + peer), str(script)],
                         capture_output=True, text=True, timeout=600, env=env)
    assert "PIPELINE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
    assert ("transport=peer" if peer else "transport=nccl") in out.stdout, out.stdout[-500:]
