"""GPU: k-quant slices (Q4_K_S / Q4_K_M / Q6_K files: Q4_K and Q6_K matrices in any mix, Q8_K activations quantised in
each matmul's prologue) -- bit-identical to the C restatement, to goldens dumped from the reference and, where oracle/_ref
is built, to the reference itself."""
import hashlib
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)
MIXES = ["q4_K_S", "q4_K_M", "q6_K"]
REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.fixture
def kq_slice(tmp_path):
    def make(shape, mix, a, b, seed=0):
        path = str(tmp_path / ("%s_%s_%d_%d_%d.bin" % (shape, mix, a, b, seed)))
        if not os.path.exists(path):
            ggjt.write_kquant_slice(path, ggjt.SHAPES[shape], a, b, mix, seed=seed)
        return path
    return make


def _run_pair(path, calls, n_embd, n_ctx=512, seed=1, digests=None):
    """GPU against the C restatement, call by call; `digests`: the GPU outputs' SHA-256 are appended."""
    from distributedllm_b200 import capi
    from kq_port import KQPortSlice

    rng = np.random.default_rng(seed)
    gpu = capi.Slice(path, 0, n_ctx)
    cpu = KQPortSlice(path, n_ctx)
    bad = tot = 0
    try:
        for n in calls:
            x = rng.standard_normal((n, n_embd), dtype=np.float32)
            a = cpu.forward(x)
            b = gpu.forward(x)
            bad += int((_bits(a) != _bits(b)).sum())
            tot += a.size
            assert np.isfinite(b).all()
            if digests is not None:
                digests.append(hashlib.sha256(np.ascontiguousarray(b, np.float32).tobytes()).hexdigest())
    finally:
        gpu.close()
        cpu.close()
    return bad, tot


@pytest.mark.parametrize("mix", MIXES)
@pytest.mark.parametrize("shape", ["tinyk", "tinyk128"])
def test_kquant_bit_exact_prefill_then_decode(kq_slice, shape, mix):
    """Layers 2-4 of 8: a slice starting mid-model; for Q4_K_M layer 3's wv / w2 are Q6_K, layers 2 and 4's are Q4_K."""
    path = kq_slice(shape, mix, 2, 4)
    bad, tot = _run_pair(path, [40, 1, 1, 7, 1, 20, 3, 1] + [1] * 40, ggjt.SHAPES[shape].n_embd)
    assert bad == 0, "%d of %d floats differ from the oracle" % (bad, tot)


def test_kquant_goldens_on_gpu(tmp_path):
    """Hidden states against the reference's own, dumped into tests/golden/slices_kquant.*."""
    from distributedllm_b200 import capi
    meta = json.load(open(os.path.join(GOLD, "slices_kquant.json")))
    gold = np.load(os.path.join(GOLD, "slices_kquant.npz"))
    assert len(meta) == 6
    for name, m in meta.items():
        path = str(tmp_path / (name + ".bin"))
        ggjt.write_kquant_slice(path, ggjt.SHAPES[m["shape"]], m["layers"][0], m["layers"][1], m["mix"], seed=0)
        sl = capi.Slice(path, 0, 512)
        for i in range(len(m["schedule"])):
            y = sl.forward(gold["%s/x%d" % (name, i)])
            bad = int((_bits(y) != _bits(gold["%s/y%d" % (name, i)])).sum())
            assert bad == 0, (name, i, bad)
        sl.close()


@pytest.mark.parametrize("mix", MIXES)
def test_kquant_weight_type_and_bytes(kq_slice, mix):
    from distributedllm_b200 import capi
    path = kq_slice("tinyk128", mix, 2, 4)
    f = ggjt.read_file(path, sliced=True)
    sl = capi.Slice(path, 0, 64)
    try:
        assert sl.info.weight_type == (ggjt.T_Q6_K if mix == "q6_K" else ggjt.T_Q4_K)
        assert sl.info.weight_bytes == sum(t.nbytes for t in f.tensors.values())
    finally:
        sl.close()


@pytest.mark.parametrize("env", [{"B200_RING": "0"}, {"B200_PDL": "0", "B200_GRAPH": "0"}, {"B200_NC": "8"}, {"B200_NC": "4"},
                                 {"B200_NC": "2"}, {"B200_TILED_ATTN": "0"}, {"B200_NQ": "1"}, {"B200_FAST_PREFILL": "1"}],
                         ids=["ring0", "pdl0graph0", "nc8", "nc4", "nc2", "tiled0", "nq1", "fast1"])
@pytest.mark.parametrize("shape", ["tinyk", "tinyk128"])
def test_kquant_scheduling_choices_are_exact(kq_slice, monkeypatch, env, shape):
    """Every scheduling switch keeps the bits; B200_NQ and B200_FAST_PREFILL do not apply to k-quant slices."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    path = kq_slice(shape, "q4_K_M", 2, 4)
    bad, tot = _run_pair(path, [33, 1, 1, 9, 1, 64, 1], ggjt.SHAPES[shape].n_embd)
    assert bad == 0, "%s: %d of %d floats differ" % (env, bad, tot)


@pytest.mark.parametrize("mix", ["q4_K_M", "q6_K"])
def test_kquant_batched_step_equals_private_contexts(kq_slice, mix):
    from distributedllm_b200 import capi
    from kq_port import KQPortSlice
    sh = ggjt.SHAPES["tinyk128"]
    path = kq_slice("tinyk128", mix, 2, 4, seed=21)
    gpu = capi.Slice(path, 0, 96, n_sessions=8)
    rng = np.random.default_rng(3)
    prompt_len, sessions = [7, 1, 33, 12], [6, 0, 3, 2]
    cpu = []
    try:
        for b in range(len(sessions)):
            ref = KQPortSlice(path, 96)
            x = rng.standard_normal((prompt_len[b], sh.n_embd), dtype=np.float32)
            assert (_bits(gpu.session_forward(sessions[b], x)) == _bits(ref.forward(x))).all()
            cpu.append(ref)
        for step in range(5):
            x = rng.standard_normal((len(sessions), sh.n_embd), dtype=np.float32)
            got = gpu.batch_forward(sessions, x)
            for b in range(len(sessions)):
                assert (_bits(got[b]) == _bits(cpu[b].forward(x[b:b + 1])[0])).all(), (step, b)
        # interleaved single-token steps of the sessions
        for step in range(3):
            for b in range(len(sessions)):
                x = rng.standard_normal((1, sh.n_embd), dtype=np.float32)
                assert (_bits(gpu.session_forward(sessions[b], x)) == _bits(cpu[b].forward(x))).all(), (step, b)
    finally:
        for c in cpu:
            c.close()
        gpu.close()


def test_kquant_llm_module_and_extra_layers_match_reference_goldens(tmp_path):
    """`llm` module: a Q4_K_M slice's hidden states, then the client side of a k-quant model: Q4_K tok_embeddings rows
    dequantised on the GPU, the Q6_K lm_head, the greedy id."""
    from distributedllm_b200.compute_node.slices import import_llm
    llm = import_llm()
    meta = json.load(open(os.path.join(GOLD, "slices_kquant.json")))
    gold = np.load(os.path.join(GOLD, "slices_kquant.npz"))
    name = "tinyk128_q4_K_M"
    m = meta[name]
    path = str(tmp_path / "s.bin")
    ggjt.write_kquant_slice(path, ggjt.SHAPES[m["shape"]], m["layers"][0], m["layers"][1], m["mix"], seed=0)
    assert llm.load_slice(path) == 0
    for i in range(len(m["schedule"])):
        out = np.array(llm.propagate_forward(gold["%s/x%d" % (name, i)].ravel().tolist()), np.float32)
        assert (_bits(out) == _bits(gold["%s/y%d" % (name, i)]).ravel()).all(), i
    assert llm.unload_slice() == 0

    g = np.load(os.path.join(GOLD, "extra_kquant.npz"))
    sh = ggjt.SHAPES["tinyk128"]
    extra = str(tmp_path / "extra.bin")
    ggjt.write_kquant_extra(extra, sh, "q4_K_M", seed=0)
    f = ggjt.read_file(extra)
    assert f.tensors["tok_embeddings.weight"].ttype == ggjt.T_Q4_K and f.tensors["output.weight"].ttype == ggjt.T_Q6_K
    emb = np.array(llm.prepare_embeddings(extra, g["tokens"].tolist()), np.float32).reshape(-1, sh.n_embd)
    assert (_bits(emb) == _bits(g["emb"])).all()
    hid = g["hidden"]
    la = np.array(llm.get_logits(extra, hid.ravel().tolist(), True), np.float32).reshape(len(hid), -1)
    assert (_bits(la) == _bits(g["logits_all"])).all(), int((_bits(la) != _bits(g["logits_all"])).sum())
    for i, want in enumerate(g["next_ids"]):
        assert llm.get_next_token(extra, hid[:i + 1].ravel().tolist()) == int(want)


@pytest.mark.parametrize("mix,layer", [("q4_K_S", 4), ("q4_K_M", 0), ("q4_K_M", 4), ("q6_K", 4)])
def test_kquant_one_7b_layer_bit_exact(tmp_path, mix, layer):
    """One layer at LLaMA-7B shape (4096 / 11008: 43 super-blocks per w2 row, an odd count) with real tile counts and ring
    depths, against the C restatement and the reference's digests (tests/golden/ref_digests_kquant.json).  Q4_K_M layer 0
    has Q6_K wv / w2 (the split qkv launch), layer 4 has none."""
    g = json.load(open(os.path.join(GOLD, "ref_digests_kquant.json")))
    sh = ggjt.SHAPES["7b"]
    path = str(tmp_path / "l.bin")
    ggjt.write_kquant_slice(path, sh, layer, layer, mix, seed=g["seed"])
    got = []
    bad, tot = _run_pair(path, g["schedule"], sh.n_embd, digests=got)
    assert bad == 0, "%d of %d floats differ" % (bad, tot)
    assert got == g["digests"]["%s_layer%d" % (mix, layer)]


def _write_with_types(path, shape, types):
    """A one-layer slice of `shape` whose matrices have the given ggml types (raw bytes zero: only the loader reads it)."""
    e, ff = shape.n_embd, shape.n_ff
    dims = {"attention.wq.weight": (e, e), "attention.wk.weight": (e, e), "attention.wv.weight": (e, e),
            "attention.wo.weight": (e, e), "feed_forward.w1.weight": (ff, e), "feed_forward.w2.weight": (e, ff),
            "feed_forward.w3.weight": (ff, e)}
    sizes = {2: (32, 18), 12: (256, 144), 13: (256, 176), 11: (256, 110), 10: (256, 84), 14: (256, 210)}
    hp = ggjt.HParams(shape.n_vocab, e, shape.n_mult, shape.n_head, 1, e // shape.n_head, ggjt.FTYPE_Q4_K_M, 0)
    with open(path, "wb") as f:
        ggjt._write_header(f, hp, ggjt.default_vocab(shape.n_vocab))
        for nm in ggjt.LAYER_TENSORS:
            name = ("layers.0." + nm).encode()
            if nm.endswith("norm.weight"):
                ne, t, raw = (e,), ggjt.T_F32, np.ones(e, np.float32).tobytes()
            else:
                rows, k = dims[nm]
                t = types.get(nm, ggjt.T_Q4_K)
                blk, sz = sizes[t]
                ne, raw = (k, rows), bytes(rows * k // blk * sz)
            f.write(struct.pack("<III", len(ne), len(name), t))
            f.write(struct.pack("<%dI" % len(ne), *ne))
            f.write(name)
            f.write(b"\0" * ((-f.tell()) & 31))
            f.write(raw)


@pytest.mark.parametrize("types,what", [({"feed_forward.w2.weight": 13}, "type 13"),
                                        ({"attention.wv.weight": 11}, "type 11"),
                                        ({"attention.wo.weight": 10}, "type 10"),
                                        ({"feed_forward.w1.weight": 2}, "type 2"),
                                        ({"attention.wq.weight": 13}, "weight type 13 unsupported")],
                         ids=["q5_K", "q3_K", "q2_K", "q4_0_mix", "q5_K_first"])
def test_kquant_load_refuses_unsupported_types(tmp_path, types, what):
    from distributedllm_b200 import capi
    path = str(tmp_path / "bad.bin")
    _write_with_types(path, ggjt.SHAPES["tinyk128"], types)
    with pytest.raises(capi.B200Error) as ei:
        capi.Slice(path, 0, 64)
    msg = str(ei.value)
    assert what in msg, msg
    assert next(iter(types)) in msg, msg                  # the message names the tensor


def test_kquant_load_refuses_dimensions_not_divisible_by_256(tmp_path):
    """tiny: n_embd 256 but n_ff 704, which no whole number of 256-wide super-blocks covers."""
    from distributedllm_b200 import capi
    path = str(tmp_path / "bad.bin")
    _write_with_types(path, ggjt.SHAPES["tiny"], {})
    with pytest.raises(capi.B200Error) as ei:
        capi.Slice(path, 0, 64)
    assert "divisible by 256" in str(ei.value) and "n_ff 704" in str(ei.value), str(ei.value)


@pytest.mark.parametrize("split,env", [(3, {}), (4, {}), (3, {"B200_NQ": "1"})],
                         ids=["last_w2_q6_K", "last_w2_q4_K", "last_w2_q6_K_nq1"])
def test_kquant_two_gpu_pipeline_peer_folded(tmp_path, split, env):
    """Two ranks on a Q4_K_M tinyk128 model, the hand-off folded into each slice's last w2 (EPI_RESID_SEND): rank 0 holds
    layers 0..split.  Q4_K_M makes w2 Q6_K in layers 0, 3, 6, 7, so split 3 ends rank 0 on a Q6_K w2 and split 4 on a Q4_K
    one (rank 1 ends on layer 7's Q6_K w2, which sends the ring result back).  B200_NQ=1 does not apply to k-quant slices
    and must leave the fold on.  Every step is compared bit for bit with the un-sliced model on one GPU."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    sys.path.insert(0, HERE)
    from test_gpu_pipeline import WORKER
    worker = WORKER.replace('sh = ggjt.SHAPES["tiny128"]', 'sh = ggjt.SHAPES["tinyk128"]')
    worker = worker.replace("a, b = layer_ranges(sh.n_layer, world)[rank]",
                            "a, b = [(0, %d), (%d, sh.n_layer - 1)][rank]" % (split, split + 1))
    worker = worker.replace("ggjt.write_synth_slice(p, sh, a, b, WT, seed=0)", 'ggjt.write_kquant_slice(p, sh, a, b, "q4_K_M", seed=0)')
    worker = worker.replace("ggjt.write_synth_slice(whole, sh, 0, sh.n_layer - 1, WT, seed=0)",
                            'ggjt.write_kquant_slice(whole, sh, 0, sh.n_layer - 1, "q4_K_M", seed=0)')
    assert worker.count("write_kquant_slice") == 2 and "(0, %d)" % split in worker
    script = tmp_path / "worker.py"
    script.write_text(worker % {"root": ROOT, "tmp": str(tmp_path)})
    e = dict(os.environ, B200_PP_PEER="1", B200_PP_FOLD="1", **env)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(29571 + split + 2 * len(env)), str(script)],
                         capture_output=True, text=True, timeout=600, env=e)
    assert "PIPELINE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
    assert "transport=peer" in out.stdout, out.stdout[-500:]


@pytest.mark.skipif(not os.path.isfile(os.path.join(REF_DIR, "quantize")), reason="oracle/_ref not built")
def test_kquant_reference_quantizer_q4_K_M_live(tmp_path):
    """Blocks the reference's own quantiser makes: `quantize q4_K_M` on a seeded F32 tinyk128 model, `slice_model` layers
    2-4, then GPU and reference hidden states bit for bit (prompt chunks within the reference's 32-token limit)."""
    from distributedllm_b200 import capi
    from oracle import oracle
    sh = ggjt.SHAPES["tinyk128"]
    full, q, sl = str(tmp_path / "f32.bin"), str(tmp_path / "q.bin"), str(tmp_path / "s.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=4)
    subprocess.run([os.path.join(REF_DIR, "quantize"), full, q, "q4_K_M"], check=True, capture_output=True)
    subprocess.run([os.path.join(REF_DIR, "slice_model"), "slice", q, "2", "4", sl], check=True, capture_output=True)
    types = {t.ttype for t in ggjt.read_file(sl).tensors.values()}
    assert types == {ggjt.T_F32, ggjt.T_Q4_K, ggjt.T_Q6_K}
    gpu, ref = capi.Slice(sl, 0, 256), oracle.RefSlice(sl, 3, 256)
    rng = np.random.default_rng(9)
    try:
        for n in [20, 1, 1, 7, 1, 1]:
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            a, b = ref.forward(x), gpu.forward(x)
            assert (_bits(a) == _bits(b)).all(), int((_bits(a) != _bits(b)).sum())
    finally:
        gpu.close()
        ref.close()
