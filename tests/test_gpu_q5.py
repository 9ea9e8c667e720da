"""GPU: Q5_0 / Q5_1 slices (a fifth bit per weight: Q4_0's chain with Q8_0 activations, Q4_1's chain with Q8_1
activations and the scalar min term) -- bit-identical to the C restatement and to goldens dumped from the reference."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q5 = [ggjt.T_Q5_0, ggjt.T_Q5_1]
IDS = ["q5_0", "q5_1"]


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _run_pair(path, calls, shape, n_ctx=512, seed=1):
    from distributedllm_b200 import capi
    from q5_port import Q5PortSlice

    rng = np.random.default_rng(seed)
    gpu = capi.Slice(path, 0, n_ctx)
    cpu = Q5PortSlice(path, n_ctx)
    bad = tot = 0
    try:
        assert gpu.info.weight_type == ggjt.read_file(path, sliced=True).tensors[
            "layers.%d.attention.wq.weight" % cpu.first_layer].ttype
        for n in calls:
            x = rng.standard_normal((n, shape.n_embd), dtype=np.float32)
            a = cpu.forward(x)
            b = gpu.forward(x)
            bad += int((_bits(a) != _bits(b)).sum())
            tot += a.size
            assert np.isfinite(b).all()
    finally:
        gpu.close()
        cpu.close()
    return bad, tot


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
@pytest.mark.parametrize("shape", ["tiny", "tiny128", "tiny3b"])
def test_q5_bit_exact_prefill_then_decode(tmp_models, shape, wtype):
    sh = ggjt.SHAPES[shape]
    path = tmp_models(shape, wtype, 1, 2)
    bad, tot = _run_pair(path, [40, 1, 1, 7, 1, 20, 3, 1] + [1] * 40, sh)
    assert bad == 0, "%d of %d floats differ from the oracle" % (bad, tot)


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
def test_q5_weight_bytes_are_file_bytes(tmp_models, wtype):
    from distributedllm_b200 import capi
    path = tmp_models("tiny3b", wtype, 0, 1)
    f = ggjt.read_file(path, sliced=True)
    sl = capi.Slice(path, 0, 64)
    try:
        assert sl.info.weight_type == wtype
        assert sl.info.weight_bytes == sum(t.nbytes for t in f.tensors.values())
    finally:
        sl.close()


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
@pytest.mark.parametrize("env", [{"B200_RING": "0"}, {"B200_NQ": "0"}, {"B200_NQ": "1"}, {"B200_PDL": "0", "B200_GRAPH": "0"},
                                 {"B200_PDL": "1", "B200_GRAPH": "1"}, {"B200_NC": "8"}, {"B200_NC": "4"}, {"B200_NC": "2"}],
                         ids=["ring0", "nq0", "nq1", "pdl0graph0", "pdl1graph1", "nc8", "nc4", "nc2"])
def test_q5_scheduling_choices_are_exact(tmp_models, monkeypatch, env, wtype):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    sh = ggjt.SHAPES["tiny3b"]
    path = tmp_models("tiny3b", wtype, 0, 2)
    bad, tot = _run_pair(path, [33, 1, 1, 9, 1, 5, 1], sh)
    assert bad == 0, "%s: %d of %d floats differ" % (env, bad, tot)


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
@pytest.mark.parametrize("switch", ["B200_FAST_PREFILL"])
def test_q5_ignores_paths_it_does_not_take(tmp_models, monkeypatch, switch, wtype):
    """The wgmma prefill covers Q4_0 / Q8_0 only: with its switch on, a Q5 slice stays on the exact kernels."""
    monkeypatch.setenv(switch, "1")
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", wtype, 0, 2)
    bad, tot = _run_pair(path, [64, 1, 1, 40, 1], sh)
    assert bad == 0, "%s=1: %d of %d floats differ" % (switch, bad, tot)


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
def test_q5_batched_step_equals_private_contexts(tmp_models, wtype):
    from distributedllm_b200 import capi
    from q5_port import Q5PortSlice
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", wtype, 0, 1, seed=21)
    gpu = capi.Slice(path, 0, 96, n_sessions=8)
    rng = np.random.default_rng(3)
    prompt_len, sessions = [7, 1, 33, 12], [6, 0, 3, 2]
    cpu = []
    for b in range(len(sessions)):
        ref = Q5PortSlice(path, 96)
        x = rng.standard_normal((prompt_len[b], sh.n_embd), dtype=np.float32)
        assert (_bits(gpu.session_forward(sessions[b], x)) == _bits(ref.forward(x))).all()
        cpu.append(ref)
    for step in range(5):
        x = rng.standard_normal((len(sessions), sh.n_embd), dtype=np.float32)
        got = gpu.batch_forward(sessions, x)
        for b in range(len(sessions)):
            assert (_bits(got[b]) == _bits(cpu[b].forward(x[b:b + 1])[0])).all(), (step, b)
    for c in cpu:
        c.close()
    gpu.close()


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
def test_q5_goldens_on_gpu(tmp_path, wtype):
    """Hidden states against the reference's own, dumped into tests/golden/slices_q5_*."""
    from distributedllm_b200 import capi
    stem = "slices_" + ggjt.TYPE_NAME[wtype]
    meta = json.load(open(os.path.join(GOLD, stem + ".json")))
    gold = np.load(os.path.join(GOLD, stem + ".npz"))
    for name, m in meta.items():
        path = str(tmp_path / (name + ".bin"))
        ggjt.write_synth_slice(path, ggjt.SHAPES[m["shape"]], m["layers"][0], m["layers"][1], m["wtype"], seed=0)
        sl = capi.Slice(path, 0, 512)
        for i in range(len(m["schedule"])):
            y = sl.forward(gold["%s/x%d" % (name, i)])
            assert (_bits(y) == _bits(gold["%s/y%d" % (name, i)])).all(), (name, i)
        sl.close()


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
def test_q5_llm_module_and_extra_layers_match_reference_goldens(tmp_path, wtype):
    """`llm` module: a Q5 slice's hidden states, then the client side of a Q5 model whose n_embd is not a multiple of 256
    (tiny3b): tok_embeddings rows dequantised on the GPU, output.weight through the Q5 slice matmul, the greedy id."""
    from distributedllm_b200.compute_node.slices import import_llm
    llm = import_llm()
    nm = ggjt.TYPE_NAME[wtype]
    meta = json.load(open(os.path.join(GOLD, "slices_%s.json" % nm)))
    gold = np.load(os.path.join(GOLD, "slices_%s.npz" % nm))
    name = "tiny128_" + nm
    m = meta[name]
    path = str(tmp_path / "s.bin")
    ggjt.write_synth_slice(path, ggjt.SHAPES[m["shape"]], m["layers"][0], m["layers"][1], wtype, seed=0)
    assert llm.load_slice(path) == 0
    for i in range(len(m["schedule"])):
        out = np.array(llm.propagate_forward(gold["%s/x%d" % (name, i)].ravel().tolist()), np.float32)
        assert (_bits(out) == _bits(gold["%s/y%d" % (name, i)]).ravel()).all(), i
    assert llm.unload_slice() == 0

    g = np.load(os.path.join(GOLD, "extra_%s.npz" % nm))
    sh = ggjt.SHAPES["tiny3b"]
    extra = str(tmp_path / "extra.bin")
    ggjt.write_synth_extra(extra, sh, wtype, seed=0)
    assert ggjt.read_file(extra).tensors["output.weight"].ttype == wtype
    emb = np.array(llm.prepare_embeddings(extra, g["tokens"].tolist()), np.float32).reshape(-1, sh.n_embd)
    assert (_bits(emb) == _bits(g["emb"])).all()
    hid = g["hidden"]
    la = np.array(llm.get_logits(extra, hid.ravel().tolist(), True), np.float32).reshape(len(hid), -1)
    assert (_bits(la) == _bits(g["logits_all"])).all(), int((_bits(la) != _bits(g["logits_all"])).sum())
    for i, want in enumerate(g["next_ids"]):
        assert llm.get_next_token(extra, hid[:i + 1].ravel().tolist()) == int(want)


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
def test_q5_one_7b_layer_bit_exact(tmp_path, wtype):
    """One layer at LLaMA-7B shape (4096 / 11008): real tile counts and ring depths."""
    sh = ggjt.SHAPES["7b"]
    path = str(tmp_path / "l.bin")
    ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=2, wtype=wtype)
    bad, tot = _run_pair(path, [9, 1, 1, 1], sh)
    assert bad == 0, "%d of %d floats differ" % (bad, tot)


@pytest.mark.parametrize("wtype", Q5, ids=IDS)
def test_q5_two_gpu_pipeline_peer_folded(tmp_path, wtype):
    """Two ranks, the hand-off folded into the last matmul (EPI_RESID_SEND) with a Q5 slice."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_pipeline import WORKER
    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT, "tmp": str(tmp_path)})
    env = dict(os.environ, B200_PP_PEER="1", B200_PP_FOLD="1", B200_TEST_WTYPE=str(wtype))
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                          "--master-addr", "127.0.0.1", "--master-port", str(29551 + wtype), str(script)],
                         capture_output=True, text=True, timeout=600, env=env)
    assert "PIPELINE_OK" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
    assert "transport=peer" in out.stdout, out.stdout[-500:]
