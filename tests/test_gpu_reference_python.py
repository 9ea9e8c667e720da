"""GPU: the REFERENCE's own Python host code running on this repo's `llm` module -- the zero-edit drop-in claim of
INTEGRATION.md section 1, on real hardware.

`oracle/_ref/py/distllm` is a build output of oracle/Makefile (the reference's distllm/*.py copied next to the compiled
reference; git-ignored, the tests skip without it -- nothing here reads the reference checkout).  With
`distributedllm_b200/` first on sys.path, `import llm` inside the reference's code binds to csrc/llm_module.cpp:

  * distllm.compute_node.slices.GGMLSlice (slices.py:74-91)          llm.load_slice / propagate_forward / clear_context
  * distllm.compute_node.serve + tcp_handler + routes + uploads       the reference's node server, unmodified
  * distllm.control_center.Connection (control_center.py:88-254)      push_slice, load_slice, propagate_forward RPCs
  * distllm.cli_api.common.DistributedLLM (common.py:89-154)          tokenize -> embed -> relay -> logits -> sample
Token ids / hidden states are compared with the CPU oracle (bit-exact hidden states make ids an equality).
"""
import os
import sys
import threading

import numpy as np
import pytest

from distributedllm_b200 import ggjt

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_PY = os.path.join(ROOT, "oracle", "_ref", "py")
needs_ref_py = pytest.mark.skipif(not os.path.isfile(os.path.join(REF_PY, "distllm", "control_center.py")),
                                  reason="reference Python snapshot (oracle/_ref/py) not shipped")


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def ref_py():
    """Our `llm` first, then the reference's package: the order the reference's Dockerfile sets with PYTHONPATH=/libs."""
    from distributedllm_b200.compute_node.slices import import_llm
    llm = import_llm()
    assert "distributedllm_b200" in os.path.abspath(llm.__file__)
    if REF_PY not in sys.path:
        sys.path.append(REF_PY)
    import distllm  # noqa: F401
    assert os.path.abspath(distllm.__file__).startswith(REF_PY)
    return llm


@needs_ref_py
def test_reference_ggmlslice_runs_on_the_b200_llm_module(ref_py, tmp_models):
    from distllm.compute_node.slices import GGMLSlice, Tensor
    from oracle import oracle
    sh = ggjt.SHAPES["tiny128"]
    path = tmp_models("tiny128", ggjt.T_Q4_0, 0, 2, seed=12)
    cpu = oracle.PortSlice(path, 512)
    sl = GGMLSlice(path)                                     # the reference's class, our llm.load_slice
    try:
        rng = np.random.default_rng(4)
        for n in (5, 1, 1):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            out = sl(Tensor((1, x.size), x.ravel().tolist()))
            assert out.shape == (1, x.size) and isinstance(out.values, list)
            assert (_bits(np.array(out.values, np.float32)) == _bits(cpu.forward(x)).ravel()).all()
        sl.clear_context()
        cpu.clear_context()
        x = rng.standard_normal((2, sh.n_embd), dtype=np.float32)
        out = sl(Tensor((1, x.size), x.ravel().tolist()))
        assert (_bits(np.array(out.values, np.float32)) == _bits(cpu.forward(x)).ravel()).all()
    finally:
        ref_py.unload_slice()


@needs_ref_py
def test_reference_node_and_client_generate_on_the_b200(ref_py, tmp_path, monkeypatch, capsys):
    """The reference's node server AND the reference's client, both unmodified; only `llm` is ours."""
    llm = ref_py
    from distllm.cli_api.common import DistributedLLM
    from distllm.compute_node import serve as rserve
    from distllm.compute_node import uploads as ruploads
    from distllm.control_center import Connection
    from oracle import oracle
    sh = ggjt.SHAPES["tiny128"]
    full = str(tmp_path / "full.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_Q4_0, seed=2)
    sl, extra = str(tmp_path / "slice.bin"), str(tmp_path / "extra.bin")
    ggjt.slice_model(full, sl, 0, sh.n_layer - 1)
    ggjt.extract_extra_layers(full, extra)
    ruploads.upload_registry.root = str(tmp_path / "uploads")          # serve.run_server does this for a fresh dir
    srv = rserve.ThreadingTCPServer(("127.0.0.1", 0), rserve.MyTCPHandler)
    threading.Thread(target=srv.serve_forever, daemon=True).start()
    try:
        addr = ("127.0.0.1", srv.server_address[1])
        conn = Connection(addr)
        with open(sl, "rb") as f:
            res = conn.push_slice(f, "tiny128", {"layer_from": 0, "layer_to": sh.n_layer - 1})
        name = res["file_name"] if isinstance(res, dict) else res
        conn.load_slice(name)
        assert conn.get_status()["status"] == "up"
        prompt, steps = "the the a in", 10
        np.random.seed(0)
        model = DistributedLLM([addr], extra)
        # T = 0 -> logits / 1e-5 -> softmax -> np.random.choice: argmax unless two logits tie within ~1e-4 (common.py:64-86)
        got = list(model.generate(prompt, max_steps=steps, temperature=0.0, repeat_penalty=1.0))
        cpu = oracle.PortSlice(sl, 512)
        toks = llm.tokenize_prompt(extra, prompt)
        want = []
        for _ in range(steps):
            emb = np.array(llm.prepare_embeddings(extra, toks), np.float32).reshape(len(toks), -1)
            t = llm.get_next_token(extra, cpu.forward(emb).ravel().tolist())
            want.append(llm.decode_token(extra, t))
            toks = [t]
        assert got == want
        ppl = model.perplexity("the the a in the")
        assert np.isfinite(ppl) and ppl > 1
    finally:
        srv.shutdown()
        srv.server_close()
        llm.unload_slice()
