"""CPU: the C restatement's lm_head and embedding rows at vocabulary sizes that are not a multiple of 32, against the
reference's digests (tests/golden/ref_digests_vocab.json, written by tests/golden/gen_golden_vocab.py).

Each case regenerates its extra-layers file and first checks the file's sha256, so a change in the writers shows up as
a fixture mismatch rather than as a restatement (or, in tests/test_gpu_vocab_sizes.py, a kernel) failure.  Where the
reference is built (oracle/_ref), one more case runs it live on a file its own `quantize` and `slice_model` wrote."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_cases as ec
from distributedllm_b200 import ggjt
from oracle import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import gen_golden_vocab as vocab_ref  # noqa: E402

CASES = json.load(open(os.path.join(HERE, "golden", "ref_digests_vocab.json")))


def test_fixture_covers_the_cases():
    assert sorted(CASES) == sorted(vocab_ref.case_list())
    for name, case in CASES.items():
        assert [len(d) for d in case["logits"]] == case["rows"], name
        assert case["embed_ids"] == vocab_ref.tail_ids(case["n_vocab"]), name
        assert case["n_vocab"] % 32 != 0, name


def port_embed(path: str, ids) -> np.ndarray:
    """Embedding rows as get_rows computes them: the row dequantised (dequantize_row_*), F16 widened."""
    return ec.dequant_rows(ggjt.read_file(path, sliced=True), "tok_embeddings.weight", ids)


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_reproduces_the_reference(tmp_path, name):
    case = CASES[name]
    path = str(tmp_path / "extra.bin")
    vocab_ref.write_extra(path, case)
    assert vocab_ref.file_sha256(path) == case["file_sha256"], "the writer changed: regenerate the fixture"
    for n, want, want_max in zip(case["rows"], case["logits"], case["argmax"]):
        y = ec.port_logits(path, vocab_ref.hidden(case, n))
        assert y.shape == (n, case["n_vocab"])
        got = [vocab_ref.digest(r) for r in y]
        assert got == want, (name, n, [i for i in range(n) if got[i] != want[i]])
        assert [vocab_ref.first_max(r) for r in y] == want_max, (name, n)
    emb = port_embed(path, case["embed_ids"])
    assert np.isfinite(emb).all()
    if case["embed"] is not None:                     # None: the reference cannot embed this type (gen_golden_vocab)
        assert [vocab_ref.digest(r) for r in emb] == case["embed"], name


@pytest.mark.skipif(not oracle.have_ref(), reason="needs the compiled reference (oracle/_ref)")
def test_reference_tools_file_at_1031_ids(tmp_path):
    """The reference's own `quantize q4_0` and `slice_model extra_layers` on a 1031-id model, whose logits and embedding
    rows the restatement reproduces bit for bit.  `quantize` gives output.weight Q6_K only when both of its dimensions
    are multiples of 256 (llama.cpp:2523-2528), so at a ragged vocabulary the lm_head stays in the file's base type."""
    sh = ggjt.ModelShape(1031, 256, 32, 4, 1)
    full, fq, extra = (str(tmp_path / n) for n in ("full.bin", "q4.bin", "extra.bin"))
    ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=3)
    subprocess.run([os.path.join(oracle.REF_DIR, "quantize"), full, fq, "q4_0"], check=True, capture_output=True)
    subprocess.run([os.path.join(oracle.REF_DIR, "slice_model"), "extra_layers", fq, extra], check=True,
                   capture_output=True)
    f = ggjt.read_file(extra, sliced=True)
    assert f.hparams.n_vocab == 1031
    assert f.tensors["output.weight"].ttype == ggjt.T_Q4_0
    assert f.tensors["tok_embeddings.weight"].ttype == ggjt.T_Q4_0
    rng = np.random.default_rng(4)
    for n in (1, 9, 13):
        x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
        if n > 1:
            x[1] = 0.0
            x[-1] *= np.float32(30.0)
        ref = oracle.ref_logits(extra, x, 1031, True)
        got = ec.port_logits(extra, x)
        assert (got.view(np.uint32) == ref.view(np.uint32)).all(), n
    ids = vocab_ref.tail_ids(1031)
    ref = oracle.ref_embed(extra, ids, sh.n_embd)
    assert np.isfinite(ref).all()
    assert (port_embed(extra, ids).view(np.uint32) == ref.view(np.uint32)).all()
