"""Generate the k-quant (Q4_K / Q6_K) golden fixtures from the REFERENCE ITSELF (run in the build container only, next to
gen_golden.py; it writes only these files):

  slices_kquant.npz / .json  hidden states of oracle/_ref on writer-made Q4_K_S / Q4_K_M / Q6_K slices of tinyk and
                 tinyk128 (layers 2-4 of 8: a slice starting mid-model that, for Q4_K_M, holds layers whose wv / w2 are
                 Q6_K and layers whose are not), prefill then decode
  extra_kquant.npz  reference get_inputs / get_llm_output / greedy ids on a tinyk128 extra-layers file with Q4_K
                 tok_embeddings and a Q6_K output.weight
  ref_digests_kquant.json  SHA-256 digests of the reference's hidden states on one LLaMA-7B-shape layer per mix (a Q4_K_M
                 layer whose wv / w2 are Q6_K and one whose are not), schedule CASES_7B
  ref_kquant_types.json  the per-tensor types the reference `quantize` writes for q4_K_S / q4_K_M / q6_K on full F32
                 models of 8 (tinyk128) and 32 (the 7B layer count) layers, and the types `slice_model` keeps in a slice

    python tests/golden/gen_golden_kquant.py      # needs /root/reference and a built oracle/_ref
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from distributedllm_b200 import ggjt  # noqa: E402
from oracle import oracle  # noqa: E402

MIXES = ("q4_K_S", "q4_K_M", "q6_K")
SCHEDULE = [9, 1, 1, 3, 1]
CASES = [("%s_%s" % (shape, mix), shape, mix, (2, 4)) for shape in ("tinyk", "tinyk128") for mix in MIXES]
# one 7B-shape layer: (mix, layer); written with seed 2, inputs from default_rng(1), calls [9, 1, 1, 1]
CASES_7B = [("q4_K_S", 4), ("q4_K_M", 0), ("q4_K_M", 4), ("q6_K", 4)]
SCHEDULE_7B = [9, 1, 1, 1]
# a 7B-deep model with small matrices: the tool's choices depend on the layer count only
DEEP = ggjt.ModelShape(512, 256, 256, 4, 32)


def gen_slices(tmp):
    out, meta = {}, {}
    for name, shape, mix, (a, b) in CASES:
        sh = ggjt.SHAPES[shape]
        path = os.path.join(tmp, name + ".bin")
        ggjt.write_kquant_slice(path, sh, a, b, mix, seed=0)
        meta[name] = {"shape": shape, "mix": mix, "layers": [a, b], "schedule": SCHEDULE,
                      "file_sha256": hashlib.sha256(open(path, "rb").read()).hexdigest()}
        rng = np.random.default_rng(1234)
        ref = oracle.RefSlice(path, n_threads=3, n_ctx=512)
        for i, n in enumerate(SCHEDULE):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            out["%s/x%d" % (name, i)] = x
            out["%s/y%d" % (name, i)] = ref.forward(x)
        ref.close()
    np.savez_compressed(os.path.join(HERE, "slices_kquant.npz"), **out)
    json.dump(meta, open(os.path.join(HERE, "slices_kquant.json"), "w"), indent=1)


def gen_extra(tmp):
    sh = ggjt.SHAPES["tinyk128"]
    extra = os.path.join(tmp, "extra_kquant.bin")
    ggjt.write_kquant_extra(extra, sh, "q4_K_M", seed=0)
    toks = np.array([1, 5, 300, 44, 511, 0, 77], np.int32)
    h = np.random.default_rng(7).standard_normal((5, sh.n_embd), dtype=np.float32)
    ids = [oracle.ref_lib().ref_next_token(extra.encode(), np.ascontiguousarray(h[:i + 1]).ctypes.data, (i + 1) * sh.n_embd)
           for i in range(5)]
    np.savez_compressed(os.path.join(HERE, "extra_kquant.npz"), tokens=toks, emb=oracle.ref_embed(extra, toks, sh.n_embd),
                        hidden=h, logits_all=oracle.ref_logits(extra, h, sh.n_vocab, True), next_ids=np.array(ids, np.int32),
                        file_sha256=np.frombuffer(hashlib.sha256(open(extra, "rb").read()).digest(), np.uint8))


def digest(a) -> str:
    """SHA-256 of the float32 bit patterns: comparing digests is comparing every bit of the array."""
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def gen_7b(tmp):
    sh = ggjt.SHAPES["7b"]
    out = {}
    for mix, layer in CASES_7B:
        path = os.path.join(tmp, "7b.bin")
        ggjt.write_kquant_slice(path, sh, layer, layer, mix, seed=2)
        ref, rng = oracle.RefSlice(path, n_threads=8, n_ctx=512), np.random.default_rng(1)
        out["%s_layer%d" % (mix, layer)] = [digest(ref.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32)))
                                            for n in SCHEDULE_7B]
        ref.close()
    json.dump({"schedule": SCHEDULE_7B, "seed": 2, "digests": out}, open(os.path.join(HERE, "ref_digests_kquant.json"), "w"), indent=1)


def gen_types(tmp):
    types = {}
    for label, sh in (("tinyk128", ggjt.SHAPES["tinyk128"]), ("deep32", DEEP)):
        full = os.path.join(tmp, "f32_%s.bin" % label)
        ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=0)
        for mix in MIXES:
            fq, sl = os.path.join(tmp, "q.bin"), os.path.join(tmp, "s.bin")
            subprocess.run([os.path.join(oracle.REF_DIR, "quantize"), full, fq, mix], check=True, capture_output=True)
            q = ggjt.read_file(fq)
            types["%s/%s/full" % (label, mix)] = {n: ggjt.TYPE_NAME[t.ttype] for n, t in q.tensors.items()}
            subprocess.run([os.path.join(oracle.REF_DIR, "slice_model"), "slice", fq, "2", "4", sl], check=True, capture_output=True)
            s = ggjt.read_file(sl)
            types["%s/%s/slice_2_4" % (label, mix)] = {n: ggjt.TYPE_NAME[t.ttype] for n, t in s.tensors.items()}
    json.dump({"n_layer": {"tinyk128": ggjt.SHAPES["tinyk128"].n_layer, "deep32": DEEP.n_layer}, "types": types},
              open(os.path.join(HERE, "ref_kquant_types.json"), "w"), indent=1, sort_keys=True)


if __name__ == "__main__":
    tmp = tempfile.mkdtemp()
    gen_slices(tmp)
    gen_extra(tmp)
    gen_7b(tmp)
    gen_types(tmp)
    print("k-quant golden fixtures written to", HERE)
