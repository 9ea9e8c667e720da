"""Generate tests/golden/ref_digests_vocab.json: the reference's logits and embeddings on extra-layers files whose
vocabulary is not a multiple of 32, kept as SHA-256 digests of their float32 bits (as in ref_digests.json).  It runs the
compiled reference (oracle/_ref: get_llm_output with all logits, get_inputs) on the CPU and needs no GPU.

  cases    n_embd 256 at V = 1031, 32001 and 49953 (Chinese-LLaMA's 49953 ids, a fine-tune's added pad token, and a
           size whose lm_head, bitmaps and sampler chunks all end part-way), with output.weight
             Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, F16   ggjt.write_synth_extra (tok_embeddings in the same type)
             Q6_K                                ggjt.write_kquant_extra(..., "q4_K_M"): Q4_K tok_embeddings
           and at LLaMA-7B shape (n_embd 4096, V = 32001) one Q6_K and one F16 file.
  calls    1, 3, 8, 9, 13 and 65 hidden rows (8 is one lm_head column group, 64 one scoring block); the 7B files
           take 1, 8 and 13.  Rows are Gaussian; from 3 rows on, the middle one is all zero and the last one is x30.
  record   the file's sha256 (a writer change then shows up as a fixture mismatch, not as a kernel failure); per call
           and row the digest of the logits and their argmax (first maximum, sample_next_token's rule); the digests
           of the embedding rows of ids 0, 1, 32*floor(V/32) - 1, 32*floor(V/32), V - 2 and V - 1
           (not for Q8_0 and F16 tok_embeddings, which the reference cannot embed: see ref_can_embed).

Running the script twice writes the same file byte for byte.  It takes about a minute on 8 x86-64 cores and writes up to
530 MB (the 7B F16 file) at a time to a temporary directory.

    python tests/golden/gen_golden_vocab.py          # needs a built oracle/_ref
"""
import hashlib
import json
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from distributedllm_b200 import ggjt  # noqa: E402
from oracle import oracle  # noqa: E402

OUT = os.path.join(HERE, "ref_digests_vocab.json")
VOCABS = (1031, 32001, 49953)
TYPES = ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "f16", "q6_K")   # output.weight
ROWS = (1, 3, 8, 9, 13, 65)
ROWS_7B = (1, 8, 13)
SEED = 13                                   # weight-file seed


def digest(a) -> str:
    """SHA-256 of the float32 bit patterns: comparing digests is comparing every bit of the array."""
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def file_sha256(path: str) -> str:
    h = hashlib.sha256()
    with open(path, "rb") as f:
        for b in iter(lambda: f.read(1 << 24), b""):
            h.update(b)
    return h.hexdigest()


def shape_of(case) -> ggjt.ModelShape:
    if case["n_embd"] == 4096:
        return ggjt.ModelShape(case["n_vocab"], 4096, 256, 32, 32)
    return ggjt.ModelShape(case["n_vocab"], 256, 256, 4, 8)


def write_extra(path: str, case) -> None:
    """The extra-layers file of a case."""
    sh = shape_of(case)
    if case["out"] == "q6_K":
        ggjt.write_kquant_extra(path, sh, "q4_K_M", seed=case["seed"])
    else:
        wt = {v: k for k, v in ggjt.TYPE_NAME.items()}[case["out"]]
        ggjt.write_synth_extra(path, sh, wt, seed=case["seed"])


def tail_ids(n_vocab: int) -> list:
    """The ids around the last partial 32-id word and the end of the vocabulary."""
    w = n_vocab // 32 * 32
    return [0, 1, w - 1, w, n_vocab - 2, n_vocab - 1]


def hidden(case, n: int) -> np.ndarray:
    """The n hidden rows of a call: Gaussian; from 3 rows on the middle one all zero and the last one x30."""
    x = np.random.default_rng([case["input_seed"], n]).standard_normal((n, case["n_embd"]), dtype=np.float32)
    if n >= 3:
        x[n // 2] = 0.0
        x[n - 1] *= np.float32(30.0)
    return x


def ref_can_embed(case) -> bool:
    """Whether the reference's get_inputs can hold the case's tok_embeddings (at most one byte per weight)."""
    return case["out"] not in ("q8_0", "f16")


def first_max(row) -> int:
    """sample_next_token's argmax: the first id whose logit beats every earlier one, starting from -1e12."""
    return int(np.argmax(row))


def case_list():
    cases = {}
    for v in VOCABS:
        for t in TYPES:
            cases["%s_%d" % (t, v)] = {"n_embd": 256, "n_vocab": v, "out": t, "seed": SEED,
                                       "input_seed": 500 + len(cases), "rows": list(ROWS)}
    for t in ("q6_K", "f16"):
        cases["7b_%s_32001" % t] = {"n_embd": 4096, "n_vocab": 32001, "out": t, "seed": SEED,
                                    "input_seed": 500 + len(cases), "rows": list(ROWS_7B)}
    return cases


def gen(tmp):
    cases, path = case_list(), os.path.join(tmp, "extra.bin")
    lib = oracle.ref_lib()
    for name, case in cases.items():
        write_extra(path, case)
        case["file_sha256"] = file_sha256(path)
        v, e = case["n_vocab"], case["n_embd"]
        case["logits"], case["argmax"] = [], []
        for n in case["rows"]:
            x = hidden(case, n)
            y = oracle.ref_logits(path, x, v, True)
            assert y.shape == (n, v) and np.isfinite(y).all(), name
            case["logits"].append([digest(r) for r in y])
            case["argmax"].append([first_max(r) for r in y])
            assert lib.ref_next_token(path.encode(), x.ctypes.data, x.size) == case["argmax"][-1][-1], name
        ids = tail_ids(v)
        case["embed_ids"] = ids
        # get_inputs sizes its weight arena at one byte per weight (tensor_processor.cpp:1725): Q8_0 and F16
        # tok_embeddings do not fit it, and the reference aborts
        case["embed"] = [digest(r) for r in oracle.ref_embed(path, ids, e)] if ref_can_embed(case) else None
        print(name, flush=True)
    os.remove(path)
    with open(OUT, "w") as f:
        json.dump(cases, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    tmp = tempfile.mkdtemp()
    try:
        gen(tmp)
    finally:
        shutil.rmtree(tmp)
    print("digests written to", OUT)
