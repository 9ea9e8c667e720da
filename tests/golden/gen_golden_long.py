"""Generate tests/golden/ref_digests_long.json: the reference's hidden states on one-layer LLaMA-7B and LLaMA-13B slices
at n_ctx 2048, kept as SHA-256 digests of their float32 bits (as in ref_digests.json).  It runs the compiled reference
(oracle/_ref, RefSlice(path, threads, 2048), calls of at most 32 tokens) on the CPU and needs no GPU.

  cases    7b_q4_0   32 heads (ggjt.write_fast_q4_slice)
           13b_q4_0  40 heads: on an H100 SXM the single-token attention reads its exp table through L2 at this width
           7b_f16    ggjt.write_fast_f16_slice: tests/test_gpu_full_size.py's config 4 layer
           each on SCHEDULE: a chunked prefill that crosses position 512 with single tokens at 511 and 512, ends at
           position 2000, then single-token steps up to the last position, 2047.  Every call has a digest.

The reference runs cleanly over the whole of n_ctx 2048: its scratch and eval budgets are sized for 2048-token contexts,
and a one-layer slice's KV cache is 1/32 (7B) or 1/40 (13B) of the full model's.

Every input comes from a seed stored next to its digests, so the GPU tests can replay it.  Running the script twice
writes the same file byte for byte.  It takes about a minute on 8 x86-64 cores (AVX2) and writes up to 400 MB (the 7B
F16 layer) at a time to a temporary directory.

    python tests/golden/gen_golden_long.py           # needs a built oracle/_ref
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

OUT = os.path.join(HERE, "ref_digests_long.json")
SEED = 7                                    # weight-file seed
N_CTX = 2048
# 480 in chunks, 31 to position 511, single tokens at 511 and 512, 31 to 544, chunks to 2000, then steps to 2047
SCHEDULE = [32] * 15 + [31, 1, 1, 31] + [32] * 45 + [16] + [1] * 48
assert sum(SCHEDULE) == N_CTX and max(SCHEDULE) <= oracle.RefSlice.MAX_CHUNK


def digest(a) -> str:
    """SHA-256 of the float32 bit patterns: comparing digests is comparing every bit of the array."""
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def write_slice(path, shape, wtype, seed=SEED):
    """The one-layer file of a case."""
    sh = ggjt.SHAPES[shape]
    if wtype == ggjt.T_F16:
        ggjt.write_fast_f16_slice(path, sh, 0, 0, seed=seed)
    else:
        ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=seed, wtype=wtype)


def case_inputs(case):
    """The inputs of a case, call by call."""
    rng = np.random.default_rng(case["input_seed"])
    e = ggjt.SHAPES[case["shape"]].n_embd
    return [rng.standard_normal((n, e), dtype=np.float32) for n in case["schedule"]]


def case_list():
    cases = {}
    for shape, wt in (("7b", ggjt.T_Q4_0), ("13b", ggjt.T_Q4_0), ("7b", ggjt.T_F16)):
        nm = "%s_%s" % (shape, ggjt.TYPE_NAME[wt])
        cases[nm] = {"shape": shape, "wtype": wt, "seed": SEED, "n_ctx": N_CTX, "input_seed": 400 + len(cases),
                     "schedule": SCHEDULE}
    return cases


def gen(tmp):
    threads = min(16, os.cpu_count() or 4)
    cases, path = case_list(), os.path.join(tmp, "layer.bin")
    for name, case in cases.items():
        write_slice(path, case["shape"], case["wtype"], case["seed"])
        ref = oracle.RefSlice(path, threads, case["n_ctx"])
        try:
            outs = [ref.forward(x) for x in case_inputs(case)]
            assert all(np.isfinite(y).all() for y in outs), name
            case["digests"] = [digest(y) for y in outs]
        finally:
            ref.close()
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
