"""Generate tests/golden/ref_digests_large.json: the reference's hidden states on one-layer LLaMA-30B and LLaMA-65B
slices, kept as SHA-256 digests of their float32 bits (as in ref_digests.json).  It runs the compiled reference
(oracle/_ref, RefSlice, calls of at most 32 tokens) on the CPU and needs no GPU.

  cases    one layer of 30b and 65b for every weight type the runtime loads (Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 from
           ggjt.write_fast_q4_slice, F16 from ggjt.write_fast_f16_slice) on the call schedule SCHEDULE; a 30b Q4_0 layer
           prefilled to position 480 in 32-token chunks, then decoded one token at a time to position 512
  batches  65b Q4_0 and Q8_0 with 12 sessions: ragged prompts, then batched steps (one token of every session).  Each
           session's reference is that session's whole sequence replayed on one RefSlice (clear, prompt, steps), so
           one copy of the weights serves all twelve.

Every input comes from a seed stored next to its digests, so tests/test_gpu_large_shapes.py can replay it.  Running
the script twice writes the same file byte for byte.  It takes about 25 s on 8 x86-64 cores (AVX2, 16 reference
threads) and writes up to 1.6 GB (the 65b F16 layer) at a time to a temporary directory.

    python tests/golden/gen_golden_large.py          # needs a built oracle/_ref
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

OUT = os.path.join(HERE, "ref_digests_large.json")
SEED = 3                                    # weight-file seed, one file per (shape, weight type)
N_CTX = 512
# At 65B, 9 is the smallest call whose w2 (256 tiles) takes 8 columns per CTA on a 132-SM H100; 5 takes 4 and 2 takes 2
SCHEDULE = [32, 9, 17, 5, 1, 1, 1, 1, 1, 1, 1, 1]
WTYPES = [ggjt.T_Q4_0, ggjt.T_Q4_1, ggjt.T_Q5_0, ggjt.T_Q5_1, ggjt.T_Q8_0, ggjt.T_F16]
BATCH_PROMPTS = [3, 17, 1, 32, 9, 5, 26, 2, 11, 8, 20, 14]
BATCH_SESSIONS = [4, 0, 11, 7, 2, 9, 1, 10, 5, 3, 8, 6]     # the batch's column b steps session BATCH_SESSIONS[b]
BATCH_STEPS = 3


def digest(a) -> str:
    """SHA-256 of the float32 bit patterns: comparing digests is comparing every bit of the array."""
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def write_slice(path, shape, wtype, seed=SEED):
    """The one-layer file every case of (shape, wtype) runs on."""
    sh = ggjt.SHAPES[shape]
    if wtype == ggjt.T_F16:
        ggjt.write_fast_f16_slice(path, sh, 0, 0, seed=seed)
    else:
        ggjt.write_fast_q4_slice(path, sh, 0, 0, seed=seed, wtype=wtype)


def case_inputs(case):
    """The inputs of a schedule case, call by call."""
    rng = np.random.default_rng(case["input_seed"])
    e = ggjt.SHAPES[case["shape"]].n_embd
    return [rng.standard_normal((n, e), dtype=np.float32) for n in case["schedule"]]


def batch_inputs(case):
    """(prompts per column, steps as [n_columns][n_embd]) of a batch case; column b belongs to session sessions[b]."""
    rng = np.random.default_rng(case["input_seed"])
    e = ggjt.SHAPES[case["shape"]].n_embd
    prompts = [rng.standard_normal((n, e), dtype=np.float32) for n in case["prompt_len"]]
    steps = [rng.standard_normal((len(case["sessions"]), e), dtype=np.float32) for _ in range(case["n_steps"])]
    return prompts, steps


def case_list():
    """name -> case, in the order the GPU tests replay them (all users of one weight file next to each other)."""
    cases = {}
    for shape in ("30b", "65b"):
        # 65b Q4_0 goes last: the GPU tests' sweep of runtime switches follows on its file
        for wt in WTYPES if shape == "30b" else WTYPES[1:] + WTYPES[:1]:
            nm = "%s_%s" % (shape, ggjt.TYPE_NAME[wt])
            cases[nm] = {"kind": "schedule", "shape": shape, "wtype": wt, "seed": SEED, "n_ctx": N_CTX,
                         "input_seed": len(cases) + 100, "schedule": SCHEDULE}
            if nm == "30b_q4_0":
                cases["30b_q4_0_deep"] = {"kind": "schedule", "shape": shape, "wtype": wt, "seed": SEED, "n_ctx": N_CTX,
                                          "input_seed": 200, "schedule": [32] * 15 + [1] * 32}
            if shape == "65b" and wt in (ggjt.T_Q4_0, ggjt.T_Q8_0):
                cases[nm + "_batch"] = {"kind": "batch", "shape": shape, "wtype": wt, "seed": SEED, "n_ctx": N_CTX,
                                        "input_seed": 300 + wt, "prompt_len": BATCH_PROMPTS, "sessions": BATCH_SESSIONS,
                                        "n_steps": BATCH_STEPS}
    return cases


def ref_schedule(path, case, threads):
    ref = oracle.RefSlice(path, threads, case["n_ctx"])
    try:
        return [ref.forward(x) for x in case_inputs(case)]
    finally:
        ref.close()


def ref_batch(path, case, threads):
    """(prompt outputs per column, step outputs [step][column]) from one RefSlice replaying each session in turn."""
    prompts, steps = batch_inputs(case)
    ref = oracle.RefSlice(path, threads, case["n_ctx"])
    out_p, out_s = [], [[None] * len(prompts) for _ in steps]
    try:
        for b in range(len(prompts)):
            ref.clear_context()
            out_p.append(ref.forward(prompts[b]))
            for i, x in enumerate(steps):
                out_s[i][b] = ref.forward(x[b:b + 1])[0]
    finally:
        ref.close()
    return out_p, out_s


def gen(tmp):
    threads = min(16, os.cpu_count() or 4)
    cases, path, have = case_list(), os.path.join(tmp, "layer.bin"), None
    for name, case in cases.items():
        key = (case["shape"], case["wtype"], case["seed"])
        if key != have:
            write_slice(path, *key)
            have = key
        if case["kind"] == "schedule":
            case["digests"] = [digest(y) for y in ref_schedule(path, case, threads)]
        else:
            out_p, out_s = ref_batch(path, case, threads)
            case["prompt_digests"] = [digest(y) for y in out_p]
            case["step_digests"] = [[digest(y) for y in s] for s in out_s]
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
