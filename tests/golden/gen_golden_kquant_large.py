"""Generate the k-quant fixtures at LLaMA-13B, 30B and 65B shapes from the compiled reference (oracle/_ref, on the CPU,
no GPU needed):

  ref_digests_kquant_large.json  SHA-256 digests of the reference's float32 outputs (as in ref_digests_large.json)
    {13b,30b,65b}_q4_K_S, _q6_K  one layer from ggjt.write_kquant_slice on gen_golden_large.SCHEDULE
    {13b,30b,65b}_q4_K_M         two adjacent layers, the first all Q4_K, the second with Q6_K wv / w2 (use_more_bits at
                                 the shape's real layer count: 13B layers 6-7 of 40, 30B 8-9 of 60, 65B 11-12 of 80), so
                                 one slice holds both qkv packings (one launch, and wq|wk beside a separate wv launch)
    13b_q4_K_M_deep              the 13B Q4_K_M file at n_ctx 2048: 32-token calls to position 2000, single steps to 2047
    65b_q4_K_M_batch             the 65B Q4_K_M file with gen_golden_large's 12-session batch plan (ragged prompts, then
                                 batched steps); each session replayed on one RefSlice after clear_context
    {13b,30b,65b}_extra          ggjt.write_kquant_extra(..., "q4_K_M"): Q4_K tok_embeddings and a Q6_K output.weight
                                 of 32000 ids; embedding rows of 7 ids (0 and 31999 among them), the logits of every row
                                 of 1, 8, 9 and 13 hidden rows (gen_golden_vocab.hidden) and their first-maximum ids
  ref_kquant_types_deep.json     the per-tensor types the reference's `quantize q4_K_S / q4_K_M / q6_K` writes on F32
                                 models with small matrices and 40, 60 and 80 layers (LLaMA-13B / 30B / 65B depths, where
                                 n_layer / 8 and 7 n_layer / 8 round), for the full file and one `slice_model` cut

Every file is recorded with its sha256 (a writer change then shows up as a fixture mismatch, not as a kernel failure)
and every input comes from a seed stored next to its digests.  Running the script twice writes the same files byte for
byte.  It takes about a minute on 8 x86-64 cores (AVX2, 8 reference threads) and writes up to 1 GB (the two-layer 65B
Q4_K_M file) at a time to a temporary directory.

    python tests/golden/gen_golden_kquant_large.py      # needs a built oracle/_ref
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
from distributedllm_b200 import ggjt  # noqa: E402
from oracle import oracle  # noqa: E402
from gen_golden_large import (BATCH_PROMPTS, BATCH_SESSIONS, BATCH_STEPS, SCHEDULE, digest, ref_batch,  # noqa: E402
                              ref_schedule)
from gen_golden_vocab import file_sha256, hidden  # noqa: E402

OUT = os.path.join(HERE, "ref_digests_kquant_large.json")
OUT_TYPES = os.path.join(HERE, "ref_kquant_types_deep.json")
SEED = 5                                    # weight-file seed
N_CTX = 512
MIXES = ("q4_K_S", "q6_K", "q4_K_M")
# Q4_K_M: (all-Q4_K layer, the next layer, whose wv / w2 are Q6_K) at the shape's layer count
PAIRS = {"13b": (6, 7), "30b": (8, 9), "65b": (11, 12)}
DEEP_SCHEDULE = [32] * 62 + [16] + [1] * 48                 # 32-token calls to position 2000, steps to 2047
EXTRA_IDS = [0, 1, 255, 256, 12345, 31998, 31999]
EXTRA_ROWS = [1, 8, 9, 13]                                   # one lm_head column group, one past it, a ragged group
TYPE_DEPTHS = (40, 60, 80)
TYPE_MIXES = ("q4_K_S", "q4_K_M", "q6_K")


def layers_of(shape, mix):
    """The layer range [a, b] of a (shape, mix) weight file."""
    a, b = PAIRS[shape]
    return [a, b] if mix == "q4_K_M" else [a, a]


def write_layers(path, case):
    """The weight file of a layer case."""
    a, b = case["layers"]
    ggjt.write_kquant_slice(path, ggjt.SHAPES[case["shape"]], a, b, case["mix"], seed=case["seed"])


def write_extra(path, case):
    ggjt.write_kquant_extra(path, ggjt.SHAPES[case["shape"]], case["mix"], seed=case["seed"])


def write_case_file(path, case):
    (write_extra if case["kind"] == "extra" else write_layers)(path, case)


def file_key(case):
    """Cases with equal keys run on the same file."""
    return case["kind"] == "extra", case["shape"], case["mix"], tuple(case.get("layers", ())), case["seed"]


def case_list():
    """name -> case, every user of one weight file next to the others (65b_q4_K_M's users last among the layer files
    of 65B: the GPU tests' sweep of runtime switches follows on that file)."""
    cases = {}
    for shape in ("13b", "30b", "65b"):
        for mix in MIXES:
            nm = "%s_%s" % (shape, mix)
            base = {"shape": shape, "mix": mix, "layers": layers_of(shape, mix), "seed": SEED}
            cases[nm] = dict(base, kind="schedule", n_ctx=N_CTX, input_seed=400 + len(cases), schedule=SCHEDULE)
            if nm == "13b_q4_K_M":
                cases[nm + "_deep"] = dict(base, kind="schedule", n_ctx=2048, input_seed=400 + len(cases),
                                           schedule=DEEP_SCHEDULE)
            if nm == "65b_q4_K_M":
                cases[nm + "_batch"] = dict(base, kind="batch", n_ctx=N_CTX, input_seed=400 + len(cases),
                                            prompt_len=BATCH_PROMPTS, sessions=BATCH_SESSIONS, n_steps=BATCH_STEPS)
        sh = ggjt.SHAPES[shape]
        cases[shape + "_extra"] = {"kind": "extra", "shape": shape, "mix": "q4_K_M", "seed": SEED, "n_embd": sh.n_embd,
                                   "n_vocab": sh.n_vocab, "input_seed": 400 + len(cases), "rows": EXTRA_ROWS,
                                   "embed_ids": EXTRA_IDS}
    return cases


def ref_extra(path, case):
    """(per call the digests of every logit row, per call the first-maximum id of every row, the embedding digests)."""
    lib = oracle.ref_lib()
    logits, argmax = [], []
    for n in case["rows"]:
        x = hidden(case, n)
        y = oracle.ref_logits(path, x, case["n_vocab"], True)
        assert y.shape == (n, case["n_vocab"]) and np.isfinite(y).all()
        logits.append([digest(r) for r in y])
        argmax.append([int(np.argmax(r)) for r in y])
        assert lib.ref_next_token(path.encode(), x.ctypes.data, x.size) == argmax[-1][-1]
    emb = oracle.ref_embed(path, case["embed_ids"], case["n_embd"])
    return logits, argmax, [digest(r) for r in emb]


def gen_digests(tmp):
    threads = min(16, os.cpu_count() or 4)
    cases, path, have = case_list(), os.path.join(tmp, "w.bin"), None
    for name, case in cases.items():
        if file_key(case) != have:
            write_case_file(path, case)
            have, sha = file_key(case), file_sha256(path)
        case["file_sha256"] = sha
        if case["kind"] == "schedule":
            case["digests"] = [digest(y) for y in ref_schedule(path, case, threads)]
        elif case["kind"] == "batch":
            out_p, out_s = ref_batch(path, case, threads)
            case["prompt_digests"] = [digest(y) for y in out_p]
            case["step_digests"] = [[digest(y) for y in s] for s in out_s]
        else:
            case["logits"], case["argmax"], case["embed"] = ref_extra(path, case)
        print(name, flush=True)
    os.remove(path)
    with open(OUT, "w") as f:
        json.dump(cases, f, indent=1)
        f.write("\n")


def type_cut(n_layer):
    """The slice_model cut of a type case: across 7 n_layer / 8 (rounded down at 60 layers), where use_more_bits
    switches on for good."""
    c = 7 * n_layer // 8
    return [c - 3, c + 1]


def gen_types(tmp):
    types, cuts = {}, {}
    for n_layer in TYPE_DEPTHS:
        label = "deep%d" % n_layer
        full = os.path.join(tmp, "f32.bin")
        ggjt.write_synth_full(full, ggjt.ModelShape(512, 256, 256, 4, n_layer), ggjt.T_F32, seed=0)
        a, b = cuts[label] = type_cut(n_layer)
        for mix in TYPE_MIXES:
            fq, sl = os.path.join(tmp, "q.bin"), os.path.join(tmp, "s.bin")
            subprocess.run([os.path.join(oracle.REF_DIR, "quantize"), full, fq, mix], check=True, capture_output=True)
            q = ggjt.read_file(fq)
            types["%s/%s/full" % (label, mix)] = {n: ggjt.TYPE_NAME[t.ttype] for n, t in q.tensors.items()}
            subprocess.run([os.path.join(oracle.REF_DIR, "slice_model"), "slice", fq, str(a), str(b), sl], check=True,
                           capture_output=True)
            s = ggjt.read_file(sl)
            types["%s/%s/slice_%d_%d" % (label, mix, a, b)] = {n: ggjt.TYPE_NAME[t.ttype] for n, t in s.tensors.items()}
            os.remove(fq)
            os.remove(sl)
        os.remove(full)
    with open(OUT_TYPES, "w") as f:
        json.dump({"n_layer": {"deep%d" % n: n for n in TYPE_DEPTHS}, "cuts": cuts, "types": types}, f, indent=1,
                  sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    tmp = tempfile.mkdtemp()
    try:
        gen_types(tmp)
        gen_digests(tmp)
    finally:
        shutil.rmtree(tmp)
    print("fixtures written to", OUT, "and", OUT_TYPES)
