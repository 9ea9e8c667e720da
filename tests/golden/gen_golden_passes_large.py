"""Generate tests/golden/ref_digests_passes_large.json: the reference's hidden states for the runtime's multi-session
passes (batched steps, mixed passes, decode rows) at LLaMA-13B, 30B and 65B layer shapes, kept as SHA-256 digests of
their float32 bits (as in ref_digests_large.json).  It runs the compiled reference (oracle/_ref, RefSlice) on the CPU
and needs no GPU.

  cases     65B: one layer of Q4_0, Q4_1, Q5_0, Q5_1, Q8_0 and F16 (gen_golden_large.write_slice) and the one-layer
            Q4_K_S / Q6_K and two-layer Q4_K_M files of gen_golden_kquant_large (Q6_K wv / w2 in the second layer);
            30B and 13B: Q4_0, Q5_1, F16 and Q4_K_M.  Every case loads its file with n_ctx 1024 and 12 sessions and runs
            the operations of ops() on it, with inputs drawn in operation order from the case's input_seed.
  13b_generate  the 13B Q4_K_M two-layer file with the 13B extra layers of the k-quant fixture: the reference's own
            greedy loop (ref_embed, RefSlice, ref_logits, first maximum) for 3 prompts over 24 steps.

ops() in words (sessions 0..11; A = 11, B = 6):
  1. a mixed pass of all 12 sessions' prompts, ragged counts 1..32 in a permuted session order (each segment within the
     attention's staged window of 512 positions: the query-tiled kernel over the pass's tile table);
  2. three batched steps over all 12 sessions in permuted orders (8 + 4 columns), then one over 9 of them (8 + 1);
  3. A pushed to position 515 and B to 500 by session_forward calls of up to 32 rows;
  4. a mixed pass of a single token, A's 29 rows past position 512 (per-query cluster kernel, per-row lengths; the
     segment ends at 544, a multiple of 32, where the row length moves the float / double split of the V sum), 20 rows
     of session 0 (query-tiled) and another single token (the fused single-token kernel);
  5. decode rows: B 24 rows across position 512, A 16 rows (the speculative maximum), session 2 40 rows near the start;
  6. a batched step over all 12 sessions, now at positions 6 to 560.

A session's output depends only on its own calls, so one RefSlice replays each session in turn (clear, then that
session's share of every operation): a mixed-pass segment is one call of its rows (at most RefSlice.MAX_CHUNK = 32), a
batched-step column one one-row call, N decode rows N one-row calls.  One digest is stored per (operation, session),
and every file's sha256 next to its case.  Running the script twice writes the same file byte for byte.  It takes
about 5 minutes on 8 x86-64 cores (AVX2, 8 reference threads) and writes up to 1.6 GB (the 65B F16 layer) at a time
to a temporary directory.

    python tests/golden/gen_golden_passes_large.py      # needs a built oracle/_ref
"""
import json
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, HERE)
from distributedllm_b200 import ggjt  # noqa: E402
from oracle import oracle  # noqa: E402
import gen_golden_kquant_large as klarge  # noqa: E402
import gen_golden_large as large  # noqa: E402
from gen_golden_large import digest  # noqa: E402
from gen_golden_vocab import file_sha256  # noqa: E402

OUT = os.path.join(HERE, "ref_digests_passes_large.json")
N_CTX = 1024
N_SESSIONS = 12
BLOCK = {"q4_0": ggjt.T_Q4_0, "q4_1": ggjt.T_Q4_1, "q5_0": ggjt.T_Q5_0, "q5_1": ggjt.T_Q5_1, "q8_0": ggjt.T_Q8_0,
         "f16": ggjt.T_F16}
KQUANT = ("q4_K_S", "q4_K_M", "q6_K")
FAMILIES = {"65b": ("q4_0", "q4_1", "q5_0", "q5_1", "q8_0", "f16", "q4_K_S", "q6_K", "q4_K_M"),
            "30b": ("q4_0", "q5_1", "f16", "q4_K_M"),
            "13b": ("q4_0", "q5_1", "f16", "q4_K_M")}
PROMPT_LEN = [3, 17, 1, 32, 9, 5, 26, 2, 11, 8, 20, 14]           # session s's prompt in the first mixed pass
MIX_ORDER = [4, 0, 11, 7, 2, 9, 1, 10, 5, 3, 8, 6]
STEP_ORDERS = [[7, 2, 10, 0, 5, 11, 3, 8, 1, 6, 9, 4], [3, 9, 0, 6, 11, 1, 4, 8, 10, 2, 7, 5],
               [5, 11, 8, 1, 2, 10, 4, 0, 6, 9, 3, 7], [6, 1, 9, 3, 11, 0, 8, 5, 2]]
FINAL_ORDER = [11, 3, 6, 0, 9, 2, 4, 8, 1, 10, 5, 7]
A, B = 11, 6
GEN_PROMPTS = [6, 1, 11]                                           # 13b_generate: prompt lengths of sessions 0, 1, 2
GEN_STEPS = 24


def ops():
    """The operations every passes case runs, in order.  Each is a dict: op 'mixed' (sessions, counts), 'batch'
    (sessions, one row each), 'session' (one session_forward call: session, count) or 'steps' (one forward_steps call:
    session, count)."""
    out = [{"op": "mixed", "sessions": MIX_ORDER, "counts": [PROMPT_LEN[s] for s in MIX_ORDER]}]
    out += [{"op": "batch", "sessions": o} for o in STEP_ORDERS]
    for s, to in ((A, 515), (B, 500)):
        at = PROMPT_LEN[s] + sum(s in o for o in STEP_ORDERS)
        while at < to:
            out.append({"op": "session", "session": s, "count": min(32, to - at)})
            at += out[-1]["count"]
    out.append({"op": "mixed", "sessions": [7, A, 0, 9], "counts": [1, 29, 20, 1]})
    out += [{"op": "steps", "session": B, "count": 24}, {"op": "steps", "session": A, "count": 16},
            {"op": "steps", "session": 2, "count": 40}]
    out.append({"op": "batch", "sessions": FINAL_ORDER})
    return out


def op_sessions(op):
    """(session, rows) of an operation in row order."""
    if op["op"] == "mixed":
        return list(zip(op["sessions"], op["counts"]))
    if op["op"] == "batch":
        return [(s, 1) for s in op["sessions"]]
    return [(op["session"], op["count"])]


def positions(case):
    """Per operation, the position of every listed session before it; and every session's n_past at the end."""
    past, out = [0] * case["n_sessions"], []
    for op in case["ops"]:
        out.append([past[s] for s, _ in op_sessions(op)])
        for s, n in op_sessions(op):
            past[s] += n
    return out, past


def inputs(case):
    """Per operation its [rows][n_embd] input, rows grouped by session in list order."""
    rng = np.random.default_rng(case["input_seed"])
    e = ggjt.SHAPES[case["shape"]].n_embd
    return [rng.standard_normal((sum(n for _, n in op_sessions(op)), e), dtype=np.float32) for op in case["ops"]]


def split(op, y):
    """An operation's output rows -> one array per listed session."""
    out, r = [], 0
    for _, n in op_sessions(op):
        out.append(y[r:r + n])
        r += n
    return out


def replay(cpu, case, xs, sessions=None):
    """{(operation index, session): output rows} from a CPU checker (RefSlice or a port) replaying each session in
    turn: clear, then that session's share of every operation -- a segment or a session_forward call as one call, a
    batched-step column as a one-row call, decode rows as one-row calls.  `sessions`: only these."""
    out = {}
    for s in range(case["n_sessions"]) if sessions is None else sessions:
        cpu.clear_context()
        for i, op in enumerate(case["ops"]):
            for (t, n), x in zip(op_sessions(op), split(op, xs[i])):
                if t != s:
                    continue
                if op["op"] == "steps":
                    out[(i, s)] = np.concatenate([cpu.forward(x[j:j + 1]) for j in range(n)])
                else:
                    assert n <= oracle.RefSlice.MAX_CHUNK
                    out[(i, s)] = cpu.forward(x)
    return out


def case_digests(case, outs):
    """Per operation, the digest of every listed session's rows."""
    return [[digest(outs[(i, s)]) for s, _ in op_sessions(op)] for i, op in enumerate(case["ops"])]


def write_case_file(path, case):
    if case["family"] in KQUANT:
        klarge.write_layers(path, case)
    else:
        large.write_slice(path, case["shape"], BLOCK[case["family"]], case["seed"])


def case_list():
    """name -> passes case; 65b_q4_0 and 65b_q4_K_M first (the GPU tests sweep runtime switches on them)."""
    cases = {}
    order = [("65b", "q4_0"), ("65b", "q4_K_M")]
    order += [(sh, f) for sh in ("65b", "30b", "13b") for f in FAMILIES[sh] if (sh, f) not in order]
    for shape, fam in order:
        c = {"kind": "passes", "shape": shape, "family": fam}
        if fam in KQUANT:
            c.update(mix=fam, layers=klarge.layers_of(shape, fam), seed=klarge.SEED)
        else:
            c.update(wtype=BLOCK[fam], seed=large.SEED)
        c.update(n_ctx=N_CTX, n_sessions=N_SESSIONS, input_seed=500 + len(cases), ops=ops())
        cases["%s_%s" % (shape, fam)] = c
    return cases


def gen_case():
    """The 13B greedy-generation case (files: the 13b_q4_K_M and 13b_extra cases of ref_digests_kquant_large.json)."""
    rng = np.random.default_rng(600)
    return {"kind": "generate", "shape": "13b", "mix": "q4_K_M", "layers": klarge.layers_of("13b", "q4_K_M"),
            "seed": klarge.SEED, "n_steps": GEN_STEPS,
            "prompts": [rng.integers(0, 32000, n).tolist() for n in GEN_PROMPTS]}


def greedy(cpu, embed, logits, prompt, n_steps):
    """The client's greedy loop on a CPU checker: embed, forward, the last row's logits, the first maximum."""
    cpu.clear_context()
    ids, toks = [], prompt
    for _ in range(n_steps):
        y = cpu.forward(embed(toks))
        ids.append(int(np.argmax(logits(y[-1:])[-1])))
        toks = [ids[-1]]
    return ids


def gen_generate(tmp, case, threads):
    path, extra = os.path.join(tmp, "g.bin"), os.path.join(tmp, "extra.bin")
    klarge.write_layers(path, case)
    ggjt.write_kquant_extra(extra, ggjt.SHAPES["13b"], case["mix"], seed=case["seed"])
    case["file_sha256"], case["extra_sha256"] = file_sha256(path), file_sha256(extra)
    n_vocab, e = ggjt.SHAPES["13b"].n_vocab, ggjt.SHAPES["13b"].n_embd
    ref = oracle.RefSlice(path, threads, 128)
    try:
        embed, logits = lambda t: oracle.ref_embed(extra, t, e), lambda y: oracle.ref_logits(extra, y, n_vocab, False)
        ids = [greedy(ref, embed, logits, p, case["n_steps"]) for p in case["prompts"]]
    finally:
        ref.close()
    case["ids"] = [list(r) for r in zip(*ids)]          # [step][session], as capi.generate_greedy returns them
    os.remove(path)
    os.remove(extra)


def gen(tmp):
    threads = min(16, os.cpu_count() or 4)
    cases, path = case_list(), os.path.join(tmp, "w.bin")
    for name, case in cases.items():
        write_case_file(path, case)
        case["file_sha256"] = file_sha256(path)
        ref = oracle.RefSlice(path, threads, case["n_ctx"])
        try:
            case["digests"] = case_digests(case, replay(ref, case, inputs(case)))
        finally:
            ref.close()
        case["n_past"] = positions(case)[1]
        os.remove(path)
        print(name, flush=True)
    cases["13b_generate"] = gen_case()
    gen_generate(tmp, cases["13b_generate"], threads)
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
