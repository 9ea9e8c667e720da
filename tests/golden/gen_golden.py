"""Generate the committed golden fixtures from the REFERENCE ITSELF (run in the build container only).

  slices.npz     hidden states of oracle/_ref (= distllm/tensor_processor.cpp compiled unmodified, see
                 oracle/Makefile) on seeded synthetic slice files, for a fixed schedule of propagate_forward calls
  slices_q4_1.*  the same for Q4_1 slices (added later; `gen_golden.py q4_1` writes only these) + extra_q4_1.npz
  extra.npz      reference get_inputs / get_llm_output / llama_tokenize on a synthetic extra-layers file
  tokenizer.json reference tokenisation of fixed strings with vendor/llama.cpp/models/ggml-vocab.bin's vocabulary
  protocol.json  frames produced by the reference's distllm/protocol.py for one instance of every message
  ref_digests.json  SHA-256 of the reference's outputs (and its greedy ids) in the tests whose inputs are too large to store
                 (`gen_golden.py digests` writes only this)

    python tests/golden/gen_golden.py          # needs /root/reference and a built oracle/_ref
"""
import base64
import hashlib
import json
import os
import struct
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from distributedllm_b200 import ggjt  # noqa: E402
from oracle import oracle  # noqa: E402

CASES = [  # name, shape, weight type, layer range, schedule of calls
    ("tiny_q4_0", "tiny", ggjt.T_Q4_0, (1, 2), [40, 1, 1, 7, 1, 20, 3, 1]),
    ("tiny128_q4_0", "tiny128", ggjt.T_Q4_0, (0, 1), [33, 1, 1, 1, 30, 1]),
    ("tiny3b_q4_0", "tiny3b", ggjt.T_Q4_0, (0, 1), [37, 1, 1, 5]),
    ("tiny_q8_0", "tiny", ggjt.T_Q8_0, (0, 1), [18, 1, 1, 16]),
    ("tiny_f16", "tiny", ggjt.T_F16, (2, 3), [35, 1, 1]),
]
CASES_Q4_1 = [
    ("tiny_q4_1", "tiny", ggjt.T_Q4_1, (1, 2), [40, 1, 1, 7, 1, 20, 3, 1]),
    ("tiny128_q4_1", "tiny128", ggjt.T_Q4_1, (0, 1), [33, 1, 1, 1, 30, 1]),
    ("tiny3b_q4_1", "tiny3b", ggjt.T_Q4_1, (0, 1), [37, 1, 1, 5]),
]


def gen_slices(tmp, cases, stem):
    out = {}
    meta = {}
    for name, shape, wt, (a, b), sched in cases:
        sh = ggjt.SHAPES[shape]
        path = os.path.join(tmp, name + ".bin")
        ggjt.write_synth_slice(path, sh, a, b, wt, seed=0)
        meta[name] = {"shape": shape, "wtype": wt, "layers": [a, b], "schedule": sched,
                      "file_sha256": hashlib.sha256(open(path, "rb").read()).hexdigest()}
        rng = np.random.default_rng(1234)
        ref = oracle.RefSlice(path, n_threads=3, n_ctx=512)
        for i, n in enumerate(sched):
            x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
            out["%s/x%d" % (name, i)] = x
            out["%s/y%d" % (name, i)] = ref.forward(x)
        ref.close()
    np.savez_compressed(os.path.join(HERE, stem + ".npz"), **out)
    json.dump(meta, open(os.path.join(HERE, stem + ".json"), "w"), indent=1)


def gen_q4_1(tmp):
    gen_slices(tmp, CASES_Q4_1, "slices_q4_1")
    # client side of a Q4_1 model: tok_embeddings rows dequantised as nibble * d + m, output.weight through the Q4_1 dot
    sh = ggjt.SHAPES["tiny"]
    extra = os.path.join(tmp, "extra_q4_1.bin")
    ggjt.write_synth_extra(extra, sh, ggjt.T_Q4_1, seed=0)
    toks = np.array([1, 5, 300, 44, 511, 0, 77], np.int32)
    h = np.random.default_rng(7).standard_normal((5, sh.n_embd), dtype=np.float32)
    np.savez_compressed(os.path.join(HERE, "extra_q4_1.npz"), tokens=toks, emb=oracle.ref_embed(extra, toks, sh.n_embd), hidden=h,
                        logits_all=oracle.ref_logits(extra, h, sh.n_vocab, True),
                        file_sha256=np.frombuffer(hashlib.sha256(open(extra, "rb").read()).digest(), np.uint8))


def digest(a) -> str:
    """SHA-256 of the float32 bit patterns: comparing digests is comparing every bit of the array."""
    return hashlib.sha256(np.ascontiguousarray(a, np.float32).tobytes()).hexdigest()


def gen_digests(tmp):
    """ref_digests.json: what the reference computed in the tests that compare against it on inputs too large to store
    (full-size layer shapes) -- the digest of every call's output and the greedy ids.  Each block replays the exact
    inputs (files, seeds, schedules) of the test that reads it."""
    import subprocess
    out = {}
    # tests/test_oracle.py::test_port_matches_live_reference
    for shape, wt in [("tiny", ggjt.T_F32), ("tiny128", ggjt.T_F16), ("tiny3b", ggjt.T_Q8_0), ("tiny3b", ggjt.T_Q4_1)]:
        path = os.path.join(tmp, "m.bin")
        ggjt.write_synth_slice(path, ggjt.SHAPES[shape], 0, 1, wt, seed=3)
        ref, rng = oracle.RefSlice(path, 3, 512), np.random.default_rng(5)
        out["port/%s_%s" % (shape, ggjt.TYPE_NAME[wt])] = [
            digest(ref.forward(rng.standard_normal((n, ggjt.SHAPES[shape].n_embd), dtype=np.float32))) for n in (34, 1, 2, 1)]
        ref.close()
    # tests/test_oracle.py::test_fast_q4_1_writer_files_are_valid_for_the_reference
    sh = ggjt.SHAPES["tiny128"]
    path = os.path.join(tmp, "fast_q4_1.bin")
    ggjt.write_fast_q4_slice(path, sh, 0, 1, 0, wtype=ggjt.T_Q4_1)
    ref, rng = oracle.RefSlice(path, 3, 512), np.random.default_rng(11)
    out["fast_q4_1_writer"] = [digest(ref.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32))) for n in (20, 1, 1)]
    ref.close()
    # tests/test_ggjt_and_abi.py::test_q4_1_quantizer_is_the_reference_quantize_tool: the tool's Q4_1 tensors
    sh = ggjt.SHAPES["tiny3b"]
    full, fq = os.path.join(tmp, "f32.bin"), os.path.join(tmp, "q41.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=0)
    subprocess.run([os.path.join(oracle.REF_DIR, "quantize"), full, fq, "q4_1"], check=True, capture_output=True)
    b = ggjt.read_file(fq)
    out["quantize_q4_1"] = {name: hashlib.sha256(b.read_raw(name)).hexdigest()
                            for name, t in b.tensors.items() if t.ttype == ggjt.T_Q4_1}
    # tests/test_gpu_llm_api.py::test_gpu_matches_live_reference
    sh = ggjt.SHAPES["tiny128"]
    path = os.path.join(tmp, "tiny128_q4_0_0_2_s5.bin")
    ggjt.write_synth_slice(path, sh, 0, 2, ggjt.T_Q4_0, 5)
    ref, rng = oracle.RefSlice(path, 3, 512), np.random.default_rng(8)
    out["gpu_tiny128"] = [digest(ref.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32))) for n in (45, 1, 1, 1)]
    ref.close()
    # tests/test_gpu_full_size.py
    threads = min(16, os.cpu_count() or 4)
    sh = ggjt.SHAPES["3b"]
    pa, pb, extra = (os.path.join(tmp, n) for n in ("a.bin", "b.bin", "extra.bin"))
    ggjt.write_fast_q4_slice(pa, sh, 0, 16, seed=3)
    ggjt.write_fast_q4_slice(pb, sh, 17, 25, seed=3)
    ggjt.write_fast_q4_extra(extra, sh, seed=3)
    refs = [oracle.RefSlice(pa, threads, 512), oracle.RefSlice(pb, threads, 512)]
    toks, ids, hidden = [1 + (i * 7919) % 31999 for i in range(16)], [], []
    for step in range(33):
        y = oracle.ref_embed(extra, toks, sh.n_embd)
        for s in refs:
            y = s.forward(y)
        hidden.append(digest(y))
        toks = [oracle.ref_lib().ref_next_token(extra.encode(), y.ctypes.data, y.size)]
        ids.append(toks[0])
    out["config1"] = {"ids": ids, "hidden": hidden}
    for s in refs:
        s.close()
    sh = ggjt.SHAPES["7b"]
    p = os.path.join(tmp, "f16.bin")
    ggjt.write_fast_f16_slice(p, sh, 0, 0, seed=4)
    ref, rng = oracle.RefSlice(p, threads, 512), np.random.default_rng(9)
    out["config4"] = [digest(ref.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32))) for n in (24, 1, 1, 9, 1)]
    ref.close()
    os.remove(p)
    sh = ggjt.SHAPES["13b"]
    p = os.path.join(tmp, "q4_13b.bin")
    ggjt.write_fast_q4_slice(p, sh, 0, 0, seed=5)
    refs, rng = [oracle.RefSlice(p, threads, 512) for _ in range(8)], np.random.default_rng(10)
    prompt = [digest(refs[b].forward(rng.standard_normal((3 + 2 * b, sh.n_embd), dtype=np.float32))) for b in range(8)]
    steps = []
    for step in range(3):
        x = rng.standard_normal((8, sh.n_embd), dtype=np.float32)
        steps.append([digest(refs[b].forward(x[b:b + 1])[0]) for b in range(8)])
    out["config5"] = {"prompt": prompt, "steps": steps}
    for r in refs:
        r.close()
    sh = ggjt.SHAPES["7b"]
    p = os.path.join(tmp, "q4_7b_2l.bin")
    ggjt.write_fast_q4_slice(p, sh, 0, 1, seed=6)
    ref, rng = oracle.RefSlice(p, threads, 512), np.random.default_rng(11)
    chunks, pos = [], 0
    while pos < 500:                     # the reference's arena caps a call at ~64 tokens
        n = min(oracle.RefSlice.MAX_CHUNK, 500 - pos)
        chunks.append([n, digest(ref.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32)))])
        pos += n
    out["config2"] = {"prefill": chunks,
                      "decode": [digest(ref.forward(rng.standard_normal((1, sh.n_embd), dtype=np.float32))) for _ in range(500, 512)]}
    ref.close()
    json.dump(out, open(os.path.join(HERE, "ref_digests.json"), "w"), indent=1)


def main():
    tmp = tempfile.mkdtemp()
    if sys.argv[1:] == ["q4_1"]:
        gen_q4_1(tmp)
        return
    if sys.argv[1:] == ["digests"]:
        gen_digests(tmp)
        return
    gen_slices(tmp, CASES, "slices")
    gen_q4_1(tmp)

    # extra layers + tokenizer on a synthetic all-Q4_0 extra file
    sh = ggjt.SHAPES["tiny"]
    extra = os.path.join(tmp, "extra.bin")
    ggjt.write_synth_extra(extra, sh, ggjt.T_Q4_0, seed=0)
    toks = np.array([1, 5, 300, 44, 511, 0, 77], np.int32)
    emb = oracle.ref_embed(extra, toks, sh.n_embd)
    h = np.random.default_rng(7).standard_normal((5, sh.n_embd), dtype=np.float32)
    np.savez_compressed(os.path.join(HERE, "extra.npz"), tokens=toks, emb=emb, hidden=h,
                        logits_all=oracle.ref_logits(extra, h, sh.n_vocab, True),
                        logits_last=oracle.ref_logits(extra, h, sh.n_vocab, False),
                        file_sha256=np.frombuffer(hashlib.sha256(open(extra, "rb").read()).digest(), np.uint8))

    # extra layers as the reference's own `quantize q4_0` writes them for n_embd % 256 == 0: output.weight is Q6_K
    # (llama.cpp:2523-2528).  The quantised file itself is committed (190 KB): k-quant quantisation is not restated here.
    import subprocess
    full = os.path.join(tmp, "full_f32.bin")
    ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=0)
    fq = os.path.join(tmp, "full_q4.bin")
    subprocess.run([os.path.join(ROOT, "oracle", "_ref", "quantize"), full, fq, "q4_0"], check=True, capture_output=True)
    eq = os.path.join(HERE, "extra_q6k.bin")
    subprocess.run([os.path.join(ROOT, "oracle", "_ref", "slice_model"), "extra_layers", fq, eq], check=True, capture_output=True)
    assert ggjt.read_file(eq).tensors["output.weight"].ttype == ggjt.T_Q6_K
    h6 = np.random.default_rng(8).standard_normal((6, sh.n_embd), dtype=np.float32)
    h6[3] *= 30.0
    h6[4, :] = 0.0
    np.savez_compressed(os.path.join(HERE, "extra_q6k.npz"), hidden=h6, logits_all=oracle.ref_logits(eq, h6, sh.n_vocab, True),
                        emb=oracle.ref_embed(eq, toks, sh.n_embd), tokens=toks)

    # tokenizer with the real 32000-entry llama vocabulary
    vocab_bin = "/root/reference/vendor/llama.cpp/models/ggml-vocab.bin"
    f = ggjt.read_file(vocab_bin, sliced=False)
    vfile = os.path.join(tmp, "vocab_extra.bin")
    hp = ggjt.HParams(f.hparams.n_vocab, 32, 32, 1, 0, 32, ggjt.FTYPE_F32, ggjt.NO_FIRST_LAYER)
    ggjt.write_file(vfile, hp, f.vocab, [])
    texts = ["Hello World", " Hello World", "Hello, World!", " this is 🦙.cpp", "w048 7tuijk dsdfhu",
             "Alan Turing is", "", "  double  spaces\nnewline\ttab", "ünïcödé ✓ 日本語", "a" * 50]
    json.dump({"vocab_sha256": hashlib.sha256(open(vocab_bin, "rb").read()).hexdigest(),
               "cases": [{"text": t, "ids": oracle.ref_tokenize(vfile, t)} for t in texts]},
              open(os.path.join(HERE, "tokenizer.json"), "w"), indent=1, ensure_ascii=False)
    # the vocabulary itself (432 KB) is needed to replay the cases: keep only (len, bytes, score) records, gzip
    import gzip
    with gzip.open(os.path.join(HERE, "llama_vocab.bin.gz"), "wb") as g:
        for text, score in f.vocab:
            g.write(struct.pack("<I", len(text)) + text + struct.pack("<f", score))

    # protocol frames from the reference implementation
    sys.path.insert(0, "/root/reference")
    from distllm import protocol as ref_protocol
    msgs = [("RequestAllSlices", {}), ("RequestStatus", {}), ("RequestLoadSlice", {"name": "orb"}),
            ("RequestPropagateForward", {"axis0": 1, "axis1": 4, "values": [0.5, -1.25, 3.0, 0.1]}),
            ("ResponsePropagateForward", {"axis0": 1, "axis1": 2, "values": [1e-8, 65504.0]}),
            ("RequestClearContext", {}), ("ResponseClearContext", {}),
            ("RequestFileSubmissionBegin", {"metadata_json": '{"type": "slice", "model": "m"}'}),
            ("ResponseFileSubmissionBegin", {"submission_id": 7}),
            ("RequestSubmitPart", {"submission_id": 7, "part_number": 2, "data": bytes(range(40))}),
            ("ResponseSubmitPart", {"part_size": 40}),
            ("RequestFileSubmissionEnd", {"submission_id": 7, "checksum": "ab" * 32}),
            ("ResponseFileSubmissionEnd", {"file_name": "orb", "total_size": 1 << 20}),
            ("JsonResponseWithStatus", {"status_json": '{"status": "up"}'}),
            ("JsonResponseWithSlices", {"slices_json": "[]"}),
            ("JsonResponseWithLoadedSlice", {"name": "orb", "model": "llama"}),
            ("ResponseWithError", {"operation": "load_slice_request", "error": "slice_not_found", "description": "ü"}),
            ("RequestGreeting", {}), ("ResponseGreeting", {})]
    frames = []
    for cls, body in msgs:
        frame = getattr(ref_protocol, cls)(**body).encode()
        jb = {k: (base64.b64encode(v).decode() if isinstance(v, bytes) else v) for k, v in body.items()}
        frames.append({"cls": cls, "body": jb, "bytes_fields": [k for k, v in body.items() if isinstance(v, bytes)],
                       "frame_b64": base64.b64encode(frame).decode()})
    json.dump(frames, open(os.path.join(HERE, "protocol.json"), "w"), indent=1)
    print("golden fixtures written to", HERE)


if __name__ == "__main__":
    main()
