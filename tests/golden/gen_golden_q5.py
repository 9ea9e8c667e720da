"""Generate the Q5_0 / Q5_1 golden fixtures from the REFERENCE ITSELF (run in the build container only, next to
gen_golden.py, whose slice dumper it reuses; it writes only these files):

  slices_q5_0.*, slices_q5_1.*  hidden states of oracle/_ref on seeded Q5 slice files (tiny / tiny128 / tiny3b)
  extra_q5_0.npz, extra_q5_1.npz  reference get_inputs / get_llm_output / greedy ids on a tiny3b Q5 extra-layers file
                 (n_embd 800 is not a multiple of 256, so `quantize` keeps output.weight in Q5)
  ref_digests_q5.json  SHA-256 of the Q5 tensors the reference `quantize` tool writes for tiny3b, and of the reference's
                 outputs on the benchmark writer's Q5 files

    python tests/golden/gen_golden_q5.py          # needs /root/reference and a built oracle/_ref
"""
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from gen_golden import digest, gen_slices  # noqa: E402
from distributedllm_b200 import ggjt  # noqa: E402
from oracle import oracle  # noqa: E402

CASES_Q5 = {wt: [("tiny_%s" % nm, "tiny", wt, (1, 2), [40, 1, 1, 7, 1, 20, 3, 1]),
                 ("tiny128_%s" % nm, "tiny128", wt, (0, 1), [33, 1, 1, 1, 30, 1]),
                 ("tiny3b_%s" % nm, "tiny3b", wt, (0, 1), [37, 1, 1, 5])]
            for wt, nm in ((ggjt.T_Q5_0, "q5_0"), (ggjt.T_Q5_1, "q5_1"))}


def gen_q5(tmp):
    dig = {}
    for wt in (ggjt.T_Q5_0, ggjt.T_Q5_1):
        nm = ggjt.TYPE_NAME[wt]
        gen_slices(tmp, CASES_Q5[wt], "slices_" + nm)
        # client side on tiny3b: n_embd 800 is not a multiple of 256, so output.weight stays Q5 (llama.cpp:2523)
        sh = ggjt.SHAPES["tiny3b"]
        extra = os.path.join(tmp, "extra_%s.bin" % nm)
        ggjt.write_synth_extra(extra, sh, wt, seed=0)
        toks = np.array([1, 5, 300, 44, 511, 0, 77], np.int32)
        h = np.random.default_rng(7).standard_normal((5, sh.n_embd), dtype=np.float32)
        ids = [oracle.ref_lib().ref_next_token(extra.encode(), np.ascontiguousarray(h[:i + 1]).ctypes.data, (i + 1) * sh.n_embd)
               for i in range(5)]
        np.savez_compressed(os.path.join(HERE, "extra_%s.npz" % nm), tokens=toks, emb=oracle.ref_embed(extra, toks, sh.n_embd),
                            hidden=h, logits_all=oracle.ref_logits(extra, h, sh.n_vocab, True), next_ids=np.array(ids, np.int32),
                            file_sha256=np.frombuffer(hashlib.sha256(open(extra, "rb").read()).digest(), np.uint8))
        # the reference `quantize` tool's Q5 tensors of a full tiny3b model
        full, fq = os.path.join(tmp, "f32.bin"), os.path.join(tmp, "q5.bin")
        ggjt.write_synth_full(full, sh, ggjt.T_F32, seed=0)
        subprocess.run([os.path.join(oracle.REF_DIR, "quantize"), full, fq, nm], check=True, capture_output=True)
        b = ggjt.read_file(fq)
        dig["quantize_" + nm] = {name: hashlib.sha256(b.read_raw(name)).hexdigest()
                                 for name, t in b.tensors.items() if t.ttype == wt}
        # the benchmark writer's blocks are valid for the reference
        sh = ggjt.SHAPES["tiny128"]
        path = os.path.join(tmp, "fast_%s.bin" % nm)
        ggjt.write_fast_q4_slice(path, sh, 0, 1, 0, wtype=wt)
        ref, rng = oracle.RefSlice(path, 3, 512), np.random.default_rng(11)
        dig["fast_%s_writer" % nm] = [digest(ref.forward(rng.standard_normal((n, sh.n_embd), dtype=np.float32))) for n in (20, 1, 1)]
        ref.close()
    json.dump(dig, open(os.path.join(HERE, "ref_digests_q5.json"), "w"), indent=1)


if __name__ == "__main__":
    gen_q5(tempfile.mkdtemp())
    print("Q5 golden fixtures written to", HERE)
