"""Generate tests/golden/ppl_windows.json: what llama.cpp's `perplexity` program prints for a tiny model, kept as data so
the GPU tests can compare LocalPipeline.perplexity_windows with it where the reference is absent.  It runs the compiled
program (oracle/_ref/perplexity, from the reference's vendor/llama.cpp/examples/perplexity) on the CPU and needs no GPU.

  model    SHAPES["tiny128"] (3 layers, 512 ids), Q4_0, ggjt.write_synth_full(seed=SEED)
  text     TEXT_WORDS words drawn from WORDS by numpy's default_rng(SEED): about 5 windows of 64 ids and a partial one
  cases    (n_ctx, n_batch) in CASES, each `perplexity -m model -f text -c n_ctx -b n_batch -t 1`
  record   the file's sha256, the number of ids, and per case the values the program prints after each window

Running the script twice writes the same file byte for byte.

    python tests/golden/gen_golden_ppl_windows.py          # needs a built oracle/_ref
"""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from distributedllm_b200 import ggjt  # noqa: E402

OUT = os.path.join(HERE, "ppl_windows.json")
BINARY = os.path.join(ROOT, "oracle", "_ref", "perplexity")
SHAPE = "tiny128"
SEED = 11
WORDS = ["the", "a", "in", "an", "on", "he", "at", "she", "tea", "rain", "net", "the", "the", "a"]
TEXT_WORDS = 190
CASES = ((64, 24), (32, 32), (40, 16))      # n_ctx not a multiple of n_batch; n_batch == n_ctx; first = n_ctx / 2 = 20


def text() -> str:
    rng = np.random.default_rng(SEED)
    return " ".join(WORDS[i] for i in rng.integers(0, len(WORDS), TEXT_WORDS))


def write_model(path: str) -> str:
    ggjt.write_synth_full(path, ggjt.SHAPES[SHAPE], ggjt.T_Q4_0, seed=SEED)
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def run_binary(model: str, text_path: str, n_ctx: int, n_batch: int) -> list:
    """The running perplexities perplexity.cpp:115 prints ("[i]x.xxxx,")."""
    r = subprocess.run([BINARY, "-m", model, "-f", text_path, "-c", str(n_ctx), "-b", str(n_batch), "-t", "1"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True, text=True)
    got = re.findall(r"\[(\d+)\]([0-9.]+|nan|inf),", r.stdout)
    assert [int(i) for i, _ in got] == list(range(1, len(got) + 1)), r.stdout
    return [v for _, v in got]


def main() -> None:
    with tempfile.TemporaryDirectory() as d:
        model, text_path = os.path.join(d, "full.bin"), os.path.join(d, "text.txt")
        digest = write_model(model)
        with open(text_path, "w") as f:
            f.write(text())
        cases = [{"n_ctx": c, "n_batch": b, "printed": run_binary(model, text_path, c, b)} for c, b in CASES]
        from oracle import oracle
        extra = os.path.join(d, "extra.bin")
        ggjt.extract_extra_layers(model, extra)
        n_ids = len(oracle.ref_tokenize(extra, text()))
    doc = {"shape": SHAPE, "wtype": "q4_0", "seed": SEED, "model_sha256": digest, "n_ids": n_ids, "cases": cases}
    with open(OUT, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote %s: %d ids, %s" % (OUT, n_ids, [(c["n_ctx"], c["n_batch"], len(c["printed"])) for c in cases]))


if __name__ == "__main__":
    main()
