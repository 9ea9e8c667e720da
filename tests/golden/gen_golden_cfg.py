"""Generate tests/golden/cfg_main.json: what llama.cpp's `main` prints when it generates with classifier-free guidance on a
tiny model, kept as data so the GPU tests can compare the device's guided generation with it where the reference is
absent.  It runs the compiled program (oracle/_ref/main, from the reference's vendor/llama.cpp/examples/main) on the CPU
and needs no GPU.

  model    SHAPES["tiny128"] (3 layers, 512 ids), Q4_0, ggjt.write_synth_full(seed=SEED)
  run      `main -m model -p PROMPT --cfg-negative-prompt NEGATIVE --cfg-scale S --cfg-smooth-factor SF --temp 0
            --repeat-penalty 1 -c 128 -n N_PREDICT -t 1 -s 1 --verbose-prompt` for each (S, SF) in CASES; 128 holds both
            prompts and every generated id, so main never swaps its context
  record   the file's sha256, the prompt and negative-prompt ids main prints (BOS and main's leading space included),
           and per case the text main prints after the prompt

Running the script twice writes the same file byte for byte.

    python tests/golden/gen_golden_cfg.py          # needs a built oracle/_ref
"""
import hashlib
import json
import os
import re
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from distributedllm_b200 import ggjt  # noqa: E402

OUT = os.path.join(HERE, "cfg_main.json")
BINARY = os.path.join(ROOT, "oracle", "_ref", "main")
SHAPE = "tiny128"
SEED = 11
PROMPT = "the rain on a net"
NEGATIVE = "she at tea in the rain"
N_CTX = 128
N_PREDICT = 24
CASES = ((1.5, 1.0), (2.0, 0.5), (4.0, 1.0), (1.25, 0.0))


def write_model(path: str) -> str:
    ggjt.write_synth_full(path, ggjt.SHAPES[SHAPE], ggjt.T_Q4_0, seed=SEED)
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def run_main(model: str, scale: float, sf: float, binary: str = BINARY):
    """-> (prompt ids, negative prompt ids, the text printed after the prompt's echo)."""
    r = subprocess.run([binary, "-m", model, "-p", PROMPT, "--cfg-negative-prompt", NEGATIVE, "--cfg-scale", repr(scale),
                        "--cfg-smooth-factor", repr(sf), "--temp", "0", "--repeat-penalty", "1", "-c", str(N_CTX),
                        "-n", str(N_PREDICT), "-t", "1", "-s", "1", "--verbose-prompt"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True)
    err = r.stderr.decode("utf-8", "replace")

    def ids(section):
        block = err.split("main: %s: '" % section, 1)[1]
        n = int(re.search(r"number of tokens in %s = (\d+)" % section, block).group(1))
        got = [int(t) for t in re.findall(r"^\s*(\d+) -> '", block.split("\n", 2)[2], re.M)[:n]]
        assert len(got) == n, err
        return got

    prompt_ids, neg_ids = ids("prompt"), ids("negative prompt")
    vocab = ggjt.default_vocab(ggjt.SHAPES[SHAPE].n_vocab)
    echo = b"".join(vocab[t][0] for t in prompt_ids)
    assert r.stdout.startswith(echo), (r.stdout, echo)
    return prompt_ids, neg_ids, r.stdout[len(echo):].decode("utf-8")


def main() -> None:
    with tempfile.TemporaryDirectory() as d:
        model = os.path.join(d, "full.bin")
        digest = write_model(model)
        cases = []
        for scale, sf in CASES:
            p, n, text = run_main(model, scale, sf)
            cases.append({"scale": scale, "smooth_factor": sf, "text": text})
    doc = {"shape": SHAPE, "wtype": "q4_0", "seed": SEED, "model_sha256": digest, "prompt": PROMPT, "negative": NEGATIVE,
           "n_predict": N_PREDICT, "prompt_ids": p, "negative_ids": n, "cases": cases}
    with open(OUT, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")
    print("wrote %s: %d + %d prompt ids, %d cases" % (OUT, len(p), len(n), len(cases)))


if __name__ == "__main__":
    main()
