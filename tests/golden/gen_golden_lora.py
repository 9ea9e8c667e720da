"""Write tests/golden/ref_digests_lora.json: for every case of tests/lora_ref.cases() and .edges(), the sha256 of each layer matrix
after llama.cpp's LoRA merge (oracle/_ref/lora_merge on the case's full model).  The CPU tests then check the host twin
against these digests where oracle/_ref is absent.

    python tests/golden/gen_golden_lora.py
"""
from __future__ import annotations

import hashlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import lora_ref  # noqa: E402

from distributedllm_b200 import ggjt  # noqa: E402

TOOL = os.path.join(ROOT, "oracle", "_ref", "lora_merge")
OUT = os.path.join(ROOT, "tests", "golden", "ref_digests_lora.json")


def oracle_digests(c, d: str) -> dict:
    m, a, b = lora_ref.write_case(d, c)
    out = os.path.join(d, "oracle.bin")
    subprocess.run([TOOL, m, a, b or "-", out, "2"], check=True, capture_output=True)
    f = ggjt.read_file(out, sliced=False)
    return {n: hashlib.sha256(f.read_raw(n)).hexdigest() for n in f.tensors if n.startswith("layers.")}


def main() -> None:
    res = {}
    for c in lora_ref.cases() + lora_ref.edges():
        with tempfile.TemporaryDirectory() as d:
            res[lora_ref.case_id(c)] = oracle_digests(c, d)
    with open(OUT, "w") as f:
        json.dump(res, f, indent=0, sort_keys=True)
    print("wrote %d cases to %s" % (len(res), OUT))


if __name__ == "__main__":
    main()
