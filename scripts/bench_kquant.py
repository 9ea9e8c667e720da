"""bench.py's measurement on the same LLaMA-7B model stored as a k-quant file: Q4_K_S, Q4_K_M or Q6_K.

    python scripts/bench_kquant.py --mix q4_K_M [bench.py options]      # or --mix q4_K_S / q6_K

Runs bench.py's GPU arm unchanged (decode tok/s, tok/s at position 511, the in-step matmul streaming rate, and, without
--no-cpu, the CPU baseline + bit-for-bit parity against the compiled reference over the same file) with two
substitutions: the synthetic slice file holds k-quant blocks with the per-tensor types the reference's `quantize` gives
that mix (ggjt.write_kquant_slice), and every figure that bench.py derives from Q4_0's 18 B per 32 weights is restated
with the file's bytes.  The streaming rate needs no restating: it divides the slice's weight bytes as the library reports
them (file bytes) by kernel time.  Q4_K_S measures Q4_K matrices, Q6_K measures Q6_K matrices, Q4_K_M their mix.
Prints ONE JSON line, as bench.py does.
"""
import argparse
import contextlib
import io
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributedllm_b200 import ggjt  # noqa: E402
import bench  # noqa: E402

MIXES = sorted(ggjt.KQUANT_MIXES)


def layer_bytes(mix, sh, layer: int) -> int:
    """Matrix bytes of one layer of a `mix` file (mix None: the Q4_0 file bench.py writes)."""
    n = 0
    for nm in ggjt.LAYER_TENSORS:
        if nm.endswith("norm.weight"):
            continue
        t = ggjt.T_Q4_0 if mix is None else ggjt.kquant_tensor_type("layers.%d.%s" % (layer, nm), mix, sh.n_layer)
        rows, k = (sh.n_embd, sh.n_embd) if nm.startswith("attention") else (sh.n_ff, sh.n_embd)
        blk, sz = ggjt.TYPE_BLOCK[t]
        n += rows * k // blk * sz
    return n


def model_bytes(mix, sh) -> int:
    """bench.py's W_all: 32 layers of matrices + their two f32 norm vectors."""
    return sum(layer_bytes(mix, sh, i) for i in range(32)) + 32 * 2 * sh.n_embd * 4


def make_slice_file(mix: str):
    def slice_file(shape_name: str, a: int, b: int) -> str:
        p = os.path.join(bench.model_dir(), "%s_%s_s%d_layers_%d_%d.bin" % (shape_name, mix, bench.SEED, a, b))
        sh = ggjt.SHAPES[shape_name]
        need = sum(layer_bytes(mix, sh, i) for i in range(a, b + 1))
        if not (os.path.isfile(p) and os.path.getsize(p) > need):
            tmp = p + ".tmp%d" % os.getpid()
            ggjt.write_kquant_slice(tmp, sh, a, b, mix, bench.SEED)
            os.replace(tmp, p)
        return p

    return slice_file


def restate(line: dict, mix: str) -> dict:
    """Replace bench.py's Q4_0-derived fields of one result line with the mix's."""
    up = mix.upper()
    sh = ggjt.SHAPES["7b"]
    dw = model_bytes(mix, sh) - model_bytes(None, sh)
    line["metric"] = line["metric"].replace("Q4_0", up)
    line["dtype"] = "%s*q8_K->f32" % mix
    cfg = line.get("config", {})
    for k in ("workload", "weights"):
        if k in cfg:
            cfg[k] = cfg[k].replace("Q4_0", up)
    roof = line.get("roofline") or {}
    if "kernel" in roof:
        roof["kernel"] = roof["kernel"].replace("Q4_0xQ8_0", "%sxQ8_K" % up)
    sr = line.get("step_roofline")
    if sr:
        b = sr["algorithmic_bytes_per_step"] + dw
        peak = sr["roofline_tokens_per_s_one_gpu"] * sr["algorithmic_bytes_per_step"]       # peak * 1e9, as bench.py used it
        sr["algorithmic_bytes_per_step"] = b
        sr["roofline_tokens_per_s_one_gpu"] = peak / b
        sr["frac_of_one_gpu"] = line["value"] / (peak / b)
        sr["frac_of_n_gpus"] = line["value"] / (line["n_gpus"] * peak / b)
        p511 = line.get("at_p511")
        if p511:
            b511 = p511["algorithmic_bytes"] + dw
            p511["algorithmic_bytes"] = b511
            p511["frac_of_one_gpu"] = p511["tokens_per_s"] / (peak / b511)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mix", required=True, choices=MIXES)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg (and with it the parity check)")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's output to DIR/hidden.npy (float32)")
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_kquant.py measures one GPU")
    args.warmup = max(args.warmup, 3)
    bench.slice_file = make_slice_file(args.mix)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        rc = bench.run_b200(args)
    for ln in buf.getvalue().splitlines():
        if ln.startswith("{"):
            print(json.dumps(restate(json.loads(ln), args.mix)), flush=True)
        else:
            print(ln)
    return rc


if __name__ == "__main__":
    sys.exit(main())
