"""bench.py's measurement on the same LLaMA-7B model stored as Q5_0 or Q5_1 blocks.

    python scripts/bench_q5.py --wtype q5_0 [bench.py options]      # or --wtype q5_1

Runs bench.py's GPU arm unchanged (decode tok/s, tok/s at position 511, the k_gemv roofline, and, without --no-cpu,
the CPU baseline + bit-for-bit parity against the compiled reference over the same file) with two substitutions: the
synthetic slice file holds Q5 blocks (ggjt.write_fast_q4_slice(wtype=...), 22 / 24 B per block), and every figure that
bench.py derives from Q4_0's 18 B per block is restated with the type's block size.  The k_gemv roofline needs no
restating: it divides the slice's weight bytes as the library reports them (file bytes) by kernel time.
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

WTYPES = {"q5_0": ggjt.T_Q5_0, "q5_1": ggjt.T_Q5_1}


def type_bytes(wt: int, n_weights: int) -> int:
    return n_weights // 32 * ggjt.TYPE_BLOCK[wt][1]


def model_bytes(wt: int, sh) -> int:
    """bench.py's W_all for weight type wt: 32 layers of matrices + their two f32 norm vectors."""
    e = sh.n_embd
    return 32 * (4 * type_bytes(wt, e * e) + 3 * type_bytes(wt, e * sh.n_ff)) + 32 * 2 * e * 4


def make_slice_file(wt: int):
    name = ggjt.TYPE_NAME[wt]

    def slice_file(shape_name: str, a: int, b: int) -> str:
        p = os.path.join(bench.model_dir(), "%s_%s_s%d_layers_%d_%d.bin" % (shape_name, name, bench.SEED, a, b))
        sh = ggjt.SHAPES[shape_name]
        per_layer = 4 * type_bytes(wt, sh.n_embd * sh.n_embd) + 3 * type_bytes(wt, sh.n_embd * sh.n_ff)
        if not (os.path.isfile(p) and os.path.getsize(p) > per_layer * (b - a + 1)):
            tmp = p + ".tmp%d" % os.getpid()
            ggjt.write_fast_q4_slice(tmp, sh, a, b, bench.SEED, wtype=wt)
            os.replace(tmp, p)
        return p

    return slice_file


def restate(line: dict, wt: int) -> dict:
    """Replace bench.py's Q4_0-derived fields of one result line with the type's."""
    name = ggjt.TYPE_NAME[wt]
    up = name.upper()
    act = "q8_1" if wt == ggjt.T_Q5_1 else "q8_0"
    sh = ggjt.SHAPES["7b"]
    dw = model_bytes(wt, sh) - model_bytes(ggjt.T_Q4_0, sh)
    line["metric"] = line["metric"].replace("Q4_0", up)
    line["dtype"] = "%s*%s->f32" % (name, act)
    cfg = line.get("config", {})
    for k in ("workload", "weights"):
        if k in cfg:
            cfg[k] = cfg[k].replace("Q4_0", up)
    roof = line.get("roofline") or {}
    if "kernel" in roof:
        roof["kernel"] = roof["kernel"].replace("Q4_0xQ8_0", "%sx%s" % (up, act.upper()))
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
    ap.add_argument("--wtype", required=True, choices=sorted(WTYPES))
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg (and with it the parity check)")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the last timed step's output to DIR/hidden.npy (float32)")
    args = ap.parse_args()
    if args.gpus != 1:
        raise SystemExit("bench_q5.py measures one GPU")
    args.warmup = max(args.warmup, 3)
    wt = WTYPES[args.wtype]
    bench.slice_file = make_slice_file(wt)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        rc = bench.run_b200(args)
    for ln in buf.getvalue().splitlines():
        if ln.startswith("{"):
            print(json.dumps(restate(json.loads(ln), wt)), flush=True)
        else:
            print(ln)
    return rc


if __name__ == "__main__":
    sys.exit(main())
