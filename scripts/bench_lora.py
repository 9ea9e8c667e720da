"""Load time of a LLaMA-7B Q4_0 slice with a LoRA adapter merged on the GPU (b200_slice_load_lora).

Adapters: rank 16 on wq / wv (alpaca-lora's targets) and rank 64 on all seven matrices.  Before any timing, the adapted
slice's hidden states are checked bit-identical to the host twin's merged slice loaded plainly (a 7B layer at rank 16, a
tiny128 slice at rank 64).  Reports the median load seconds of each arm (arms alternate), the k_lora_merge kernel time
(torch.profiler, a separate load), llama.cpp's CPU merge time on this host's cores for a few 7B layers when
oracle/_ref/lora_merge exists, and the card's name and power limit.

    python scripts/bench_lora.py [--layers 32] [--reps 3] [--oracle-layers 4]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from distributedllm_b200 import capi, ggjt  # noqa: E402

TOOL = os.path.join(ROOT, "oracle", "_ref", "lora_merge")
ALPACA = ("attention.wq.weight", "attention.wv.weight")
ALL7 = ("attention.wq.weight", "attention.wk.weight", "attention.wv.weight", "attention.wo.weight",
        "feed_forward.w1.weight", "feed_forward.w2.weight", "feed_forward.w3.weight")


def write_adapter(path, shape, layers, r, alpha, mats, seed=0):
    e, ff = shape.n_embd, shape.n_ff
    dims = {"attention.wq.weight": (e, e), "attention.wk.weight": (e, e), "attention.wv.weight": (e, e),
            "attention.wo.weight": (e, e), "feed_forward.w1.weight": (ff, e), "feed_forward.w2.weight": (e, ff),
            "feed_forward.w3.weight": (ff, e)}
    rng = np.random.default_rng([seed, r])

    def gen():
        for layer in layers:
            for m in mats:
                rows, k = dims[m]
                name = "layers.%d.%s" % (layer, m)
                yield name + ".loraA", (rng.standard_normal((k, r), dtype=np.float32) * np.float32(0.02))
                yield name + ".loraB", (rng.standard_normal((rows, r), dtype=np.float32) * np.float32(0.02))
    ggjt.write_lora(path, r, alpha, gen())


def check_equal(d, shape_name, r, mats, n_ctx=128):
    import lora_ref
    sh = ggjt.SHAPES[shape_name]
    p, a, m = (os.path.join(d, "chk_%s_%s.bin" % (shape_name, k)) for k in ("s", "a", "m"))
    if shape_name == "7b":
        ggjt.write_fast_q4_slice(p, sh, 0, 0, seed=1)
    else:
        ggjt.write_synth_slice(p, sh, 0, 1, ggjt.T_Q4_0, seed=1)
    write_adapter(a, sh, range(2), r, 2 * r, mats)
    lora_ref.merge_file(p, m, a)
    s1 = capi.Slice(p, 0, n_ctx, lora=a)
    s2 = capi.Slice(m, 0, n_ctx)
    x = np.random.default_rng(0).standard_normal((9, sh.n_embd), dtype=np.float32)
    ok = all(np.array_equal(s1.forward(v).view(np.uint32), s2.forward(v).view(np.uint32)) for v in (x[:8], x[8:]))
    s1.close(), s2.close()
    for f in (p, a, m):
        os.remove(f)
    if not ok:
        raise SystemExit("hidden states differ (%s, rank %d): no timing" % (shape_name, r))
    return ok


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--oracle-layers", type=int, default=4)
    args = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    res = {"gpu": smi[0] if smi else "unknown", "layers": args.layers}
    sh = ggjt.SHAPES["7b"]
    with tempfile.TemporaryDirectory() as d:
        res["checked_equal"] = check_equal(d, "7b", 16, ALPACA) and check_equal(d, "tiny128", 64, ALL7)
        sp = os.path.join(d, "slice.bin")
        ggjt.write_fast_q4_slice(sp, sh, 0, args.layers - 1, seed=0)
        arms = {"plain": None, "r16_wq_wv": os.path.join(d, "a16.bin"), "r64_all7": os.path.join(d, "a64.bin")}
        write_adapter(arms["r16_wq_wv"], sh, range(args.layers), 16, 32, ALPACA)
        write_adapter(arms["r64_all7"], sh, range(args.layers), 64, 128, ALL7)
        capi.lib().b200_device_init(0)
        capi.Slice(sp, 0, 512).close()                     # page cache and modules warm for every arm
        times = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, a in arms.items():
                t0 = time.perf_counter()
                s = capi.Slice(sp, 0, 512, lora=a)
                times[k].append(time.perf_counter() - t0)
                s.close()
        res["load_s_median"] = {k: float(np.median(v)) for k, v in times.items()}
        res["load_s_all"] = times
        import torch
        from torch.profiler import ProfilerActivity, profile
        for k in ("r16_wq_wv", "r64_all7"):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                capi.Slice(sp, 0, 512, lora=arms[k]).close()
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if "k_lora_merge" in e.name]
            res["k_lora_merge_ms_" + k] = {"launches": len(ev),
                                           "total": sum(e.device_time_total for e in ev) / 1e3}
        if os.path.isfile(TOOL):
            n = args.oracle_layers
            full = os.path.join(d, "full.bin")
            sub = ggjt.ModelShape(sh.n_vocab, sh.n_embd, sh.n_mult, sh.n_head, n)
            hp = ggjt.HParams(sub.n_vocab, sub.n_embd, sub.n_mult, sub.n_head, n, sub.n_embd // sub.n_head,
                              ggjt.FTYPE_Q4_0, None)
            src = ggjt.read_file(sp)
            ex = os.path.join(d, "extra.bin")
            ggjt.write_fast_q4_extra(ex, sh, seed=0)
            exf = ggjt.read_file(ex)

            def tensors():
                for f, names in ((exf, ("tok_embeddings.weight", "norm.weight", "output.weight")),
                                 (src, [t for t in src.tensors if int(t.split(".")[1]) < n])):
                    for name in names:
                        t = f.tensors[name]
                        yield name, t.ttype, t.ne, f.read_raw(name)
            ggjt.write_file(full, hp, src.vocab, tensors())
            cores = os.cpu_count()
            # llama.cpp refuses adapter tensors the model lacks: adapters for the n layers it has
            small = {"r16_wq_wv": (16, 32, ALPACA), "r64_all7": (64, 128, ALL7)}
            for k, (r, alpha, mats) in small.items():
                ap_k = os.path.join(d, "oracle_%s.bin" % k)
                write_adapter(ap_k, sh, range(n), r, alpha, mats)
                p = subprocess.run([TOOL, full, ap_k, "-", os.path.join(d, "merged.bin"), str(cores)],
                                   capture_output=True, text=True)
                if p.returncode != 0:
                    res["llama_cpp_cpu_merge_ms_" + k] = "failed: " + p.stderr[-300:]
                    continue
                ms = float(p.stdout.split()[-1])
                res["llama_cpp_cpu_merge_ms_" + k] = {"layers": n, "threads": cores, "ms": ms, "ms_per_layer": ms / n}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
