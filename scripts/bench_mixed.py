"""A prompt chunk riding along with eight decode steps: one mixed pass against two separate passes.

    python scripts/bench_mixed.py [--reps 30] [--chunks 16,64,256]

LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU, one slice with 9 sessions.  Sessions 0..7 are prefilled to
256 positions and decode one token each; session 8 receives a prompt chunk of C tokens at position 0.  Two arms, alternated
in the same process, each timed with CUDA events on the slice's stream (b200_slice_mark) and reported as the median over
the repetitions:
  A  one mixed pass, counts [1] * 8 + [C]                       (b200_mixed_forward_device)
  B  a batched step of the 8, then the chunk of session 8 alone (b200_batch_forward_device + b200_session_forward_device)
Every session is rewound before each repetition, so positions are the same in every one; every shape is warmed up first.
Each arm is timed from an idle stream (reading the elapsed time synchronises, and the rewinds synchronise too), so both
arms' times are end to end: they include the host enqueue of every launch and the upload of the pass's column table (a
pageable host-to-device copy: one in A, one for B's batched step), not only kernel time.
The outputs of the last A and B repetitions are compared bit for bit.  Prints the GPU's name and power limit, one line per
chunk size, then one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributedllm_b200 import capi, ggjt  # noqa: E402
import bench  # noqa: E402

N_DEC, PAST, N_CTX = 8, 256, 512


def gpu_card() -> dict:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit": out[1], "max_sm_clock": out[2]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--chunks", default="16,64,256")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    E = sh.n_embd
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, N_CTX, n_sessions=N_DEC + 1)
    rng = np.random.default_rng(0)
    for k in range(N_DEC):
        sl.session_forward(k, rng.standard_normal((PAST, E), dtype=np.float32))
    dec = list(range(N_DEC))
    results = []
    for C in [int(c) for c in args.chunks.split(",")]:
        x = torch.from_numpy(rng.standard_normal((N_DEC + C, E), dtype=np.float32)).cuda()
        out_a = torch.empty_like(x)
        out_b = torch.empty_like(x)
        torch.cuda.synchronize()
        row = 4 * E

        def rewind():
            for k in dec:
                sl.session_rewind(k, PAST)
            sl.session_rewind(N_DEC, 0)

        def arm_a():
            sl.mixed_forward_device(dec + [N_DEC], [1] * N_DEC + [C], x.data_ptr(), out_a.data_ptr())

        def arm_b():
            sl.batch_forward_device(dec, x.data_ptr(), out_b.data_ptr())
            capi.check(capi.lib().b200_session_forward_device(sl.handle, N_DEC, capi.C.c_void_p(x.data_ptr() + N_DEC * row), C,
                                                              capi.C.c_void_p(out_b.data_ptr() + N_DEC * row), 0))

        times = {"A": [], "B": []}
        for rep in range(args.warmup + args.reps):
            for name, arm in (("A", arm_a), ("B", arm_b)) if rep % 2 == 0 else (("B", arm_b), ("A", arm_a)):
                rewind()
                sl.mark(0)
                arm()
                sl.mark(1)
                ms = sl.mark_elapsed_ms()
                if rep >= args.warmup:
                    times[name].append(ms)
        sl.sync()
        torch.cuda.synchronize()
        a = out_a.cpu().numpy().view(np.uint32)
        b = out_b.cpu().numpy().view(np.uint32)
        differ = int((a != b).sum())
        ma, mb = statistics.median(times["A"]), statistics.median(times["B"])
        print("C=%3d  A mixed pass %.3f ms (%.3f..%.3f)  B batch + chunk %.3f ms (%.3f..%.3f)  B/A %.3f  outputs %s (%d floats differ)"
              % (C, ma, min(times["A"]), max(times["A"]), mb, min(times["B"]), max(times["B"]), mb / ma,
                 "bit-identical" if differ == 0 else "DIFFER", differ), flush=True)
        results.append({"chunk": C, "mixed_ms_median": ma, "separate_ms_median": mb, "separate_over_mixed": mb / ma,
                        "mixed_ms_range": [min(times["A"]), max(times["A"])],
                        "separate_ms_range": [min(times["B"]), max(times["B"])], "differing_floats": differ})
    sl.close()
    print(json.dumps({"bench": "mixed_pass", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, one GPU",
                      "decoders": N_DEC, "decoder_position": PAST, "reps": args.reps, "gpu": card, "results": results}))
    return 0 if all(r["differing_floats"] == 0 for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
