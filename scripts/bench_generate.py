"""Greedy generation through the host against greedy generation on the device.

    python scripts/bench_generate.py [--reps 5] [--steps 256] [--batches 1,8]

LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU, with an extra-layers file whose output.weight is Q6_K, as
`quantize q4_0` writes it at 7B (ggjt.write_kquant_extra).  Prompt: the 16 tokens 1 + (i * 7919 mod 31999), then --steps
generated tokens, for each of B sessions (session k's prompt is shifted by k so the sessions differ).  Two arms, alternated
in the same process, each timed end to end with a host clock around work that ends in a device synchronise:
  A  the host loop through the C ABI: b200_extra_embed -> b200_mixed_forward / b200_batch_forward -> b200_extra_logits +
     argmax per session (B = 1: b200_session_forward and b200_extra_next_token, the client's path)
  B  the device loop: one b200_generate_greedy call
Every session is cleared before each repetition.  Tokens/s counts generated tokens over all sessions.  The arms' ids must
be identical.  Then, in a profiled window of its own, the Q6_K lm_head alone (b200_extra_logits on --rows rows): the
device time of its kernels from torch.profiler, copies excluded.  Prints the GPU's name and power limit, one line per
batch and per row count, then one JSON line.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributedllm_b200 import capi, ggjt  # noqa: E402
import bench  # noqa: E402


def gpu_card() -> dict:
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().split(", ")
    return {"name": out[0], "power_limit": out[1], "max_sm_clock": out[2]}


def prompts_for(batch):
    return [[1 + ((i + 3 * k) * 7919) % 31999 for i in range(16)] for k in range(batch)]


def host_loop(sl, extra, prompts, n_steps):
    B = len(prompts)
    sessions = list(range(B))
    ids = np.zeros((n_steps, B), np.int32)
    if B == 1:
        toks = prompts[0]
        for step in range(n_steps):
            x = sl.session_forward(0, extra.embed(toks))
            ids[step, 0] = extra.next_token(x)
            toks = [int(ids[step, 0])]
        return ids
    x = sl.mixed_forward(sessions, [len(p) for p in prompts], extra.embed([t for p in prompts for t in p]))
    last = np.cumsum([len(p) for p in prompts]) - 1
    ids[0] = np.argmax(extra.logits(x[last]), axis=1)
    for step in range(1, n_steps):
        x = sl.batch_forward(sessions, extra.embed(ids[step - 1]))
        ids[step] = np.argmax(extra.logits(x), axis=1)
    return ids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--rows", default="1,8,128,512", help="lm_head row counts to time")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_generate.py needs a GPU")
    card = gpu_card()
    print("gpu: %s, power limit %s, max SM clock %s" % (card["name"], card["power_limit"], card["max_sm_clock"]), flush=True)
    sh = ggjt.SHAPES["7b"]
    batches = [int(b) for b in args.batches.split(",") if b]
    n_ctx = 512
    assert 16 + args.steps - 1 <= n_ctx
    sl = capi.Slice(bench.slice_file("7b", 0, sh.n_layer - 1), 0, n_ctx, n_sessions=max(batches + [1]))
    with tempfile.TemporaryDirectory() as d:
        extra_path = os.path.join(d, "extra_7b_q6k.bin")
        ggjt.write_kquant_extra(extra_path, sh, "q4_K_M", seed=bench.SEED)
        extra = capi.Extra(extra_path, 0)
    results = []
    for B in batches:
        prompts = prompts_for(B)
        arms = {"A": lambda: host_loop(sl, extra, prompts, args.steps),
                "B": lambda: capi.generate_greedy([sl], extra, list(range(B)), prompts, args.steps)}
        times = {"A": [], "B": []}
        out = {}
        for rep in range(1 + args.reps):                    # repetition 0 warms up every shape
            for name in ("A", "B") if rep % 2 == 0 else ("B", "A"):
                sl.session_clear(-1)
                sl.sync()
                t0 = time.perf_counter()
                out[name] = arms[name]()
                sl.sync()
                dt = time.perf_counter() - t0
                if rep > 0:
                    times[name].append(B * args.steps / dt)
        same = bool((out["A"] == out["B"]).all())
        ta, tb = statistics.median(times["A"]), statistics.median(times["B"])
        print("B=%d  A host loop %.1f tok/s (%.1f..%.1f)  B device loop %.1f tok/s (%.1f..%.1f)  B/A %.3f  ids %s"
              % (B, ta, min(times["A"]), max(times["A"]), tb, min(times["B"]), max(times["B"]), tb / ta,
                 "identical" if same else "DIFFER"), flush=True)
        results.append({"batch": B, "host_loop_tok_s": ta, "device_loop_tok_s": tb, "device_over_host": tb / ta,
                        "host_loop_range": [min(times["A"]), max(times["A"])],
                        "device_loop_range": [min(times["B"]), max(times["B"])], "ids_identical": same,
                        "distinct_ids": int(len(set(out["B"].ravel().tolist())))})
    # the lm_head alone: device time of its kernels (torch.profiler, copies excluded), in a profiled window of its own
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    lm = {}
    for n in [int(r) for r in args.rows.split(",") if r]:
        x = rng.standard_normal((n, sh.n_embd), dtype=np.float32)
        for _ in range(3):
            extra.logits(x)
        calls = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(calls):
                extra.logits(x)
        kern = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            if t and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
                kern[ev.key] = t / calls / 1e3
        lm[n] = sum(kern.values())
        print("lm_head (Q6_K, 32000 x 4096) %3d row(s): %.4f ms of kernels per call, %.4f ms per row  [%s]"
              % (n, lm[n], lm[n] / n, ", ".join("%s %.4f" % (k.split("(")[0][:40], v) for k, v in kern.items())), flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "generate_greedy", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "prompt_tokens": 16, "steps": args.steps, "reps": args.reps, "gpu": card, "results": results,
                      "lm_head_ms_per_call": {str(k): v for k, v in lm.items()}}))
    return 0 if all(r["ids_identical"] for r in results) else 1


if __name__ == "__main__":
    sys.exit(main())
