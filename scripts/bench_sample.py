"""Sampled generation through the host against sampled generation on the device.

    python scripts/bench_sample.py [--reps 5] [--steps 256] [--batches 1,8]

bench_generate.py's model: LLaMA-7B Q4_0 (bench.py's synthetic 32-layer file) on one GPU, with a Q6_K output.weight,
a 16-token prompt and --steps generated tokens for each of B sessions.  Three arms, alternated in the same process, each
timed end to end with a host clock around work that ends in a device synchronise:
  A  the host loop: b200_extra_embed -> b200_mixed_forward / b200_batch_forward (B = 1: b200_session_forward) ->
     b200_extra_logits -> client.Sampler per session on numpy.random.Philox(key=seed_k), T 0.7, rp 1.1
  B  the device loop: one b200_generate_sample call, same settings and keys
  C  the device loop, greedy: one b200_generate_greedy call
Every session is cleared before each repetition.  Tokens/s counts generated tokens over all sessions.  A and B must agree
under the ambiguity rule: ids equal wherever the draw u lies more than 1e-9 from every boundary of the host's CDF
(checked in the warm-up repetition; a session is compared up to its first ambiguous draw).  Then, in a profiled window of
its own, k_sample_rows alone (b200_extra_sample on --rows rows of 32000 logits): its device time from torch.profiler,
copies excluded.  Prints the GPU's name and power limit, one line per batch and per row count, then one JSON line.
Exits non-zero if A and B disagree outside the ambiguity rule.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributedllm_b200 import capi, ggjt  # noqa: E402
from distributedllm_b200.client import Sampler, _softmax  # noqa: E402
import bench  # noqa: E402
from bench_generate import gpu_card, prompts_for  # noqa: E402

T, RP = 0.7, 1.1


def margin(logits, prev, u):
    """Distance from u to the nearest boundary of the host's CDF (Sampler's arithmetic, then Generator.choice's)."""
    ids = np.arange(len(logits))
    seen = np.isin(ids, prev)
    cdf = _softmax(np.asarray(logits) / ((seen * RP + ~seen) * (T + 10 ** (-5)))).cumsum()
    cdf /= cdf[-1]
    return float(np.min(np.abs(cdf - u)))


def host_loop(sl, extra, prompts, n_steps, seeds, check=False):
    """-> (ids [n_steps][B], per session the number of draws before its first ambiguous one (check only))."""
    B = len(prompts)
    sessions = list(range(B))
    samplers = [Sampler(T, RP, rng=np.random.Generator(np.random.Philox(key=s))) for s in seeds]
    ids = np.zeros((n_steps, B), np.int32)
    safe = [n_steps] * B

    def pick(step, logits):
        for k in range(B):
            if check and safe[k] == n_steps:
                u = (int(np.random.Philox(key=seeds[k]).random_raw(step + 1)[step]) >> 11) * 2.0 ** -53
                if margin(logits[k], samplers[k].previous_ids, u) <= 1e-9:
                    safe[k] = step
            ids[step, k] = samplers[k](logits[k])

    if B == 1:
        toks = prompts[0]
        for step in range(n_steps):
            x = sl.session_forward(0, extra.embed(toks))
            pick(step, extra.logits(x)[-1:])
            toks = [int(ids[step, 0])]
        return ids, safe
    x = sl.mixed_forward(sessions, [len(p) for p in prompts], extra.embed([t for p in prompts for t in p]))
    pick(0, extra.logits(x[np.cumsum([len(p) for p in prompts]) - 1]))
    for step in range(1, n_steps):
        x = sl.batch_forward(sessions, extra.embed(ids[step - 1]))
        pick(step, extra.logits(x))
    return ids, safe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--rows", default="1,8,64", help="k_sample_rows row counts to time")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sample.py needs a GPU")
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
    results, ok = [], True
    for B in batches:
        prompts = prompts_for(B)
        seeds = [1000 + 7 * k for k in range(B)]
        arms = {"A": lambda: host_loop(sl, extra, prompts, args.steps, seeds)[0],
                "B": lambda: capi.generate_sample([sl], extra, list(range(B)), prompts, args.steps, T, RP, seeds),
                "C": lambda: capi.generate_greedy([sl], extra, list(range(B)), prompts, args.steps)}
        sl.session_clear(-1)
        host_ids, safe = host_loop(sl, extra, prompts, args.steps, seeds, check=True)
        times = {a: [] for a in arms}
        out, sampled = {}, []
        for rep in range(1 + args.reps):                    # repetition 0 warms up every shape
            order = ("A", "B", "C") if rep % 2 == 0 else ("C", "B", "A")
            for name in order:
                sl.session_clear(-1)
                sl.sync()
                t0 = time.perf_counter()
                out[name] = arms[name]()
                sl.sync()
                dt = time.perf_counter() - t0
                if rep > 0:
                    times[name].append(B * args.steps / dt)
                if name == "B":
                    sampled.append(out["B"])
        dev = out["B"]
        disagree = sum(int((host_ids[:safe[k], k] != dev[:safe[k], k]).sum()) for k in range(B))
        ambiguous = sum(1 for s in safe if s < args.steps)
        same_device = all((o == dev).all() for o in sampled)
        ok &= disagree == 0 and same_device
        med = {a: statistics.median(v) for a, v in times.items()}
        print("B=%d  A host loop + Sampler %.1f tok/s (%.1f..%.1f)  B device sampling %.1f tok/s (%.1f..%.1f)  "
              "C device greedy %.1f tok/s (%.1f..%.1f)  B/A %.3f  B/C %.3f  A vs B: %d ids differ outside the ambiguity "
              "rule, %d sessions hit an ambiguous draw; device ids %s across repetitions, %d distinct"
              % (B, med["A"], min(times["A"]), max(times["A"]), med["B"], min(times["B"]), max(times["B"]),
                 med["C"], min(times["C"]), max(times["C"]), med["B"] / med["A"], med["B"] / med["C"], disagree, ambiguous,
                 "identical" if same_device else "DIFFER", len(set(dev.ravel().tolist()))), flush=True)
        results.append({"batch": B, "host_sampler_tok_s": med["A"], "device_sample_tok_s": med["B"],
                        "device_greedy_tok_s": med["C"], "host_sampler_range": [min(times["A"]), max(times["A"])],
                        "device_sample_range": [min(times["B"]), max(times["B"])],
                        "device_greedy_range": [min(times["C"]), max(times["C"])],
                        "ids_differ_outside_ambiguity": disagree, "ambiguous_sessions": ambiguous,
                        "device_repeatable": same_device, "distinct_ids": int(len(set(dev.ravel().tolist())))})
    # k_sample_rows alone: device time from torch.profiler (copies excluded), in a profiled window of its own
    from torch.profiler import ProfilerActivity, profile
    rng = np.random.default_rng(0)
    kern_ms = {}
    for n in [int(r) for r in args.rows.split(",") if r]:
        x = (rng.standard_normal((n, sh.n_vocab)) * 3).astype(np.float32)
        seeds = list(range(1, n + 1))
        hist = [rng.integers(0, sh.n_vocab, 64).tolist() for _ in range(n)]
        for _ in range(3):
            extra.sample(x, T, RP, seeds, 0, hist)
        calls = 20
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for c in range(calls):
                extra.sample(x, T, RP, seeds, c, hist)
        kern = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            if t and "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
                kern[ev.key] = t / calls / 1e3
        kern_ms[n] = sum(kern.values())
        print("k_sample_rows %2d row(s) of %d: %.4f ms per call  [%s]"
              % (n, sh.n_vocab, kern_ms[n], ", ".join("%s %.4f" % (k.split("(")[0][:40], v) for k, v in kern.items())),
              flush=True)
    extra.close()
    sl.close()
    print(json.dumps({"bench": "generate_sample", "model": "LLaMA-7B Q4_0 (synthetic), 32 layers, Q6_K output.weight, one GPU",
                      "temperature": T, "repeat_penalty": RP, "prompt_tokens": 16, "steps": args.steps, "reps": args.reps,
                      "gpu": card, "results": results, "k_sample_rows_ms": {str(k): v for k, v in kern_ms.items()}}))
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
