"""Prefill throughput probe (needs an H100): a 4-layer LLaMA-7B Q4_0 slice, one 512-token prompt in 64- / 512-token calls.
    exact   the bit-exact multi-column k_gemv path            fast2   wgmma + tensor-map TMA, 128 x 256 tiles (fastgemm2.cuh)
Prints ms per call and the 32-layer-equivalent tokens/s; checks fast modes against exact (relative RMS)."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import bench
from distributedllm_b200 import capi, ggjt

L = int(os.environ.get("PROF_LAYERS", "4"))
sh = ggjt.SHAPES["7b"]
wt = os.environ.get("PROBE_WT", "q4_0")
path = bench.slice_file("7b", 0, L - 1)
x = bench.synth_inputs(512, sh.n_embd, 1)
ref = None
for name, env, chunk in (("exact", {}, 64), ("fast2", {"B200_FAST_PREFILL": "1"}, 512), ("fast2/256", {"B200_FAST_PREFILL": "1"}, 256)):
    os.environ.update(env)
    sl = capi.Slice(path, 0, 512)
    outs = []
    for rep in range(3):
        sl.clear_context()
        sl.sync()
        t0 = time.perf_counter()
        outs = [sl.forward(x[i:i + chunk]) for i in range(0, 512, chunk)]
        sl.sync()
        dt = time.perf_counter() - t0
    y = np.concatenate(outs)
    if ref is None:
        ref = y
    rel = float(np.sqrt(np.mean((y - ref) ** 2)) / np.sqrt(np.mean(ref ** 2)))
    print("%-10s chunk %3d: %7.2f ms per 512 tokens on %d layers -> %8.0f tok/s (32-layer equivalent)   rel RMS vs exact %.2e"
          % (name, chunk, 1e3 * dt, L, 512 / (dt * 32 / L), rel), flush=True)
    sl.close()
    for k in env:
        os.environ.pop(k)
