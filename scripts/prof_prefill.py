"""Prefill throughput of the 7B slice: exact mode (NC=8 dp4a columns) vs fast mode (wgmma), N tokens in one call."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from distributedllm_b200 import capi
import bench
L = int(os.environ.get("PROF_LAYERS", "4")); N = int(os.environ.get("PROF_TOKENS", "512"))
path = bench.slice_file("7b", 0, L - 1)
sl = capi.Slice(path, 0, 512)
x = bench.synth_inputs(N, sl.n_embd, 1)
bench._h2d(sl, x)
for mode in (0, 1):
    sl.set_fast_prefill(bool(mode), 32)
    ts = []
    for it in range(4):
        sl.clear_context()
        sl.mark(0); sl.forward_device(sl.dev_in, N, sl.dev_out); sl.mark(1); sl.sync()
        ts.append(sl.mark_elapsed_ms())
    ms = min(ts[1:])
    flops = 2.0 * N * L * (4 * 4096 * 4096 + 3 * 4096 * 11008)
    print("%s prefill: %d tokens x %d layers  %.3f ms  -> %.0f tok/s (32-layer equiv %.0f tok/s), %.1f TFLOP/s" %
          ("fast(wgmma)  " if mode else "exact(dp4a) ", N, L, ms, N / (ms / 1e3), N / (ms * 32 / L / 1e3), flops / (ms / 1e3) / 1e12))
    sl.profile(True)
    sl.clear_context(); sl.forward_device(sl.dev_in, N, sl.dev_out)
    ms_c, cnt = sl.profile_read(); sl.profile(False)
    names = ("qkv", "rope", "attn", "wo", "w13", "w2", "advance")
    print("   per class ms (all layers): " + "  ".join("%s %.3f(%d)" % (n, m, c) for n, m, c in zip(names, ms_c, cnt) if c))
sl.close()
