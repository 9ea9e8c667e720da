"""Timing probe for the persistent decode step (needs an H100): 7B Q4_0, 32 layers, decode at p ~ 260.
    python scripts/persist_probe.py [cfg ...]      cfg = name:ENV=VAL,ENV=VAL   (B200_* variables read at load)
Prints ms/step per configuration and checks every configuration's outputs against the first (bit patterns)."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from distributedllm_b200 import capi, ggjt  # noqa: E402

cfgs = sys.argv[1:] or ["multi:B200_PERSIST=0", "persist:B200_PERSIST=1"]
sh = ggjt.SHAPES["7b"]
path = bench.slice_file("7b", 0, sh.n_layer - 1)
xp = bench.synth_inputs(256, sh.n_embd, 1)
xs = bench.synth_inputs(64, sh.n_embd, 2)
want = None
for cfg in cfgs:
    name, _, envs = cfg.partition(":")
    for kv in filter(None, envs.split(",")):
        k, v = kv.split("=")
        os.environ[k] = v
    t0 = time.perf_counter()
    sl = capi.Slice(path, 0, 512)
    load_s = time.perf_counter() - t0
    for i in range(0, 256, 64):
        sl.forward(xp[i:i + 64])
    outs = [sl.forward(xs[i:i + 1]) for i in range(8)]
    if want is None:
        want = outs
    bad = sum(int((a.view(np.uint32) != b.view(np.uint32)).sum()) for a, b in zip(outs, want))
    sl.rewind(256)
    bench._h2d(sl, xs[0:1])
    for i in range(8):
        sl.forward_device(sl.dev_in, 1, sl.dev_out)
    sl.sync()
    sl.rewind(256)
    sl.mark(0)
    for i in range(64):
        sl.forward_device(sl.dev_in, 1, sl.dev_out)
    sl.mark(1)
    sl.sync()
    ms = sl.mark_elapsed_ms() / 64
    print("%-28s %8.4f ms/step  %7.1f tok/s  %6.2f us/layer   mismatching floats vs first cfg: %d   load %.2f s"
          % (name, ms, 1e3 / ms, 1e3 * ms / sh.n_layer, bad, load_s), flush=True)
    sl.close()
    for kv in filter(None, envs.split(",")):
        os.environ.pop(kv.split("=")[0], None)
