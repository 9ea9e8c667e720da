"""Per-phase timeline of the persistent decode step (needs an H100): 7B Q4_0, 32 layers, decode at p ~ 260.
Stamps per (CTA, layer): 0 qkv wait done | 1 qkv prologue done | 2 qkv tiles done | 3 attn wait done | 4 attn done |
see `names` below; slot 15 = clock cycles thread 0 waited for ring stages in the layer."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ["B200_PERSIST"] = "1"
os.environ["B200_PTRACE"] = "1"
import bench  # noqa: E402
from distributedllm_b200 import capi, ggjt  # noqa: E402

sh = ggjt.SHAPES["7b"]
nl = int(os.environ.get("TRACE_LAYERS", "8"))
path = bench.slice_file("7b", 0, nl - 1)
sl = capi.Slice(path, 0, 512)
xp = bench.synth_inputs(256, sh.n_embd, 1)
for i in range(0, 256, 64):
    sl.forward(xp[i:i + 64])
bench._h2d(sl, xp[0:1])
for i in range(6):
    sl.forward_device(sl.dev_in, 1, sl.dev_out)
sl.sync()
st = sl.ptrace_read().astype(np.int64)             # [cta][layer][16]
names = ["qkv wait", "qkv pro", "qkv mma", "att wait", "att", "wo wait", "wo preq", "wo mma", "w13 wait", "w13 pro", "w13 mma", "w2 wait",
         "w2 preq", "w2 mma", "w2 publish"]
t0 = st[:, 0, 0][st[:, 0, 0] > 0].min()
print("layer | phase end (us from step start): median / max over the CTAs that ran it   [duration median / max]")
for il in range(min(nl, 4), min(nl, 6)):
    prev = None
    for k, nm in enumerate(names):
        v = st[:, il, k]
        ok = v > 0
        if not ok.any():
            continue
        rel = (v[ok] - t0) / 1e3
        line = "%2d %-10s n=%3d  end %8.2f / %8.2f" % (il, nm, ok.sum(), np.median(rel), rel.max())
        if k > 0:
            pv = st[:, il, k - 1]
            both = ok & (pv > 0)
            if both.any():
                d = (v[both] - pv[both]) / 1e3
                line += "   dur %6.2f / %6.2f (min %5.2f)" % (np.median(d), d.max(), d.min())
        print(line)
wc = st[:, min(nl, 4):min(nl, 6), 15].astype(np.float64)
print("cycles group 0 / warp 0 spent waiting for ring stages, per layer: median %.0f  max %.0f  (x 0.51 ns)" % (np.median(wc), wc.max()))
per_layer = (st[:, 1:, 0].max(axis=0)[1:] - st[:, 1:, 0].max(axis=0)[:-1]) / 1e3 if nl > 2 else []
print("layer period (last CTA's qkv-wait-done to next):", np.round(per_layer, 2))
