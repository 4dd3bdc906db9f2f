#!/usr/bin/env python3
"""Per-layer kernel times of a workload (events around every launch, no CUDA graph), each beside its floor:
max(bytes / HBM bandwidth, int8 ops / int8 tensor peak), with bytes and ops from the layer shapes as bench.py counts them
(input + output activations, weights and bias; 2 ops per MAC).  The per-kernel-family sums follow the table."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tengine_b200 import abi, workloads  # noqa: E402
from tengine_b200 import runtime as rt  # noqa: E402

HBM_GBS = 3350.0  # H100 SXM data sheet, HBM3
INT8_TOPS_SHEET = 1979.0  # H100 SXM data sheet, dense int8

batch = int(sys.argv[1]) if len(sys.argv) > 1 else 256
net = sys.argv[2] if len(sys.argv) > 2 else "mobilenet_v1"
dt = abi.DT_UINT8 if (len(sys.argv) > 3 and sys.argv[3] == "uint8") else abi.DT_INT8
res = 416 if net == "yolov3_tiny" else (640 if net == "yolov5s" else 224)
g, b = getattr(workloads, net)(dt, batch=batch, res=res)
ctx = rt.Context(0)
try:
    tops = ctx.probe_int8_tops()
    tops_src = "measured (tb200_probe_int8_tops)"
except Exception:
    tops = 0.0
if tops <= 100:
    tops, tops_src = INT8_TOPS_SHEET, "data sheet"
graph = rt.Graph(ctx, g, abi.PRERUN_NO_GRAPH)
graph.upload(0, b.random_input(1))
graph.sync()
for _ in range(3):
    graph.profile()
ms = np.mean([graph.profile() for _ in range(5)], axis=0)
print(f"floors: HBM {HBM_GBS:.0f} GB/s (data sheet), int8 {tops:.0f} TOP/s ({tops_src})")
fam = {}
for i, (k, t) in enumerate(zip(graph.layer_kernels(), ms)):
    L = g.layers[i]
    byts = float(g.numel(L["inputs"][0]) + g.numel(L["output"]))
    ops = 0.0
    if L["weight"] is not None:
        byts += L["weight"].size + (4 * g.dims(L["output"])[1] if L["bias"] is not None else 0)
        ops = 2.0 * g.numel(L["output"]) * (L["weight"].size // g.dims(L["output"])[1])
    t_hbm, t_ops = byts / (HBM_GBS * 1e9) * 1e6, ops / (tops * 1e12) * 1e6
    floor = max(t_hbm, t_ops)
    f = fam.setdefault(k, [0, 0.0, 0.0])
    f[0] += 1
    f[1] += t * 1000
    f[2] += floor
    print(f"layer {i:2d} {k:26s} {t * 1000:8.1f} us   floor {floor:7.1f} us ({'hbm' if t_hbm >= t_ops else 'int8'}, x{t * 1000 / floor if floor else 0:5.1f})"
          f"   out {tuple(g.dims(L['output']))}")
total = ms.sum() * 1000
for k, (n, t, fl) in sorted(fam.items(), key=lambda kv: -kv[1][1]):
    print(f"family {k:26s} {n:3d} layers {t:8.1f} us ({100 * t / total:4.1f} %)   floor {fl:7.1f} us")
print("total", total)
