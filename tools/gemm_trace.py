#!/usr/bin/env python3
"""Per-role waiting time of every tensor-core GEMM launch of a workload (debug aid; TB200_GEMM_TRACE=1 makes the launcher
synchronise and print cycle counters, so the graph is built without CUDA-graph capture)."""
import os
import sys

os.environ["TB200_GEMM_TRACE"] = "1"
os.environ.setdefault("TB200_LIB", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "build", "trace", "libtengine_b200_trace.so"))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tengine_b200 import abi, workloads  # noqa: E402
from tengine_b200 import runtime as rt  # noqa: E402

batch = int(sys.argv[1]) if len(sys.argv) > 1 else 256
g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=batch, res=224)
ctx = rt.Context(0)
graph = rt.Graph(ctx, g, abi.PRERUN_NO_GRAPH)
graph.upload(0, b.random_input(1))
graph.sync()
graph.profile()
ms = graph.profile()
kern = graph.layer_kernels()
for i, (k, t) in enumerate(zip(kern, ms)):
    print(f"layer {i:2d} {k:24s} {t * 1000:8.1f} us")
