#!/usr/bin/env python3
"""On-GPU probe of the tensor-core GEMM path: for each 1x1-conv shape run the tensor-core path and the CUDA-core
cross-check path through the C ABI and compare bytes.  Each shape runs in its own subprocess so that a device trap in one
configuration does not poison the others.  Usage: python tools/gemm_probe.py [--one n,c,h,w,oc]"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(1, 16, 8, 8, 16), (1, 32, 16, 16, 64), (2, 64, 9, 9, 32), (1, 128, 12, 12, 128), (1, 256, 14, 14, 256),
          (1, 512, 7, 7, 1024), (2, 1024, 7, 7, 1000), (1, 48, 5, 5, 24), (8, 32, 112, 112, 64), (1, 1024, 1, 1, 1000)]


def one(shape):
    from tengine_b200 import abi
    from tengine_b200 import runtime as rt
    from tengine_b200.graphdef import GraphDef

    n, c, h, w, oc = shape
    rng = np.random.default_rng(1)
    g = GraphDef(abi.DT_INT8)
    x = g.input(n, c, h, w, 0.02)
    wq = rng.integers(-127, 128, (oc, c, 1, 1)).astype(np.int8)
    ws = rng.uniform(0.001, 0.01, oc)
    b = rng.integers(-2000, 2000, oc).astype(np.int32)
    y = g.conv(x, wq, b, ws, 0.02 * 0.0055 * np.sqrt(c) * 73 * 73 / 100, activation=0)
    g.mark_output(y)
    xin = rng.integers(-127, 128, (n, c, h, w)).astype(np.int8)
    ctx = rt.Context(0)
    gr = rt.Graph(ctx, g, abi.PRERUN_NO_TENSORCORE)
    ref = gr.run([xin])[0]
    gr.close()
    # numpy check of the cross-check path itself (int8 HCL recipe)
    acc = np.einsum("nchw,oc->nohw", xin.astype(np.int64), wq[:, :, 0, 0].astype(np.int64)) + b.reshape(1, -1, 1, 1)
    f = (acc.astype(np.float32) * np.float32(0.02)) * ws.astype(np.float32).reshape(1, -1, 1, 1)
    f = np.maximum(f, 0)
    q = f / np.float32(g.tensors[y]["scale"])
    qn = np.clip(np.where(q >= 0, np.floor(q + 0.5), np.ceil(q - 0.5)), -127, 127).astype(np.int8)
    print(f"shape {shape}: cudacore vs numpy mismatches {(qn != ref).sum()} / {ref.size}", flush=True)
    gr = rt.Graph(ctx, g)
    print("  kernel:", gr.layer_kernels(), flush=True)
    got = gr.run([xin])[0]
    gr.close()
    bad = got != ref
    print(f"  tensor-core vs cudacore mismatches {bad.sum()} / {ref.size}", flush=True)
    if bad.any():
        idx = np.argwhere(bad)
        print("  first bad (n,oc,h,w):", idx[:6].tolist(), "got", got[bad][:6].tolist(), "want", ref[bad][:6].tolist())
        print("  bad by oc%16:", np.bincount(idx[:, 1] % 16, minlength=16).tolist())
        pix = (idx[:, 2] * w + idx[:, 3]) + idx[:, 0] * h * w
        print("  bad by row%8:", np.bincount(pix % 8, minlength=8).tolist(), " rows>=128:", int((pix >= 128).sum()))
    ctx.close()


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--one":
        one(tuple(int(v) for v in sys.argv[2].split(",")))
        sys.exit(0)
    for s in SHAPES:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", ",".join(map(str, s))], capture_output=True,
                           text=True, timeout=180)
        print(r.stdout.strip())
        if r.returncode != 0:
            print(f"  shape {s}: FAILED rc={r.returncode}: {r.stderr.strip()[-600:]}")
