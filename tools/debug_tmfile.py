#!/usr/bin/env python3
"""Debug helper: the same model through (a) the direct ABI and (b) run_graph() on device B200 from the tmfile, each in its own
process with the engine's per-layer output hashes (TB200_DEBUG_HASH=2); prints the first layers whose hashes differ.
usage: debug_tmfile.py [direct|tmfile]   (no argument: run both and compare)"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run(route):
    from oracle.pyoracle import Oracle, Reference, run_tmfile
    from tengine_b200 import abi, workloads
    from tengine_b200 import runtime as rt

    g, b = workloads.resnet50(abi.DT_UINT8, batch=4, softmax=True)
    outs = [g.outputs[0], g.layers[-1]["inputs"][0]]
    g.mark_output(outs[1])
    x = b.random_input(21)
    want = Oracle().run(g, [x], uint8_mode=0)
    if route == "direct":
        ctx = rt.Context(0)
        gr = rt.Graph(ctx, g)
        got = gr.run([x])
        print("kernels:", gr.layer_kernels(), file=sys.stderr)
        gr.close()
    else:
        ref = Reference(libdir=os.path.join(ROOT, "oracle", "_ref", "tengine"))
        got, _ = run_tmfile(ref, os.path.join(ROOT, "oracle/_ref/models/resnet50_uint8.tmfile"), x, [g.dims(t) for t in outs], device="B200")
    for o, t, nm in zip(got, outs, ("prob", "fc")):
        d = np.abs(o.astype(int) - want[t].astype(int))
        print(route, nm, "max diff", d.max(), "count", int((d > 0).sum()), flush=True)


if len(sys.argv) > 1:
    run(sys.argv[1])
else:
    logs = {}
    for route in ("direct", "tmfile"):
        env = dict(os.environ, TB200_DEBUG_HASH="2")
        r = subprocess.run([sys.executable, os.path.abspath(__file__), route], capture_output=True, text=True, env=env)
        print(r.stdout.strip())
        logs[route] = [l for l in r.stderr.splitlines() if l.startswith("[tb200 dbg]")]
        print(route, len(logs[route]), "debug lines; stderr tail:", r.stderr.strip().splitlines()[-2:] if not logs[route] else "")
    a, b = logs["direct"], logs["tmfile"]
    # layer numbering is the same (same node order); compare by position
    shown = 0
    for la, lb in zip(a, b):
        if la.split("hash")[-1] != lb.split("hash")[-1] or ("pack layer" in la and la != lb):
            print("DIFF\n  direct:", la, "\n  tmfile:", lb)
            shown += 1
            if shown >= 4:
                break
    if not shown:
        print("all", len(a), "hash lines equal")
