#!/usr/bin/env python3
"""Stage-by-stage check of the single-process multi-GPU path on a real multi-GPU box.  Torch-free (graphs come pickled from
tools/debug_multi_graphs.pkl, so a fresh box does not spend a minute importing torch); every variant runs in its own subprocess
with a watchdog that dumps the Python stack and exits when a stage hangs.
usage: debug_multi.py [n_gpus]            all variants
       debug_multi.py --one <variant>     (internal) one variant in this process"""
import faulthandler
import os
import pickle
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
T0 = time.time()
WATCHDOG = float(os.environ.get("DEBUG_MULTI_WATCHDOG", "25"))


def stage(msg):
    print(f"  [{time.time() - T0:5.1f}s] {msg}", flush=True)
    faulthandler.cancel_dump_traceback_later()
    faulthandler.dump_traceback_later(WATCHDOG, exit=True)


def one(devices, net):
    import numpy as np

    from tengine_b200 import runtime as rt

    g, x = pickle.load(open(os.path.join(ROOT, "tools", "debug_multi_graphs.pkl"), "rb"))[net]
    stage(f"devices visible {rt.device_count()}, group {devices}, net {net}")
    ctx = rt.Context(devices=devices)
    stage(f"context created, weight broadcast = {ctx.broadcast_kind if len(devices) > 1 else 'n/a'}")
    from tengine_b200 import abi

    flags = abi.PRERUN_NO_GRAPH if os.environ.get("DEBUG_MULTI_FLAGS") == "nograph" else abi.PRERUN_DEFAULT
    gr = rt.Graph(ctx, g, flags)
    stage(f"prerun done, shards {gr.shards()}")
    y = gr.run([x])
    stage("first run done")
    y2 = gr.run([x])
    stage("second run done")
    gr.close()
    ctx.close()
    one_ctx = rt.Context(devices=[devices[0]])
    g1 = rt.Graph(one_ctx, g)
    y1 = g1.run([x])
    g1.close()
    one_ctx.close()
    ok = all(np.array_equal(a, c) and np.array_equal(a, d) for a, c, d in zip(y, y1, y2))
    stage(f"group == single GPU {devices[0]}: {ok}")
    faulthandler.cancel_dump_traceback_later()
    print("  VARIANT OK" if ok else "  VARIANT MISMATCH", flush=True)


VARIANTS = {  # name -> (devices as a function of n, net, extra environment)
    "nccl_mobilenet": (lambda n: list(range(n)), "mobilenet", {}),
    "nccl_yolo_u8": (lambda n: list(range(n)), "yolo", {}),
    "memcpy_peer_mobilenet": (lambda n: list(range(n)), "mobilenet", {"TB200_NO_NCCL": "1"}),
    "gpu1_alone": (lambda n: [1], "mobilenet", {}),
    "nccl_no_graph_capture": (lambda n: list(range(n)), "mobilenet", {"DEBUG_MULTI_FLAGS": "nograph"}),
}

if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--one":
        name, n = sys.argv[2], int(sys.argv[3])
        devs, net, _ = VARIANTS[name]
        one(devs(n), net)
        sys.exit(0)
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    names = sys.argv[2].split(",") if len(sys.argv) > 2 else list(VARIANTS)
    good = 0
    for name in names:
        env = dict(os.environ)
        env.update(VARIANTS[name][2])
        print(f"=== {name} {VARIANTS[name][2]}", flush=True)
        try:
            r = subprocess.run([sys.executable, "-X", "faulthandler", os.path.abspath(__file__), "--one", name, str(n)], env=env, timeout=4 * WATCHDOG,
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            out = r.stdout
        except subprocess.TimeoutExpired as e:
            out = (e.stdout or "") + "\n  TIMEOUT (killed)"
        lines = out.splitlines()
        print("\n".join(l[:400] for l in lines[-25:]), flush=True)
        good += "VARIANT OK" in out
    print(f"{good} of {len(names)} variants OK", flush=True)
    if good == len(names):
        print("OK", flush=True)
