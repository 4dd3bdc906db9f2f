#!/usr/bin/env python3
"""Times running a prepared graph on fewer images than it was prepared for (tb200_graph_set_batch), on one GPU.

MobileNet-v1 int8 at 224x224 (random weights, seeded), prepared at 256.  For each n in {1, 8, 32, 64, 128, 255}, alternated in one
process, with a host clock around work that ends in a synchronise:
 (a) set_batch(n) + launch + sync, n being the cached other batch (the switch back from 256 costs a drain and nothing else);
 (b) the padded full batch a caller pays without set_batch: launch + sync at 256;
 (c) launch + sync of a graph prepared at n, the lower bound;
 (d) the first set_batch(n): every step list rebuilt and the CUDA graphs captured for n (the previous cached batch was another n);
 (e) a fresh prerun at n (graph planned, weights packed and uploaded, CUDA graphs captured).
The same for tb200_graph_run with pageable numpy buffers (registered in place by the first call): set_batch(n) + run of n images
(a) against a run of the padded 256 (b).  Median, minimum and maximum of the repetitions ((e): of --prerun-reps).  The outputs at
n are checked against the full batch's first n images and against the graph prepared at n.  Prints the card name and power limit
first, and fails without a GPU.  usage: partial_batch_times.py [--reps N] [--prerun-reps N] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

BATCH, NS = 256, (1, 8, 32, 64, 128, 255)


def stats(ts):
    return {"ms_median": float(np.median(ts)) * 1e3, "ms_min": float(np.min(ts)) * 1e3, "ms_max": float(np.max(ts)) * 1e3}


def timed(f):
    t0 = time.perf_counter()
    f()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--prerun-reps", type=int, default=3)
    ap.add_argument("--out", help="directory for partial_batch_times.json")
    a = ap.parse_args()
    from tengine_b200 import abi, workloads
    from tengine_b200 import runtime as rt

    if rt.device_count() < 1:
        print("no CUDA device: every number is not measured", file=sys.stderr)
        return 2
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    print("card (name, power limit, max SM clock):", card)

    ctx = rt.Context(0)
    make = lambda n: workloads.mobilenet_v1(abi.DT_INT8, batch=n, res=224)[0]  # noqa: E731
    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=BATCH, res=224)
    x = b.random_input(1)
    out_shape = g.dims(g.outputs[0])
    gr = rt.Graph(ctx, g)
    full = gr.run([x])[0]
    prepared = {n: rt.Graph(ctx, make(n)) for n in NS}
    res = {"card": card, "model": "mobilenet_v1 int8 224x224", "prepared_batch": BATCH, "reps": a.reps, "prerun_reps": a.prerun_reps}
    T = {n: {k: [] for k in ("a", "b", "c", "d", "e", "run_a", "run_b")} for n in NS}
    # pageable caller buffers of n images and of the padded batch, registered by a first run
    xs = {n: np.array(x[:n]) for n in NS}
    ys = {n: np.empty((n,) + tuple(out_shape[1:]), full.dtype) for n in NS}
    y_full = np.empty(out_shape, full.dtype)

    def launch_sync(graph):
        graph.launch()
        graph.sync()

    for n in NS:  # warm every shape and buffer the timed window uses
        prepared[n].run([xs[n]])
        launch_sync(prepared[n])
        gr.set_batch(n)
        gr.run([xs[n]], [ys[n]])
        launch_sync(gr)
        gr.set_batch(BATCH)
    gr.run([x], [y_full])
    for rep in range(a.reps):
        for n in NS:
            gr.set_batch(BATCH)
            T[n]["d"].append(timed(lambda: gr.set_batch(n)))  # the cached other batch was the previous n: rebuild + capture
            launch_sync(gr)
            gr.set_batch(BATCH)
            T[n]["b"].append(timed(lambda: launch_sync(gr)))
            T[n]["a"].append(timed(lambda: (gr.set_batch(n), launch_sync(gr))))
            T[n]["c"].append(timed(lambda: launch_sync(prepared[n])))
            gr.set_batch(BATCH)
            T[n]["run_b"].append(timed(lambda: gr.run([x], [y_full])))
            T[n]["run_a"].append(timed(lambda: (gr.set_batch(n), gr.run([xs[n]], [ys[n]]))))
    equal = True
    for n in NS:
        gr.set_batch(n)
        y_n = gr.run([xs[n]])[0]
        equal &= bool(np.array_equal(y_n, full[:n]) and np.array_equal(y_n, prepared[n].run([xs[n]])[0]))
    gr.set_batch(BATCH)
    for rep in range(a.prerun_reps):
        for n in NS:
            gn = make(n)
            t0 = time.perf_counter()
            h = rt.Graph(ctx, gn)
            T[n]["e"].append(time.perf_counter() - t0)
            h.close()
    names = {"a": "set_batch_launch_sync", "b": "padded_full_batch_launch_sync", "c": "prepared_at_n_launch_sync",
             "d": "first_set_batch", "e": "fresh_prerun", "run_a": "run_pageable_set_batch", "run_b": "run_pageable_padded_full_batch"}
    for n in NS:
        res[str(n)] = {names[k]: stats(v) for k, v in T[n].items()}
        print(f"n={n}", json.dumps(res[str(n)]))
    res["results_equal"] = equal
    print("outputs at n equal the full batch's first n and the graph prepared at n:", equal)
    print(f"{'n':>4} {'(a) ms':>8} {'(b) ms':>8} {'(c) ms':>8} {'(d) ms':>8} {'(e) ms':>9} {'run(a)':>8} {'run(b)':>8}   (medians)")
    for n in NS:
        r = res[str(n)]
        print(f"{n:>4} " + " ".join(f"{r[names[k]]['ms_median']:>{9 if k == 'e' else 8}.3f}" for k in ("a", "b", "c", "d", "e", "run_a", "run_b")))
    for h in prepared.values():
        h.close()
    gr.close(), ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "partial_batch_times.json"), "w") as f:
            json.dump(res, f, indent=1)
    return 0 if equal else 1


if __name__ == "__main__":
    sys.exit(main())
