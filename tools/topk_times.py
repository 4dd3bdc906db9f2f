#!/usr/bin/env python3
"""Times ranking a classification output on the device (tb200_graph_topk) against downloading it and ranking on the host, on one GPU.

MobileNet-v1 int8 at 224x224, batch 256, 1000 classes (random weights, seeded), after one launch.  Two outputs are ranked: the graph's
own (`logits`), and a Softmax-shaped one (`softmax`: nearly every class at probability 0, a few peaks, several tied) laid into a
second graph of the same output shape -- the tie-heavy case, where the example's quicksort is quadratic.
 (a) tb200_graph_topk(k = 5): host clock around the synchronous call; and the kernel alone (tb200k_class_topk on device memory of the
     same bytes, in a process of its own), CUDA events around 200 launches.
 (b) tb200_graph_download + sync, then the example's own sort per image on one host thread: oracle/_ref/libtopk_example.so where it
     exists, else a plain C loop of the same algorithm compiled by this script into a temporary directory.
(a) and (b) alternate in the same process; median, minimum and maximum of the repetitions are reported.  The results of both are
compared.  Prints the card name and power limit first, and fails without a GPU.  usage: topk_times.py [--reps N] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

BATCH, CLASSES, K = 256, 1000, 5

HOST_SORT_C = r"""
typedef struct { int id; float score; } rec;
static void sort_desc(rec* a, int left, int right)
{
    int i = left, j = right;
    rec key;
    if (left >= right) return;
    key = a[left];
    while (left < right)
    {
        while (left < right && key.score >= a[right].score) --right;
        a[left] = a[right];
        while (left < right && key.score <= a[left].score) ++left;
        a[right] = a[left];
    }
    a[left] = key;
    sort_desc(a, i, left - 1);
    sort_desc(a, left + 1, j);
}
#include <stdlib.h>
int topk_example_sorted(const float* data, int n, int* ids, float* scores)
{
    rec* a = (rec*)malloc(n * sizeof(rec));
    for (int i = 0; i < n; i++) a[i].id = i, a[i].score = data[i];
    sort_desc(a, 0, n - 1);
    for (int i = 0; i < n; i++) ids[i] = a[i].id, scores[i] = a[i].score;
    free(a);
    return 0;
}
"""


def host_sort_lib(tmp):
    """(library, what it is): the compiled example where it travelled, else the same loop compiled here."""
    ref = os.path.join(ROOT, "oracle", "_ref", "libtopk_example.so")
    if os.path.exists(ref):
        path, what = ref, "examples/common/tengine_operations.c sort_cls_score (oracle/_ref/libtopk_example.so)"
    else:
        src, path = os.path.join(tmp, "host_sort.c"), os.path.join(tmp, "libhost_sort.so")
        open(src, "w").write(HOST_SORT_C)
        subprocess.check_call(["gcc", "-O2", "-std=gnu99", "-fPIC", "-shared", src, "-o", path])
        what = "a plain C loop of the same quicksort, gcc -O2"
    L = C.CDLL(path)
    L.topk_example_sorted.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L, what


def softmax_shaped(rng):
    q = np.zeros((BATCH, CLASSES, 1, 1), np.int8)
    for n in range(BATCH):
        pos = rng.permutation(CLASSES)[:15]
        q[n, pos, 0, 0] = [90, 14, 14, 14, 3, 3] + [1] * 9
    return q


def child_kernel(path, scale):
    """The kernel alone (tb200k_class_topk) on a device copy of the saved output bytes in the device layout: CUDA events around 200
    launches.  A process of its own, where torch owns the device from the start and no graph call precedes its allocations."""
    import torch

    from tengine_b200 import runtime as rt

    torch.cuda.init()
    y = np.load(path)
    cp = (CLASSES + 15) // 16 * 16
    lay = np.zeros((BATCH, 1, 1, cp), np.int8)
    lay[..., :CLASSES] = y.reshape(BATCH, 1, 1, CLASSES)
    din = torch.from_numpy(lay).cuda()
    dout = torch.zeros((BATCH, K, 2), dtype=torch.int32, device="cuda")
    launch = lambda: rt.class_topk(din.data_ptr(), BATCH, CLASSES, 1, 1, False, scale, 0, K, dout.data_ptr(), None)
    launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(200):
        launch()
    e1.record()
    e1.synchronize()
    return {"kernel_us_per_launch": e0.elapsed_time(e1) * 1e3 / 200, "ids": dout.cpu().numpy()[..., 1].tolist()}


def run_child(args):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)] + args, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError(f"{args}: exit {r.returncode}\n{r.stdout[-2000:]}{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def stats(ts):
    return {"ms_median": float(np.median(ts)) * 1e3, "ms_min": float(np.min(ts)) * 1e3, "ms_max": float(np.max(ts)) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", help="directory for topk_times.json")
    ap.add_argument("--child-kernel", help=argparse.SUPPRESS)
    ap.add_argument("--scale", type=float, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child_kernel:
        print(json.dumps(child_kernel(a.child_kernel, np.float32(a.scale))))
        return 0
    from tengine_b200 import abi, workloads
    from tengine_b200 import runtime as rt
    from tengine_b200.graphdef import GraphDef

    if rt.device_count() < 1:
        print("no CUDA device: every number is not measured", file=sys.stderr)
        return 2
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    print("card (name, power limit, max SM clock):", card)
    from oracle import topk

    ctx = rt.Context(0)
    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=BATCH, res=224, classes=CLASSES)
    t = g.tensors[g.outputs[0]]
    gr = rt.Graph(ctx, g)
    gr.run([b.random_input(1)])
    # the Softmax-shaped bytes as the output of a graph of their own, same shape and scale 1 / 128
    ident = GraphDef(abi.DT_INT8)
    ident.mark_output(ident.identity(ident.input(BATCH, CLASSES, 1, 1, 0.0078125, 0)))
    gs = rt.Graph(ctx, ident)
    gs.run([softmax_shaped(np.random.default_rng(3))])
    res = {"card": card, "batch": BATCH, "classes": CLASSES, "k": K}
    with tempfile.TemporaryDirectory() as tmp:
        L, res["host_sort"] = host_sort_lib(tmp)
        for name, graph, scale in (("logits", gr, np.float32(t["scale"])), ("softmax", gs, np.float32(0.0078125))):
            y = np.empty((BATCH, CLASSES, 1, 1), np.int8)
            ids, scores = np.empty(CLASSES, np.int32), np.empty(CLASSES, np.float32)
            host_ids = np.empty((BATCH, K), np.int32)

            def host():
                graph.download(0, y)
                graph.sync()
                f = topk.dequantise(y.reshape(BATCH, CLASSES), scale, 0, False)
                for n in range(BATCH):
                    L.topk_example_sorted(f[n].ctypes.data, CLASSES, ids.ctypes.data, scores.ctypes.data)
                    host_ids[n] = ids[:K]

            dev, hst = [], []
            graph.topk(0, K), host()  # warm-up
            for _ in range(a.reps):
                t0 = time.perf_counter()
                got = graph.topk(0, K)
                dev.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                host()
                hst.append(time.perf_counter() - t0)
            np.save(os.path.join(tmp, name + ".npy"), y)
            kern = run_child(["--child-kernel", os.path.join(tmp, name + ".npy"), "--scale", repr(float(scale))])
            res[name] = {"device_graph_topk": stats(dev), "download_plus_host_sort": stats(hst), "kernel_us_per_launch": kern["kernel_us_per_launch"],
                         "bytes_back_device": BATCH * K * 8, "bytes_back_host": BATCH * CLASSES,
                         "results_equal": bool(np.array_equal(got[1], host_ids) and np.array_equal(np.array(kern["ids"], np.int32), host_ids))}
            print(name, json.dumps(res[name]))
    gr.close(), gs.close(), ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "topk_times.json"), "w") as f:
            json.dump(res, f, indent=1)
    return 0 if all(res[n]["results_equal"] for n in ("logits", "softmax")) else 1


if __name__ == "__main__":
    sys.exit(main())
