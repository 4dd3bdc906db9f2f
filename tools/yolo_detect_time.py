#!/usr/bin/env python3
"""Times detection post-processing on the device against downloading the raw heads, on one GPU.

1. YOLOv5s int8 at 640x640, batch 8 and 64 (random weights, seeded): wall time of tb200_graph_yolov5_detect (synchronous: decode,
   sort, NMS, copy of the kept boxes) and of downloading the three head tensors into host memory, which post-processing on the host
   would need first.  The score threshold is chosen from the heads so that about 300 anchors per image pass: a random-weight head
   passes far more anchors at the example's 0.25 than a trained one does.
2. The decode kernel's time from torch.profiler CUDA activities, in a run of its own, against the head bytes / 3.35 TB/s (H100 SXM
   data-sheet HBM3 bandwidth).  The decode skips the class bytes of anchors whose objectness cannot pass the threshold, so it may
   read fewer bytes than that bound assumes.
3. YOLOv3-tiny int8 at 416x416: wall time of tb200_graph_yolo_detect with the library of the parent commit
   (--parent-lib) and with this tree's library, alternated, at batch 16 (the bench default) and 128, each in its own process (TB200_LIB), with a hash of the detections.

Prints the card name and power limit first.  usage: yolo_detect_time.py [--parent-lib PATH] [--reps N] [--out DIR]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
V5_HEADS = [(2, 32, [116, 90, 156, 198, 373, 326]), (1, 16, [30, 61, 62, 45, 59, 119]), (0, 8, [10, 13, 16, 30, 33, 23])]  # tm_yolov5s.cpp:143
V3_ANCHORS = [10, 14, 23, 27, 37, 58, 81, 82, 135, 169, 344, 319]
V3_HEADS = [(1, 32, V3_ANCHORS[6:12]), (0, 16, V3_ANCHORS[0:6])]  # yolov3_tiny outputs are (26x26, 13x13)


def _threshold(outs, scales, zeros, per_image=300):
    """A score threshold that about `per_image` anchors of the busiest image pass (sigmoid(obj) * sigmoid(best class), float32)."""
    from oracle import yolo_post

    scores = []
    for q, s, z in zip(outs, scales, zeros):
        b = np.arange(256)
        x = ((b.astype(np.float32) if q.dtype == np.uint8 else b.astype(np.uint8).view(np.int8).astype(np.float32)) - np.float32(z)) * np.float32(s)
        sig = np.array([yolo_post._sigmoid(v) for v in x.astype(np.float32)], np.float32)
        n, c, h, w = q.shape
        r = q.reshape(n, 3, c // 3, h, w)
        best = np.take_along_axis(r[:, :, 5:], r[:, :, 5:].argmax(axis=2)[:, :, None], axis=2)[:, :, 0]
        scores.append((sig[r[:, :, 4].view(np.uint8)] * sig[best.view(np.uint8)]).reshape(n, -1))
    sc = np.concatenate(scores, axis=1)
    return float(np.max(np.quantile(sc, 1.0 - per_image / sc.shape[1], axis=1)))


def _graph(net, batch):
    from tengine_b200 import abi, workloads
    from tengine_b200 import runtime as rt

    res = 640 if net == "yolov5s" else 416
    g, b = getattr(workloads, net)(abi.DT_INT8, batch=batch, res=res)
    ctx = rt.Context(0)
    gr = rt.Graph(ctx, g)
    outs = gr.run([b.random_input(1)])
    scales = [np.float32(g.tensors[t]["scale"]) for t in g.outputs]
    zeros = [int(g.tensors[t]["zero_point"]) for t in g.outputs]
    return ctx, gr, g, outs, _threshold(outs, scales, zeros)


def _wall(fn, reps):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, float(np.min(ts)) * 1e3


def child_v5(batch, reps):
    ctx, gr, g, outs, prob = _graph("yolov5s", batch)
    detect = lambda: gr.yolo_detect(V5_HEADS, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, max_candidates=8192, version=5)
    host = [np.empty_like(o) for o in outs]

    def download():
        for i, h in enumerate(host):
            gr.download(i, h)
        gr.sync()

    det_ms, det_min = _wall(detect, reps)
    dl_ms, dl_min = _wall(download, reps)
    kept = [len(d) for d in detect()]
    head_bytes = sum(int(np.prod(o.shape)) for o in outs)
    gr.close(), ctx.close()
    return {"net": "yolov5s_int8_640", "batch": batch, "prob_threshold": prob, "kept_per_image_mean": float(np.mean(kept)), "head_bytes": head_bytes,
            "detect_ms_median": det_ms, "detect_ms_min": det_min, "download_heads_ms_median": dl_ms, "download_heads_ms_min": dl_min}


def child_profile(batch, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    ctx, gr, g, outs, prob = _graph("yolov5s", batch)
    detect = lambda: gr.yolo_detect(V5_HEADS, num_classes=80, prob_threshold=prob, nms_threshold=0.45, max_per_image=1024, max_candidates=8192, version=5)
    detect()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            detect()
    dec = [e for e in prof.events() if "yolo_decode_kernel" in e.name]
    nms = [e for e in prof.events() if "yolo_nms_kernel" in e.name]
    us = lambda ev: sum(e.device_time for e in ev) / reps  # per detect call (three decode launches)
    stored = sum(int(np.prod(o.shape)) // o.shape[1] * ((o.shape[1] + 15) // 16 * 16) for o in outs)  # NHWC rows padded to 16
    gr.close(), ctx.close()
    return {"net": "yolov5s_int8_640", "batch": batch, "decode_launches_per_call": len(dec) / reps, "decode_us_per_call": us(dec),
            "nms_us_per_call": us(nms), "head_bytes_stored": stored, "hbm_bound_us": stored / HBM_BYTES_PER_S * 1e6,
            "decode_share_of_hbm_bound": stored / HBM_BYTES_PER_S * 1e6 / max(us(dec), 1e-9)}


def child_v3(batch, reps):
    ctx, gr, g, outs, prob = _graph("yolov3_tiny", batch)
    detect = lambda: gr.yolo_detect(V3_HEADS, num_classes=80, prob_threshold=prob, nms_threshold=0.25, max_per_image=1024, max_candidates=8192)
    det_ms, det_min = _wall(detect, reps)
    boxes = np.array([b for d in detect() for b in d], np.float32)
    gr.close(), ctx.close()
    return {"net": "yolov3_tiny_int8_416", "batch": batch, "lib": os.environ.get("TB200_LIB", "tree"), "detect_ms_median": det_ms, "detect_ms_min": det_min,
            "boxes": len(boxes), "sha256": hashlib.sha256(boxes.tobytes()).hexdigest()[:16]}


def _run_child(args, env=None):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)] + args, capture_output=True, text=True, env=env, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError(f"{args}: exit {r.returncode}\n{r.stdout[-2000:]}{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", help="libtengine_b200.so built from the parent commit (YOLOv3-tiny comparison)")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", help="directory for results.json")
    ap.add_argument("--child", choices=["v5", "v3", "profile"])
    ap.add_argument("--batch", type=int, default=8)
    a = ap.parse_args()
    if a.child:
        fn = {"v5": child_v5, "v3": child_v3, "profile": child_profile}[a.child]
        print(json.dumps(fn(a.batch, a.reps)))
        return 0
    from tengine_b200 import runtime as rt

    if rt.device_count() < 1:
        print("no CUDA device: every number is not measured", file=sys.stderr)
        return 2
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    print("card (name, power limit, max SM clock):", card)
    res = {"card": card, "v5": [], "profile": [], "v3": []}
    for batch in (8, 64):
        r = _run_child(["--child", "v5", "--batch", str(batch), "--reps", str(a.reps)])
        print(json.dumps(r))
        res["v5"].append(r)
    for batch in (8, 64):
        r = _run_child(["--child", "profile", "--batch", str(batch), "--reps", str(a.reps)])
        print(json.dumps(r))
        res["profile"].append(r)
    if a.parent_lib:
        own = os.path.join(ROOT, "tengine_b200", "libtengine_b200.so")
        for batch in (16, 128):
            for _ in range(3):
                for lib in (own, a.parent_lib):
                    try:
                        r = _run_child(["--child", "v3", "--batch", str(batch), "--reps", str(a.reps)], env=dict(os.environ, TB200_LIB=lib))
                    except RuntimeError as e:  # reported, not measured
                        r = {"net": "yolov3_tiny_int8_416", "batch": batch, "lib": lib, "error": str(e).strip().splitlines()[-1]}
                    print(json.dumps(r))
                    res["v3"].append(r)
    else:
        print("YOLOv3-tiny parent comparison: not measured (no --parent-lib)")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "yolo_detect_time.json"), "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
