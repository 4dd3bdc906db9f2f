#!/usr/bin/env python3
"""Times detection preprocessing on the device (tb200_graph_upload_detect_images) on one GPU.

YOLOv5s int8 at 640x640 (graph input [64, 12, 320, 320], random weights, seeded), batch 64, letterbox + Focus with the example's
default mean and scale, fed from 64 seeded RGB images in page-locked memory: 1280x720 (a downscale) and 640x480 (letterbox at the same
scale).  For each source size, reports:
1. wall time of upload_detect_images + launch + yolov5_detect + detections_to_source (threshold set so that about 300 candidates per
   image pass, as the random weights would otherwise pass every anchor), alternated in the same process with the host
   path the caller had before: the numpy restatement of the example's preprocessing (oracle/detect_pre.py, NOT OpenCV: its speed
   says nothing about the example's own C++), tb200_graph_upload of the result, then the same launch / detect / back-mapping; the
   boxes of both paths are compared;
2. the detect_pre kernel's time from torch.profiler CUDA activities, in a run of its own, against the bytes it must move / 3.35 TB/s
   (H100 SXM data-sheet HBM3 bandwidth): the source rows the resize reads plus the input bytes it writes;
3. the host-to-device bytes of the source pixels against the copy bandwidth measured here (torch, page-locked, same size).

Prints the card name and power limit first.  usage: detect_pre_time.py [--reps N] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BATCH, RES = 64, 640
SOURCES = {"1280x720": (720, 1280), "640x480": (480, 640)}
MAX_PER_IMAGE = 1024


def _setup(src):
    from oracle import detect_pre as dp
    from oracle import yolov5_post
    from tengine_b200 import abi, workloads
    from tengine_b200 import runtime as rt

    h, w = SOURCES[src]
    g, _ = workloads.yolov5s(abi.DT_INT8, batch=BATCH, res=RES)
    ctx = rt.Context(0)
    gr = rt.Graph(ctx, g)
    pixels = rt.PinnedBuffer((BATCH, h, w, 3), np.uint8)
    pixels.array[:] = np.random.default_rng(1).integers(0, 256, (BATCH, h, w, 3), dtype=np.uint8)
    descs = (abi.Image * BATCH)()
    for i, d in enumerate(descs):
        d.offset, d.w, d.h, d.c = i * h * w * 3, w, h, 3
    pre = abi.DetectPre()
    pre.mode, pre.focus = abi.PRE_LETTERBOX, 1
    for k in range(3):
        pre.mean[k], pre.scale[k] = dp.DEFAULT_MEAN[k], dp.DEFAULT_SCALE[k]
    geo = (abi.DetectGeometry * BATCH)()
    params = abi.YoloParams()
    heads = [(2, 32, yolov5_post.HEADS_BY_STRIDE[32]), (1, 16, yolov5_post.HEADS_BY_STRIDE[16]), (0, 8, yolov5_post.HEADS_BY_STRIDE[8])]
    params.num_heads = 3
    for i, (oi, stride, anchors) in enumerate(heads):
        params.heads[i].output_index, params.heads[i].stride = oi, stride
        for k in range(6):
            params.heads[i].anchors[k] = float(anchors[k])
    params.num_classes, params.nms_threshold, params.max_candidates = 80, 0.45, 0  # tm_yolov5s.cpp:559
    dets = (abi.Detection * (BATCH * MAX_PER_IMAGE))()
    counts = (C.c_int32 * BATCH)()
    L = rt.lib()
    L.tb200_graph_yolov5_detect.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]

    def upload():
        rt._check(L.tb200_graph_upload_detect_images(gr.h, 0, pixels.ptr, pixels.nbytes, descs, C.byref(pre), geo))

    # random weights pass almost every anchor at the example's 0.25: raise the threshold so that about 300 candidates per image remain,
    # as a trained model would leave, instead of overflowing the candidate list
    upload()
    gr.launch()
    scores = []
    for i, o in enumerate(g.outputs):
        q = np.empty(g.dims(o), np.int8)
        gr.download(i, q)
        gr.sync()
        x = (q.astype(np.float32) - np.float32(g.tensors[o]["zero_point"])) * np.float32(g.tensors[o]["scale"])
        x = x.reshape(BATCH, 3, 85, *q.shape[2:])
        sig = lambda v: 1.0 / (1.0 + np.exp(-v))
        scores.append((sig(x[:, :, 4]) * sig(x[:, :, 5:].max(axis=2))).reshape(BATCH, -1))
    scores = np.concatenate(scores, axis=1)
    params.prob_threshold = float(np.max(np.quantile(scores, 1.0 - 300.0 / scores.shape[1], axis=1)))

    def detect():
        gr.launch()
        rt._check(L.tb200_graph_yolov5_detect(gr.h, C.byref(params), dets, MAX_PER_IMAGE, counts))
        rt._check(L.tb200_detections_to_source(abi.PRE_LETTERBOX, geo, BATCH, dets, MAX_PER_IMAGE, counts))
        return [[(d.x, d.y, d.w, d.h, d.prob, d.label) for d in dets[i * MAX_PER_IMAGE:i * MAX_PER_IMAGE + max(counts[i], 0)]] + [int(counts[i])]
                for i in range(BATCH)]

    return ctx, gr, g, pixels, upload, detect


def _bytes_moved(src):
    """Source rows the resize reads (two per output row, shared between neighbours) plus the graph input it writes."""
    from oracle import detect_pre as dp

    h, w = SOURCES[src]
    _, _, rw, rh, _, _, _ = dp.geometry(dp.LETTERBOX, w, h, RES, RES)
    sy, _, _ = dp.linear_coef(rh, h, False)
    rows = len(set(np.clip(sy, 0, h - 1).tolist()) | set(np.clip(sy + 1, 0, h - 1).tolist()))
    return BATCH * rows * w * 3, BATCH * 12 * (RES // 2) ** 2


def child_profile(src, reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.init()
    ctx, gr, g, pixels, upload, _ = _setup(src)
    upload()
    gr.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            upload()
            gr.sync()
    ev = [e for e in prof.events() if "detect_pre_kernel" in e.name]
    us = sum(e.device_time for e in ev) / reps
    read, written = _bytes_moved(src)
    pixels.free(), gr.close(), ctx.close()
    bound = (read + written) / HBM_BYTES_PER_S * 1e6
    return {"source": src, "launches_per_call": len(ev) / reps, "kernel_us": us, "source_bytes_read": read, "input_bytes_written": written,
            "hbm_bound_us": bound, "share_of_hbm_bound": bound / max(us, 1e-9)}


def child_copy(src, reps):
    import torch

    h, w = SOURCES[src]
    host = torch.empty(BATCH * h * w * 3, dtype=torch.uint8).pin_memory()
    dev = torch.empty_like(host, device="cuda")
    dev.copy_(host, non_blocking=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dev.copy_(host, non_blocking=True)
    b.record()
    b.synchronize()
    s = a.elapsed_time(b) / 1e3 / reps
    return {"source": src, "source_bytes": host.numel(), "h2d_ms": s * 1e3, "h2d_gb_per_s": host.numel() / s / 1e9}


def _run_child(args):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)] + args, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError(f"{args}: exit {r.returncode}\n{r.stdout[-2000:]}{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def wall(src, reps, host_reps):
    from oracle import detect_pre as dp

    ctx, gr, g, pixels, upload, detect = _setup(src)
    t = g.tensors[g.inputs[0]]
    x = np.empty(g.dims(g.inputs[0]), np.int8)

    def device_path():
        upload()
        return detect()

    def host_path():
        x[:] = dp.preprocess_batch(pixels.array, dp.LETTERBOX, RES, RES, dp.DEFAULT_MEAN, dp.DEFAULT_SCALE, np.float32(t["scale"]), 0, False, True)
        gr.upload(0, x)
        return detect()

    dev_boxes, host_boxes = device_path(), host_path()  # warm-up, and the comparison
    td, th = [], []
    for r in range(max(reps, host_reps)):  # alternated
        t0 = time.perf_counter()
        device_path()
        td.append(time.perf_counter() - t0)
        if r < host_reps:
            t0 = time.perf_counter()
            host_path()
            th.append(time.perf_counter() - t0)
    kept = [b[-1] for b in dev_boxes]
    pixels.free(), gr.close(), ctx.close()
    return {"source": src, "device_path_ms_median": float(np.median(td)) * 1e3, "device_path_ms_min": float(np.min(td)) * 1e3,
            "device_reps": len(td), "host_restatement_path_ms_median": float(np.median(th)) * 1e3, "host_reps": len(th),
            "boxes_equal": dev_boxes == host_boxes, "boxes_per_image_min_max": [min(kept), max(kept)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--host-reps", type=int, default=3, help="repetitions of the (slow) numpy host path")
    ap.add_argument("--out", help="directory for detect_pre_time.json")
    ap.add_argument("--child", choices=["profile", "copy"])
    ap.add_argument("--source", choices=sorted(SOURCES), default="1280x720")
    a = ap.parse_args()
    if a.child:
        print(json.dumps({"profile": child_profile, "copy": child_copy}[a.child](a.source, a.reps)))
        return 0
    from tengine_b200 import runtime as rt

    if rt.device_count() < 1:
        print("no CUDA device: every number is not measured", file=sys.stderr)
        return 2
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    print("card (name, power limit, max SM clock):", card)
    res = {"card": card, "runs": []}
    for src in SOURCES:
        r = {"wall": wall(src, a.reps, a.host_reps)}
        print(json.dumps(r["wall"]))
        r["kernel"] = _run_child(["--child", "profile", "--source", src, "--reps", str(a.reps)])
        print(json.dumps(r["kernel"]))
        r["copy"] = _run_child(["--child", "copy", "--source", src, "--reps", str(a.reps)])
        print(json.dumps(r["copy"]))
        res["runs"].append(r)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "detect_pre_time.json"), "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
