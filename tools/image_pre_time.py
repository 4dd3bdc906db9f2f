#!/usr/bin/env python3
"""Times classification preprocessing on the device (tb200_graph_upload_images) on one GPU.

MobileNet-v1 int8 at 224x224, batch 256 (random weights, seeded), fed from 256 seeded 500x375 RGB images in page-locked memory
(144 MB per batch), with the examples' default mean and scale.  Reports:
1. wall time of upload_images + launch + download + sync, against tb200_graph_run on the already-quantised input (same graph);
   the outputs of both paths are compared;
2. the image_pre kernel's time from torch.profiler CUDA activities, in a run of its own, against the bytes it must move / 3.35 TB/s
   (H100 SXM data-sheet HBM3 bandwidth): the NCHW bytes it writes plus the source rows the resize reads;
3. the host-to-device bytes of one upload_images against the copy bandwidth measured here (torch, page-locked, same size);
4. where oracle/_ref/libimage_example.so exists: the unmodified example's get_input_int8_data per image on one core (its stbi_load of
   a binary PPM included, and that load alone).

Prints the card name and power limit first.  usage: image_pre_time.py [--reps N] [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import numpy as np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
BATCH, RES, SRC_H, SRC_W = 256, 224, 375, 500


def _images(seed=1):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (BATCH, SRC_H, SRC_W, 3), dtype=np.uint8)


def _setup():
    from oracle import image_pre
    from tengine_b200 import abi, workloads
    from tengine_b200 import runtime as rt

    g, _ = workloads.mobilenet_v1(abi.DT_INT8, batch=BATCH, res=RES)
    ctx = rt.Context(0)
    gr = rt.Graph(ctx, g)
    t = g.tensors[g.inputs[0]]
    pixels = rt.PinnedBuffer((BATCH, SRC_H, SRC_W, 3), np.uint8)
    pixels.array[:] = _images()
    descs = (abi.Image * BATCH)()
    for i, d in enumerate(descs):
        d.offset, d.w, d.h, d.c = i * SRC_H * SRC_W * 3, SRC_W, SRC_H, 3
    import ctypes as C

    mean = (C.c_float * 3)(*image_pre.DEFAULT_MEAN)
    scale = (C.c_float * 3)(*image_pre.DEFAULT_SCALE)

    def upload():
        rt._check(rt.lib().tb200_graph_upload_images(gr.h, 0, pixels.ptr, pixels.nbytes, descs, mean, scale))

    return ctx, gr, g, t, pixels, upload


def _wall(fn, reps):
    fn()  # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)) * 1e3, float(np.min(ts)) * 1e3


def child_profile(reps):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from oracle import image_pre

    torch.cuda.init()
    ctx, gr, g, t, pixels, upload = _setup()
    upload()
    gr.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            upload()
            gr.sync()
    ev = [e for e in prof.events() if "image_pre_kernel" in e.name]
    us = sum(e.device_time for e in ev) / reps
    sy, _, _ = image_pre.resize_coef(RES, SRC_H)
    rows = len(set(sy.tolist()) | set((sy + 1).tolist()))
    moved = BATCH * 3 * RES * RES + BATCH * rows * SRC_W * 3
    pixels.free(), gr.close(), ctx.close()
    return {"launches_per_call": len(ev) / reps, "kernel_us": us, "bytes_moved": moved, "hbm_bound_us": moved / HBM_BYTES_PER_S * 1e6,
            "share_of_hbm_bound": moved / HBM_BYTES_PER_S * 1e6 / max(us, 1e-9)}


def child_copy(reps):
    import torch

    src = torch.empty(BATCH * SRC_H * SRC_W * 3, dtype=torch.uint8).pin_memory()
    dst = torch.empty_like(src, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    b.record()
    b.synchronize()
    s = a.elapsed_time(b) / 1e3 / reps
    return {"bytes": src.numel(), "h2d_ms": s * 1e3, "h2d_gb_per_s": src.numel() / s / 1e9}


def host_example(reps):
    import make_golden_image_pre as gen

    from oracle import image_pre

    if not os.path.exists(gen.LIB):
        return {"host_example": "not measured (oracle/_ref/libimage_example.so absent)"}
    L = gen.example_lib()
    img = _images()[0]
    out = np.zeros((3, RES, RES), np.int8)
    import ctypes as C

    m, s = (C.c_float * 3)(*image_pre.DEFAULT_MEAN), (C.c_float * 3)(*image_pre.DEFAULT_SCALE)
    with tempfile.TemporaryDirectory() as tmp:
        path = gen.write_image(L, os.path.join(tmp, "img"), img)
        full = _wall(lambda: L.get_input_int8_data(path.encode(), out.ctypes.data, RES, RES, m, s, C.c_float(1 / 127)), reps)
        load = _wall(lambda: gen.stbi_load(L, path), reps)
    return {"host_get_input_int8_data_ms_per_image": full[0], "host_stbi_load_ppm_ms_per_image": load[0],
            "host_images_per_s_one_core": 1e3 / full[0]}


def _run_child(args):
    r = subprocess.run([sys.executable, os.path.abspath(__file__)] + args, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError(f"{args}: exit {r.returncode}\n{r.stdout[-2000:]}{r.stderr[-3000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", help="directory for image_pre_time.json")
    ap.add_argument("--child", choices=["profile", "copy"])
    a = ap.parse_args()
    if a.child:
        print(json.dumps({"profile": child_profile, "copy": child_copy}[a.child](a.reps)))
        return 0
    from tengine_b200 import runtime as rt

    if rt.device_count() < 1:
        print("no CUDA device: every number is not measured", file=sys.stderr)
        return 2
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    print("card (name, power limit, max SM clock):", card)
    res = {"card": card}

    from oracle import image_pre

    ctx, gr, g, t, pixels, upload = _setup()
    out_dev = np.empty(g.dims(g.outputs[0]), np.int8)

    def from_images():
        upload()
        gr.launch()
        gr.download(0, out_dev)
        gr.sync()

    x = image_pre.preprocess_batch(pixels.array, RES, RES, image_pre.DEFAULT_MEAN, image_pre.DEFAULT_SCALE, np.float32(t["scale"]), 0, False)
    out_run = np.empty_like(out_dev)
    run = lambda: gr.run([x], [out_run])
    wall = {}
    for name, fn in (("upload_images_launch_download", from_images), ("graph_run_prequantised", run)):
        med, mn = _wall(fn, a.reps)
        wall[name] = {"ms_median": med, "ms_min": mn, "images_per_s_median": BATCH / med * 1e3}
    from_images()
    run()
    wall["outputs_equal"] = bool(np.array_equal(out_dev, out_run))
    res["wall"] = wall
    print(json.dumps(wall))
    pixels.free(), gr.close(), ctx.close()

    res["kernel"] = _run_child(["--child", "profile", "--reps", str(a.reps)])
    print(json.dumps(res["kernel"]))
    cp = _run_child(["--child", "copy", "--reps", str(a.reps)])
    h2d = BATCH * SRC_H * SRC_W * 3 + BATCH * 24  # pixels + descriptors
    cp["upload_images_h2d_bytes"] = h2d
    cp["upload_images_h2d_ms_at_that_bandwidth"] = h2d / (cp["h2d_gb_per_s"] * 1e9) * 1e3
    res["copy"] = cp
    print(json.dumps(cp))
    res["host"] = host_example(max(3, a.reps // 4))
    print(json.dumps(res["host"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "image_pre_time.json"), "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
