"""Plan fingerprint of the library named by TB200_LIB (default: the in-tree build).

For every graph below and every prerun flag it prints one JSON line: the kernel of each layer, the launch count, the arena
sizes, work(), the shards, the pack-cache file (name and sha256) and the sha256 of the outputs of one run.  Two builds that
plan, pack and compute alike print identical output, so a change to the planner can be checked against its parent:

    TB200_LIB=/path/to/parent.so python tools/plan_fingerprint.py > parent.jsonl
    python tools/plan_fingerprint.py > new.jsonl && cmp parent.jsonl new.jsonl

Needs an H100.
"""
import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tengine_b200 import abi, workloads  # noqa: E402
from tengine_b200 import runtime as rt  # noqa: E402

FLAGS = {"default": abi.PRERUN_DEFAULT, "no_tensorcore": abi.PRERUN_NO_TENSORCORE, "no_graph": abi.PRERUN_NO_GRAPH}


def graphs():
    """(name, (graph, builder), GPUs).  The bench workloads at reduced size cover the three node fusions: eltwise -> ReLU
    (ResNet-50), ReLU -> max pooling (YOLOv3-tiny) and SiLU (int8 YOLOv5s, tail_net)."""
    for dt, dn in ((abi.DT_INT8, "int8"), (abi.DT_UINT8, "uint8")):
        yield f"mobilenet_v1_{dn}", workloads.mobilenet_v1(dt, batch=4, res=64, width=0.5, classes=100), 1
        yield f"resnet50_{dn}", workloads.resnet50(dt, batch=2, res=64, width=0.25, classes=50), 1
        yield f"yolov3_tiny_{dn}", workloads.yolov3_tiny(dt, batch=2, res=128, width=0.25), 1
        yield f"yolov5s_{dn}", workloads.yolov5s(dt, batch=2, res=128, width=0.25), 1
        yield f"tiny_net_{dn}", workloads.tiny_net(dt, batch=2), 1
        yield f"tail_net_{dn}", workloads.tail_net(dt, batch=2), 1
        yield f"tiny_net_{dn}_2shards", workloads.tiny_net(dt, batch=5), 2
    # batch >= 64: the pipelined run is cut into chunks of 1/4 and 3/4 of the batch
    yield "mobilenet_v1_int8_b64", workloads.mobilenet_v1(abi.DT_INT8, batch=64, res=64, width=0.5, classes=100), 1


def fingerprint(ctx, g, x, flags):
    with tempfile.TemporaryDirectory() as cache:
        rt.set_pack_cache_dir(cache)
        gr = rt.Graph(ctx, g, flags)
        try:
            packs = sorted(f for f in os.listdir(cache) if f.endswith(".pack"))
            pack = {f: hashlib.sha256(open(os.path.join(cache, f), "rb").read()).hexdigest() for f in packs}
            out = hashlib.sha256(b"".join(o.tobytes() for o in gr.run([x]))).hexdigest()
            return {"layer_kernels": gr.layer_kernels(), "num_launches": gr.num_launches(), "arena_bytes": list(gr.arena_bytes()),
                    "work": list(gr.work()), "shards": [list(s) for s in gr.shards()], "pack_cache": pack, "outputs_sha256": out}
        finally:
            gr.close()
            rt.set_pack_cache_dir(None)


def main():
    ctxs = {1: rt.Context(0), 2: rt.Context(devices=[0, 0])}  # device 0 twice: two shards on a one-GPU box
    try:
        for name, (g, b), ngpu in graphs():
            x = b.random_input(1)
            for fname, flags in FLAGS.items():
                rec = {"graph": name, "flags": fname, **fingerprint(ctxs[ngpu], g, x, flags)}
                print(json.dumps(rec, sort_keys=True), flush=True)
    finally:
        for c in ctxs.values():
            c.close()


if __name__ == "__main__":
    main()
