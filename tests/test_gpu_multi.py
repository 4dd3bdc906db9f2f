"""Multi-GPU behind the boundary (SURVEY.md 8(e)): ONE process, one tb200 context over several GPUs, the batch of every
run cut into contiguous slices of dim 0, weights packed once on GPU 0 and copied to the other GPUs by cudaMemcpyPeerAsync at
prerun, no collective afterwards.  Checked: every shard's bytes (rank > 0 included) equal the oracle's, layer by layer.

On a box with one GPU the group lists device 0 more than once; the peer copies, the NO_WEIGHTS prerun of shards > 0, slicing
of the caller's buffers, per-shard streams and the merge of the outputs are the code that runs on 2/4/8 GPUs.  With >= 2 GPUs
a group of distinct devices is tested too."""
import os

import numpy as np
import pytest

from tengine_b200 import abi, workloads
from tests.helpers import layer_outputs

pytestmark = pytest.mark.gpu


def _devices(n):
    from tengine_b200 import runtime as rt

    have = rt.device_count()
    return [i % have for i in range(n)]


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
@pytest.mark.parametrize("ngpu,batch", [(2, 5), (3, 7), (4, 4)])
def test_sharded_run_every_layer_vs_oracle(oracle, dtype, ngpu, batch):
    from tengine_b200 import runtime as rt

    mctx = rt.Context(devices=_devices(ngpu))
    try:
        assert mctx.num_gpus == ngpu
        g, b = workloads.tiny_net(dtype, batch=batch, seed=5)
        x = b.random_input(8)
        gr = rt.Graph(mctx, g, abi.PRERUN_NO_GRAPH)
        try:
            sh = gr.shards()
            assert len(sh) == ngpu and sum(s[2] for s in sh) == batch and [s[1] for s in sh] == list(np.cumsum([0] + [s[2] for s in sh[:-1]]))
            assert max(s[2] for s in sh) - min(s[2] for s in sh) <= 1
            outs = gr.run([x])
            tensors = {t: gr.read_tensor(t) for t in layer_outputs(g)}
        finally:
            gr.close()
        want = oracle.run(g, [x], uint8_mode=0)
        for li, L in enumerate(g.layers):
            assert np.array_equal(tensors[L["output"]], want[L["output"]]), f"layer {li} {abi.OP_NAMES[L['op']]}"
        for o, t in zip(outs, g.outputs):
            assert np.array_equal(o, want[t])
    finally:
        mctx.close()


def test_sharded_mobilenet_graph_replay_and_pageable_buffers(oracle):
    """Captured CUDA graphs + pipelined chunks per shard, caller buffers that are plain (pageable) numpy arrays: the first run
    page-locks them in place, later runs reuse the registration; a different buffer the next time works too."""
    from tengine_b200 import runtime as rt

    mctx = rt.Context(devices=_devices(2))
    try:
        g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=66, res=64, width=0.5, classes=100)
        x = b.random_input(1)
        gr = rt.Graph(mctx, g)
        try:
            assert [s[2] for s in gr.shards()] == [33, 33]
            y1 = gr.run([x])[0]
            y2 = gr.run([x])[0]  # same input buffer (registered), fresh output buffer
            x2 = x.copy()
            y3 = gr.run([x2])[0]
        finally:
            gr.close()
        g1, _ = workloads.mobilenet_v1(abi.DT_INT8, batch=2, res=64, width=0.5, classes=100)
        for i in (0, 32, 33, 64):  # both sides of the shard boundary
            want = oracle.run(g1, [x[i:i + 2]])[g1.outputs[0]]
            assert np.array_equal(y1[i:i + 2], want), i
        assert np.array_equal(y1, y2) and np.array_equal(y1, y3)
    finally:
        mctx.close()


def test_real_multi_gpu_group(oracle):
    from tengine_b200 import runtime as rt

    if rt.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (run with gpurun --gpus 2)")
    n = min(rt.device_count(), 8)
    mctx = rt.Context(devices=list(range(n)))
    try:
        assert mctx.broadcast_kind == "memcpy_peer"
        g, b = workloads.yolov3_tiny(abi.DT_UINT8, batch=2 * n + 1, res=96, width=0.25, head=27, seed=6)
        x = b.random_input(2)
        gr = rt.Graph(mctx, g)
        try:
            assert sorted({s[0] for s in gr.shards()}) == list(range(n))
            outs = gr.run([x])
        finally:
            gr.close()
        want = oracle.run(g, [x], uint8_mode=0)
        for o, t in zip(outs, g.outputs):
            assert np.array_equal(o, want[t])
    finally:
        mctx.close()


def test_arena_slots_are_reused_and_producers_own_their_pad_lanes(ctx, oracle):
    """The activation arena hands a tensor's slot on after its last consumer (cpu_pool.c's role).  Correctness then needs every
    kernel to write the pad lanes of its output itself: run with the arena poisoned (0xA5) instead of zeroed."""
    from tengine_b200 import runtime as rt

    for dtype in (abi.DT_INT8, abi.DT_UINT8):
        for g, b in (workloads.tiny_net(dtype, batch=3, seed=2), workloads.tail_net(dtype, batch=3),
                     workloads.yolov3_tiny(dtype, batch=2, res=96, width=0.25, head=27, seed=6),
                     workloads.resnet50(dtype, batch=2, res=64, width=0.25, classes=24, seed=5, softmax=True)):
            x = b.random_input(5)
            gr = rt.Graph(ctx, g, abi.PRERUN_POISON_ARENA)
            try:
                act, unshared, _ = gr.arena_bytes()
                outs = gr.run([x])
                outs2 = gr.run([x])
            finally:
                gr.close()
            assert act < unshared
            want = oracle.run(g, [x], uint8_mode=0)
            for o, o2, t in zip(outs, outs2, g.outputs):
                assert np.array_equal(o, want[t]) and np.array_equal(o2, want[t])
    g, _ = workloads.resnet50(abi.DT_UINT8, batch=8)
    gr = rt.Graph(ctx, g)
    act, unshared, _ = gr.arena_bytes()
    gr.close()
    assert act * 3 < unshared, (act, unshared)


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
def test_tail_ops_every_layer_vs_oracle(ctx, oracle, dtype):
    """Sigmoid / HardSwish (byte tables built at prerun with the reference's C arithmetic), Eltwise-PROD, Flatten of a C x H x W
    tensor (NHWC -> NCHW order), FC, Softmax: every layer bit-exact against the oracle (which is pinned to the reference)."""
    from tengine_b200 import runtime as rt

    g, b = workloads.tail_net(dtype, batch=3)
    x = b.random_input(4)
    gr = rt.Graph(ctx, g, abi.PRERUN_NO_GRAPH)
    try:
        gr.run([x])
        tensors = {t: gr.read_tensor(t) for t in layer_outputs(g)}
        kernels = gr.layer_kernels()
    finally:
        gr.close()
    want = oracle.run(g, [x], uint8_mode=0)
    for li, L in enumerate(g.layers):
        assert np.array_equal(tensors[L["output"]], want[L["output"]]), f"layer {li} {abi.OP_NAMES[L['op']]} ({kernels[li]})"
    assert {"byte_lut", "softmax", "reshape_nchw_order"} <= set(kernels)


def test_uint8_fc_bias_scale(ctx, oracle):
    from tengine_b200 import runtime as rt
    from tengine_b200.graphdef import GraphDef

    rng = np.random.default_rng(3)
    g = GraphDef(abi.DT_UINT8)
    x = g.input(3, 64, 2, 2, 0.02, 128)
    y = g.fc(x, rng.integers(0, 256, (40, 256)).astype(np.uint8), rng.integers(-30000, 30000, 40).astype(np.int32), [0.004], 0.05, 120,
             weight_zero=119)
    g.layers[-1]["bias_scale"] = float(np.float32(0.02 * 0.004 * 1.37))
    g.mark_output(y)
    xin = rng.integers(0, 256, (3, 64, 2, 2)).astype(np.uint8)
    for flags in (abi.PRERUN_DEFAULT, abi.PRERUN_NO_TENSORCORE):
        gr = rt.Graph(ctx, g, flags)
        got = gr.run([xin])[0]
        gr.close()
        assert np.array_equal(got, oracle.run(g, [xin], uint8_mode=0)[y])


def test_pack_cache_round_trip(ctx, oracle, tmp_path):
    """SURVEY.md 8(f)-3: the packed weight arena is written under a hash of everything it depends on; a second prerun of the same
    model reads it back (same bytes on the device, same results); a model with other weights gets another entry."""
    import time

    from tengine_b200 import runtime as rt

    rt.set_pack_cache_dir(str(tmp_path))
    try:
        g, b = workloads.resnet50(abi.DT_UINT8, batch=2, res=64, width=0.5, classes=30, seed=9)
        x = b.random_input(1)
        want = oracle.run(g, [x], uint8_mode=0)[g.outputs[0]]
        t0 = time.perf_counter()
        gr = rt.Graph(ctx, g)
        t_pack = time.perf_counter() - t0
        assert gr.pack_cache_state() == 1
        y1 = gr.run([x])[0]
        gr.close()
        files = sorted(os.listdir(tmp_path))
        assert len(files) == 1 and files[0].endswith(".pack")
        t0 = time.perf_counter()
        gr = rt.Graph(ctx, g)
        t_hit = time.perf_counter() - t0
        assert gr.pack_cache_state() == 2
        y2 = gr.run([x])[0]
        gr.close()
        assert np.array_equal(y1, want) and np.array_equal(y2, want)
        g2, _ = workloads.resnet50(abi.DT_UINT8, batch=2, res=64, width=0.5, classes=30, seed=10)  # other weights
        gr = rt.Graph(ctx, g2)
        assert gr.pack_cache_state() == 1
        gr.close()
        assert len(os.listdir(tmp_path)) == 2
        print(f"prerun with packing {t_pack * 1e3:.1f} ms, from the cache {t_hit * 1e3:.1f} ms")
    finally:
        rt.set_pack_cache_dir(None)
    gr = rt.Graph(ctx, g)
    assert gr.pack_cache_state() == 0
    gr.close()


@pytest.mark.parametrize("gpus", [1, 2])
def test_yolo_detect_on_device_equals_the_examples_post_processing(oracle, gpus):
    """SURVEY.md 8(f)-4: region decode + threshold + sort + NMS on the device, from the quantised head tensors in HBM, against the
    CPU restatement of examples/tm_yolov3_tiny_uint8.cpp's post-processing (oracle/yolo_post.py) on the same bytes: the same boxes
    in the same order, bit-identical floats."""
    from oracle import yolo_post
    from tengine_b200 import runtime as rt

    g, b = workloads.yolov3_tiny(abi.DT_UINT8, batch=5, res=160, width=0.5, seed=8)
    x = b.random_input(3)
    c = rt.Context(devices=_devices(gpus)) if gpus > 1 else rt.Context(0)
    anchors = [10, 14, 23, 27, 37, 58, 81, 82, 135, 169, 344, 319]
    # the example's order: the stride-32 head (anchors[6:12]) first, then stride 16 (anchors[0:6]); graph outputs are (26x26, 13x13)-like
    heads = [(1, 32, anchors[6:12]), (0, 16, anchors[0:6])]
    try:
        gr = rt.Graph(c, g)
        outs = gr.run([x])
        # low threshold: random-weight heads rarely reach the example's 0.4
        got = gr.yolo_detect(heads, num_classes=80, prob_threshold=0.27, nms_threshold=0.25, max_per_image=512)
        gr.close()
    finally:
        c.close()
    want_raw = oracle.run(g, [x], uint8_mode=0)
    for o, t in zip(outs, g.outputs):
        assert np.array_equal(o, want_raw[t])
    scales = [g.tensors[t]["scale"] for t in g.outputs]
    zeros = [g.tensors[t]["zero_point"] for t in g.outputs]
    want = yolo_post.detect(outs, scales, zeros, heads, 80, 0.27, 0.25)
    assert sum(len(w) for w in want) > 20, "test vacuous: nothing passes the threshold"
    for i, (gd, wd) in enumerate(zip(got, want)):
        assert len(gd) == len(wd), (i, len(gd), len(wd))
        for a, w in zip(gd, wd):
            assert a[5] == w[5] and all(np.float32(a[k]) == np.float32(w[k]) for k in range(5)), (i, a, w)
