"""Classification post-processing on the device: tb200k_class_topk and tb200_graph_topk against the output of the unmodified
example (tests/golden/topk_example.npz) and the restatement (oracle/topk.py), ids and score bits.

- tb200k_class_topk on device tensors in the padded NHWC layout holding every fixture case, several images per call, pad lanes
  poisoned, [E, 1, 1] and C x H x W shapes with C not a multiple of 16.
- tb200_graph_topk after real runs (reduced MobileNet-v1 int8 / uint8, the Softmax-ended tail_net), on one shard and on two.
- Every invalid call returns its code before any launch and leaves `out` untouched."""
import os

import numpy as np
import pytest

from oracle import topk
from tengine_b200 import abi, workloads

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "topk_example.npz")
_names = list(np.load(FIXTURE)["names"])


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _factor(e):
    """(c, h, w) with c * h * w == e, h * w > 1 and c not a multiple of 16 where e allows it."""
    for hw in (4, 9, 6, 2, 3, 5, 7, 11, 13):
        if e % hw == 0 and (e // hw) % 16:
            h = 2 if hw % 2 == 0 else (3 if hw == 9 else 1)
            return e // hw, h, hw // h
    return e, 1, 1


def _device_layout(q_nchw, poison):
    n, c, h, w = q_nchw.shape
    cp = (c + 15) // 16 * 16
    out = np.full((n, h, w, cp), poison, q_nchw.dtype)
    out[..., :c] = q_nchw.transpose(0, 2, 3, 1)
    return out


def _class_topk(ctx, q_nchw, scale, zp, u8, k, poison):
    import torch

    from tengine_b200 import runtime as rt

    n, c, h, w = q_nchw.shape
    din = torch.from_numpy(_device_layout(q_nchw, poison)).cuda()
    dout = torch.zeros((n, k, 2), dtype=torch.int32, device="cuda")
    rt.class_topk(din.data_ptr(), n, c, h, w, u8, scale, zp, k, dout.data_ptr(), ctx.stream)
    torch.cuda.synchronize()
    rec = dout.cpu().numpy()
    return rec[..., 0].view(np.float32), rec[..., 1]


@pytest.mark.parametrize("spatial", [False, True], ids=["Ex1x1", "CxHxW"])
@pytest.mark.parametrize("name", _names)
def test_kernel_reproduces_the_examples_committed_order(ctx, name, spatial):
    d = np.load(FIXTURE)
    i = _names.index(name)
    q = d[f"q_{i}"]
    s, zp, u8 = d[f"quant_{i}"]
    s, zp, u8 = np.float32(s), int(zp), bool(u8)
    e = q.size
    c, h, w = _factor(e) if spatial else (e, 1, 1)
    # three images per call: the case itself between its reverse and a rotation of it, so every CTA has its own answer
    batch = np.stack([q[::-1], q, np.roll(q, 7)]).reshape(3, c, h, w)
    want_s, want_i = topk.topk(batch, s, zp, u8, min(64, e))
    for k in sorted({1, min(5, e), min(64, e)}):
        got_s, got_i = _class_topk(ctx, batch, s, zp, u8, k, poison=(0x7F if not u8 else 0xFF))
        assert np.array_equal(got_i[1], d[f"ids_{i}"][:k]), (name, k)
        assert np.array_equal(_bits(got_s[1]), _bits(d[f"scores_{i}"][:k])), (name, k)
        assert np.array_equal(got_i, want_i[:, :k]) and np.array_equal(_bits(got_s), _bits(want_s[:, :k])), (name, k)


def test_kernel_at_the_largest_class_count(ctx):
    rng = np.random.default_rng(5)
    q = rng.integers(-127, 128, (2, abi.TOPK_MAX_CLASSES, 1, 1)).astype(np.int8)
    got_s, got_i = _class_topk(ctx, q, np.float32(0.01), 0, False, abi.TOPK_MAX, poison=0x7F)
    want_s, want_i = topk.topk(q, np.float32(0.01), 0, False, abi.TOPK_MAX)
    assert np.array_equal(got_i, want_i) and np.array_equal(_bits(got_s), _bits(want_s))


def _graphs():
    return [("mobilenet_int8", lambda: workloads.mobilenet_v1(abi.DT_INT8, batch=9, res=64, width=0.5, classes=100), [0]),
            ("mobilenet_uint8", lambda: workloads.mobilenet_v1(abi.DT_UINT8, batch=8, res=64, width=0.5, classes=100), [0]),
            ("tail_net_int8", lambda: workloads.tail_net(abi.DT_INT8, batch=5), [0, 1]),
            ("tail_net_uint8", lambda: workloads.tail_net(abi.DT_UINT8, batch=5), [0, 1])]


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("case", _graphs(), ids=[c[0] for c in _graphs()])
def test_graph_topk_equals_the_restatement_of_the_downloaded_output(case, shards):
    from tengine_b200 import runtime as rt

    _, make, outputs = case
    g, b = make()
    u8 = g.data_type == abi.DT_UINT8
    x = b.random_input(3)
    c = rt.Context(devices=[0] * shards) if shards > 1 else rt.Context(0)
    try:
        gr = rt.Graph(c, g)
        try:
            assert len(gr.shards()) == shards
            for how in ("run", "launch"):
                if how == "run":
                    gr.run([x])
                else:
                    gr.upload(0, x)
                    gr.launch()
                for oi in outputs:
                    t = g.tensors[g.outputs[oi]]
                    y = np.empty(g.dims(g.outputs[oi]), g.np_dtype)
                    for k in (5, 1):
                        got_s, got_i = gr.topk(oi, k)
                        gr.download(oi, y)
                        gr.sync()
                        want_s, want_i = topk.topk(y, np.float32(t["scale"]), int(t["zero_point"]), u8, k)
                        assert got_i.shape == (y.shape[0], k) and got_i.dtype == np.int32 and got_s.dtype == np.float32
                        assert np.array_equal(got_i, want_i), (how, oi, k)  # every image at its own row, the second shard's included
                        assert np.array_equal(_bits(got_s), _bits(want_s)), (how, oi, k)
        finally:
            gr.close()
    finally:
        c.close()


def test_errors_leave_out_untouched(ctx):
    import torch

    from tengine_b200 import runtime as rt
    from tengine_b200.graphdef import GraphDef

    L = rt.lib()
    g, b = workloads.tail_net(abi.DT_INT8, batch=2)
    gr = rt.Graph(ctx, g)
    big = GraphDef(abi.DT_INT8)
    big.mark_output(big.identity(big.input(1, 8, 65, 64, 0.02, 0)))  # 33280 classes per image
    gbig = rt.Graph(ctx, big)
    try:
        gr.run([b.random_input(1)])
        sentinel = 0x5A5A5A5A
        out = np.full((2 * 64, 2), sentinel, np.uint32)
        cases = [
            ("null graph", abi.ERR_INVALID, lambda: L.tb200_graph_topk(None, 0, 5, out.ctypes.data)),
            ("null out", abi.ERR_INVALID, lambda: L.tb200_graph_topk(gr.h, 0, 5, None)),
            ("output index", abi.ERR_INVALID, lambda: L.tb200_graph_topk(gr.h, 2, 5, out.ctypes.data)),
            ("negative index", abi.ERR_INVALID, lambda: L.tb200_graph_topk(gr.h, -1, 5, out.ctypes.data)),
            ("k 0", abi.ERR_INVALID, lambda: L.tb200_graph_topk(gr.h, 0, 0, out.ctypes.data)),
            ("k above E", abi.ERR_INVALID, lambda: L.tb200_graph_topk(gr.h, 0, 11, out.ctypes.data)),
            ("k above the maximum", abi.ERR_INVALID, lambda: L.tb200_graph_topk(gr.h, 1, abi.TOPK_MAX + 1, out.ctypes.data)),
            ("too many classes", abi.ERR_UNSUPPORTED, lambda: L.tb200_graph_topk(gbig.h, 0, 5, out.ctypes.data)),
        ]
        for name, code, call in cases:
            assert call() == code, (name, L.tb200_last_error())
            assert (out == sentinel).all(), name
        din = torch.zeros((2, 1, 1, 16), dtype=torch.int8, device="cuda")
        dout = torch.full((2 * 64, 2), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        kcases = [
            ("null in", abi.ERR_INVALID, (None, 2, 10, 1, 1, 0, 0.5, 0, 5, dout.data_ptr())),
            ("null out", abi.ERR_INVALID, (din.data_ptr(), 2, 10, 1, 1, 0, 0.5, 0, 5, None)),
            ("n 0", abi.ERR_INVALID, (din.data_ptr(), 0, 10, 1, 1, 0, 0.5, 0, 5, dout.data_ptr())),
            ("k 0", abi.ERR_INVALID, (din.data_ptr(), 2, 10, 1, 1, 0, 0.5, 0, 0, dout.data_ptr())),
            ("k above E", abi.ERR_INVALID, (din.data_ptr(), 2, 10, 1, 1, 0, 0.5, 0, 11, dout.data_ptr())),
            ("k above the maximum", abi.ERR_INVALID, (din.data_ptr(), 2, 10, 1, 1, 1, 0.5, 0, 65, dout.data_ptr())),
            ("inf scale", abi.ERR_INVALID, (din.data_ptr(), 2, 10, 1, 1, 0, float("inf"), 0, 5, dout.data_ptr())),
            ("too many classes", abi.ERR_UNSUPPORTED, (din.data_ptr(), 2, 32769, 1, 1, 0, 0.5, 0, 5, dout.data_ptr())),
        ]
        for name, code, args in kcases:
            assert L.tb200k_class_topk(*args, ctx.stream) == code, (name, L.tb200_last_error())
            torch.cuda.synchronize()
            assert bool((dout == 0x5A5A5A5A).all()), name
        # and the graph still answers
        y = np.empty(g.dims(g.outputs[0]), g.np_dtype)
        gr.download(0, y)
        gr.sync()
        t = g.tensors[g.outputs[0]]
        assert np.array_equal(gr.topk(0, 5)[1], topk.topk(y, np.float32(t["scale"]), int(t["zero_point"]), False, 5)[1])
    finally:
        gr.close(), gbig.close()
