"""Parity of the CUDA path against the CPU oracle and the committed reference fixtures, through the C ABI
(tb200_graph_prerun / run / read_tensor).  Bar: bit-exact for int8; uint8 bit-exact against the exact-integer
oracle (mode 0) and within +-1 LSB of the reference's fp32 simulation.  Needs an H100: run with `-m gpu`."""
import numpy as np
import pytest

from tengine_b200 import abi, workloads
from tengine_b200.graphdef import GraphDef
from tests.helpers import dequant, kat_graphs, layer_outputs, load_golden

pytestmark = pytest.mark.gpu


def _run_all_layers(ctx, g, x, flags):
    from tengine_b200 import runtime as rt

    gr = rt.Graph(ctx, g, flags | abi.PRERUN_NO_GRAPH)
    try:
        outs = gr.run([x])
        tensors = {t: gr.read_tensor(t) for t in layer_outputs(g)}
        return outs, tensors, gr.layer_kernels()
    finally:
        gr.close()


FLAGS = [abi.PRERUN_DEFAULT, abi.PRERUN_NO_TENSORCORE]


# the KATs of the convolution / FC / pooling tests (single graph input); the glue-op KATs added later pin the oracle on the CPU
_GPU_KATS = [k for k in kat_graphs() if k[0] in ("uint8_conv3x3_pad1", "uint8_depthwise3x3_pad1", "uint8_fc", "uint8_maxpool3x3s2_const", "int8_conv3x3_bias")]


@pytest.mark.parametrize("flags", FLAGS, ids=["tensorcore", "cudacore"])
@pytest.mark.parametrize("kat", _GPU_KATS, ids=lambda k: k[0])
def test_reference_kats(ctx, kat, flags):
    name, g, xins, expected, tol = kat
    xin = xins[0]
    outs, _, _ = _run_all_layers(ctx, g, xin, flags)
    real = dequant(g, g.outputs[0], outs[0])
    assert np.abs(real - expected).max() <= tol + 1e-6


@pytest.mark.parametrize("flags", FLAGS, ids=["tensorcore", "cudacore"])
@pytest.mark.parametrize("name", ["ref_tiny_int8", "ref_mobilenet025_int8"])
def test_int8_bit_exact_vs_reference_fixture(ctx, name, flags):
    g, x, ref = load_golden(name)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, flags)
    for li, L in enumerate(g.layers):
        t = L["output"]
        assert np.array_equal(tensors[t], ref[t]), f"{name}: layer {li} ({kernels[li]}) differs from the reference"
    for o, t in zip(outs, g.outputs):
        assert np.array_equal(o, ref[t])
    if flags == abi.PRERUN_DEFAULT and "mobilenet" in name:
        assert any("tcgen05" in k for k in kernels), kernels


@pytest.mark.parametrize("name", ["ref_resnet50_small_int8", "ref_yolov3_tiny_small_int8"])
def test_int8_benchmark_graphs_vs_reference_fixture(ctx, name):
    """Reduced ResNet-50 / YOLOv3-tiny (7x7 stem on the gather kernel, implicit GEMMs, same-scale max pooling and ReLU as byte
    operations, leaky ReLU, eltwise, concat, upsample): every layer equals the bytes the UNMODIFIED reference produced."""
    g, x, ref = load_golden(name)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, abi.PRERUN_DEFAULT)
    for li, L in enumerate(g.layers):
        t = L["output"]
        assert np.array_equal(tensors[t], ref[t]), f"{name}: layer {li} ({kernels[li]}) differs from the reference"
    assert any("tcgen05" in k for k in kernels), kernels


@pytest.mark.parametrize("name", ["ref_tiny_uint8", "ref_mobilenet025_uint8"])
def test_uint8_vs_reference_fixture(ctx, oracle, name):
    g, x, ref = load_golden(name)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, abi.PRERUN_DEFAULT)
    exact = oracle.run(g, [x], uint8_mode=0)
    for li, L in enumerate(g.layers):
        t = L["output"]
        assert np.array_equal(tensors[t], exact[t]), f"{name}: layer {li} ({kernels[li]}) differs from the exact-integer oracle"
    # against the reference's own bytes: errors of +-1 LSB propagate, so allow a small budget on the final output
    d = np.abs(outs[0].astype(int) - ref[g.outputs[0]].astype(int))
    assert d.max() <= 2, int(d.max())


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
@pytest.mark.parametrize("flags", FLAGS, ids=["tensorcore", "cudacore"])
def test_tiny_net_every_layer_vs_oracle(ctx, oracle, dtype, flags):
    g, b = workloads.tiny_net(dtype, batch=3, seed=33)
    x = b.random_input(4)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, flags)
    want = oracle.run(g, [x], uint8_mode=0)
    for li, L in enumerate(g.layers):
        t = L["output"]
        assert np.array_equal(tensors[t], want[t]), f"layer {li} {abi.OP_NAMES[L['op']]} ({kernels[li]})"


def _one_conv(rng, dtype, n, c, h, w, oc, k, s, p, group, act, recipe, bias=True, dilation=1):
    g = GraphDef(dtype)
    u8 = dtype == abi.DT_UINT8
    x = g.input(n, c, h, w, 0.02, 131 if u8 else 0)
    kk = (c // group) * k * k
    if u8:
        wq, ws, wz = rng.integers(0, 256, (oc, c // group, k, k)).astype(np.uint8), [0.004], 117
        so = 0.02 * 0.004 * np.sqrt(kk) * 74 * 74 / 100
    else:
        wq, ws, wz = rng.integers(-127, 128, (oc, c // group, k, k)).astype(np.int8), rng.uniform(0.001, 0.01, oc), 0
        so = 0.02 * 0.0055 * np.sqrt(kk) * 73 * 73 / 100
    b = rng.integers(-2000, 2000, oc).astype(np.int32) if bias else None
    y = g.conv(x, wq, b, ws, so, 110 if u8 else 0, stride=s, pad=p, dilation=dilation, group=group, activation=act, recipe=recipe,
               weight_zero=wz)
    g.mark_output(y)
    xin = rng.integers(0, 256, (n, c, h, w)).astype(np.uint8) if u8 else rng.integers(-127, 128, (n, c, h, w)).astype(np.int8)
    return g, xin


# 1x1 GEMM shapes: every K-block / swizzle mode (K 16..1024), ragged M (not a multiple of 128), odd channel counts
GEMM_CASES = [
    (1, 16, 7, 7, 16), (2, 32, 9, 9, 64), (1, 48, 5, 5, 24), (3, 64, 11, 13, 128), (1, 80, 6, 6, 40), (2, 128, 14, 14, 128),
    (1, 256, 14, 14, 512), (1, 512, 7, 7, 1024), (2, 1024, 7, 7, 1000), (1, 1024, 1, 1, 1000), (5, 128, 3, 3, 255), (1, 384, 13, 13, 256),
    (4, 32, 112, 112, 64),
]


@pytest.mark.parametrize("case", GEMM_CASES, ids=lambda c: "n%d_k%d_%dx%d_oc%d" % c)
@pytest.mark.parametrize("act,recipe,dtype", [(0, abi.RECIPE_HCL, abi.DT_INT8), (6, abi.RECIPE_REF, abi.DT_INT8),
                                              (-1, abi.RECIPE_HCL, abi.DT_INT8), (0, abi.RECIPE_HCL, abi.DT_UINT8),
                                              (-1, abi.RECIPE_REF, abi.DT_UINT8)])
def test_tcgen05_gemm_1x1_bit_exact(ctx, oracle, case, act, recipe, dtype):
    """uint8 runs the same UMMA with unsigned operands; the zero points are folded exactly (ones-row sum of x,
    per-channel sum of w): bit-exact against the exact-integer oracle."""
    from tengine_b200 import runtime as rt

    n, c, h, w, oc = case
    rng = np.random.default_rng(sum(case))
    g, x = _one_conv(rng, dtype, n, c, h, w, oc, 1, 1, 0, 1, act, recipe)
    gr = rt.Graph(ctx, g)
    try:
        assert gr.layer_kernels() == ["gemm_i8_tcgen05"]
        got = gr.run([x])[0]
    finally:
        gr.close()
    want = oracle.run(g, [x], uint8_mode=0)[g.outputs[0]]
    if dtype == abi.DT_INT8:
        assert (np.abs(want.astype(int)) == 127).mean() < 0.3
    assert np.array_equal(got, want)


CONV_CASES = [
    # n, c, h, w, oc, k, s, p, group
    (2, 3, 32, 32, 32, 3, 2, 1, 1),     # stem (NCHW input, C=3)
    (1, 3, 31, 29, 16, 7, 2, 3, 1),     # 7x7 stem, odd sizes
    (2, 16, 15, 15, 24, 3, 1, 1, 1),    # 3x3 s1
    (2, 32, 16, 16, 48, 3, 2, 1, 1),    # 3x3 s2
    (1, 32, 16, 16, 32, 3, 1, 1, 32),   # depthwise s1
    (3, 64, 15, 15, 64, 3, 2, 1, 64),   # depthwise s2, batch 3
    (2, 8, 9, 9, 16, 3, 1, 1, 2),       # grouped
    (1, 24, 10, 10, 40, 5, 1, 2, 1),    # 5x5
    (1, 20, 9, 9, 255, 1, 1, 0, 1),     # odd Cout (YOLO head), Cin not multiple of 16
    (2, 16, 12, 12, 16, 3, 1, 2, 1),    # pad > (k-1)/2
    (2, 3, 64, 48, 64, 7, 2, 3, 1),     # 7x7 stem, TMA-staged window (W % 16 == 0)
    (3, 3, 40, 32, 16, 3, 1, 1, 1),     # 3x3 s1 stem, several tiles per image, ragged tile rows
    (2, 3, 37, 48, 24, 3, 2, 0, 1),     # stem without padding
    (2, 32, 21, 19, 64, 3, 1, 1, 1),    # 32-channel 3x3 (window kernel, NHWC 32 B/pixel), ragged tiles
    (2, 24, 18, 18, 40, 3, 2, 1, 1),    # 24 real channels in a 32-byte pixel: pad lanes must stay out of the uint8 sums
    (1, 12, 20, 20, 16, 3, 1, 1, 1),    # 12 real channels in a 16-byte pixel
    (2, 32, 18, 18, 256, 3, 2, 1, 1),   # 32-channel 3x3 whose window kernel would not fit shared memory (implicit GEMM)
    (1, 32, 17, 17, 192, 3, 1, 1, 1),   # the same at stride 1
    (1, 16, 14, 14, 256, 3, 2, 1, 1),   # 16-channel 3x3, wide output: the global-memory gather kernel
]


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n%d_c%d_%dx%d_oc%d_k%d_s%d_p%d_g%d" % c)
def test_conv_kernels_bit_exact(ctx, oracle, dtype, case):
    from tengine_b200 import runtime as rt

    n, c, h, w, oc, k, s, p, group = case
    rng = np.random.default_rng(sum(case) + dtype)
    for act, recipe in ((0, abi.RECIPE_HCL), (6, abi.RECIPE_REF)):
        g, x = _one_conv(rng, dtype, n, c, h, w, oc, k, s, p, group, act, recipe, bias=(act == 0))
        gr = rt.Graph(ctx, g)
        try:
            got = gr.run([x])[0]
            kern = gr.layer_kernels()[0]
        finally:
            gr.close()
        want = oracle.run(g, [x], uint8_mode=0)[g.outputs[0]]
        assert np.array_equal(got, want), (kern, act, recipe)


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
@pytest.mark.parametrize("case", [(2, 32, 15, 15, 48, 3, 1, 2, 1, 2), (1, 16, 17, 17, 24, 3, 2, 3, 1, 3), (2, 64, 12, 12, 64, 3, 1, 2, 64, 2),
                                  (1, 8, 11, 11, 16, 3, 1, 2, 2, 2)],
                         ids=["dil2", "dil3_s2", "depthwise_dil2", "grouped_dil2"])
def test_dilated_conv_bit_exact(ctx, oracle, dtype, case):
    """dilation > 1 (conv_kernel_ref_int8.c:104-121 tap addressing): the general direct kernel, dense / depthwise / grouped."""
    from tengine_b200 import runtime as rt

    n, c, h, w, oc, k, s, p, group, dil = case
    rng = np.random.default_rng(sum(case) + dtype)
    g, x = _one_conv(rng, dtype, n, c, h, w, oc, k, s, p, group, 0, abi.RECIPE_REF, dilation=dil)
    gr = rt.Graph(ctx, g)
    try:
        got = gr.run([x])[0]
        kern = gr.layer_kernels()[0]
    finally:
        gr.close()
    want = oracle.run(g, [x], uint8_mode=0)[g.outputs[0]]
    assert np.array_equal(got, want), kern


def test_empty_and_bad_inputs_fail_cleanly(ctx):
    from tengine_b200 import runtime as rt

    g = GraphDef(abi.DT_INT8)
    x = g.input(1, 8, 4, 4, 0.1)
    y = g.conv(x, np.zeros((8, 8, 1, 1), np.int8), None, np.ones(8, np.float32), 0.1)
    g.tensors[y]["dims"] = (1, 8, 3, 3)  # wrong output shape for a 1x1 conv
    g.mark_output(y)
    with pytest.raises(rt.TB200Error) as e:
        rt.Graph(ctx, g)
    assert e.value.code == abi.ERR_INVALID


def test_mobilenet_v1_int8_batch_properties(ctx, oracle):
    """Full-size C2 workload (MobileNet-v1 224x224, batch 256 is too slow for the CPU oracle): check (a) a batch of 8
    against the oracle on every layer, (b) at batch 64 that every image equals its own batch-1 run (images are
    independent units) and that the CUDA-core cross-check path gives the same bytes as the tcgen05 path."""
    from tengine_b200 import runtime as rt

    g8, b8 = workloads.mobilenet_v1(abi.DT_INT8, batch=8)
    x8 = b8.random_input(8)
    outs, tensors, kernels = _run_all_layers(ctx, g8, x8, abi.PRERUN_DEFAULT)
    want = oracle.run(g8, [x8])
    for li, L in enumerate(g8.layers):
        assert np.array_equal(tensors[L["output"]], want[L["output"]]), f"layer {li} ({kernels[li]})"
    assert sum("tcgen05" in k for k in kernels) == 15  # stem + 13 pointwise + fc

    g64, b64 = workloads.mobilenet_v1(abi.DT_INT8, batch=64)
    x64 = b64.random_input(64)
    gr = rt.Graph(ctx, g64)
    y64 = gr.run([x64])[0]
    gr.close()
    gr = rt.Graph(ctx, g64, abi.PRERUN_NO_TENSORCORE)
    y64_cc = gr.run([x64])[0]
    gr.close()
    assert np.array_equal(y64, y64_cc)
    g1, _ = workloads.mobilenet_v1(abi.DT_INT8, batch=1, dw_recipe=abi.RECIPE_REF)
    gr = rt.Graph(ctx, g1)
    for i in (0, 17, 63):
        y1 = gr.run([x64[i:i + 1]])[0]
        assert np.array_equal(y1[0], y64[i])
    gr.close()
    assert len(np.unique(y64)) > 50


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
@pytest.mark.parametrize("net", ["resnet50", "yolov3_tiny"])
def test_reference_benchmark_graphs_every_layer(ctx, oracle, net, dtype):
    """C3 / C4 of BASELINE.json at reduced width (same layer kinds, order and shapes' structure as the reference's
    resnet50 / yolov3_tiny benchmark tmfiles): every layer against the oracle, bit-exact (uint8: exact-integer oracle)."""
    if net == "resnet50":
        g, b = workloads.resnet50(dtype, batch=2, res=96, width=0.25, classes=40, seed=5)
    else:
        g, b = workloads.yolov3_tiny(dtype, batch=2, res=96, width=0.25, head=27, seed=6)
    x = b.random_input(2)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, abi.PRERUN_DEFAULT)
    want = oracle.run(g, [x], uint8_mode=0)
    for li, L in enumerate(g.layers):
        assert np.array_equal(tensors[L["output"]], want[L["output"]]), f"{net} layer {li} {abi.OP_NAMES[L['op']]} ({kernels[li]})"


FULL = [("resnet50", abi.DT_UINT8, 3), ("resnet50", abi.DT_INT8, 2), ("yolov3_tiny", abi.DT_UINT8, 2), ("yolov3_tiny", abi.DT_INT8, 2)]


@pytest.mark.parametrize("net,dtype,batch", FULL, ids=lambda v: str(v))
def test_full_size_benchmark_graphs_every_layer(ctx, oracle, net, dtype, batch):
    """C3 (ResNet-50 224x224) and C4 (YOLOv3-tiny 416x416) of BASELINE.json at their REAL width and resolution -- K up to 4608,
    OC up to 2048, several N tiles with non-resident weights, the 16-bit clamp-range proof deciding MODE per layer -- at a batch
    the CPU oracle finishes in seconds: every layer bit-exact (uint8: against the exact-integer oracle)."""
    g, b = getattr(workloads, net)(dtype, batch=batch)
    x = b.random_input(3)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, abi.PRERUN_DEFAULT)
    want = oracle.run(g, [x], uint8_mode=0)
    for li, L in enumerate(g.layers):
        assert np.array_equal(tensors[L["output"]], want[L["output"]]), f"{net} layer {li} {abi.OP_NAMES[L['op']]} ({kernels[li]})"
    for o, t in zip(outs, g.outputs):
        assert np.array_equal(o, want[t])
        assert len(np.unique(o)) > 20
    assert sum("tcgen05" in k for k in kernels) >= (13 if net == "yolov3_tiny" else 54)


@pytest.mark.parametrize("net,dtype,batch", [("resnet50", abi.DT_UINT8, 128), ("yolov3_tiny", abi.DT_UINT8, 128)], ids=lambda v: str(v))
def test_full_size_batch_independence(ctx, oracle, net, dtype, batch):
    """At the real batch the CPU oracle is too slow; images are independent units, so every image of the big batch must equal
    the same image run in a small batch that the previous test pins to the oracle (captured CUDA graph, pipelined run)."""
    from tengine_b200 import runtime as rt

    g, b = getattr(workloads, net)(dtype, batch=batch)
    x = b.random_input(9)
    gr = rt.Graph(ctx, g)
    big = gr.run([x])
    gr.close()
    g2, _ = getattr(workloads, net)(dtype, batch=2)
    gr = rt.Graph(ctx, g2)
    try:
        for i in (0, batch // 2 - 1, batch - 2):
            small = gr.run([x[i:i + 2]])
            for o_big, o_small in zip(big, small):
                assert np.array_equal(o_big[i:i + 2], o_small), f"{net}: images {i},{i + 1} differ between batch {batch} and batch 2"
    finally:
        gr.close()
    want = oracle.run(g2, [x[:2]], uint8_mode=0)
    for o_big, t in zip(big, g2.outputs):
        assert np.array_equal(o_big[:2], want[t])


@pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])
def test_yolov5s_every_layer(ctx, oracle, dtype):
    """C5 (YOLOv5s 640x640: conv + sigmoid*x / HardSwish, C3 blocks, SPP 5/9/13 max pools, 4-input concat, PANet head) at full
    size, batch 2: every layer bit-exact against the oracle; then the default plan (captured graph, fused nodes, slot reuse)."""
    from tengine_b200 import runtime as rt

    g, b = workloads.yolov5s(dtype, batch=2)
    x = b.random_input(4)
    outs, tensors, kernels = _run_all_layers(ctx, g, x, abi.PRERUN_DEFAULT)
    want = oracle.run(g, [x], uint8_mode=0)
    for li, L in enumerate(g.layers):
        assert np.array_equal(tensors[L["output"]], want[L["output"]]), f"yolov5s layer {li} {abi.OP_NAMES[L['op']]} ({kernels[li]})"
    gr = rt.Graph(ctx, g)
    fast = gr.run([x])
    gr.close()
    for o, t in zip(fast, g.outputs):
        assert np.array_equal(o, want[t]) and len(np.unique(o)) > 50


def test_eltwise_relu_fusion_is_used_and_exact(ctx, oracle):
    from tengine_b200 import runtime as rt

    g, b = workloads.resnet50(abi.DT_UINT8, batch=2, res=64, width=0.5, classes=30, seed=9)
    x = b.random_input(1)
    gr = rt.Graph(ctx, g)
    try:
        assert gr.layer_kernels().count("fused_into_producer") == 16  # every bottleneck's standalone ReLU
        got = gr.run([x])[0]
    finally:
        gr.close()
    assert np.array_equal(got, oracle.run(g, [x], uint8_mode=0)[g.outputs[0]])


def test_pipelined_run_equals_unpipelined(ctx):
    """tb200_graph_run cuts the batch into chunks and overlaps H2D / kernels / D2H; same bytes as the single-chunk plan."""
    import os
    from tengine_b200 import runtime as rt

    g, b = workloads.mobilenet_v1(abi.DT_INT8, batch=32, res=96, width=0.5, classes=50)
    x = b.random_input(7)
    outs = []
    for chunks in ("1", "4", "2"):
        os.environ["TB200_PIPELINE_CHUNKS"] = chunks
        try:
            gr = rt.Graph(ctx, g)
            outs.append(gr.run([x])[0])
            outs.append(gr.run([x])[0])  # twice: buffers are reused
            gr.close()
        finally:
            os.environ.pop("TB200_PIPELINE_CHUNKS", None)
    os.environ["TB200_PIPELINE_SPLIT"] = "5,11,16"  # uneven chunks
    try:
        gr = rt.Graph(ctx, g)
        outs.append(gr.run([x])[0])
        gr.close()
    finally:
        os.environ.pop("TB200_PIPELINE_SPLIT", None)
    for o in outs[1:]:
        assert np.array_equal(o, outs[0])
