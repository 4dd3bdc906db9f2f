"""The device against the UNMODIFIED reference (oracle/_ref, built by build() and run on the CPU here), directly, without the
oracle or the exact restatement in between.

  - every entry of tests/kernel_edges.py the reference can judge (all but the abi_only convs), every layer (fused entries: the
    graph output): int8 bit-exact; uint8 within 1 LSB, apart from kernel_edges.REFERENCE_DIVERGENCES (at most its listed LSB);
  - every uint8 conv / FC layer of full-size ResNet-50 (224x224) and YOLOv3-tiny (416x416), as a one-layer graph at batch 1 fed
    the oracle's input tensor of that layer: within 1 LSB of the reference, or listed in WORKLOAD_DIVERGENCES with its reason.
    The reference sums the products in fp32, which is exact only while the sum stays below 2^24; a failure names the layer's K
    and its largest |accumulator| against 2^24.
Needs an H100 (-m gpu) and oracle/_ref; skipped without the latter."""
import numpy as np
import pytest

from tengine_b200 import abi, workloads
from tests import kernel_edges as ke
from tests import ties
from tests.helpers import single_layer_graph

pytestmark = pytest.mark.gpu


def _lsb(a, b):
    return int(np.abs(a.astype(np.int32) - b.astype(np.int32)).max())


def _run_device(ctx, g, inputs, flags, fused=False):
    from tengine_b200 import runtime as rt

    gr = rt.Graph(ctx, g, abi.PRERUN_POISON_ARENA | (0 if fused else abi.PRERUN_NO_GRAPH) | flags)
    try:
        outs = gr.run(inputs)
        kernels = gr.layer_kernels()
        # under node fusion only the graph outputs exist; otherwise every layer's tensor is read back
        got = dict(zip(g.outputs, outs)) if fused else {L["output"]: gr.read_tensor(L["output"]) for L in g.layers}
    finally:
        gr.close()
    return got, kernels


@pytest.mark.parametrize("name", ke.reference_entries())
def test_edge_entry_on_device_against_reference(ctx, reference, name):
    e = ke.ENTRIES[name]
    case = ke.build(name)
    g = case.g
    got, kernels = _run_device(ctx, g, case.inputs, e.flags, e.fused)
    assert kernels[e.layer] == e.kernel, (name, kernels)
    ref, _ = reference.run(g, case.inputs, want=list(got))
    u8 = g.data_type == abi.DT_UINT8
    layer_of = {L["output"]: li for li, L in enumerate(g.layers)}
    over = {layer_of[t]: _lsb(got[t], ref[t]) for t in got if _lsb(got[t], ref[t]) > int(u8)}
    if name not in ke.REFERENCE_DIVERGENCES:
        assert not over, f"{name}: the device differs from the reference by (layer: LSB) {over}"
        return
    layer, most, why = ke.REFERENCE_DIVERGENCES[name]
    assert over and set(over) == {layer} and over[layer] <= most, \
        f"{name}: the device differs from the reference by (layer: LSB) {over}; listed ({layer}: 2..{most}): {why}"


# Full-size uint8 workloads: (net, layer index) -> why that layer may be more than 1 LSB from the reference (none found).
WORKLOAD_DIVERGENCES = {}


def _workload(net):
    if net == "resnet50":
        return workloads.resnet50(abi.DT_UINT8, batch=1)
    return workloads.yolov3_tiny(abi.DT_UINT8, batch=1)


def accumulator_stats(g, L, x):
    """K (products per output) and the largest |sum of (x - zx)(w - zw)| of a uint8 conv / FC layer over input x, exactly."""
    zx = g.tensors[L["inputs"][0]]["zero_point"]
    zw = L["weight_zero"]
    w = L["weight"]
    if L["op"] == abi.OP_FC:
        n = x.shape[0]
        acc = (x.reshape(n, -1).astype(np.float64) - zx) @ (w.reshape(w.shape[0], -1).astype(np.float64) - zw).T
        return x[0].size, float(np.abs(acc).max())
    acc = ties.conv_acc(x, w.reshape(w.shape[0], -1, L["kernel_h"], L["kernel_w"]), L, zx, zw)
    return w[0].size, float(np.abs(acc).max())


def workload_layers(net):
    """Every conv / FC layer of the full-size uint8 `net` at batch 1: (layer index, one-layer graph, its input from the oracle's
    run of the whole graph, K, largest |accumulator|)."""
    from oracle.pyoracle import Oracle

    g, b = _workload(net)
    x = b.random_input(7)
    full = Oracle().run(g, [x], uint8_mode=0)
    out = []
    for li, L in enumerate(g.layers):
        if L["op"] not in (abi.OP_CONV, abi.OP_FC):
            continue
        h, src = single_layer_graph(g, li)
        xin = full[src[0]]
        out.append((li, h, [xin], *accumulator_stats(g, L, xin)))
    return out


@pytest.mark.parametrize("net", ["resnet50", "yolov3_tiny"])
def test_uint8_workload_layers_on_device_against_reference(ctx, reference, net):
    bad, rows, flat = [], [], []
    layers = workload_layers(net)
    assert len(layers) == (54 if net == "resnet50" else 13), len(layers)
    for li, h, xs, k, acc in layers:
        got, _ = _run_device(ctx, h, xs, 0)
        ref, _ = reference.run(h, xs)
        t = h.outputs[0]
        d = _lsb(got[t], ref[t])
        rows.append(f"{net} layer {li}: K {k}, max |acc| {acc:.4g} = {acc / 2 ** 24:.3f} x 2^24, {d} LSB "
                    f"({int((got[t] != ref[t]).sum())} of {ref[t].size} bytes differ)")
        if d > 1 and (net, li) not in WORKLOAD_DIVERGENCES:
            bad.append(rows[-1])
        if len(np.unique(ref[t])) <= 8:
            flat.append(li)
    print("\n".join(rows))
    assert not bad, "\n".join(bad)
    assert not flat, f"{net}: layers {flat} have 8 output values or fewer: a 1-LSB bound says little there"
