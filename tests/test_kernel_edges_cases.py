"""The edge case table of tests/kernel_edges.py on the CPU: each entry reaches the plan geometry it is meant to (per the Python
restatement of the planners), every boundary is probed from both sides, the tie-dense cases are not vacuous, and the exact
reference agrees with the oracle on every case."""
import numpy as np
import pytest

from tests import kernel_edges as ke
from tests import ties

NAMES = list(ke.ENTRIES)


def _geometry(name):
    e = ke.ENTRIES[name]
    case = ke.build(name)
    return e, case, ke.reached(case, e)


@pytest.mark.parametrize("name", NAMES)
def test_entry_reaches_its_geometry(name):
    e, case, geo = _geometry(name)
    for k, v in e.edges.items():
        assert k in geo, f"{name}: the geometry has no {k!r}: {geo}"
        assert geo[k] == v, f"{name}: {k} = {geo[k]}, meant {v}; geometry {geo}"
    if geo["kind"] in ke.KERNEL_NAME or geo["kind"] == "dw":
        assert ke.kernel_name(geo) == e.kernel, (name, geo)
    if e.fused:
        assert e.kernel == "fused_into_producer"


def test_every_boundary_is_reached_on_each_side():
    seen = {k: set() for k in ke.BOUNDARIES}
    for name, e in ke.ENTRIES.items():
        for k, v in e.edges.items():
            if k in seen:
                seen[k].add(v)
        if e.kernel in ke.CONV_KERNELS:
            seen["abi_only"].add(e.abi_only)
    missing = {k: sorted(map(str, want - seen[k])) for k, want in ke.BOUNDARIES.items() if want - seen[k]}
    assert not missing, f"boundary sides no entry reaches: {missing}"


@pytest.mark.parametrize("name", NAMES)
def test_entry_has_the_recipe_tengine_picks_unless_abi_only(name):
    """A conv entry carries the recipe b200_device.cc conv_recipe gives its shape (what the unmodified reference runs), or is
    marked abi_only: a recipe that only a C-ABI caller can ask for."""
    e = ke.ENTRIES[name]
    case = ke.build(name)
    L = case.g.layers[e.layer]
    if L["op"] != ke.abi.OP_CONV:
        assert not e.abi_only, f"{name}: abi_only on a layer that is not a convolution"
        return
    tengine = ke.conv_recipe(case.g, L)
    assert (L["recipe"] != tengine) == e.abi_only, \
        f"{name}: recipe {L['recipe']}, conv_recipe gives {tengine}, abi_only={e.abi_only}"


def test_conv_recipe_restates_the_device_glue():
    """Group 1 is HCL; a depthwise conv is HCL only for int8 at batch 1, 3x3, stride 1 or 2, each axis padded alike on both
    sides (pad_h may differ from pad_w); every other grouped conv, and every uint8 one, is REF."""
    from tengine_b200.graphdef import GraphDef

    def recipe(dtype, n, c, oc, k, stride, pad, group, dilation=1):
        g = GraphDef(dtype)
        u8 = dtype == ke.abi.DT_UINT8
        x = g.input(n, c, 12, 12, 0.5, 128 if u8 else 0)
        w = np.zeros((oc, c // group, k, k), np.uint8 if u8 else np.int8)
        g.conv(x, w, None, [0.5] * (1 if u8 else oc), 0.5, 128 if u8 else 0, stride=stride, pad=pad, group=group, dilation=dilation)
        return ke.conv_recipe(g, g.layers[0])

    H, R, I8, U8 = ke.abi.RECIPE_HCL, ke.abi.RECIPE_REF, ke.abi.DT_INT8, ke.abi.DT_UINT8
    assert recipe(I8, 4, 16, 32, 3, 1, 1, 1) == H and recipe(U8, 4, 16, 32, 5, 2, 0, 1) == H
    assert recipe(I8, 1, 32, 32, 3, 1, 1, 32) == H and recipe(I8, 1, 32, 32, 3, 2, (1, 1, 0, 0), 32) == H
    assert recipe(I8, 2, 32, 32, 3, 1, 1, 32) == R  # batched
    assert recipe(U8, 1, 32, 32, 3, 1, 1, 32) == R  # uint8
    assert recipe(I8, 1, 32, 32, 5, 1, 2, 32) == R  # 5x5
    assert recipe(I8, 1, 32, 32, 3, 3, 1, 32) == R  # stride 3
    assert recipe(I8, 1, 32, 32, 3, 1, 2, 32, dilation=2) == R
    assert recipe(I8, 1, 32, 32, 3, 1, (0, 1, 1, 1), 32) == R  # one-sided padding
    assert recipe(I8, 1, 32, 32, 3, 1, 1, 4) == R  # grouped, not depthwise
    assert recipe(I8, 1, 32, 64, 3, 1, 1, 32) == R  # group == C but OC != C


def test_par_all_boundary_sits_at_par_max():
    """ocp 2048 keeps every channel's epilogue constants resident, one more N tile of channels (2064) does not."""
    assert ke.gemm_geometry(2048, 0, m=16, k=64)["par_all"] == 1
    assert ke.gemm_geometry(2064, 0, m=16, k=64)["par_all"] == 0


def test_window_limits_sit_where_shared_memory_ends():
    """window_nhwc_fits: 32-byte pixels fit up to OCp 176 at stride 1 and 144 at stride 2; 16-byte pixels at stride 2 up to 224
    (the gather kernel takes 240); a 7x7 NCHW window over 3 channels at OCp 256 fits at xoff 0, not at xoff 13."""
    assert [ke.window_nhwc_fits(32, o, 1) for o in (176, 192)] == [True, False]
    assert [ke.window_nhwc_fits(32, o, 2) for o in (144, 160)] == [True, False]
    assert [ke.window_nhwc_fits(16, o, 2) for o in (224, 240)] == [True, False]
    assert ke.window_nhwc_fits(16, 256, 1)
    g = dict(n=1, c=3, cp=16, w=32, oh=8, ow=16, k=7, stride=2, ocp=256, nhwc=0)
    assert ke.window_geometry(pw0=0, **g)["valid"] and not ke.window_geometry(pw0=3, **g)["valid"]


def test_window_and_gather_entries_are_listed():
    """The NCHW stems over 1 and 2 channels with a 7x7 kernel (k-steps 2 and 4 of the 5 a 147-byte row could fill) through both
    kernels, and window entries of 3 or more images for the partial-batch test."""
    ks = {(ke.ENTRIES[n].kernel, ke.layer_geometry(ke.build(n).g, ke.build(n).g.layers[0]).get("ks")) for n in ke.window_entries()}
    assert {(k, s) for k in (ke.WI, ke.GA) for s in (2, 4)} <= ks
    assert len(ke.window_batch_entries()) >= 4


@pytest.mark.parametrize("name", [n for n in NAMES if ke.ENTRIES[n].ties])
def test_tie_dense_case_is_not_vacuous(name):
    e = ke.ENTRIES[name]
    case = ke.build(name)
    _, rs = ties.exact_run(case.g, case.inputs)
    # fused pairs: the ties are the first node's (a same-scale ReLU / max pooling after it rounds nothing)
    t = case.g.layers[e.tie_layer]["output"]
    ties.check_not_vacuous(case, rs[t])


@pytest.mark.parametrize("name", [n for n in NAMES if ke.ENTRIES[n].ref == "exact"])
def test_exact_reference_equals_oracle(oracle, name):
    case = ke.build(name)
    want, _ = ties.exact_run(case.g, case.inputs)
    got = oracle.run(case.g, case.inputs, uint8_mode=0)
    for L in case.g.layers:
        t = L["output"]
        assert np.array_equal(got[t], want[t]), f"{name}: tensor {t} differs in {int((got[t] != want[t]).sum())} bytes"


def test_gemm_entries_are_listed():
    """The GEMM entries the GPU test ties to the library's own plan print, and the uint8 ones of its negative control."""
    assert len(ke.gemm_entries()) >= 30
    u8 = ke.uint8_gemm_entries()
    assert u8 and all(ke.build(n).g.data_type == ke.abi.DT_UINT8 for n in u8)


FAR = [n for n in NAMES if "_far_" in n]


@pytest.mark.parametrize("name", FAR)
def test_far_end_entries_leave_the_exact_reference(oracle, name):
    """|x - zx| = |w - zw| near 255 puts the accumulator past 2^24, where the reference rounds it to fp32 before it scales it:
    ties.exact_layer refuses the layer instead of disagreeing quietly, and the oracle's outputs still spread."""
    case = ke.build(name)
    assert case.notes["acc_max"] >= 255 ** 2 * 4608 * 0.8, case.notes
    with pytest.raises(AssertionError, match="2\\^24"):
        ties.exact_run(case.g, case.inputs)
    out = oracle.run(case.g, case.inputs, uint8_mode=0)[case.g.outputs[0]]
    assert len(np.unique(out)) >= 16, np.unique(out)


def test_large_accumulator_entries_are_listed():
    """At K = 4608 and 25088, with both uint8 operand regimes that carry a correction term."""
    assert {ke.ENTRIES[n].edges["k_blocks"] for n in FAR} == {36, 196}
    assert {ke.ENTRIES[n].edges["b_signed"] for n in FAR} == {0, 1}


def test_negative_control_splits_on_cplane():
    """The uint8 GEMM entries of the GPU negative control: some with a cplane term (they must fail without it), some without
    (zw 0 or 128: they must pass); an entry left out has one output byte only, by its exact reference."""
    nc = ke.negative_control_entries()
    assert any(nc.values()) and not all(nc.values())
    assert {ke.gemm_geometry_of(ke.build(n), ke.ENTRIES[n])["u8_operands"] for n, c in nc.items() if not c} == {"unsigned_b", "no_cplane"}
    for n in ke.uint8_gemm_entries():
        case = ke.build(n)
        if ke.ENTRIES[n].ref != "exact":
            assert n in nc
            continue
        want, _ = ties.exact_run(case.g, case.inputs)
        constant = len(np.unique(want[case.g.outputs[0]])) == 1
        assert constant == (n not in nc), (n, constant)
