"""The tie-dense layers of tests/ties.py on the CPU: the numpy exact reference equals the oracle bit for bit, and (where oracle/_ref
is built) the oracle equals the UNMODIFIED reference bit for bit, int8 and uint8 alike.

The usual +-1 LSB allowance for uint8 (the reference simulates uint8 in fp32 and its summation order rounds) does not apply
here: with power-of-two scales and these small accumulators every fp32 product and partial sum of the reference is exact, so
its fp32 simulation computes the same rational t as the integer one and any difference is a real disagreement at a tie."""
import numpy as np
import pytest

from tengine_b200 import abi
from tests import ties


def _cases():
    rng = lambda s: np.random.default_rng(1000 + s)  # noqa: E731
    H, R = abi.RECIPE_HCL, abi.RECIPE_REF
    return [
        ties.int8_conv(rng(1), 2, 32, 9, 11, 40, k=1, mode=1),
        ties.int8_conv(rng(2), 2, 32, 9, 11, 40, k=1, mode=0, activation=0),
        ties.int8_conv(rng(3), 1, 16, 10, 9, 24, k=3, pad=1, recipe=H, activation=6, mode=1),
        ties.int8_conv(rng(4), 1, 16, 10, 9, 24, k=3, pad=1, recipe=R, activation=6, mode=0),
        ties.int8_conv(rng(5), 1, 16, 11, 10, 24, k=3, stride=2, pad=1, recipe=R, mode=1),
        ties.int8_conv(rng(6), 2, 32, 9, 9, 32, k=3, pad=1, group=32, mode=1),  # depthwise
        ties.int8_conv(rng(7), 1, 32, 8, 8, 48, k=1, mode=2),
        ties.int8_fc(rng(8), 3, 96, 50, mode=0),
        ties.int8_fc(rng(9), 3, 96, 50, mode=2),
        ties.uint8_conv(rng(10), 2, 32, 9, 11, 40, k=1, mode=0),
        ties.uint8_conv(rng(11), 1, 16, 10, 9, 24, k=3, pad=1, recipe=H, activation=0),
        ties.uint8_conv(rng(12), 1, 16, 10, 9, 24, k=3, pad=1, recipe=R),
        ties.uint8_conv(rng(13), 2, 32, 9, 9, 32, k=3, pad=1, group=32),  # depthwise
        ties.uint8_conv(rng(14), 1, 32, 8, 8, 48, k=1, mode=2),
        ties.uint8_conv(rng(15), 3, 24, 2, 2, 40, fc=True),
        ties.eltwise(rng(16), False, abi.ELT_SUM), ties.eltwise(rng(17), True, abi.ELT_SUM),
        ties.eltwise(rng(18), False, abi.ELT_PROD), ties.eltwise(rng(19), True, abi.ELT_PROD),
        ties.relu(rng(20), False), ties.relu(rng(21), True), ties.relu(rng(22), False, 2), ties.relu(rng(23), True, 2),
        ties.pool(rng(24), False, abi.POOL_AVG, 2, 2), ties.pool(rng(25), True, abi.POOL_AVG, 2, 2, pad=1),
        ties.pool(rng(26), False, abi.POOL_AVG, 2, 2, pad=1, caffe=1), ties.pool(rng(27), True, abi.POOL_AVG, 2, 2, caffe=1),
        ties.pool(rng(28), False, abi.POOL_AVG, 4, 4, global_pool=True, shape=(2, 64, 4, 4), scale_ratio=0.25),
        ties.pool(rng(29), False, abi.POOL_MAX, 2, 2, scale_ratio=2), ties.pool(rng(30), True, abi.POOL_MAX, 3, 2, pad=1, scale_ratio=2),
        ties.concat(rng(31), False), ties.concat(rng(32), True),
    ]


CASES = _cases()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_exact_reference_equals_oracle(oracle, case):
    want, rs = ties.exact_run(case.g, case.inputs)
    out = case.g.outputs[0]
    ties.check_not_vacuous(case, rs[out])
    got = oracle.run(case.g, case.inputs, uint8_mode=0)
    assert np.array_equal(got[out], want[out])
    if case.g.data_type == abi.DT_UINT8:
        # the fp32 simulation of the reference (oracle mode 1) is exact at these scales too
        assert np.array_equal(oracle.run(case.g, case.inputs, uint8_mode=1)[out], want[out])


def test_zero_point_placement_matters_at_negative_ties():
    """uint8 ReLU and concat add the zero point inside round(), the convolution outside: at negative ties the two placements
    give different bytes, and the exact reference follows each op's own."""
    rng = np.random.default_rng(7)
    for case in (ties.relu(rng, True, 2), ties.concat(rng, True), ties.uint8_conv(rng, 1, 16, 6, 6, 24)):
        _, rs = ties.exact_run(case.g, case.inputs)
        r = rs[case.g.outputs[0]]
        assert (r.exact() != r.zp_swapped()).sum() >= 8, case.name


def _pointwise_kernel(g, L):
    """The kernel launch_pointwise runs for a ReLU / eltwise layer: the same-scale ReLU (kernels_direct.cu:863), the fast kernel
    whose value range is proven (:879), else the literal per-element pointwise_kernel."""
    u8 = g.data_type == abi.DT_UINT8
    t0, to = g.tensors[L["inputs"][0]], g.tensors[L["output"]]
    c = t0["dims"][1]
    s0, so, slope = np.float32(t0["scale"]), np.float32(to["scale"]), np.float32(L["negative_slope"])
    mode, s1 = 0, np.float32(0)
    if L["op"] == abi.OP_ELTWISE:
        mode, s1 = (1 if L["elt_type"] == abi.ELT_SUM else 2), np.float32(g.tensors[L["inputs"][1]]["scale"])
    if mode == 0 and slope == 0 and s0 == so and (not u8 or (t0["zero_point"] == to["zero_point"] and c % 16 == 0)):
        return "relu_same_scale_kernel"
    in0, a0, a1, so = (255.0 if u8 else 128.0), abs(float(s0)), abs(float(s1)), float(so)
    tmax = (in0 * a0 / so, in0 * (a0 + a1) / so, in0 * a0 * in0 * a1 / so)[mode]
    if 1e-30 < so < 1e30 and tmax + 256.0 < 32000.0 and (mode != 0 or 0 <= slope < 1) and c >= 16:
        return "pointwise_fast_kernel"
    return "pointwise_kernel"


def test_pointwise_cases_reach_their_kernels():
    """The *_pwexact cases of the device tie tests reach the literal pointwise_kernel by their channel count, the other ReLU /
    eltwise cases a fast kernel; all of them are tie-dense."""
    from tests.test_gpu_requant_ties import CASES as DEVICE_CASES, build

    names = [n for n in DEVICE_CASES if n.startswith(("eltwise_", "relu_", "leaky_relu_"))]
    assert sum(n.endswith("_pwexact") for n in names) == 6
    for name in names:
        case, _ = build(name)
        assert (_pointwise_kernel(case.g, case.g.layers[0]) == "pointwise_kernel") == name.endswith("_pwexact"), name
        _, rs = ties.exact_run(case.g, case.inputs)
        ties.check_not_vacuous(case, rs[case.g.outputs[0]])


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_oracle_equals_unmodified_reference(reference, oracle, case):
    want = oracle.run(case.g, case.inputs, uint8_mode=0)
    got, _ = reference.run(case.g, case.inputs)
    for t in case.g.outputs:
        assert np.array_equal(got[t], want[t]), case.name
