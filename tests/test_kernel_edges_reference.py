"""The edge case table of tests/kernel_edges.py against the UNMODIFIED reference (oracle/_ref), every layer of every entry the
reference can judge (all but the abi_only convs, whose recipe Tengine never picks for their shape).  The device is compared with
the oracle and the exact restatement elsewhere; this ties those stand-ins to the reference at the same edges.

  int8:  the oracle equals the reference bit for bit;
  uint8: the oracle's fp32 simulation (uint8_mode 1) equals the reference bit for bit, and the device's arithmetic (uint8_mode 0,
         the exact integer sum) is within 1 LSB of it, except on the entries of kernel_edges.REFERENCE_DIVERGENCES, which must
         still diverge, on their listed layer only and by no more than their listed maximum.
CPU only; skipped where oracle/_ref is not built."""
import numpy as np
import pytest

from tengine_b200 import abi
from tests import kernel_edges as ke
from tests.helpers import layer_outputs

NAMES = ke.reference_entries()


def _lsb(a, b):
    return int(np.abs(a.astype(np.int32) - b.astype(np.int32)).max())


@pytest.mark.parametrize("name", NAMES)
def test_entry_against_reference(oracle, reference, name):
    case = ke.build(name)
    g = case.g
    want = layer_outputs(g)
    ref, _ = reference.run(g, case.inputs, want=want)
    u8 = g.data_type == abi.DT_UINT8
    sim = oracle.run(g, case.inputs, uint8_mode=1 if u8 else 0)
    for li, t in enumerate(want):
        assert np.array_equal(sim[t], ref[t]), \
            f"{name}: layer {li} ({abi.OP_NAMES[g.layers[li]['op']]}) differs from the reference by up to {_lsb(sim[t], ref[t])} LSB " \
            f"in {int((sim[t] != ref[t]).sum())} of {ref[t].size} bytes" + (" (oracle uint8_mode 1)" if u8 else "")
    if not u8:
        assert name not in ke.REFERENCE_DIVERGENCES, f"{name}: int8 entries are bit-exact; the divergence table lists uint8 only"
        return
    dev = oracle.run(g, case.inputs, uint8_mode=0)
    over = {li: _lsb(dev[t], ref[t]) for li, t in enumerate(want) if _lsb(dev[t], ref[t]) > 1}
    if name not in ke.REFERENCE_DIVERGENCES:
        assert not over, f"{name}: the exact integer arithmetic is more than 1 LSB from the reference (layer: LSB) {over}"
        return
    layer, most, why = ke.REFERENCE_DIVERGENCES[name]
    assert over, f"{name}: listed as diverging ({why}) but within 1 LSB of the reference now: drop it from the table"
    assert set(over) == {layer} and over[layer] <= most, f"{name}: diverges by (layer: LSB) {over}, listed ({layer}: <= {most})"


def test_divergence_table_lists_reference_entries():
    for name, (layer, most, why) in ke.REFERENCE_DIVERGENCES.items():
        assert name in NAMES and ke.build(name).g.data_type == abi.DT_UINT8, name
        assert 0 <= layer < len(ke.build(name).g.layers) and most > 1 and why


def test_reference_judges_the_ref_clamp_where_tengine_runs_it():
    """[-1, 1] and ReLU6 under REF on the kernels conv_ref really serves (grouped direct convs, the generic depthwise, the int8
    depthwise 3x3 the HCL one turns down): enough entries here, of both dtypes, at both uint8 output zero points."""
    seen = set()
    for n in NAMES:
        e = ke.ENTRIES[n]
        if e.edges.get("act") in ("ref1", "ref6") and e.kernel in (ke.DR, ke.DD, ke.D_):
            seen.add((e.edges["act"], e.kernel, "_u8_" in n, e.edges.get("zo")))
    assert {(a, k, u8) for a, k, u8, _ in seen} >= {(a, ke.DR, u8) for a in ("ref1", "ref6") for u8 in (False, True)} | \
        {(a, ke.DD, True) for a in ("ref1", "ref6")} | {(a, k, False) for a in ("ref1", "ref6") for k in (ke.DD, ke.D_)}
    assert {zo for a, _, u8, zo in seen if a == "ref1" and u8} >= {0, 255}
