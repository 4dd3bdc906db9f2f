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
    return e, case, ke.geometry(case.g, case.g.layers[e.layer])


@pytest.mark.parametrize("name", NAMES)
def test_entry_reaches_its_geometry(name):
    e, case, geo = _geometry(name)
    for k, v in e.edges.items():
        assert k in geo, f"{name}: the geometry has no {k!r}: {geo}"
        assert geo[k] == v, f"{name}: {k} = {geo[k]}, meant {v}; geometry {geo}"
    if geo["kind"] in ("gemm", "igemm", "dw"):
        assert ke.kernel_name(geo) == e.kernel, (name, geo)
    if e.fused:
        assert e.kernel == "fused_into_producer"


def test_every_boundary_is_reached_on_each_side():
    seen = {k: set() for k in ke.BOUNDARIES}
    for name, e in ke.ENTRIES.items():
        for k, v in e.edges.items():
            if k in seen:
                seen[k].add(v)
    missing = {k: sorted(map(str, want - seen[k])) for k, want in ke.BOUNDARIES.items() if want - seen[k]}
    assert not missing, f"boundary sides no entry reaches: {missing}"


def test_par_all_boundary_sits_at_par_max():
    """ocp 2048 keeps every channel's epilogue constants resident, one more N tile of channels (2064) does not."""
    assert ke.gemm_geometry(2048, 0, m=16, k=64)["par_all"] == 1
    assert ke.gemm_geometry(2064, 0, m=16, k=64)["par_all"] == 0


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
