"""The edge cases of tests/kernel_edges.py on the device: every layer bit-exact against the exact reference (or the oracle, for
ops outside ties.exact_layer), with the kernel each entry is meant to reach asserted by name.

Two child processes (`python -m tests.test_gpu_kernel_edges <entry>...`) cover what the library reads once per process:
  - TB200_DEBUG_LAUNCH: the GEMM's printed plan equals kernel_edges.gemm_geometry for every GEMM entry, so the Python
    restatement cannot drift from the code unnoticed;
  - TB200_DEBUG_NO_CPLANE (documented to give wrong uint8 results): the uint8 GEMM entries must FAIL there -- a sweep that passed
    under a known-wrong kernel would prove nothing."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tengine_b200 import abi
from tests import kernel_edges as ke
from tests import ties

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MARK = "kernel_edges case "


def run_entry(ctx, oracle, name):
    """Run entry `name` on the device and compare.  Returns a message or None."""
    from tengine_b200 import runtime as rt

    e = ke.ENTRIES[name]
    case = ke.build(name)
    g = case.g
    if e.ref == "exact":
        want, rs = ties.exact_run(g, case.inputs)
    else:
        want, rs = oracle.run(g, case.inputs, uint8_mode=0), {}
    flags = abi.PRERUN_POISON_ARENA | (0 if e.fused else abi.PRERUN_NO_GRAPH)
    gr = rt.Graph(ctx, g, flags)
    try:
        outs = gr.run(case.inputs)
        kernels = gr.layer_kernels()
        # under node fusion only the graph outputs exist; otherwise every layer's tensor is read back
        got = {t: o for t, o in zip(g.outputs, outs)} if e.fused else {L["output"]: gr.read_tensor(L["output"]) for L in g.layers}
    finally:
        gr.close()
    if kernels[e.layer] != e.kernel:
        return f"{name}: layer {e.layer} ran {kernels[e.layer]}, meant {e.kernel} (all: {kernels})"
    for li, L in enumerate(g.layers):
        t = L["output"]
        if t not in got:
            continue
        bad = got[t] != want[t]
        if bad.any():
            tie = rs[t].tie_mask() if t in rs else np.zeros_like(bad)
            return (f"{name}: layer {li} ({kernels[li]}) differs from the {e.ref} reference in {int(bad.sum())} of {bad.size} bytes, "
                    f"{int((bad & tie).sum())} of them at exact ties; first at {np.argwhere(bad)[0].tolist()}")
    for t, o in zip(g.outputs, outs):
        if not np.array_equal(o, want[t]):
            return f"{name}: graph output {t} differs from the reference"
    return None


@pytest.mark.parametrize("name", list(ke.ENTRIES))
def test_edge_case(ctx, oracle, name):
    msg = run_entry(ctx, oracle, name)
    assert msg is None, msg


def _child(names, env, timeout=900):
    e = dict(os.environ)
    e.update(env)
    return subprocess.run([sys.executable, "-m", "tests.test_gpu_kernel_edges"] + names, cwd=ROOT, env=e, capture_output=True,
                          text=True, timeout=timeout)


_LAUNCH = re.compile(r"tengine_b200: launch gemm_i8_tcgen05_kernel<U8=(\d),MODE=(\d),CS=(\d),BORDER=(\d)> out_mode=(\d+) conv=(\d) "
                     r"n_tiles=(\d+) b_res=(\d) fixq=\d mt=(\d) par_all=(\d)")


def test_gemm_plan_equals_restatement():
    names = ke.gemm_entries()
    r = _child(names, {"TB200_DEBUG_LAUNCH": "1"})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    printed, cur = {}, None
    for line in r.stderr.splitlines():
        if line.startswith(MARK):
            cur = line[len(MARK):].strip()
            continue
        m = _LAUNCH.match(line)
        if m and cur:
            printed.setdefault(cur, []).append(tuple(int(v) for v in m.groups()))
    bad = []
    for name in names:
        case = ke.build(name)
        geo = ke.geometry(case.g, case.g.layers[ke.ENTRIES[name].layer])
        want = (geo["cs"], geo["border"], geo["out_mode"], int(geo["kind"] == "igemm"), geo["n_tiles"], geo["b_res"], geo["mt"],
                geo["par_all"])
        got = [(p[2],) + p[3:] for p in printed.get(name, [])]
        if not got or any(x != want for x in got):
            bad.append(f"{name}: printed (cs, border, out_mode, conv, n_tiles, b_res, mt, par_all) {got}, restated {want}")
    assert not bad, "\n".join(bad)


def test_negative_control_without_the_uint8_correction():
    """TB200_DEBUG_NO_CPLANE drops the cplane * sum(x) term of the uint8 tensor-core kernels: every uint8 GEMM entry must fail."""
    names = ke.uint8_gemm_entries()
    r = _child(names, {"TB200_DEBUG_NO_CPLANE": "1"})
    assert r.returncode == 1, r.stdout[-3000:] + r.stderr[-3000:]
    failed = [ln for ln in r.stdout.splitlines() if ln.startswith("FAIL ")]
    assert len(failed) == len(names), r.stdout


def _main(names):
    from oracle.pyoracle import Oracle
    from tengine_b200 import runtime as rt

    ctx, oracle = rt.Context(0), Oracle()
    fails = 0
    try:
        for name in names:
            sys.stderr.write(MARK + name + "\n")
            sys.stderr.flush()
            msg = run_entry(ctx, oracle, name)
            print(("FAIL " + msg) if msg else ("ok " + name), flush=True)
            fails += msg is not None
    finally:
        ctx.close()
    return 1 if fails else 0


if __name__ == "__main__":
    sys.exit(_main(sys.argv[1:]))
