"""The edge cases of tests/kernel_edges.py on the device: every layer bit-exact against the exact reference (or the oracle, for
ops outside ties.exact_layer), with the kernel each entry is meant to reach asserted by name.

Child processes (`python -m tests.test_gpu_kernel_edges <entry>...`) cover what the library reads once per process:
  - TB200_DEBUG_LAUNCH: the printed plans of the GEMM, the window and the gather kernel equal kernel_edges.gemm_geometry,
    window_geometry and gather_geometry for every entry of theirs, so the Python restatement cannot drift from the code unnoticed;
  - TB200_DEBUG_NO_CPLANE (documented to give wrong uint8 results): the uint8 GEMM entries with a cplane term must FAIL there --
    a sweep that passed under a known-wrong kernel would prove nothing -- and those without one (zw 0 or 128) must pass."""
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
    flags = abi.PRERUN_POISON_ARENA | (0 if e.fused else abi.PRERUN_NO_GRAPH) | e.flags
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
                     r"n_tiles=(\d+) b_res=(\d) fixq=\d mt=(\d) par_all=(\d) block_n=(\d+) b_signed=(\d) cplane=(-?\d+)")


def test_gemm_plan_equals_restatement():
    names = ke.gemm_entries()
    r = _child(names, {"TB200_DEBUG_LAUNCH": "1"})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    printed, cur, uu = {}, None, set()
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
                geo["par_all"], geo["block_n"], geo["b_signed"], geo["cplane"])
        got = [(p[2],) + p[3:] for p in printed.get(name, [])]
        if not got or any(x != want for x in got):
            bad.append(f"{name}: printed (cs, border, out_mode, conv, n_tiles, b_res, mt, par_all, block_n, b_signed, cplane) {got}, "
                       f"restated {want}")
        elif geo.get("mma_uu"):
            uu.add((got[0][8], got[0][6]))
    assert not bad, "\n".join(bad)
    # the u8.u8 MMA (B unsigned: zw 0) ran in every (block_n, mt) instantiation of gemm_mma_dispatch
    assert uu == set(ke.MMA_PAIRS), sorted(set(ke.MMA_PAIRS) - uu)


_WINDOW = re.compile(r"tengine_b200: launch conv_window_tc_kernel<MODE=\d,U8=\d,LAYOUT=(\d)> layout=(\d) xoff=(\d+) box_w=(\d+) box_h=(\d+) "
                     r"ks=(\d+) smem=(\d+) tiles_w=(\d+) tiles_h=(\d+) grid=(\d+)")
_GATHER = re.compile(r"tengine_b200: launch conv_gather_tc_kernel<MODE=\d,U8=\d,KHW=(\d)> ks=(\d+) ntiles=(\d+)")


def test_window_and_gather_plans_equal_restatement():
    """Every window / gather entry launches its kernel once, with the plan window_geometry / gather_geometry restate; the window
    kernel's grid is at most one CTA per tile."""
    names = ke.window_entries()
    r = _child(names, {"TB200_DEBUG_LAUNCH": "1"})
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    printed, cur = {}, None
    for line in r.stderr.splitlines():
        if line.startswith(MARK):
            cur = line[len(MARK):].strip()
            continue
        for kind, rx in (("window", _WINDOW), ("gather", _GATHER)):
            m = rx.match(line)
            if m and cur:
                printed.setdefault(cur, []).append((kind,) + tuple(int(v) for v in m.groups()))
    bad = []
    for name in names:
        case = ke.build(name)
        L = case.g.layers[ke.ENTRIES[name].layer]
        geo = ke.geometry(case.g, L)
        if geo["kind"] == "window":
            want = ("window", geo["layout"], geo["layout"], geo["xoff"], geo["box_w"], geo["box_h"], geo["ks"], geo["smem_bytes"],
                    geo["tiles_w"], geo["tiles_h"])
            got = [p[:-1] for p in printed.get(name, [])]
            if any(p[0] == "window" and not 1 <= p[-1] <= geo["ntiles"] for p in printed.get(name, [])):
                bad.append(f"{name}: grid {[p[-1] for p in printed[name]]} for {geo['ntiles']} tiles")
        else:
            khw = 3 if L["kernel_h"] == 3 else 7
            want = ("gather", khw, geo["ks"], geo["ntiles"])
            got = printed.get(name, [])
        if len(got) != 1 or got[0] != want:
            bad.append(f"{name}: printed {got}, restated {want}")
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("name", ke.window_batch_entries())
def test_window_entry_on_part_of_the_batch(ctx, name):
    """fill_conv_step builds each slice's window tensor map from the slice's own n: a graph prepared for n images runs on the
    first n - 1 (tb200_graph_set_batch) and then on all n again, bit-exact to the reference each time."""
    from tengine_b200 import runtime as rt

    e = ke.ENTRIES[name]
    case = ke.build(name)
    g, x = case.g, case.inputs[0]
    want, _ = ties.exact_run(g, case.inputs)
    n = x.shape[0]
    gr = rt.Graph(ctx, g, abi.PRERUN_POISON_ARENA | abi.PRERUN_NO_GRAPH | e.flags)
    try:
        for b in (n - 1, n):
            gr.set_batch(b)
            outs = gr.run([x[:b]])
            assert gr.layer_kernels()[e.layer] == e.kernel
            for o, t in zip(outs, g.outputs):
                assert o.shape[0] == b and np.array_equal(o, want[t][:b]), (name, b, int((o != want[t][:b]).sum()))
    finally:
        gr.close()


def test_negative_control_without_the_uint8_correction():
    """TB200_DEBUG_NO_CPLANE drops the cplane * sum(x) term of the uint8 tensor-core kernels: every uint8 GEMM entry with a
    cplane term (zw not 0 or 128) must fail, and every one without it must still pass (entries whose output is one saturated
    byte cannot show it and are left out)."""
    want = ke.negative_control_entries()
    names = list(want)
    r = _child(names, {"TB200_DEBUG_NO_CPLANE": "1"})
    assert r.returncode == 1, r.stdout[-3000:] + r.stderr[-3000:]
    status = {}
    for ln in r.stdout.splitlines():
        if ln.startswith("ok "):
            status[ln[3:].strip()] = False
        elif ln.startswith("FAIL "):
            status[ln[5:].split(":", 1)[0]] = True
    assert status == want, {n: (status.get(n), want[n]) for n in names if status.get(n) != want[n]}


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
