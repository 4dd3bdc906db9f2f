"""The generated graphs of tests/graph_gen.py on the CPU: which planner edges they reach, an arena that never lets two live values
share a byte, and the oracle running every graph (against the unmodified reference where oracle/_ref is built)."""
import copy
import functools

import numpy as np
import pytest

from tengine_b200 import abi
from tests import graph_gen as gg

SEEDS = range(150)
DTYPES = pytest.mark.parametrize("dtype", [abi.DT_INT8, abi.DT_UINT8], ids=["int8", "uint8"])


@functools.lru_cache(maxsize=None)
def case(seed, dtype, batch=None):
    return gg.generate(seed, dtype, batch)


@DTYPES
def test_generated_graphs_reach_every_planner_edge(dtype):
    reached = set()
    for s in SEEDS:
        reached |= gg.plan(case(s, dtype)[0]).keys
    unreachable = set(gg.UNREACHABLE[dtype])
    assert not reached & unreachable, sorted(reached & unreachable)
    missing = set(gg.COVERAGE) - unreachable - reached
    assert not missing, sorted(missing)
    assert reached <= set(gg.COVERAGE) | {"fuse_elt_relu:dims"}, sorted(reached - set(gg.COVERAGE))


@DTYPES
def test_generated_graphs_stay_in_bounds(dtype):
    for s in SEEDS:
        g, xs, _ = case(s, dtype)
        assert 4 <= len(g.layers) <= 14 and 1 <= len(g.inputs) <= 3 and 1 <= len(g.outputs) <= 4, s
        assert g.dims(g.inputs[0])[1] == 3 and all(1 <= g.dims(t)[0] <= 5 for t in g.inputs), s
        assert [x.shape for x in xs] == [g.dims(t) for t in g.inputs]


def check_arena(g, p):
    """Two values whose live ranges (graph_gen.live_ranges) overlap never share a byte; every slot starts on 1 KiB; the arena is
    no larger than the sum of its slots."""
    bad = []
    vals = gg.live_ranges(g, p)
    for name, lo, hi, off, nb in vals:
        if off % 1024:
            bad.append(f"{name} at {off}: not 1 KiB aligned")
        if off + nb > p.act_bytes:
            bad.append(f"{name} [{off}, {off + nb}) past the arena's {p.act_bytes} bytes")
    for i, (na, la, ha, oa, ba) in enumerate(vals):
        for nb_, lb, hb, ob, bb in vals[i + 1:]:
            if la <= hb and lb <= ha and oa < ob + bb and ob < oa + ba:
                bad.append(f"{na} (layers {la}..{ha}, bytes {oa}..{oa + ba}) overlaps {nb_} (layers {lb}..{hb}, bytes {ob}..{ob + bb})")
    if p.act_bytes > p.unshared_bytes:
        bad.append(f"arena {p.act_bytes} bytes > {p.unshared_bytes} unshared")
    return bad


@DTYPES
@pytest.mark.parametrize("flags", [abi.PRERUN_DEFAULT, abi.PRERUN_NO_GRAPH], ids=["default", "no_graph"])
def test_arena_plan_never_overlaps_live_values(dtype, flags):
    bad = []
    for s in SEEDS:
        g = case(s, dtype)[0]
        bad += [f"seed {s}: {m}" for m in check_arena(g, gg.plan(g, flags))]
    assert not bad, "\n".join(bad[:20])


def test_arena_check_catches_an_output_placed_over_its_input():
    """The overlap check is not vacuous: a plan whose layer writes over an input it still reads fails it."""
    g = case(2, abi.DT_INT8)[0]
    p = gg.plan(g)
    li = next(i for i, L in enumerate(p.layers) if L["op"] not in (gg.NOP, abi.OP_RESHAPE) and p.tensors[L["output"]].has_slot
              and any(p.tensors[t].has_slot for t in L["inputs"]))
    L = p.layers[li]
    p.tensors[L["output"]].off = p.tensors[L["inputs"][0]].off
    assert check_arena(g, p)


@DTYPES
def test_oracle_runs_every_generated_graph_unsaturated(oracle, dtype):
    worst = []
    for s in SEEDS:
        g, xs, _ = case(s, dtype)
        out = oracle.run(g, xs, uint8_mode=0)
        f = gg.saturated_fraction(g, out)
        if f >= 0.3:
            worst.append((s, round(f, 3)))
    assert not worst, worst


# Generated graphs the unmodified reference refuses to run: (dtype, seed) -> (layer, op).  Each time an Eltwise reads a Reshape's
# output, which the reference holds as a 2-D tensor and its eltwise kernel turns down ("unsupported dim num: 2").
REFERENCE_REFUSES = {(abi.DT_INT8, 86): (4, "eltwise"), (abi.DT_INT8, 104): (3, "eltwise"), (abi.DT_INT8, 117): (4, "eltwise"),
                     (abi.DT_UINT8, 27): (5, "eltwise")}


def _prefix(g, n):
    """The graph of g's first n layers, every layer's tensor an output."""
    h = copy.copy(g)
    h.layers = g.layers[:n]
    h.outputs = [L["output"] for L in h.layers]
    return h


def _refused_layer(reference, g, xs):
    """The first layer the reference refuses: its first n layers run and its first n + 1 do not (None: it runs them all)."""
    for n in range(1, len(g.layers) + 1):
        try:
            reference.run(_prefix(g, n), xs)
        except RuntimeError:
            return n - 1
    return None


def test_oracle_equals_reference_on_generated_graphs(oracle, reference):
    """Every seed of both types at batch 1 (the reference's batched int8 3x3 path is known to be wrong), every layer's tensor:
    int8 bit-exact; uint8 within 1 LSB of the reference in both oracle modes (0: the exact integer arithmetic the device
    computes, 1: the fp32 simulation).  A seed the reference refuses must still be refused, at its listed layer: an Eltwise
    reading a Reshape."""
    bad = []
    for dtype in (abi.DT_INT8, abi.DT_UINT8):
        u8 = dtype == abi.DT_UINT8
        for s in SEEDS:
            g, xs, _ = case(s, dtype, 1)
            want = [L["output"] for L in g.layers]
            listed = REFERENCE_REFUSES.get((dtype, s))
            try:
                ref, _ = reference.run(g, xs, want=want)
            except RuntimeError:
                li = _refused_layer(reference, g, xs)
                L = g.layers[li] if li is not None else None
                from_reshape = L is not None and any(P["op"] == abi.OP_RESHAPE and P["output"] in L["inputs"] for P in g.layers)
                if listed is None or li != listed[0] or abi.OP_NAMES[L["op"]] != listed[1] or not from_reshape:
                    bad.append(f"dtype {dtype} seed {s}: the reference refuses layer {li} ({abi.OP_NAMES[L['op']] if L else '?'}), "
                               f"listed {listed}")
                continue
            if listed is not None:
                bad.append(f"dtype {dtype} seed {s}: listed as refused at {listed}, but the reference runs it")
                continue
            for mode in (0, 1) if u8 else (0,):
                got = oracle.run(g, xs, uint8_mode=mode)
                for li, t in enumerate(want):
                    d = int(np.abs(got[t].astype(np.int32) - ref[t].astype(np.int32)).max())
                    if d > int(u8):
                        bad.append(f"dtype {dtype} seed {s} mode {mode} layer {li} {abi.OP_NAMES[g.layers[li]['op']]}: {d} LSB in "
                                   f"{int((got[t] != ref[t]).sum())} bytes")
                        break
    assert not bad, "\n".join(bad)
