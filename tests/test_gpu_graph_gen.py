"""The generated graphs of tests/graph_gen.py on the device, against the CPU oracle (uint8 against the exact-integer oracle, mode 0).

Per graph: every layer's tensor with nothing fused or shared (NO_GRAPH), then the default plan -- fused nodes, reused arena
slots, a captured CUDA graph -- twice, with the layers it folds equal to graph_gen.plan's, and on part of the batch
(tb200_graph_set_batch) and back.  The arena is poisoned first (POISON_ARENA), so a value read before it is written, or
after another overwrote it, shows.  Some graphs run on the CUDA cores only, some at batch 32 and 64, where tb200_graph_run
pipelines the batch in two chunks.

A child process (`python -m tests.test_gpu_graph_gen <dtype>:<seed>...`) prepares graphs under TB200_DEBUG_LAUNCH, which the
library reads once per process: the arena offsets, slot sizes and fused pairs it prints equal graph_gen.plan's."""
import functools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from tengine_b200 import abi
from tests import graph_gen as gg

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DT = {"int8": abi.DT_INT8, "uint8": abi.DT_UINT8}
SEEDS = [(d, s) for d in DT for s in range(150)]
NO_TC_SEEDS = [(d, s) for d, s in SEEDS if s % 5 == 0]
BIG_SEEDS = [(d, s) for d in DT for s in (1, 2, 3)]
DEBUG_SEEDS = [(d, s) for d in DT for s in range(8)]
POISON = abi.PRERUN_POISON_ARENA


@functools.lru_cache(maxsize=None)
def case(dtype, seed, batch=None):
    return gg.generate(seed, DT[dtype], batch)


def _name(c):
    return f"{c[0]}:{c[1]}"


def _every_layer(ctx, g, xs, want, flags, what):
    from tengine_b200 import runtime as rt

    gr = rt.Graph(ctx, g, flags | abi.PRERUN_NO_GRAPH | POISON)
    try:
        outs = gr.run(xs)
        kernels = gr.layer_kernels()
        for li, L in enumerate(g.layers):
            got = gr.read_tensor(L["output"])
            assert np.array_equal(got, want[L["output"]]), \
                f"{what}: layer {li} {abi.OP_NAMES[L['op']]} ({kernels[li]}) differs in {int((got != want[L['output']]).sum())} bytes"
        for o, t in zip(outs, g.outputs):
            assert np.array_equal(o, want[t]), f"{what}: graph output {t}"
    finally:
        gr.close()


@pytest.mark.parametrize("dtype,seed", SEEDS, ids=list(map(_name, SEEDS)))
def test_graph_gen_on_device(ctx, oracle, dtype, seed):
    from tengine_b200 import runtime as rt

    g, xs, _ = case(dtype, seed)
    what = f"{dtype} seed {seed}"
    want = oracle.run(g, xs, uint8_mode=0)
    _every_layer(ctx, g, xs, want, abi.PRERUN_DEFAULT, what)
    gr = rt.Graph(ctx, g, POISON)
    try:
        kernels = gr.layer_kernels()
        for run in range(2):
            for o, t in zip(gr.run(xs), g.outputs):
                assert np.array_equal(o, want[t]), f"{what}: graph output {t} of the default plan ({kernels}), run {run}"
        folded = {li for li, k in enumerate(kernels) if k == "fused_into_producer"}
        assert folded == gg.plan(g).folded(), f"{what}: the library folds layers {sorted(folded)} ({kernels})"
        n = xs[0].shape[0]
        if n >= 3:
            for b in (n - 1, n):
                gr.set_batch(b)
                for o, t in zip(gr.run([x[:b] for x in xs]), g.outputs):
                    assert np.array_equal(o, want[t][:b]), f"{what}: graph output {t} on {b} of {n} images"
    finally:
        gr.close()


@pytest.mark.parametrize("dtype,seed", NO_TC_SEEDS, ids=list(map(_name, NO_TC_SEEDS)))
def test_graph_gen_on_cuda_cores(ctx, oracle, dtype, seed):
    g, xs, _ = case(dtype, seed)
    _every_layer(ctx, g, xs, oracle.run(g, xs, uint8_mode=0), abi.PRERUN_NO_TENSORCORE, f"{dtype} seed {seed}, CUDA cores")


@pytest.mark.parametrize("batch", [32, 64])
@pytest.mark.parametrize("dtype,seed", BIG_SEEDS, ids=list(map(_name, BIG_SEEDS)))
def test_graph_gen_pipelined_batch(ctx, oracle, dtype, seed, batch):
    """plan_chunks cuts a batch of 32 in halves and one of 64 in a quarter and three quarters: tb200_graph_run over the chunks,
    and upload / launch / download over the whole batch, equal the oracle."""
    from tengine_b200 import runtime as rt

    g, xs, _ = case(dtype, seed, batch)
    want = oracle.run(g, xs, uint8_mode=0)
    gr = rt.Graph(ctx, g, POISON)
    try:
        for o, t in zip(gr.run(xs), g.outputs):
            assert np.array_equal(o, want[t]), f"{dtype} seed {seed} batch {batch}: graph output {t} of run"
        for i, x in enumerate(xs):
            gr.upload(i, x)
        gr.launch()
        ys = [np.empty(g.dims(t), g.np_dtype) for t in g.outputs]
        for i, y in enumerate(ys):
            gr.download(i, y)
        gr.sync()
        for y, t in zip(ys, g.outputs):
            assert np.array_equal(y, want[t]), f"{dtype} seed {seed} batch {batch}: graph output {t} of launch"
    finally:
        gr.close()


MARK = "graph_gen case "
_TENSOR = re.compile(r"tengine_b200: plan tensor (\d+) off=(\d+) slot=(\d+) producer=(-?\d+) last_use=(-?\d+)$")
_SCRATCH = re.compile(r"tengine_b200: plan scratch layer=(\d+) off=(\d+) slot=(\d+)$")
_FUSE = re.compile(r"tengine_b200: plan fuse (\w+) layer=(\d+) folded=(\d+)$")


def test_graph_gen_plan_equals_restatement():
    names = list(map(_name, DEBUG_SEEDS))
    r = subprocess.run([sys.executable, "-m", "tests.test_gpu_graph_gen"] + names, cwd=ROOT, capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, TB200_DEBUG_LAUNCH="1"))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    printed, cur = {}, None
    for line in r.stderr.splitlines():
        if line.startswith(MARK):
            cur = printed.setdefault(line[len(MARK):].strip(), dict(tensors={}, scratch={}, pairs=[]))
        elif cur is not None and (m := _TENSOR.match(line)):
            cur["tensors"][int(m[1])] = tuple(int(v) for v in m.groups()[1:])
        elif cur is not None and (m := _SCRATCH.match(line)):
            cur["scratch"][int(m[1])] = (int(m[2]), int(m[3]))
        elif cur is not None and (m := _FUSE.match(line)):
            cur["pairs"].append((m[1], int(m[2]), int(m[3])))
    bad = []
    for (dtype, seed), name in zip(DEBUG_SEEDS, names):
        g = case(dtype, seed)[0]
        p = gg.plan(g)
        got = printed.get(name)
        if got is None or len(got["tensors"]) != len(g.tensors):
            bad.append(f"{name}: printed {got}")
            continue
        for i, t in enumerate(p.tensors):
            want = (t.off if t.has_slot else 0, t.slot, t.producer, t.last_use)
            if got["tensors"][i] != want:
                bad.append(f"{name}: tensor {i} printed (off, slot, producer, last_use) {got['tensors'][i]}, restated {want}")
        if got["scratch"] != p.scratch:
            bad.append(f"{name}: reshape scratch printed {got['scratch']}, restated {p.scratch}")
        if got["pairs"] != p.pairs:
            bad.append(f"{name}: fused pairs printed {got['pairs']}, restated {p.pairs}")
    assert not bad, "\n".join(bad)


def _main(names):
    from tengine_b200 import runtime as rt

    ctx = rt.Context(0)
    try:
        for name in names:
            dtype, seed = name.split(":")
            sys.stderr.write(MARK + name + "\n")
            sys.stderr.flush()
            rt.Graph(ctx, case(dtype, int(seed))[0]).close()
    finally:
        ctx.close()
    return 0


if __name__ == "__main__":
    sys.exit(_main(sys.argv[1:]))
