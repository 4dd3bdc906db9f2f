#!/usr/bin/env python3
"""Run a tests/golden fixture through the REAL Tengine runtime of the integration build (oracle/_ref/tengine/libtengine-lite.so:
unmodified reference + the B200 nn_device) on a named device, via init_tengine()/create_graph()/set_context_device()/
prerun_graph_multithread()/run_graph() (oracle/ref_shim.c).  Writes the requested tensors to an .npz.
usage: run_fixture.py <fixture name> <device: CPU|B200> <out.npz> [all|outputs]"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.pyoracle import Reference  # noqa: E402  (test infrastructure: drives the Tengine C API)
from tests.helpers import layer_outputs, load_golden  # noqa: E402


def main():
    name, device, out = sys.argv[1:4]
    what = sys.argv[4] if len(sys.argv) > 4 else "outputs"
    g, x, _ = load_golden(name)
    rt = Reference(libdir=os.path.join(ROOT, "oracle", "_ref", "tengine"))
    want = layer_outputs(g) if what == "all" else list(g.outputs)
    r, ms = rt.run(g, [x], want=want, device=None if device == "CPU" else device, threads=8, warmup=1, loops=2)
    np.savez(out, ms=np.array(ms), **{f"t{t}": v for t, v in r.items()})


if __name__ == "__main__":
    main()
