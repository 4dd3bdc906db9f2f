"""Host-side logic that needs no GPU: workload builders, bench.py helpers, the reference-arm worker plumbing."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tengine_b200 import abi, workloads

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_inplace_scales_mirror_the_quantisation_tool():
    """tools/quantize/quant_save_graph.cpp:136-200 (default `inplace = true`): max pooling and ReLU outputs carry the
    quantisation of their input; leaky ReLU and average pooling are calibrated on their own."""
    g, _ = workloads.yolov3_tiny(abi.DT_UINT8, batch=1, res=64, width=0.25, head=27, seed=3)
    seen_pool = seen_leaky = 0
    for L in g.layers:
        tin, tout = g.tensors[L["inputs"][0]], g.tensors[L["output"]]
        if L["op"] == abi.OP_POOL and L["pool_method"] == abi.POOL_MAX:
            assert (tin["scale"], tin["zero_point"]) == (tout["scale"], tout["zero_point"])
            seen_pool += 1
        if L["op"] == abi.OP_RELU and L.get("negative_slope", 0.0) != 0.0:
            seen_leaky += 1
    assert seen_pool >= 5 and seen_leaky >= 5
    g2, _ = workloads.resnet50(abi.DT_INT8, batch=1, res=64, width=0.25, classes=10, seed=3)
    relus = [L for L in g2.layers if L["op"] == abi.OP_RELU]
    assert relus and all(g2.tensors[L["inputs"][0]]["scale"] == g2.tensors[L["output"]]["scale"] for L in relus)
    # the every-op test net keeps independent scales so that the general pooling / ReLU kernels stay covered
    g3, _ = workloads.tiny_net(abi.DT_INT8, batch=1)
    assert any(L["op"] == abi.OP_POOL and g3.tensors[L["inputs"][0]]["scale"] != g3.tensors[L["output"]]["scale"] for L in g3.layers)


def test_reference_worker_is_torch_free_and_reports_json(tmp_path):
    """bench.py's reference arm runs `python -m oracle.ref_worker` once per CPU: it must not import torch (start-up time x
    128 processes) and must print one JSON line."""
    from oracle.pyoracle import Reference

    if not Reference.available():
        pytest.skip("oracle/_ref not built")
    g, b = workloads.tiny_net(abi.DT_INT8, batch=1)
    d = g.to_dict()
    d["input"] = b.random_input(1)
    npz = tmp_path / "g.npz"
    np.savez(npz, **d)
    env = dict(os.environ, OMP_NUM_THREADS="1", REF_SHIM_CPUS=str(sorted(os.sched_getaffinity(0))[0]), PYTHONPATH=ROOT)
    code = ("import sys, runpy; sys.argv = ['ref_worker', %r, '2', '1']; runpy.run_module('oracle.ref_worker', run_name='__main__'); "
            "assert 'torch' not in sys.modules" % str(npz))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr[-800:]
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["images"] == 2 and out["loop_s"] > 0 and out["min_ms"] > 0


def test_ncu_traffic_tool_reproduces_the_stored_traffic_file(tmp_path):
    """tools/ncu_traffic_json.py on a stored per-launch summary of one whole MobileNet-v1 int8 step (batch 256) gives the stored
    per-family DRAM bytes and launch counts (tests/golden/ncu_*: an Nsight Compute capture of an earlier build, used as input data)."""
    import subprocess

    out = tmp_path / "t.json"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "ncu_traffic_json.py"),
                        os.path.join(ROOT, "tests", "golden", "ncu_summary_mobilenet_v1_int8_b256.csv"), str(out), "mobilenet_v1_int8", "256"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    got = json.load(open(out))
    want = json.load(open(os.path.join(ROOT, "tests", "golden", "ncu_traffic_mobilenet_v1_int8_b256.json")))
    for fam, f in want["families"].items():
        assert fam in got["families"], fam
        assert got["families"][fam]["launches_per_step"] == f["launches_per_step"]
        assert got["families"][fam]["dram_bytes_per_step"] == pytest.approx(f["dram_bytes_per_step"], rel=1e-6)


def test_dump_outputs_stays_within_the_limit_and_is_reproducible(tmp_path, monkeypatch):
    """bench.py --dump-outputs: the files of all outputs together never exceed DUMP_LIMIT bytes, small outputs are stored whole and
    in shape, an output over its share holds exactly the elements at dump_sample_positions (YOLOv5s-like head sizes, scaled down)."""
    sys.path.insert(0, ROOT)
    import bench

    monkeypatch.setattr(bench, "DUMP_LIMIT", 1 << 20)
    rng = np.random.default_rng(0)
    ys = [rng.integers(-127, 128, s, dtype=np.int8) for s in ((2, 255, 40, 40), (2, 255, 20, 20), (2, 255, 10, 10))]

    class FakeGraph:
        def download(self, i, out):
            out[...] = ys[i]

        def sync(self):
            pass

    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), FakeGraph(), [np.empty_like(y) for y in ys])
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == ["output0.npy", "output1.npy", "output2.npy"]
    assert sum(os.path.getsize(tmp_path / "a" / f) for f in files) <= bench.DUMP_LIMIT
    for i, (f, y) in enumerate(zip(files, ys)):
        a, b = np.load(tmp_path / "a" / f), np.load(tmp_path / "b" / f)
        assert a.dtype == np.float32 and np.array_equal(a, b)
        if a.shape == y.shape:
            assert np.array_equal(a, y.astype(np.float32))
        else:
            assert a.ndim == 1 and np.array_equal(a, y.reshape(-1)[bench.dump_sample_positions(y.size, a.size, i)].astype(np.float32))
    assert np.load(tmp_path / "a" / "output0.npy").ndim == 1  # the large head was sampled
