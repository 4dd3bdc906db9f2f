"""The drop-in boundary, end to end: the REAL Tengine runtime (unmodified reference sources + the B200 nn_device of
tengine_b200/device/, built by integration/build_tengine_b200.py into oracle/_ref/tengine/) executes graphs on device "B200"
through init_tengine()/create_graph()/prerun_graph_multithread()/run_graph(), and the UNMODIFIED example binaries
tm_classification_int8 / tm_benchmark run against it.  Results are compared with the same library's CPU device."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "oracle", "_ref", "tengine")
MODELS = os.path.join(ROOT, "oracle", "_ref", "models")


def _refresh_cuda_library_copy():
    """libtengine-lite.so finds the CUDA library beside itself (rpath $ORIGIN): that copy must be THE library under test, not the
    one of the last integration build (a stale copy once hid a multi-GPU fix from the unmodified-app tests)."""
    import filecmp
    import shutil

    src, dst = os.path.join(ROOT, "tengine_b200", "libtengine_b200.so"), os.path.join(BUILD, "libtengine_b200.so")
    if os.path.isdir(BUILD) and os.path.exists(src) and not (os.path.exists(dst) and filecmp.cmp(src, dst, shallow=False)):
        shutil.copy2(src, dst)


_refresh_cuda_library_copy()


def _have_integration():
    return os.path.exists(os.path.join(BUILD, "libtengine-lite.so")) and os.path.exists(os.path.join(BUILD, "libref_shim.so"))


def test_integration_library_registers_b200_and_fails_loudly_without_gpu(tmp_path):
    """CPU-only check: the device is registered in-tree, the splitter hands it the graph, and without a GPU pre_run fails
    with an error (no silent CPU fallback)."""
    if not _have_integration():
        pytest.skip("integration build absent (needs /root/reference): python integration/build_tengine_b200.py")
    from tengine_b200 import runtime as rt

    if rt.device_count() > 0:
        pytest.skip("an H100 is visible")
    out = tmp_path / "o.npz"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "run_fixture.py"), "ref_tiny_int8", "B200", str(out)],
                       capture_output=True, text=True)
    assert r.returncode != 0
    assert "no CUDA device visible" in (r.stderr + r.stdout)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "run_fixture.py"), "ref_tiny_int8", "CPU", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-500:]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["ref_tiny_int8", "ref_mobilenet025_int8", "ref_tiny_uint8", "ref_mobilenet025_uint8"])
def test_graph_on_b200_device_through_tengine_runtime(tmp_path, name):
    if not _have_integration():
        pytest.skip("integration build absent")
    outs = {}
    for dev in ("CPU", "B200"):
        out = tmp_path / f"{dev}.npz"
        r = subprocess.run([sys.executable, os.path.join(ROOT, "integration", "run_fixture.py"), name, dev, str(out)],
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, (dev, r.stderr[-1500:])
        outs[dev] = dict(np.load(out))
    for k in outs["CPU"]:
        if k == "ms":
            continue
        d = np.abs(outs["CPU"][k].astype(int) - outs["B200"][k].astype(int))
        if "int8" in name and "uint8" not in name:
            assert d.max() == 0, (k, int(d.max()))
        else:
            assert d.max() <= 2, (k, int(d.max()))  # uint8: the CPU path is an fp32 simulation (+-1 LSB per layer)


@pytest.mark.gpu
def test_unmodified_tm_classification_int8_on_b200():
    """examples/tm_classification_int8.c, compiled unmodified, passes no context (create_graph(NULL, ...)): the
    TG_DEFAULT_DEVICE=B200 seam routes its graph to the device.  Same top-5 as the CPU device."""
    exe = os.path.join(BUILD, "tm_classification_int8")
    model = os.path.join(MODELS, "mobilenet_v1_int8.tmfile")
    img = os.path.join(MODELS, "test.bmp")
    if not (os.path.exists(exe) and os.path.exists(model) and os.path.exists(img)):
        pytest.skip("integration build / model files absent")
    res = {}
    for dev in ("CPU", "B200"):
        env = dict(os.environ)
        env.pop("TG_DEFAULT_DEVICE", None)
        if dev == "B200":
            env["TG_DEFAULT_DEVICE"] = "B200"
        r = subprocess.run([exe, "-m", model, "-i", img, "-g", "224,224", "-r", "2", "-t", "8"], capture_output=True, text=True,
                           env=env, timeout=600)
        assert r.returncode == 0, r.stderr[-800:]
        txt = r.stdout + r.stderr
        top = [l.strip() for l in txt.splitlines() if "," in l and l.strip()[0].isdigit() or l.strip().startswith("-")]
        res[dev] = [l for l in txt.splitlines() if l.count(",") == 1 and l.strip().replace(".", "").replace(",", "").replace(" ", "").replace("-", "").isdigit()]
        assert len(res[dev]) == 5, txt[-800:]
    assert res["CPU"] == res["B200"]


@pytest.mark.gpu
def test_unmodified_tm_benchmark_on_b200():
    exe = os.path.join(BUILD, "tm_benchmark")
    model = os.path.join(MODELS, "mobilenet_v1_int8.tmfile")
    if not (os.path.exists(exe) and os.path.exists(model)):
        pytest.skip("integration build / model files absent")
    r = subprocess.run([exe, "-d", "B200", "-m", model, "-i", "8,3,224,224", "-f", "2", "-r", "5", "-t", "8"], capture_output=True,
                       text=True, timeout=600)
    txt = r.stdout + r.stderr
    assert r.returncode == 0 and "min =" in txt, txt[-800:]


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["mobilenet_v1_uint8", "resnet50_uint8"])
def test_unmodified_tm_classification_uint8_on_b200(model):
    """examples/tm_classification_uint8.c, compiled unmodified (create_graph(NULL, ...), TENGINE_MODE_UINT8): the
    TG_DEFAULT_DEVICE=B200 seam routes the uint8 graph -- for ResNet-50 including max-pool, eltwise, ReLU, Flatten-less FC
    and Softmax -- to the device.  The CPU path is an fp32 simulation (+-1 LSB per layer), so scores are compared with a
    tolerance of a few output LSBs instead of as strings."""
    exe = os.path.join(BUILD, "tm_classification_uint8")
    path = os.path.join(MODELS, model + ".tmfile")
    img = os.path.join(MODELS, "test.bmp")
    if not (os.path.exists(exe) and os.path.exists(path) and os.path.exists(img)):
        pytest.skip("integration build / model files absent (python oracle/make_models.py)")
    res = {}
    for dev in ("CPU", "B200"):
        env = dict(os.environ)
        env.pop("TG_DEFAULT_DEVICE", None)
        if dev == "B200":
            env["TG_DEFAULT_DEVICE"] = "B200"
        r = subprocess.run([exe, "-m", path, "-i", img, "-g", "224,224", "-r", "2", "-t", "8"], capture_output=True, text=True, env=env, timeout=600)
        txt = r.stdout + r.stderr
        assert r.returncode == 0, txt[-800:]
        rows = [l.split(",") for l in txt.splitlines() if l.count(",") == 1 and l.strip().replace(".", "").replace(",", "").replace(" ", "").replace("-", "").isdigit()]
        assert len(rows) == 5, txt[-800:]
        res[dev] = [(float(a), int(b)) for a, b in rows]
    top_cpu, top_dev = res["CPU"][0][0], res["B200"][0][0]
    assert abs(top_cpu - top_dev) <= 0.05 * max(abs(top_cpu), 1e-3) + 0.05, (res["CPU"], res["B200"])


def _tmfile_case(name):
    from tengine_b200 import abi, workloads

    if name == "yolov3_tiny_uint8":
        g, b = workloads.yolov3_tiny(abi.DT_UINT8, batch=4)
        return g, b, list(g.outputs)
    g, b = workloads.resnet50(abi.DT_UINT8, batch=4, softmax=True)
    fc = g.layers[-1]["inputs"][0]
    g.mark_output(fc)  # prob, fc1000: a softmax over random-weight logits turns a 1-LSB difference into another arg-max
    return g, b, list(g.outputs)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["yolov3_tiny_uint8", "resnet50_uint8"])
@pytest.mark.parametrize("gpus", [1, 2])
def test_full_size_tmfile_through_run_graph_on_b200(oracle, tmp_path, name, gpus):
    """C3 / C4 as model FILES: written by the reference's own tmfile writer (tools/save_graph, through oracle/ref_shim_save.cpp),
    loaded by the reference's serializer and executed by run_graph() on device "B200" -- one GPU, and a two-GPU group selected
    through the set_context_device option blob (tb200_device_option; on a one-GPU box TG_B200_GPU_LIST=0,0 makes the group two
    shards on the same GPU).  Batch 4.  The bytes must equal the exact-integer oracle's on the same graph.
    (The file is written HERE from the graph the oracle gets: the workloads' activation scales come from a torch fp32
    calibration pass whose last bit depends on the host CPU, so a file made on another machine describes a slightly different
    network -- that, not the device, was the 1-LSB difference this test showed with pre-generated files.)"""
    from tengine_b200 import runtime as rt

    if not _have_integration():
        pytest.skip("integration build absent")
    g, b, outs = _tmfile_case(name)
    x = b.random_input(21)
    path = str(tmp_path / (name + ".tmfile"))
    # A fresh process holds ONE Tengine library, the integration build: it writes the file and runs it.  (In this process another
    # test may already have mapped the plain reference library, whose soname is the same, so the dynamic loader would hand that
    # one -- without the B200 device -- to the integration build's shim.)
    d = g.to_dict()
    d["input"] = x
    npz, out_npz = str(tmp_path / "case.npz"), str(tmp_path / "got.npz")
    np.savez(npz, **d)
    env = {"TG_B200_GPU_LIST": "0,0"} if (gpus == 2 and rt.device_count() < 2) else {}
    code = ("import sys, numpy as np\n"
            "from oracle.pyoracle import Reference, run_tmfile, save_tmfile\n"
            "from tengine_b200.graphdef import GraphDef\n"
            "npz, path, out, libdir, gpus = sys.argv[1:6]\n"
            "d = dict(np.load(npz)); g = GraphDef.from_dict(d)\n"
            "ref = Reference(libdir=libdir)\n"
            "save_tmfile(ref, g, path)\n"
            "got, ms = run_tmfile(ref, path, d['input'], [g.dims(t) for t in g.outputs], device='B200', num_gpus=int(gpus), env=%r, warmup=1, loops=2)\n"
            "np.savez(out, *got)\n" % env)
    r = subprocess.run([sys.executable, "-c", code, npz, path, out_npz, BUILD, str(gpus if gpus > 1 else 0)], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    saved = np.load(out_npz)
    got = [saved[f"arr_{i}"] for i in range(len(outs))]
    want = oracle.run(g, [x], uint8_mode=0)
    for o, t in zip(got, outs):
        assert np.array_equal(o, want[t]), (name, t, int(np.abs(o.astype(int) - want[t].astype(int)).max()))
    assert len(np.unique(got[-1])) > 30


@pytest.mark.gpu
def test_unmodified_tm_benchmark_two_gpu_group():
    """tm_benchmark -d B200 unmodified, the GPU group chosen by the environment (TG_B200_GPUS / TG_B200_GPU_LIST)."""
    from tengine_b200 import runtime as rt

    exe = os.path.join(BUILD, "tm_benchmark")
    model = os.path.join(MODELS, "mobilenet_v1_int8.tmfile")
    if not (os.path.exists(exe) and os.path.exists(model)):
        pytest.skip("integration build / model files absent")
    env = dict(os.environ)
    if rt.device_count() >= 2:
        env["TG_B200_GPUS"] = "2"
    else:
        env["TG_B200_GPU_LIST"] = "0,0"
    r = subprocess.run([exe, "-d", "B200", "-m", model, "-i", "16,3,224,224", "-f", "2", "-r", "5", "-t", "8"], capture_output=True, text=True,
                       timeout=600, env=env)
    txt = r.stdout + r.stderr
    assert r.returncode == 0 and "min =" in txt, txt[-800:]
