"""What ptxas made of the persistent int8 GEMM (tengine_b200/csrc/gemm_tcgen05.cu), read from its -Xptxas -v report: the 14
kernel variants are compiled, none of them has its wgmma serialised by the compiler, and none spills to local memory."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "tengine_b200", "csrc")
LOG = os.path.join(CSRC, "gemm_tcgen05.o.ptxas.log")
KERNEL = "gemm_i8_tcgen05_kernel"
VARIANTS = 14  # <U8, MODE, CS, BORDER> combinations launch_gemm_i8 dispatches to


def _nvcc():
    p = shutil.which("nvcc")
    if p:
        return p
    p = "/usr/local/cuda/bin/nvcc"
    return p if os.path.exists(p) else None


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    """The report `make` writes next to the object file, else a fresh compile of the file with -Xptxas -v."""
    if os.path.exists(LOG) and os.path.getmtime(LOG) >= os.path.getmtime(os.path.join(CSRC, "gemm_tcgen05.cu")):
        return open(LOG).read()
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("codegen") / "gemm_tcgen05.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", "gemm_tcgen05.cu", "-o", str(out)],
                       cwd=CSRC, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return r.stdout + r.stderr


def _entries(log):
    """{mangled kernel name: (spill stores, spill loads)} of every compiled GEMM kernel entry."""
    lines = log.splitlines()
    out = {}
    for i, line in enumerate(lines):
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if not m or KERNEL not in m.group(1):
            continue
        for nxt in lines[i + 1:i + 4]:
            s = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", nxt)
            if s:
                out[m.group(1)] = (int(s.group(1)), int(s.group(2)))
                break
        else:
            out[m.group(1)] = None
    return out


def test_every_variant_is_compiled(ptxas_log):
    e = _entries(ptxas_log)
    assert len(e) == VARIANTS, sorted(e)


def test_no_serialised_wgmma(ptxas_log):
    bad = [line for line in ptxas_log.splitlines()
           if KERNEL in line and ("C7520" in line or ("wgmma" in line and "serializ" in line))]
    assert not bad, "\n".join(bad[:5])


def test_no_spills(ptxas_log):
    e = _entries(ptxas_log)
    assert e, "no GEMM kernel in the ptxas report"
    spilled = {k: v for k, v in e.items() if v != (0, 0)}
    assert not spilled, spilled
