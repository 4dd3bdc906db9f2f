"""The C-ABI library: loads, exports exactly what include/tengine_b200.h declares, and refuses to compute without a GPU."""
import ctypes
import os
import re

import pytest

from tengine_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_and_python_mirror_agree():
    hdr = open(os.path.join(ROOT, "include", "tengine_b200.h")).read()
    declared = sorted(set(re.findall(r"TB200_API\s+[\w\s\*]+?\b(tb200k?_\w+)\s*\(", hdr)))
    assert declared == sorted(abi.EXPORTS)


def test_library_exports_every_symbol():
    from tengine_b200 import runtime as rt

    L = rt.lib()
    for name in abi.EXPORTS:
        assert hasattr(L, name), name
    assert L.tb200_abi_version() == abi.ABI_VERSION


def test_struct_sizes_match_header():
    # compile a tiny C program against the header and compare sizeof()
    import subprocess
    import tempfile

    src = '#include <stdio.h>\n#include "tengine_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", sizeof(tb200_tensor_desc), sizeof(tb200_layer_desc), sizeof(tb200k_epilogue), sizeof(tb200k_conv_shape));return 0;}'
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        out = subprocess.check_output([os.path.join(d, "t")]).split()
    assert [int(x) for x in out] == [ctypes.sizeof(abi.TensorDesc), ctypes.sizeof(abi.LayerDesc),
                                     ctypes.sizeof(abi.KEpilogue), ctypes.sizeof(abi.KConvShape)]


def test_no_cpu_fallback_without_gpu():
    from tengine_b200 import runtime as rt

    if rt.device_count() > 0:
        pytest.skip("an H100 is visible")
    with pytest.raises(rt.TB200Error) as e:
        rt.Context(0)
    assert e.value.code == abi.ERR_NO_DEVICE


def test_product_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "tengine_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc", ".cpp", ".hpp")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                assert "pyoracle" not in txt and "tb200_oracle" not in txt and "ref_shim" not in txt, os.path.join(dirpath, f)
