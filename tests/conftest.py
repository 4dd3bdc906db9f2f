import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")
    # On a multi-GPU box some tests reach the library's NCCL path through the Tengine runtime (not through tengine_b200/runtime.py,
    # which maps torch's bundled NCCL first): do the same here, once, so that a later `import torch` in this process still finds
    # the NCCL build it was linked against (a process can hold only one libnccl.so.2).
    try:
        from tengine_b200 import runtime as rt

        if os.path.exists(rt.LIB_PATH) and rt.device_count() > 1:
            rt._preload_bundled_nccl()
    except Exception:
        pass


@pytest.fixture(scope="session")
def oracle():
    from oracle.pyoracle import Oracle

    return Oracle()


@pytest.fixture(scope="session")
def reference():
    from oracle.pyoracle import Reference

    if not Reference.available():
        pytest.skip("oracle/_ref not built (needs /root/reference: make -C oracle)")
    return Reference()


@pytest.fixture(scope="session")
def ctx():
    from tengine_b200 import runtime as rt

    c = rt.Context(0)
    yield c
    c.close()
