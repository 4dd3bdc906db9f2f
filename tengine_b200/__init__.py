"""tengine_b200 -- H100 (sm_90a) int8/uint8 convolution + GEMM device backend for Tengine.

The product is the C-ABI library `libtengine_b200.so` (include/tengine_b200.h) built from tengine_b200/csrc/
and the C++ Tengine device glue under tengine_b200/device/.  This package only loads that library for the
Python tests and bench.py.  There is no Python/CPU compute fallback: if the library is missing, importing
`tengine_b200.runtime` raises.
"""
from . import abi  # noqa: F401
from .graphdef import GraphDef  # noqa: F401

__all__ = ["abi", "GraphDef"]
