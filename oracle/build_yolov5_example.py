#!/usr/bin/env python3
"""Build oracle/_ref/libyolov5_example.so: the detection post-processing of the UNMODIFIED examples/tm_yolov5s.cpp, callable through
oracle/yolov5_example_shim.cpp (TEST INFRASTRUCTURE).  Same recipe as libyolo_example.so in oracle/build_ref.py: -O2 -std=c++11 on
x86-64 (no -mfma, so no FMA contraction), the C++ OpenCV the example names replaced by oracle/cvstub, linked with the reference's
examples/common/tengine_operations.c and oracle/_ref/libtengine-lite.so for the helpers its main() calls.  Runs after
oracle/build_ref.py (it needs oracle/_ref/gen/include and libtengine-lite.so) and only where the reference tree exists; no reference
source is copied, the output goes to the git-ignored oracle/_ref/.

Usage: python oracle/build_yolov5_example.py [--ref /root/reference]"""
import argparse
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libyolov5_example.so")
CC = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"


def build(ref="/root/reference"):
    """Returns the library's path, or None where it cannot be built (no reference tree, or oracle/_ref not built yet)."""
    example = os.path.join(ref, "examples", "tm_yolov5s.cpp")
    shim = os.path.join(HERE, "yolov5_example_shim.cpp")
    if not os.path.exists(example) or not os.path.exists(os.path.join(OUT, "libtengine-lite.so")):
        return LIB if os.path.exists(LIB) else None
    deps = (shim, example, os.path.join(HERE, "cvstub", "opencv2", "core", "core.hpp"), __file__)
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in deps):
        return LIB
    inc = [f"-I{os.path.join(OUT, 'gen', 'include')}", f"-I{ref}/source", f"-I{os.path.join(OUT, 'gen', 'source')}", f"-I{ref}/examples/common",
           f"-I{ref}/examples"]
    ops_o = os.path.join(OUT, "yolov5_example_tengine_operations.o")
    r = subprocess.run([CC, "-O2", "-w", "-std=gnu99", "-fPIC", "-c"] + inc + [f"{ref}/examples/common/tengine_operations.c", "-o", ops_o],
                       capture_output=True, text=True)
    if r.returncode == 0:
        r = subprocess.run([CXX, "-O2", "-w", "-std=c++11", "-fPIC", "-shared", f"-I{os.path.join(HERE, 'cvstub')}"] + inc +
                           [shim, ops_o, "-o", LIB, f"-L{OUT}", "-ltengine-lite", "-Wl,-rpath,$ORIGIN", "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        print(f"[oracle] WARNING: could not build libyolov5_example.so:\n{r.stderr[-1500:]}", file=sys.stderr)
        return None
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    print(build(ap.parse_args().ref))
