#!/usr/bin/env python3
"""Build oracle/_ref/libtopk_example.so: the ranking step of the UNMODIFIED classification examples (print_topk and its static
sort_cls_score in examples/common/tengine_operations.c), callable through oracle/topk_example_shim.c (TEST INFRASTRUCTURE).  Same
recipe as oracle/build_image_example.py: gcc -O2 -std=gnu99 on x86-64 (no -mfma), the reference's file compiled from where it lies,
linked with oracle/_ref/libtengine-lite.so.  Runs after oracle/build_ref.py (it needs oracle/_ref/gen/include and libtengine-lite.so)
and only where the reference tree exists; no reference source is copied, the output goes to the git-ignored oracle/_ref/.

Usage: python oracle/build_topk_example.py [--ref /root/reference]"""
import argparse
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libtopk_example.so")
CC = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def build(ref="/root/reference"):
    """Returns the library's path, or None where it cannot be built (no reference tree, or oracle/_ref not built yet)."""
    ops = os.path.join(ref, "examples", "common", "tengine_operations.c")
    shim = os.path.join(HERE, "topk_example_shim.c")
    if not os.path.exists(ops) or not os.path.exists(os.path.join(OUT, "libtengine-lite.so")):
        return LIB if os.path.exists(LIB) else None
    deps = [ops, shim, __file__]
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in deps):
        return LIB
    inc = [f"-I{os.path.join(OUT, 'gen', 'include')}", f"-I{ref}/source", f"-I{os.path.join(OUT, 'gen', 'source')}", f"-I{ref}/examples/common"]
    r = subprocess.run([CC, "-O2", "-w", "-std=gnu99", "-fPIC", "-shared"] + inc + [shim, "-o", LIB, f"-L{OUT}", "-ltengine-lite",
                                                                                  "-Wl,-rpath,$ORIGIN", "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        print(f"[oracle] WARNING: could not build libtopk_example.so:\n{r.stderr[-1500:]}", file=sys.stderr)
        return None
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    print(build(ap.parse_args().ref))
