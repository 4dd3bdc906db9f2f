#!/usr/bin/env python3
"""Build oracle/_ref/libimage_example.so: the input preprocessing of the UNMODIFIED examples/tm_classification_int8.c and
examples/tm_classification_uint8.c, callable through oracle/image_example_shim.c (TEST INFRASTRUCTURE).  Same recipe as the
examples' own binaries in oracle/build_ref.py: gcc -O2 -std=gnu99 on x86-64 (no -mfma, so no FMA contraction), linked with the
reference's examples/common/tengine_operations.c and oracle/_ref/libtengine-lite.so.  Runs after oracle/build_ref.py (it needs
oracle/_ref/gen/include and libtengine-lite.so) and only where the reference tree exists; no reference source is copied, the output
goes to the git-ignored oracle/_ref/.

Usage: python oracle/build_image_example.py [--ref /root/reference]"""
import argparse
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libimage_example.so")
CC = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"


def build(ref="/root/reference"):
    """Returns the library's path, or None where it cannot be built (no reference tree, or oracle/_ref not built yet)."""
    examples = [os.path.join(ref, "examples", f"tm_classification_{t}.c") for t in ("int8", "uint8")]
    ops = os.path.join(ref, "examples", "common", "tengine_operations.c")
    shim = os.path.join(HERE, "image_example_shim.c")
    if not all(os.path.exists(p) for p in examples + [ops]) or not os.path.exists(os.path.join(OUT, "libtengine-lite.so")):
        return LIB if os.path.exists(LIB) else None
    deps = examples + [ops, shim, __file__]
    if os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in deps):
        return LIB
    inc = [f"-I{os.path.join(OUT, 'gen', 'include')}", f"-I{ref}/source", f"-I{os.path.join(OUT, 'gen', 'source')}", f"-I{ref}/examples/common",
           f"-I{ref}/examples"]
    r = subprocess.run([CC, "-O2", "-w", "-std=gnu99", "-fPIC", "-shared"] + inc + [shim, ops, "-o", LIB, f"-L{OUT}", "-ltengine-lite",
                                                                                  "-Wl,-rpath,$ORIGIN", "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        print(f"[oracle] WARNING: could not build libimage_example.so:\n{r.stderr[-1500:]}", file=sys.stderr)
        return None
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--ref", default="/root/reference")
    print(build(ap.parse_args().ref))
