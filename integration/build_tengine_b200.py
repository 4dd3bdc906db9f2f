#!/usr/bin/env python3
"""Integration build (test/demo infrastructure, not part of the product package): the reference Tengine library WITH the B200 device compiled in, exactly as its CMake would do for
`source/device/b200/` + one `_REGISTER_DEVICE_LIST` entry (source/device/CMakeLists.txt:63-188), but driven by gcc directly.

  oracle/_ref/tengine/libtengine-lite.so            reference objects (oracle/_ref/obj, untouched sources) + b200_device.cc
                                              + source/api/c_api.c recompiled against a generated device/register.h that also lists
                                              register_b200_device()
  oracle/_ref/tengine/tm_classification_int8, tm_classification_uint8, tm_benchmark   the UNMODIFIED apps, linked against it

Needs /root/reference (headers + sources are compiled where they lie; nothing is copied into this repo).
c_api.c, c_api.h, the serializer, examples/ and benchmark/ are byte-identical to the reference.
"""
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "tengine_b200", "device")  # the device sources (would be source/device/b200/ in-tree)
sys.path.insert(0, ROOT)
from oracle import build_ref as br  # noqa: E402

OUT = os.path.join(ROOT, "oracle", "_ref", "tengine")


def main(ref="/root/reference"):
    br.build(ref, verbose=False)
    os.makedirs(OUT, exist_ok=True)
    gen = os.path.join(OUT, "gen")
    lists = br.source_lists(ref)
    # the registry CMake would generate with the extra _REGISTER_DEVICE_LIST entry
    br.gen_headers(ref, gen, lists, [os.path.join(ref, "source/device/cpu/cpu_device.c"), os.path.join(HERE, "b200_device.cc")])
    inc = br.include_flags(ref, gen)
    # api/c_api.c is the translation unit that includes the generated device/register.h (c_api.c:33); the SOURCE is
    # untouched, only the generated registry it sees differs -- exactly what a CMake build with the device enabled does
    dev_c = os.path.join(ref, "source/api/c_api.c")
    dev_o = os.path.join(OUT, "c_api.c.o")
    subprocess.check_call([br.CC] + br.CFLAGS + inc + ["-c", dev_c, "-o", dev_o])
    b200_o = os.path.join(OUT, "b200_device.cc.o")
    subprocess.check_call([br.CXX, "-O2", "-fPIC", "-std=c++14", "-w"] + inc + [f"-I{ROOT}/include", "-c",
                           os.path.join(HERE, "b200_device.cc"), "-o", b200_o])
    objs = [br.obj_path(os.path.join(br.OUT, "obj"), ref, s) for s in lists["srcs"] if s != dev_c] + [dev_o, b200_o]
    rsp = os.path.join(OUT, "objs.rsp")
    open(rsp, "w").write("\n".join(objs))
    # libtengine_b200.so sits beside the integration library so that $ORIGIN resolves it on any box
    shutil.copy2(os.path.join(ROOT, "tengine_b200", "libtengine_b200.so"), os.path.join(OUT, "libtengine_b200.so"))
    lib = os.path.join(OUT, "libtengine-lite.so")
    subprocess.check_call([br.CXX, "-shared", "-fopenmp", "-o", lib, "@" + rsp, f"-L{OUT}", "-ltengine_b200",
                           "-Wl,-rpath,$ORIGIN", "-lm", "-ldl", "-lpthread"])
    # unmodified apps + the test shim against the integration library
    save_out = br.OUT
    try:
        br.OUT = OUT
        os.makedirs(os.path.join(OUT, "gen/source"), exist_ok=True)
        br.build_apps(ref, verbose=False)
    finally:
        br.OUT = save_out
    from oracle import build_shim

    build_shim.main(ref, OUT)
    print(f"[integration] {lib} (+ apps, shim) built")


if __name__ == "__main__":
    main()
