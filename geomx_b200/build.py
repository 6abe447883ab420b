"""In-tree build of the native libraries.

  * ``geomx_b200/lib/libgeomx_kernels.so`` — every CUDA kernel, compiled for **sm_90a only** (H100)
    (``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo``), flat C ABI loaded with ctypes.
  * ``geomx_b200/lib/_C*.so`` — the C++ runtime (HiPS transport / servers / engine / serializer / profiler / IO), pybind11.

``python -m geomx_b200.build [--force] [--kernels-only|--runtime-only]``; ``__graft_entry__.build()`` calls ``build_all``.
Objects are cached by source mtime so rebuilds are incremental.  The built ``.so`` files are git-ignored: every checkout builds its own.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
LIB = os.path.join(ROOT, "lib")
OBJ = os.path.join(ROOT, "build_obj")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("CXX", "g++")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr"]
CXX_FLAGS = ["-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-pthread", "-fvisibility=hidden"]
# GEOMX_SANITIZE=address|thread|undefined builds an instrumented runtime (run python with LD_PRELOAD=$(gcc -print-file-name=libasan.so) etc.);
# GEOMX_DEBUG=1 adds -g -O0.  (reference: CMake USE_ASAN, Makefile DEBUG=1)
_SAN = os.environ.get("GEOMX_SANITIZE", "")
if _SAN:
    CXX_FLAGS = [f for f in CXX_FLAGS if f != "-O2"] + ["-O1", "-g", "-fno-omit-frame-pointer", "-fsanitize=" + _SAN]
if os.environ.get("GEOMX_DEBUG", "0") == "1":
    CXX_FLAGS = [f for f in CXX_FLAGS if not f.startswith("-O")] + ["-O0", "-g"]


def _newer(src, dst, extra=()):
    if not os.path.exists(dst):
        return True
    t = os.path.getmtime(dst)
    return any(os.path.getmtime(s) > t for s in (src,) + tuple(extra))


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s" % (" ".join(cmd), r.stdout))
    return r.stdout


def build_kernels(force=False, verbose=False):
    kdir = os.path.join(CSRC, "kernels")
    os.makedirs(LIB, exist_ok=True); os.makedirs(OBJ, exist_ok=True)
    srcs = sorted(f for f in os.listdir(kdir) if f.endswith(".cu"))
    hdrs = tuple(os.path.join(kdir, f) for f in os.listdir(kdir) if f.endswith((".cuh", ".h")))
    objs, jobs = [], []
    for f in srcs:
        src = os.path.join(kdir, f); obj = os.path.join(OBJ, f[:-3] + ".o")
        objs.append(obj)
        if force or _newer(src, obj, hdrs):
            jobs.append([NVCC] + NVCC_FLAGS + ["-c", src, "-o", obj])
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as pool:
        for out in pool.map(_run, jobs):
            if verbose and out.strip():
                print(out)
    out = os.path.join(LIB, "libgeomx_kernels.so")
    if jobs or not os.path.exists(out):
        _run([NVCC, "-shared", "-o", out] + objs + ARCH + ["-lcudart"])
    return out


def build_runtime(force=False, verbose=False):
    import pybind11
    rdirs = [os.path.join(CSRC, "hips"), os.path.join(CSRC, "runtime")]
    os.makedirs(LIB, exist_ok=True); os.makedirs(OBJ, exist_ok=True)
    ext = sysconfig.get_config_var("EXT_SUFFIX")
    out = os.path.join(LIB, "_C" + ext)
    hdrs, srcs = [], []
    for d in rdirs:
        if not os.path.isdir(d):
            continue
        for f in sorted(os.listdir(d)):
            p = os.path.join(d, f)
            (srcs if f.endswith(".cc") else hdrs if f.endswith((".h", ".hpp")) else []).append(p)
    if not srcs:
        return None
    inc = ["-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"], "-I", CSRC]
    objs, jobs = [], []
    for src in srcs:
        obj = os.path.join(OBJ, "rt_" + os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _newer(src, obj, tuple(hdrs)):
            jobs.append([CXX] + CXX_FLAGS + inc + ["-c", src, "-o", obj])
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as pool:
        for o in pool.map(_run, jobs):
            if verbose and o.strip():
                print(o)
    if jobs or not os.path.exists(out):
        # link the SHARED libstdc++ explicitly: some toolchains (e.g. a relocated g++ that only ships libstdc++.a) would otherwise embed a
        # second, static copy next to the one torch already loaded — two iostream/locale runtimes in one process crash on first use
        _run([CXX, "-shared", "-o", out] + objs + ["-pthread", "-l:libstdc++.so.6", "-ldl"] + (["-fsanitize=" + _SAN] if _SAN else []))
    return out


def build_capi(force=False, verbose=False):
    """``lib/libgeomx_capi.so``: the flat C ABI (GXKVStore* / GXNDArray* / GXSymbol* / GXExecutor* / GXAutograd* / GXRecordIO* / GXDataIter* /
    GXPred* / profiler / engine / storage) WITHOUT Python — the same sources as ``_C``, minus the pybind11 module, compiled with
    ``-DGEOMX_NO_PYTHON`` and with neither the pybind11 nor the CPython include directory on the command line.  This is what a C / C++ /
    other-language front end links (header: ``geomx_b200/include/geomx/c_api.h``; the role of the reference's libmxnet.so C API)."""
    rdirs = [os.path.join(CSRC, "hips"), os.path.join(CSRC, "runtime")]
    os.makedirs(LIB, exist_ok=True); os.makedirs(OBJ, exist_ok=True)
    out = os.path.join(LIB, "libgeomx_capi.so")
    hdrs, srcs = [], []
    for d in rdirs:
        for f in sorted(os.listdir(d)):
            p = os.path.join(d, f)
            if f.endswith(".cc") and f != "py_module.cc":
                srcs.append(p)
            elif f.endswith((".h", ".hpp")):
                hdrs.append(p)
    objs, jobs = [], []
    for src in srcs:
        obj = os.path.join(OBJ, "capi_" + os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _newer(src, obj, tuple(hdrs)):
            jobs.append([CXX] + CXX_FLAGS + ["-DGEOMX_NO_PYTHON", "-I", CSRC, "-c", src, "-o", obj])
    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as pool:
        for o in pool.map(_run, jobs):
            if verbose and o.strip():
                print(o)
    if jobs or not os.path.exists(out):
        # no CUDA here: the device predictor (runtime/predict_device.h) dlopens libgeomx_kernels.so when dev_type 2 is asked for
        _run([CXX, "-shared", "-o", out] + objs + ["-pthread", "-l:libstdc++.so.6", "-ldl", "-Wl,--no-undefined"] + (["-fsanitize=" + _SAN] if _SAN else []))
    return out


def build_all(force=False, verbose=False):
    k = build_kernels(force, verbose)
    r = build_runtime(force, verbose)
    build_capi(force, verbose)
    return k, r


if __name__ == "__main__":
    force = "--force" in sys.argv
    if "--runtime-only" not in sys.argv:
        print(build_kernels(force, True))
    if "--kernels-only" not in sys.argv:
        print(build_runtime(force, True))
        print(build_capi(force, True))
