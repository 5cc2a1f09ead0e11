"""Builds the native pieces in-tree (no JIT cache: the .so files travel with the repo).

  lib/libhbcu.so          CUDA kernels + C-ABI (include/hbcu.h), nvcc, sm_90a only
  lib/libhbcu_filters.so  the product's host side: the hb_filter_*_cuda objects in C (gcc) and their libhb-facing
                          helpers, linked against libhbcu.so; everything libhb itself provides (hb_buffer_*, hb_dict_*,
                          hb_log ...) is an undefined symbol of this library
  lib/libhbshim.so        TEST SCAFFOLDING: the stand-in for libhb those symbols resolve to outside a HandBrake build
                          (hb_runtime.c) plus the test harness and the bench driver; never part of an integration

`python -m handbrake_b200.build` or `build_all()`.
"""
import os
import shutil
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
REPO = ROOT.parent
LIB = ROOT / "lib"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-fmad=false",                  # the reference is built without FMA contraction (SURVEY.md 8a)
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]
CU_SOURCES = ["hbcu_core.cu", "hbcu_frames.cu", "nlmeans.cu", "comb_detect.cu", "decomb.cu", "eedi2.cu", "lapsharp.cu", "unsharp.cu", "hqdn3d.cu", "detelecine.cu", "blend.cu", "motion_metric.cu", "format.cu", "rotate.cu", "deinterlace.cu"]
SHIM_SOURCES = ["hb_runtime.c", "hb_harness.c", "hb_bench.c"]
C_SOURCES = ["hbcu_registry.c", "hbcu_pinned.c", "hbcu_device_frames.c", "nlmeans_cuda.c", "comb_detect_cuda.c", "decomb_cuda.c", "lapsharp_cuda.c", "unsharp_cuda.c", "denoise_cuda.c", "detelecine_cuda.c", "blend_cuda.c", "vfr_cuda.c", "format_cuda.c", "rotate_cuda.c", "deinterlace_cuda.c"]
CFLAGS = ["-O2", "-std=gnu99", "-fPIC", "-Wall", "-Wno-unused-function", "-D__LIBHB__", "-pthread"]


def _newer(target, deps):
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def _run(cmd, verbose):
    if verbose:
        print(" ".join(str(c) for c in cmd), flush=True)
    r = subprocess.run([str(c) for c in cmd], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("build step failed: " + " ".join(str(c) for c in cmd))
    if verbose and r.stderr.strip():
        print(r.stderr)


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found")
    return p


def build_cuda(force=False, verbose=False):
    LIB.mkdir(exist_ok=True)
    obj_dir = LIB / "obj"
    obj_dir.mkdir(exist_ok=True)
    csrc = ROOT / "csrc"
    headers = list(csrc.glob("*.h")) + list(csrc.glob("*.cuh")) + [REPO / "include" / "hbcu.h"]
    objs, jobs = [], []
    for name in CU_SOURCES:
        src = csrc / name
        obj = obj_dir / (name + ".o")
        if force or _newer(obj, [src] + headers):
            jobs.append([nvcc_path()] + NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", obj])
        objs.append(obj)
    if jobs:
        # translation units are independent: compile them side by side (nlmeans.cu alone takes minutes)
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1)) as pool:
            for f in [pool.submit(_run, j, verbose) for j in jobs]:
                f.result()
    out = LIB / "libhbcu.so"
    if force or _newer(out, objs):
        _run([nvcc_path(), "-shared", "-o", out] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static", "-Xlinker", "--exclude-libs=ALL"], verbose)
    return out


def build_shim(force=False, verbose=False):
    LIB.mkdir(exist_ok=True)
    libhb = ROOT / "libhb"
    srcs = [libhb / s for s in SHIM_SOURCES]
    headers = list(libhb.glob("**/*.h"))
    out = LIB / "libhbshim.so"
    if force or _newer(out, srcs + headers):
        _run(["gcc"] + CFLAGS + ["-shared", "-o", out] + srcs + ["-I", libhb, "-I", REPO / "include", "-lm", "-lpthread"], verbose)
    return out


def build_filters(force=False, verbose=False):
    shim = build_shim(force, verbose)
    libhb = ROOT / "libhb"
    srcs = [libhb / s for s in C_SOURCES]
    headers = list(libhb.glob("**/*.h")) + [REPO / "include" / "hbcu.h"]
    out = LIB / "libhbcu_filters.so"
    if force or _newer(out, srcs + headers + [LIB / "libhbcu.so", shim]):
        # -lhbshim stands where a HandBrake build has libhb itself: the filter objects carry no runtime of their own
        _run(["gcc"] + CFLAGS + ["-shared", "-o", out] + srcs +
             ["-I", libhb, "-I", REPO / "include", "-L", LIB, "-lhbcu", "-lhbshim", "-Wl,-rpath,$ORIGIN", "-Wl,-z,defs", "-lm", "-lpthread"], verbose)
    return out


def build_all(force=False, verbose=False):
    return build_cuda(force, verbose), build_filters(force, verbose)


if __name__ == "__main__":
    a, b = build_all(force="--force" in sys.argv, verbose=True)
    print("built", a, b)
