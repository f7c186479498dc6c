"""In-tree build of libr8bgpu.so (the C-ABI library) for sm_90a (H100).

nvcc cross-compiles without a GPU.  The library is written next to this file, where the
package loads it from; it is git-ignored.
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libr8bgpu.so")
SHIM_SOURCES = ["r8bsrc_shim.cpp", os.path.join("..", "..", "include", "r8b", "CDSPResampler.h"), os.path.join("..", "..", "include", "r8b", "DLL", "r8bsrc.h")]
SOURCES = ["r8b_capi.cu", "r8b_kernels.cu", "r8b_fused.cu", "r8b_fused2.cu", "r8b_format.cu", "r8b_format_bytes.cu", "r8b_format_dsd.cu", "r8b_dsd_mod.cu", "r8b_state.cu", "r8b_oneshot.cu", "r8b_adjoint.cu", "r8b_plan.cpp", "r8b_design.cpp", "r8b_hosttab.cpp", "r8b_multi.cpp"]
HEADERS = ["r8b_fft.cuh", "r8b_bclarge.cuh","r8b_interp.cuh", "r8b_fused_common.cuh", "r8b_fused2_core.cuh", "r8b_poly.cuh", "r8b_hbfuse.cuh", "r8b_kernels.h", "r8b_dither.cuh", "r8b_codec.cuh", "r8b_dsd.cuh", "r8b_dsdmod.cuh", "r8b_format.cuh", "r8b_plan.h", "r8b_hosttab.h", "r8b_multi.h", "r8b_design.h", "r8b_tables.inc",
           os.path.join("..", "..", "include", "r8bgpu.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17", "--shared",
    "-Xcompiler", "-fPIC,-fvisibility=hidden,-ffp-contract=off,-fno-fast-math",
    "-Xptxas", "-v",
]


def find_nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    return None


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS + SHIM_SOURCES] + [os.path.abspath(__file__)]
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


DLL_LIB = os.path.join(HERE, "libr8bsrc.so")


def build_dll_shim():
    """libr8bsrc.so: the reference's r8b_* DLL entry points (DLL/r8bsrc.h) over the header front-end and libr8bgpu.so."""
    gxx = shutil.which("g++")
    if gxx is None:
        return None
    src = os.path.join(CSRC, "r8bsrc_shim.cpp")
    r = subprocess.run([gxx, "-O2", "-std=c++11", "-fPIC", "-shared", "-fvisibility=hidden", "-o", DLL_LIB + ".tmp", src,
                        "-L", HERE, "-lr8bgpu", "-Wl,-rpath,$ORIGIN"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("building libr8bsrc.so failed")
    os.replace(DLL_LIB + ".tmp", DLL_LIB)
    return DLL_LIB


def build(force=False, verbose=False):
    """Compile the library if it is missing or stale.  Returns the path of the .so."""
    alt = os.environ.get("R8BGPU_LIB_PATH")  # experiments: a library built elsewhere with other -D knobs
    if alt and os.path.exists(alt):
        return alt
    if not force and not needs_build():
        if not os.path.exists(DLL_LIB) and os.path.exists(LIB):
            build_dll_shim()
        return LIB
    nvcc = find_nvcc()
    if nvcc is None:
        if os.path.exists(LIB):
            return LIB  # GPU box without a toolchain: use the prebuilt library
        raise RuntimeError("nvcc not found and no prebuilt libr8bgpu.so present")
    extra = ["-DR8BGPU_PHASE_TIMERS"] if os.environ.get("R8BGPU_PHASE_TIMERS") else []
    extra += os.environ.get("R8BGPU_EXTRA_DEFS", "").split()  # experiments, e.g. "-DR8BGPU_HB_NT=512 -DR8BGPU_HB_MINB=2"
    cmd = [nvcc] + NVCC_FLAGS + extra + ["-o", LIB + ".tmp"] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log = os.path.join(HERE, "build.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("nvcc failed (see %s)" % log)
    os.replace(LIB + ".tmp", LIB)
    build_dll_shim()
    if verbose:
        sys.stdout.write(r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
