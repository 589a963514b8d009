"""In-tree build of the CUDA library and the torch operator module.

    python -m warp_rnnt_b200.build            # both
    python -m warp_rnnt_b200.build --lib      # librnnt_b200.so only (no torch needed)

Artifacts (git-ignored):
    warp_rnnt_b200/lib/librnnt_b200.so   nvcc -gencode arch=compute_90a,code=sm_90a  (C ABI)
    warp_rnnt_b200/lib/_C.so             g++ binding.cpp against torch + librnnt_b200.so
sm_90a (H100) only: no other arch, no PTX fallback, no CPU path.
"""
import os
import shutil
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "librnnt_b200.so")
EXT = os.path.join(LIBDIR, "_C.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

CU_SOURCES = ["wavefront.cu", "expand.cu", "fused.cu", "logits.cu", "joint.cu", "simple.cu", "tdt.cu", "frames.cu",
              "api.cu"]
CU_HEADERS = ["common.cuh", "kernels.cuh", os.path.join(INCLUDE, "rnnt_b200.h")]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: the CUDA extension cannot be built (there is no CPU fallback)")


def cu_sources():
    return [os.path.join(CSRC, s) for s in CU_SOURCES if os.path.exists(os.path.join(CSRC, s))]


STAMP = os.path.join(LIBDIR, "sources.sha256")


def sources_digest():
    """Content hash of everything the two artefacts are built from (mtimes do not survive copies to another box)."""
    import hashlib
    h = hashlib.sha256()
    files = cu_sources() + [d if os.path.isabs(d) else os.path.join(CSRC, d) for d in CU_HEADERS] + \
        [os.path.join(CSRC, "binding.cpp")]
    for f in sorted(files):
        if os.path.exists(f):
            h.update(os.path.basename(f).encode())
            h.update(open(f, "rb").read())
    return h.hexdigest()


def up_to_date():
    """True when lib/ holds both artefacts AND they were built from the sources as they are now."""
    if not (os.path.exists(LIB) and os.path.exists(EXT) and os.path.exists(STAMP)):
        return False
    try:
        return open(STAMP).read().strip() == sources_digest()
    except OSError:
        return False


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))




def build_lib(force=False, verbose=False):
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = cu_sources()
    deps = srcs + [d if os.path.isabs(d) else os.path.join(CSRC, d) for d in CU_HEADERS]
    if not (force or _stale(LIB, deps)):
        return LIB
    cmd = [_nvcc(), "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
           "-Xcompiler", "-fPIC", "-shared", "-Xlinker", "-soname=librnnt_b200.so", "-o", LIB] + srcs
    if verbose:
        cmd += ["-Xptxas", "-v"]
    subprocess.check_call(cmd)
    return LIB


def build_ext(force=False):
    """binding.cpp -> lib/_C.so (needs torch headers; ~1 min)."""
    src = os.path.join(CSRC, "binding.cpp")
    if not (force or _stale(EXT, [src, os.path.join(INCLUDE, "rnnt_b200.h")])):
        return EXT
    build_lib()
    import torch
    from torch.utils import cpp_extension as ce
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
           "-DTORCH_EXTENSION_NAME=_C", "-DTORCH_API_INCLUDE_EXTENSION_H",
           "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI)]
    for name in ("COMPILER_TYPE", "STDLIB", "BUILD_ABI"):
        v = getattr(torch._C, "_PYBIND11_" + name, None)
        if v is not None:
            cmd.append('-DPYBIND11_%s="%s"' % (name, v))
    for inc in ce.include_paths("cuda") + [sysconfig.get_paths()["include"]]:
        cmd += ["-isystem", inc]
    cmd += [src, "-o", EXT]
    for lp in ce.library_paths("cuda"):
        cmd += ["-L" + lp, "-Wl,-rpath," + lp]
    cmd += ["-L" + LIBDIR, "-lrnnt_b200", "-Wl,-rpath,$ORIGIN",
            "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart"]
    subprocess.check_call(cmd)
    return EXT


def build_all(force=False, verbose=False):
    force = force or not up_to_date()
    build_lib(force, verbose)
    build_ext(force)
    with open(STAMP, "w") as f:
        f.write(sources_digest() + "\n")
    return LIB, EXT


if __name__ == "__main__":
    force = "--force" in sys.argv
    if "--lib" in sys.argv:
        print(build_lib(force, verbose="-v" in sys.argv))
    else:
        print(*build_all(force, verbose="-v" in sys.argv))
