"""Build the UNMODIFIED reference (1ytic/warp-rnnt) for sm_90a into oracle/_ref/ -- checker only.

    python oracle/build_ref.py        # RNNT_REFERENCE_DIR=<checkout of 1ytic/warp-rnnt> overrides the default

Compiles the reference's own sources in $RNNT_REFERENCE_DIR, default /root/reference (core.cu,
core_gather.cu, core_compact.cu, pytorch_binding/binding.cpp) with nvcc / g++ directly; nothing
is copied into this repository and the reference's setup.py (which refuses to run without a
visible GPU, setup.py:21-22) is not used.  Output: oracle/_ref/warp_rnnt_ref_C.so, a torch
extension exposing the reference's `_C` API (rnnt_loss / rnnt_loss_compact /
rnnt_loss_compact_backward).  oracle/_ref/ is git-ignored; without a reference checkout nothing is built and a
prebuilt oracle/_ref/ is used if there is one.

TEST INFRASTRUCTURE ONLY: used by tests/golden/make_reference_outputs.py (which records the reference's outputs
that the GPU tests compare with), by tests/test_gpu_parity.py (the reference's binding.cpp on our C ABI, when
present) and by bench.py --impl reference.  The product never loads it.
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("RNNT_REFERENCE_DIR", "/root/reference")
OUT_DIR = os.path.join(HERE, "_ref")
OUT = os.path.join(OUT_DIR, "warp_rnnt_ref_C.so")
NAME = "warp_rnnt_ref_C"


def build(force=False):
    if not os.path.isdir(REF):
        return None                      # no reference checkout: use a prebuilt file if there is one
    if os.path.exists(OUT) and not force:
        return OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    import torch
    from torch.utils import cpp_extension as ce
    objs = []
    for cu in ("core.cu", "core_gather.cu", "core_compact.cu"):
        o = os.path.join(OUT_DIR, cu.replace(".cu", ".o"))
        subprocess.check_call(["nvcc", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a",
                               "-Xcompiler", "-fPIC", "-I" + REF, "-c", os.path.join(REF, cu), "-o", o])
        objs.append(o)
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w",
           "-DTORCH_EXTENSION_NAME=" + NAME, "-DTORCH_API_INCLUDE_EXTENSION_H",
           "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI), "-I" + REF]
    for name in ("COMPILER_TYPE", "STDLIB", "BUILD_ABI"):
        v = getattr(torch._C, "_PYBIND11_" + name, None)
        if v is not None:
            cmd.append('-DPYBIND11_%s="%s"' % (name, v))
    for inc in ce.include_paths("cuda") + [sysconfig.get_paths()["include"]]:
        cmd += ["-isystem", inc]
    cmd += [os.path.join(REF, "pytorch_binding", "binding.cpp")] + objs + ["-o", OUT]
    for lp in ce.library_paths("cuda"):
        cmd += ["-L" + lp, "-Wl,-rpath," + lp]
    cmd += ["-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart"]
    subprocess.check_call(cmd)
    for o in objs:
        os.remove(o)
    return OUT


COMPAT_NAME = "warp_rnnt_compat_C"
COMPAT_OUT = os.path.join(OUT_DIR, COMPAT_NAME + ".so")


def build_compat(force=False):
    """Drop-in proof at the C-ABI level: the reference's OWN pytorch_binding/binding.cpp, compiled
    unmodified, linked against warp_rnnt_b200/lib/librnnt_b200.so (which exports core.h:29-60's
    five entry points) instead of core.cu / core_gather.cu / core_compact.cu."""
    if not os.path.isdir(REF):
        return None
    if os.path.exists(COMPAT_OUT) and not force:
        return COMPAT_OUT
    os.makedirs(OUT_DIR, exist_ok=True)
    import torch
    from torch.utils import cpp_extension as ce
    libdir = os.path.join(os.path.dirname(HERE), "warp_rnnt_b200", "lib")
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-w",
           "-DTORCH_EXTENSION_NAME=" + COMPAT_NAME, "-DTORCH_API_INCLUDE_EXTENSION_H",
           "-D_GLIBCXX_USE_CXX11_ABI=%d" % int(torch._C._GLIBCXX_USE_CXX11_ABI), "-I" + REF]
    for name in ("COMPILER_TYPE", "STDLIB", "BUILD_ABI"):
        v = getattr(torch._C, "_PYBIND11_" + name, None)
        if v is not None:
            cmd.append('-DPYBIND11_%s="%s"' % (name, v))
    for inc in ce.include_paths("cuda") + [sysconfig.get_paths()["include"]]:
        cmd += ["-isystem", inc]
    cmd += [os.path.join(REF, "pytorch_binding", "binding.cpp"), "-o", COMPAT_OUT]
    for lp in ce.library_paths("cuda"):
        cmd += ["-L" + lp, "-Wl,-rpath," + lp]
    cmd += ["-L" + libdir, "-lrnnt_b200", "-Wl,-rpath,$ORIGIN/../../warp_rnnt_b200/lib",
            "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch", "-ltorch_python", "-lcudart"]
    subprocess.check_call(cmd)
    return COMPAT_OUT


def _load(name, path):
    if not os.path.exists(path):
        return None
    import importlib.machinery
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    loader = importlib.machinery.ExtensionFileLoader(name, path)
    spec = importlib.util.spec_from_file_location(name, path, loader=loader)
    mod = importlib.util.module_from_spec(spec)
    loader.exec_module(mod)
    return mod


def load():
    """Import the prebuilt reference extension; None when it is not available."""
    return _load(NAME, OUT)


def load_compat():
    """The reference's binding.cpp on top of librnnt_b200.so; None when it is not available."""
    return _load(COMPAT_NAME, COMPAT_OUT)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
    print(build_compat(force="--force" in sys.argv))
