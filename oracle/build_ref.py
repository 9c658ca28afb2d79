"""ORACLE — test infrastructure only.

Compile the UNMODIFIED reference extension (MyRender/CloudProjection/{pcpr_cuda.cpp,point_render.cu}) from a checkout of
the reference (READ_REFERENCE_ROOT, default /root/reference) into oracle/_ref/pcpr*.so with a direct nvcc/g++ recipe (not
the reference's setup.py).  tests/golden/make_ref_pcpr_golden.py runs it on a GPU and stores its outputs, which
tests/test_gpu_reference_kernel.py compares against.
No reference SOURCE is copied into this repository.
"""
import os
import subprocess
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
OUT_DIR = os.path.join(HERE, "_ref")
REFERENCE_ROOT = os.environ.get("READ_REFERENCE_ROOT", "/root/reference")
SRC = os.path.join(REFERENCE_ROOT, "MyRender", "CloudProjection")


def so_path():
    return os.path.join(OUT_DIR, "pcpr" + sysconfig.get_config_var("EXT_SUFFIX"))


def build(force=False):
    import torch
    from torch.utils import cpp_extension as ce
    out = so_path()
    if os.path.exists(out) and not force:
        return out
    if not os.path.isdir(SRC):
        raise RuntimeError("reference sources not present")
    os.makedirs(OUT_DIR, exist_ok=True)
    inc = []
    for p in ce.include_paths(device_type="cuda") if "device_type" in ce.include_paths.__code__.co_varnames else ce.include_paths(True):
        inc += ["-I", p]
    inc += ["-I", sysconfig.get_paths()["include"], "-I", SRC]
    defs = ["-DTORCH_EXTENSION_NAME=pcpr", "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=" + str(int(torch._C._GLIBCXX_USE_CXX11_ABI))]
    o1, o2 = os.path.join(OUT_DIR, "pcpr_cuda.o"), os.path.join(OUT_DIR, "point_render.o")
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-w"] + defs + inc + ["-c", os.path.join(SRC, "pcpr_cuda.cpp"), "-o", o1])
    subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-O2", "-std=c++17", "-w", "-Xcompiler", "-fPIC",
                           "-gencode", "arch=compute_90,code=sm_90"] + defs + inc +
                          ["-c", os.path.join(SRC, "point_render.cu"), "-o", o2])
    libdir = os.path.join(os.path.dirname(torch.__file__), "lib")
    subprocess.check_call(["g++", "-shared", o1, o2, "-o", out, "-L" + libdir, "-L/usr/local/cuda/lib64",
                           "-lc10", "-ltorch", "-ltorch_cpu", "-ltorch_python", "-lc10_cuda", "-ltorch_cuda", "-lcudart",
                           "-Wl,-rpath," + libdir])
    return out


def load():
    """Import the built reference module (needs a GPU to run anything)."""
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    p = so_path()
    if not os.path.exists(p):
        return None
    spec = importlib.util.spec_from_file_location("pcpr", p)
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


if __name__ == "__main__":
    print(build(force=True))
