"""Build the C-ABI CUDA library in-tree with nvcc for sm_90a (no JIT, no torch build system).

    python -m read_b200.build [--force] [--verbose]

The .so and the object files are build products (git-ignored).
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libread_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, diag=False):
    """diag=True builds libread_b200_diag.so with -DREAD_DIAG (work-skipping knobs + role timelines for timing experiments;
    never loaded by the product: scripts opt in with READ_B200_LIB=...)."""
    if diag:
        return _build(LIB.replace(".so", "_diag.so"), "_obj_diag", ["-DREAD_DIAG"], verbose)
    if not force and not _stale():
        return LIB
    return _build(LIB, "_obj", [], verbose)


def _build(LIB, objdir, extra, verbose):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, objdir), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- {os.path.basename(src)}\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libread_b200.so")
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv, diag="--diag" in sys.argv))
