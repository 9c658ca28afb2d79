"""The int32-index oracle z-buffer (tests/zbuffer_i32.c) for the tests of clouds of more than 2^24 + 1 points.

The C file is compiled with oracle/'s flags into a private temporary directory on first use (the source tree may be read-only),
and removed when the process exits."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "zbuffer_i32.c")
_lib = None


def _load():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="read_b200_oracle_i32_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "liboracle_zbuffer_i32.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-o", so, _SRC, "-lm"])
        lib = ctypes.CDLL(so)
        f32p = ctypes.POINTER(ctypes.c_float)
        lib.oracle_pcpr_forward_i32.argtypes = [f32p, ctypes.c_int64, f32p, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                                ctypes.POINTER(ctypes.c_int32), f32p]
        lib.oracle_pcpr_forward_i32.restype = None
        _lib = lib
    return _lib


def pcpr_forward_i32(xyz, total_m, w, h):
    """``oracle.pcpr_forward`` with an int32 index map (exact for every id < 2^31; the float map is exact up to 2^24 + 1 points):
    xyz [N,3] f32, total_m [B,4,4] f32 -> (index [B,h,w] int32, depth [B,h,w] f32), numpy."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    total_m = np.ascontiguousarray(total_m, dtype=np.float32)
    assert xyz.ndim == 2 and xyz.shape[1] == 3 and xyz.shape[0] < 2 ** 31
    assert total_m.ndim == 3 and total_m.shape[1:] == (4, 4), "batch_size check"
    B = total_m.shape[0]
    index = np.empty((B, h, w), np.int32)
    depth = np.empty((B, h, w), np.float32)
    fp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
    _load().oracle_pcpr_forward_i32(fp(xyz), xyz.shape[0], fp(total_m), B, int(w), int(h),
                                    index.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)), fp(depth))
    return index, depth
