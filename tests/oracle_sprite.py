"""The point-sprite oracle z-buffer (tests/zbuffer_sprite.c), the parity target of the point-sprite tests.

The C file is compiled with oracle/'s flags into a private temporary directory on first use (the source tree may be read-only),
and removed when the process exits."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "zbuffer_sprite.c")
_lib = None
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _load():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="read_b200_oracle_sprite_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "liboracle_sprite.so")
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-mfma", "-o", so, _SRC, "-lm"])
        lib = ctypes.CDLL(so)
        vp = ctypes.c_void_p
        lib.oracle_sprite_project.argtypes = [vp, ctypes.c_int64, vp, ctypes.c_int, ctypes.c_int, vp, vp, vp, vp, vp, vp]
        lib.oracle_sprite_project.restype = None
        _lib = lib
    return _lib


def level_sizes(W, H, L):
    return [(int(W * (0.5 ** i)), int(H * (0.5 ** i))) for i in range(L)]


def sprite_zbuf(xyz, total_m, W, H, levels, point_sizes=None):
    """xyz [N,3] f32, total_m [B,4,4] f32, levels [(N, relative)] per level, point_sizes [N] or None -> per level the [B,h,w] uint64
    keys (depth bits << 32 | id; EMPTY where no point), numpy."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    total_m = np.ascontiguousarray(total_m, dtype=np.float32).reshape(-1, 4, 4)
    B, L = total_m.shape[0], len(levels)
    sizes = level_sizes(W, H, L)
    w = np.array([s[0] for s in sizes], np.int32)
    h = np.array([s[1] for s in sizes], np.int32)
    N = np.array([n for n, _ in levels], np.float32)
    rel = np.array([1 if r else 0 for _, r in levels], np.int32)
    ps = None if point_sizes is None else np.ascontiguousarray(point_sizes, dtype=np.float32)
    assert ps is None or ps.shape == (xyz.shape[0],)
    z = np.empty(sum(B * a * b for a, b in sizes), np.uint64)
    p = lambda a: None if a is None else a.ctypes.data
    _load().oracle_sprite_project(p(xyz), xyz.shape[0], p(total_m), B, L, p(w), p(h), p(N), p(rel), p(ps), p(z))
    out, off = [], 0
    for (a, b) in sizes:
        out.append(z[off:off + B * a * b].reshape(B, b, a))
        off += B * a * b
    return out


def resolve(keys, index_dtype=np.float32):
    """[B,h,w] uint64 keys -> (index, depth) maps as the rasterizer's resolve writes them (0 / 0 where empty)."""
    empty = keys == EMPTY
    idx = np.where(empty, 0, keys & np.uint64(0xFFFFFFFF)).astype(np.int64).astype(index_dtype)
    dep = np.where(empty, 0, keys >> np.uint64(32)).astype(np.uint32).view(np.float32)
    return idx, dep


def sprite_maps(xyz, total_m, W, H, levels, point_sizes=None):
    """Per level (index [B,h,w] f32, depth [B,h,w] f32)."""
    return [resolve(k) for k in sprite_zbuf(xyz, total_m, W, H, levels, point_sizes)]
