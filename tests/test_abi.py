"""The C-ABI library loads and exports every symbol include/read_b200.h declares (no compute without a GPU)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from read_b200 import _lib


def _declared():
    src = open(os.path.join(ROOT, "include", "read_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    names = re.findall(r"\b(read_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


def test_library_is_built_and_loads():
    lib = _lib.load()
    assert lib.read_version() >= 100


def test_every_declared_symbol_is_exported_and_bound():
    lib = _lib.load()
    declared = _declared()
    assert len(declared) >= 25
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/read_b200.h but not exported"
    assert sorted(_lib.EXPORTS) == declared, set(_lib.EXPORTS) ^ set(declared)


def test_pyramid_geometry_host_functions():
    lib = _lib.load()
    # myrender.py:33-34 sizes; kitti6 viewport and 1080p
    w, h = ctypes.c_int(), ctypes.c_int()
    lib.read_level_size(1216, 368, 4, ctypes.byref(w), ctypes.byref(h))
    assert (w.value, h.value) == (76, 23)
    lib.read_level_size(1920, 1080, 4, ctypes.byref(w), ctypes.byref(h))
    assert (w.value, h.value) == (120, 67)
    P = sum((1920 >> l) * (1072 >> l) for l in range(4))
    assert P == 2733600                                  # SURVEY.md §8: P for C3
    assert lib.read_pyramid_entries(1, 1920, 1072, 4) == P
    assert lib.read_pyramid_entries(3, 1920, 1072, 4) == 3 * P
    assert lib.read_pyramid_level_offset(2, 64, 32, 2) == 2 * (64 * 32 + 32 * 16)
    assert lib.read_pyramid_entries(1, 64, 64, 99) == -1


def test_direct_mask_nested_vs_odd_levels():
    lib = _lib.load()
    assert lib.read_raster_direct_mask(1920, 1072, 4) == 0b0001       # every level an exact halving
    assert lib.read_raster_direct_mask(1920, 1080, 5) == 0b10001      # 135 -> 67 is not
    assert lib.read_raster_direct_mask(1216, 368, 5) == 0b00001
    assert lib.read_raster_direct_mask(100, 50, 3) == 0b101           # 50,25,12 / 100,50,25 : level 2 odd


def test_generic_packing_geometry():
    lib = _lib.load()
    assert lib.read_generic_npad(3) == 64 and lib.read_generic_npad(32) == 64 and lib.read_generic_npad(56) == 128
    assert lib.read_tc_weight_elems(32, 32, 3) == 9 * 32 * 64
    assert lib.read_tc_weight_elems(3, 32, 3) == 9 * 32 * 16          # final layer: Cout padded to 8 (N = 16)
    assert lib.read_tc_weight_elems(56, 32, 1) == -1                  # not a TMA-kernel shape (gather kernel takes it)
    assert lib.read_tcg_weight_elems(56, 32, 1) == 64 * 112           # K padded to one 64-block, N = 2*56


def test_conv_validation_errors_without_gpu():
    lib = _lib.load()
    d = _lib.ReadConvDesc()
    plan = _lib.c_vp()
    rc = lib.read_conv_plan_create(ctypes.byref(d), ctypes.byref(plan))
    assert rc == -1 and b"conv" in lib.read_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc)


def test_ctypes_mirror_matches_the_header_layout(tmp_path):
    """read_conv_desc / read_src cross the C ABI by pointer: the ctypes mirror in read_b200/_lib.py must have the header's
    size and field offsets (compiled here with the host C compiler, no GPU involved)."""
    import subprocess
    fields = [n for n, _ in _lib.ReadConvDesc._fields_]
    prog = ['#include <stdio.h>', '#include <stddef.h>', '#include "read_b200.h"', 'int main(void) {',
            '  printf("sizeof_desc %zu\\n", sizeof(read_conv_desc));', '  printf("sizeof_src %zu\\n", sizeof(read_src));']
    prog += [f'  printf("{f} %zu\\n", offsetof(read_conv_desc, {f}));' for f in fields]
    prog += ['  return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(prog))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(line.split() for line in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["sizeof_desc"]) == ctypes.sizeof(_lib.ReadConvDesc)
    assert int(got["sizeof_src"]) == ctypes.sizeof(_lib.ReadSrc)
    for f in fields:
        assert int(got[f]) == getattr(_lib.ReadConvDesc, f).offset, f


def _desc_1x1(cout, srcs, out_mode=None, addin=False):
    d = _lib.ReadConvDesc()
    d.act_dtype, d.n_src = _lib.ACT_BF16, len(srcs)
    cin = 0
    for i, (c, h, w, mode, f) in enumerate(srcs):
        d.src[i].ptr, d.src[i].C, d.src[i].H, d.src[i].W = 0x1000, c, h, w
        d.src[i].mode, d.src[i].factor = mode, f
        cin += c
    d.B, d.Hin, d.Win, d.Cin, d.Hout, d.Wout, d.Cout = 1, 64, 64, cin, 64, 64, cout
    d.k, d.stride, d.pad = 1, 1, 0
    d.out_mode = _lib.OUT_NHWC if out_mode is None else out_mode
    if addin:
        d.addin, d.addin_H, d.addin_W = 0x2000, 32, 32
    return d


def test_tc_supported_predicate_for_concat_raw_and_addin():
    """Which layers the TMA-fed wgmma kernel accepts (host-side predicate only): 1x1 virtual concats of identity /
    nearest-down sources in 32-channel granules, RAW terms and add-ins for Cout 16 / 32 / 64, stride-2 3x3 / 4x4."""
    lib = _lib.load()
    ID, DOWN, UP = _lib.SRC_IDENTITY, _lib.SRC_NEAREST_DOWN, _lib.SRC_NEAREST_UP
    ok = lambda d: lib.read_conv_tc_supported(ctypes.byref(d))
    assert ok(_desc_1x1(32, [(32, 64, 64, ID, 1), (32, 64, 64, ID, 1)])) == 1                    # Convs.2
    assert ok(_desc_1x1(64, [(32, 128, 128, DOWN, 2), (64, 64, 64, ID, 1)])) == 1                # AFF1's fine sources
    assert ok(_desc_1x1(64, [(32, 128, 128, DOWN, 2), (64, 32, 32, UP, 2)])) == 0                # nearest-up: gather kernel
    assert ok(_desc_1x1(64, [(8, 64, 64, ID, 1), (56, 64, 64, ID, 1)])) == 0                     # SCM concat: 8-channel source
    assert ok(_desc_1x1(32, [(64, 64, 64, ID, 1)], out_mode=_lib.OUT_RAW_NHWC)) == 1             # RAW term
    assert ok(_desc_1x1(32, [(32, 64, 64, ID, 1)], addin=True)) == 1                             # final AFF0 term
    assert ok(_desc_1x1(128, [(128, 64, 64, ID, 1)], out_mode=_lib.OUT_RAW_NHWC)) == 0           # RAW only for Cout <= 64
    assert ok(_desc_1x1(128, [(128, 64, 64, ID, 1)], addin=True)) == 0
    d = _desc_1x1(64, [(32, 64, 64, ID, 1)])
    d.k, d.stride, d.pad, d.Hout, d.Wout = 3, 2, 1, 32, 32
    assert ok(d) == 1                                                                            # feat_extract.1
    d.k = 4
    assert ok(d) == 1                                                                            # 4x4 stride 2, pad 1
    d.k, d.Hout = 3, 31
    assert ok(d) == 0
    # RAW / add-in exist on the TMA kernel only: the gather kernel refuses them
    assert lib.read_conv_tcg_supported(ctypes.byref(_desc_1x1(32, [(32, 64, 64, ID, 1)], addin=True))) == 0
