"""The built library really contains the Hopper instructions DESIGN.md claims (checked on the SASS of libread_b200.so, no GPU needed):
warpgroup MMAs (HGMMA) fed by ldmatrix (LDSM), TMA tile loads (UTMALDG), the cp.async-gathered A operand of the gather kernel
(LDGSTS) and the bulk copy of the streaming rasterizer (UBLKCP); and that the work-skipping diagnostic knobs are absent from the
shipped build."""
import collections
import os
import re
import shutil
import subprocess

import pytest

from read_b200 import _lib

CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"


@pytest.fixture(scope="module")
def sass():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("libread_b200.so not built")
    out = subprocess.run([CUOBJDUMP, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=300).stdout
    per_fn, cur = collections.defaultdict(collections.Counter), None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"\*/\s+(?:@!?U?P\w+\s+)?([A-Z][A-Z0-9_.]*)", line)
        if m and cur:
            per_fn[cur][m.group(1)] += 1
    return per_fn


def _kernels(per_fn, needle):
    ks = {k: v for k, v in per_fn.items() if needle in k}
    assert ks, f"no kernel named *{needle}* in the library"
    return ks


def _has(counter, prefix):
    return sum(n for op, n in counter.items() if op.startswith(prefix))


def test_conv_kernels_use_wgmma_and_tma(sass):
    for name, ops in _kernels(sass, "gated_conv_tc_kernel").items():
        assert _has(ops, "HGMMA") > 0 and _has(ops, "LDSM") > 0 and _has(ops, "UTMALDG") > 0, name
        assert _has(ops, "SYNCS") > 0, name                                  # mbarrier rings between producer and consumers


def test_gather_kernel_and_rasterizer(sass):
    for name, ops in _kernels(sass, "gated_conv_tc_gather_kernel").items():
        assert _has(ops, "HGMMA") > 0 and _has(ops, "LDSM") > 0 and _has(ops, "LDGSTS") > 0, name     # cp.async-gathered A operand
    for name, ops in _kernels(sass, "raster_stream_kernel").items():
        assert _has(ops, "UBLKCP") > 0 and _has(ops, "SYNCS") > 0, name        # cp.async.bulk ring + mbarriers
        assert _has(ops, "RED") + _has(ops, "ATOM") > 0, name                 # 64-bit min into the packed z-buffer


def test_shipped_library_rejects_the_diagnostic_knobs():
    lib = _lib.load()
    for knob in (b"tc_debug", b"tcg_debug"):
        assert lib.read_set_option(knob, 1) != 0                              # unknown to the shipped build (READ_DIAG only)
    assert lib.read_set_option(b"raster_mode", 4) != 0 and lib.read_set_option(b"raster_mode", 5) != 0
    assert lib.read_set_option(b"raster_mode", 2) == 0 and lib.read_set_option(b"tc_pdl", 1) == 0
    assert lib.read_set_option(b"no_such_option", 1) != 0
