"""-m gpu: the TMA kernel's epilogue stage (residual / FAM multiplier loaded by TMA, out / out2 stored by TMA) on ragged shapes with
B = 2, where the per-warpgroup store boxes cross the right edge, the bottom edge and the batch boundary of the output."""
import pytest
import torch

from read_b200 import _lib as L
from test_gpu_conv import run_conv

pytestmark = pytest.mark.gpu

CASES = [
    # C32: N = 64, 64-byte rows (SWIZZLE_64B); 37 rows = two full tile rows + 5, 29 columns = three full tile columns + 5
    ("3x3 C32 @37x29 + residual + out2", [(32, 37, 29, "id", 1)], 32, 3, True),
    # C16: N = 32, 32-byte rows (SWIZZLE_32B); rows 9..15 of the last tile row lie outside, so its second warpgroup stores nothing
    ("3x3 16->16 @9x13 + residual + out2", [(16, 9, 13, "id", 1)], 16, 3, False),
    # C64: N = 128, 128-byte rows (SWIZZLE_128B)
    ("3x3 C64 @21x35 + residual + out2", [(64, 21, 35, "id", 1)], 64, 3, True),
    # C256: two n-tiles, each box covers its 64-channel slice
    ("3x3 C256 @19x11 + residual + out2, two n-tiles", [(256, 19, 11, "id", 1)], 256, 3, False),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_tma_epilogue_residual_and_out2_ragged(case):
    _, srcs, cout, k, elu = case
    got, want, got2, want2 = run_conv(srcs, cout, k, 1, elu, True, L.CONV_TCGEN05, residual=True, out2=True)
    assert torch.isfinite(got).all() and torch.isfinite(got2).all(), "TMA kernel left outputs unwritten (NaN sentinel)"
    tol = 2 ** -8 * float(want.abs().max()) + 4e-3
    assert float((got - want).abs().max()) < tol
    assert float((got2 - want2).abs().max()) < tol
