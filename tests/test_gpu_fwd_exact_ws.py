"""Exact checks of the TMA conv kernel's weight-stationary body (csrc/conv_tc.cu: gated_conv_tc_ws_kernel, the 3x3 stride-1
32 -> 32 layers) at the edges test_gpu_fwd_exact.py's small images do not reach, by its method (tests/fwd_exact_util.py):

* several tiles per CTA, so the two consumer warpgroups alternate, and odd tile counts per CTA, so one warpgroup's last turn
  finds no tile (one, two and three persistent CTAs and the full grid, in both tile orders);
* enough tiles per CTA that the halo ring (13 stages) and the four epilogue stages wrap several times;
* ELU with a residual and neither, at ragged W and H and B = 1 and 2.

A CONV_TCGEN05 plan does not say which kernel body it runs, so one more test reads the launched kernel's name from the profiler.
"""
import pytest

import fwd_exact_util as X
from test_gpu_fwd_exact import _run_case, gate_pinned  # noqa: F401  (gate_pinned is a module fixture)
from test_gpu_fwd_exact_ws64 import _kernels_launched

pytestmark = pytest.mark.gpu

WS_CASES = [
    # 6 x 3 = 18 tiles: 18 / 9 / 6 per CTA at max_ctas 1 / 2 / 3
    X.Case("ws 3x3 32->32 +res elu 18 tiles", "tma", ((32, "id", 1),), 32, 3, 1, 1, 33, 41, elu=1, residual=True),
    # 2 x (3 x 5) = 30 tiles: 30 / 15 / 10 per CTA
    X.Case("ws 3x3 32->32 30 tiles", "tma", ((32, "id", 1),), 32, 3, 1, 2, 47, 35),
    # 1 x 7 = 7 tiles, one pixel wide: 7 / 4+3 / 3+2+2 per CTA
    X.Case("ws 3x3 32->32 +res W1", "tma", ((32, "id", 1),), 32, 3, 1, 1, 100, 1, residual=True),
]


@pytest.mark.parametrize("case", WS_CASES, ids=lambda c: c.id)
def test_ws_forward_is_exact(case, gate_pinned):  # noqa: F811
    _run_case(case, gate_pinned)


@pytest.mark.parametrize("case, body", [
    (WS_CASES[0], "gated_conv_tc_ws_kernel"),
    # the training path's recomputed [f | m] of the same shape keeps the general body
    (X.Case("RAW 3x3 32->32", "tma", ((32, "id", 1),), 32, 3, 1, 1, 17, 9, out="raw"), "gated_conv_tc_kernel"),
], ids=lambda v: v.id if isinstance(v, X.Case) else v)
def test_32_channel_layer_runs_its_body(case, body):
    names = _kernels_launched(case)
    assert len(names) == 1 and body in next(iter(names)), f"{case.id}: launched {names}, expected {body}"
