"""Exact checks of the TMA conv kernel's 64-channel weight-stationary body (csrc/conv_tc.cu: gated_conv_tc_ws64_kernel, the 3x3
stride-1 64 -> 64 layers) at the edges test_gpu_fwd_exact.py's small images do not reach, by its method (tests/fwd_exact_util.py):

* several tiles per CTA, so both accumulator sets of each warpgroup take turns, and odd tile counts per CTA, so the last turn
  issues no next tile (one, two and three persistent CTAs and the full grid, in both tile orders);
* enough tiles per CTA that the two-stage halo ring and the two epilogue stages wrap several times;
* ELU with a residual and neither, at ragged W and H and B = 1 and 2.

A CONV_TCGEN05 plan does not say which kernel body it runs, so one more test reads the launched kernel's name from the profiler.
"""
import pytest
import torch

import fwd_exact_util as X
from test_gpu_fwd_exact import Launch, _gen, _run_case, gate_pinned  # noqa: F401  (gate_pinned is a module fixture)

pytestmark = pytest.mark.gpu

WS64_CASES = [
    # 6 x 3 = 18 tiles: 18 / 9 / 6 per CTA at max_ctas 1 / 2 / 3
    X.Case("ws64 3x3 64->64 +res elu 18 tiles", "tma", ((64, "id", 1),), 64, 3, 1, 1, 33, 41, elu=1, residual=True),
    # 2 x (3 x 5) = 30 tiles: 30 / 15 / 10 per CTA
    X.Case("ws64 3x3 64->64 30 tiles", "tma", ((64, "id", 1),), 64, 3, 1, 2, 47, 35),
    # 1 x 7 = 7 tiles, one pixel wide: 7 / 4+3 / 3+2+2 per CTA
    X.Case("ws64 3x3 64->64 +res W1", "tma", ((64, "id", 1),), 64, 3, 1, 1, 100, 1, residual=True),
    # 2 x (2 x 3) = 12 tiles, ragged on both edges, ELU without a residual: 12 / 6 / 4 per CTA
    X.Case("ws64 3x3 64->64 elu 12 tiles", "tma", ((64, "id", 1),), 64, 3, 1, 2, 31, 17, elu=1),
]


@pytest.mark.parametrize("case", WS64_CASES, ids=lambda c: c.id)
def test_ws64_forward_is_exact(case, gate_pinned):  # noqa: F811
    _run_case(case, gate_pinned)


def _kernels_launched(c):
    ln = Launch(c, X.make(c, _gen(c)))
    ln.run()                                         # plans and loads the module outside the profiled window
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        ln.run()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "gated_conv" in e.name}


@pytest.mark.parametrize("case, body", [
    (WS64_CASES[0], "gated_conv_tc_ws64_kernel"),
    # the training path's recomputed [f | m] of the same shape keeps the general body
    (X.Case("RAW 3x3 64->64", "tma", ((64, "id", 1),), 64, 3, 1, 1, 17, 9, out="raw"), "gated_conv_tc_kernel"),
], ids=lambda v: v.id if isinstance(v, X.Case) else v)
def test_64_channel_layer_runs_its_body(case, body):
    names = _kernels_launched(case)
    assert len(names) == 1 and body in next(iter(names)), f"{case.id}: launched {names}, expected {body}"
