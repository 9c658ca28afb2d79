"""Exact checks of the TMA conv kernel's role-swapped body with streamed weights (csrc/conv_tc.cu: gated_conv_tc_wss_kernel<R>,
the 3x3 stride-1 128 -> 128 and 256 -> 256 layers) at the edges test_gpu_fwd_exact.py's small images do not reach, by its method
(tests/fwd_exact_util.py):

* several work units (16 x R-pixel tile, n-tile of 64 output channels) per CTA, and unit counts that do not divide evenly (one,
  two and three persistent CTAs and the full grid, in both tile orders);
* enough units per CTA that the two-stage halo ring, the weight ring and the two epilogue stages wrap several times;
* ELU with a residual and neither, at W and H that are multiples of neither 16 nor 17, one pixel wide, and B = 1 and 2;
* tiles of R = 16 and R = 17 rows, as the plan's rule picks them for the GPU's SM count (wss_rows below).

A CONV_TCGEN05 plan does not say which kernel body it runs, so one more test reads the launched kernel's name from the profiler.
"""
import pytest
import torch

import fwd_exact_util as X
from test_gpu_fwd_exact import _run_case, gate_pinned  # noqa: F401  (gate_pinned is a module fixture)
from test_gpu_fwd_exact_ws64 import _kernels_launched

pytestmark = pytest.mark.gpu


def wss_rows(c, sms):
    """Tile rows of the plan (conv_tc.cu: tc_wss_rows): the fewest pixel slots on the busiest CTA, ceil(units / SMs) x 16 R, and
    on a tie the fewer halo rows."""
    def key(r):
        ty = -(-c.hout // r)
        units = -(-c.wout // 16) * ty * c.B * (c.cout // 64)
        return -(-units // sms) * 16 * r, ty * (r + 2)
    return min((16, 17), key=key)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


WSS_CASES = [
    # 3 x 3 tiles x 2 n-tiles = 18 units (R = 16): 18 / 9 / 6 per CTA at max_ctas 1 / 2 / 3
    X.Case("wss 3x3 128->128 +res elu 18 units", "tma", ((128, "id", 1),), 128, 3, 1, 1, 35, 41, elu=1, residual=True),
    # R = 17 on 132 SMs: 2 x (6 x 2) tiles x 4 n-tiles = 96 units, where R = 16 makes 144 (two rounds)
    X.Case("wss 3x3 256->256 B2 96 units", "tma", ((256, "id", 1),), 256, 3, 1, 2, 33, 90),
    # one pixel wide: 7 tiles x 2 n-tiles = 14 units
    X.Case("wss 3x3 128->128 +res W1", "tma", ((128, "id", 1),), 128, 3, 1, 1, 100, 1, residual=True),
    # 2 x (2 x 2) tiles x 4 n-tiles = 32 units, ELU without a residual
    X.Case("wss 3x3 256->256 elu 32 units", "tma", ((256, "id", 1),), 256, 3, 1, 2, 20, 23, elu=1),
    # R = 17 on 132 SMs: 23 x 2 tiles x 2 n-tiles = 92 units, where R = 16 makes 138
    X.Case("wss 3x3 128->128 +res elu 92 units", "tma", ((128, "id", 1),), 128, 3, 1, 1, 33, 359, elu=1, residual=True),
]


@pytest.mark.parametrize("case", WSS_CASES, ids=lambda c: c.id)
def test_wss_forward_is_exact(case, gate_pinned):  # noqa: F811
    _run_case(case, gate_pinned)


def test_cases_pick_both_tile_heights():
    sms = _sms()
    assert {wss_rows(c, sms) for c in WSS_CASES} == {16, 17}, f"on {sms} SMs the cases do not reach both R = 16 and R = 17"


@pytest.mark.parametrize("case, body", [
    (WSS_CASES[0], "gated_conv_tc_wss_kernel"),
    (WSS_CASES[1], "gated_conv_tc_wss_kernel"),
    (WSS_CASES[4], "gated_conv_tc_wss_kernel"),
    # the training path's recomputed [f | m] of the same shape keeps the general body
    (X.Case("RAW 3x3 128->128", "tma", ((128, "id", 1),), 128, 3, 1, 1, 17, 9, out="raw"), "gated_conv_tc_kernel"),
], ids=lambda v: v.id if isinstance(v, X.Case) else v)
def test_streamed_layer_runs_its_body(case, body):
    # a profiler session now and then reports no kernel events at all after a long run of other tests in the process; an
    # empty capture says nothing about the body, so it is taken again (a wrong body still fails)
    for _ in range(3):
        names = _kernels_launched(case)
        if names:
            break
    assert len(names) == 1 and body in next(iter(names)), f"{case.id}: launched {names}, expected {body}"
    if body == "gated_conv_tc_wss_kernel":
        r = wss_rows(case, _sms())
        assert f"gated_conv_tc_wss_kernel<{r}>" in next(iter(names)), f"{case.id}: launched {names}, expected R = {r}"
