"""No GPU: the float64 replay of the bf16 training Functions (tests/train_fn_exact_util.py) restates the modules, and every
exact-tier case meets its precondition and its coverage rule."""
import functools

import pytest
import torch

import train_fn_exact_util as T


@functools.lru_cache(maxsize=None)
def _operands(case):
    return T.exact_operands(case)


def _rel(got, want):
    scale = float(want.abs().max()) if want.numel() else 0.0
    return float((got - want).abs().max()) / scale if scale > 0 else float((got - want).abs().max())


@pytest.mark.parametrize("case", T.EXACT_CASES, ids=lambda c: c.id)
def test_replay_without_rounding_is_float64_autograd(case):
    """With every rounding the identity the replay is float64 autograd of the same GatedConv modules: the output, every input
    gradient and all six parameter gradients of every conv, to 1e-12 relative."""
    mods, xs, res, gout = _operands(case)
    r = T.replay(case, mods, xs, res, gout, R=T.ident)
    out, dxs, dres, grads = T.autograd_ref(case, mods, xs, res, gout)
    assert _rel(r["out"], out) <= 1e-12, case.id
    for a, b in zip(r["dxs"], dxs):
        assert (a is None) == (b is None), case.id
        if a is not None:
            assert _rel(a, b) <= 1e-12, case.id
    if case.residual:
        assert _rel(r["dres"], dres) <= 1e-12, case.id
    assert len(grads) == len(r["grads"]) == 6 * case.n_convs
    for i, (a, b) in enumerate(zip(r["grads"], grads)):
        assert a.shape == b.shape and _rel(a, b) <= 1e-12, (case.id, i // 6, T.NAMES[i % 6])


@pytest.mark.parametrize("case", T.EXACT_CASES, ids=lambda c: c.id)
def test_exact_case_meets_its_precondition(case):
    """Every fp32 sum of every stage is a multiple of its unit below 2^24 units, every gate pinned open, every ELU input
    positive; the Function's output holds at least NONREP_FLOOR values that bf16 cannot (the rounding is tested)."""
    mods, xs, res, gout = _operands(case)
    worst = T.precondition(case, mods, xs, res, gout)
    shares = T.nonrep_shares(T.replay(case, mods, xs, res, gout))
    print(f"\n{case.id}: worst {max(worst.values()):.3g} units ({max(worst, key=worst.get)}); bf16-unrepresentable shares "
          + ", ".join(f"{k} {v:.2f}" for k, v in shares.items()))
    assert shares["out"] >= T.NONREP_FLOOR, (case.id, shares)


@pytest.mark.parametrize("family", ["stack", "single", "multi"])
def test_every_rounding_point_is_tested_and_every_filter_block_covered(family):
    """Across a family's cases: every conv has nonzero f-filters at all k x k taps and in every 8-channel input and output
    block (a misrouted tap, block, source or item changes some element), and each bf16 rounding point of the chain holds
    values bf16 cannot in at least ROUND_FLOOR of some case's elements ([df | dm] only where gamma is not a power of two: the
    stacks keep gamma = +-1 so their values stay exact through 8 convs)."""
    cases = [c for c in T.EXACT_CASES if c.family == family]
    best = {}
    for c in cases:
        mods, xs, res, gout = _operands(c)
        for i, (taps, ib, nib, ob, nob) in enumerate(T.filter_coverage(mods)):
            assert taps == c.k * c.k and ib == nib and ob == nob, (c.id, i, taps, ib, nib, ob, nob)
        for k, v in T.nonrep_shares(T.replay(c, mods, xs, res, gout)).items():
            best[k] = max(best.get(k, 0.0), v)
    print(f"\n{family}: best bf16-unrepresentable share per rounding point: " + ", ".join(f"{k} {v:.2f}" for k, v in best.items()))
    for k, v in best.items():
        if family == "stack" and k == "[df | dm]":
            continue
        assert v >= T.ROUND_FLOOR, (family, k, v)


@functools.lru_cache(maxsize=None)
def _bounded(case):
    return T.bounded_operands(case)


@pytest.mark.parametrize("mode", T.BOUNDED_MODES)
@pytest.mark.parametrize("case", T.BOUNDED_CASES, ids=lambda c: c.id)
def test_bounded_tier_sees_one_pixel_and_one_item(case, mode):
    """Each bounded-tier bound is at most a quarter of the change some element sees when one pixel is dropped, doubled or read
    from its neighbour, or (per item) item 0 is normalised with item 1's statistics.  A one-ulp change of one bf16 output-gradient
    element is printed, not required: it moves [df | dm] by about its own rounding, which a bound that admits bf16's half ulp
    cannot resolve in every case (the exact tier holds those)."""
    mods, xs, res, gout = _bounded(case)
    r = T.defect_ratios(case, mods, xs, res, gout, mode)
    print(f"\n{case.id} {mode}: change / bound " + ", ".join(f"{k} {v:.3g}" for k, v in r.items()))
    for k, v in r.items():
        if k != "one-ulp output gradient":
            assert v >= T.DEFECT_MARGIN, (case.id, mode, k, v)


@pytest.mark.parametrize("case", T.BOUNDED_CASES, ids=lambda c: c.id)
def test_bounded_operands_reach_the_hard_gate_regions(case):
    """The bounded tier's operands reach what the exact tier pins away: saturated and cancelling gates (|m + b_m| >= 10), m
    filters that matter, and (on an ELU conv) ELU's negative branch."""
    mods, xs, res, gout = _bounded(case)
    x, accf, accm, A, g = T._gated(case, mods[0], xs)
    p = T.params64(mods[0])
    m = accm + p["bm"][:, None, None]
    f = accf + p["bf"][:, None, None]
    assert bool((m.abs() >= 10).any()) and bool((m.abs() < 3).any()), case.id
    assert bool((p["wm"] != 0).any()), case.id
    if case.elu:
        assert bool((f < -1).any()), case.id
