"""Host checks (no GPU) of bn_fwd_exact_util, the checkers of test_gpu_bn_fwd_exact.py: every case's integer sums exact in fp32, the
case lists reach every partition edge, each statistics bound is at most a quarter of the change one dropped, doubled or
neighbouring item's pixel or a P - 1 divisor makes, an emulation of the kernel's arithmetic passes the bounds while the same
emulation with a planted defect fails them, and the apply replay tells a contracted FMA apart on at least 10 % of the elements."""
import numpy as np
import pytest
import torch

import bn_fwd_exact_util as B
from bwd_exact_util import assert_exact

SMS_LIST = (132, 114, 66)                   # H100 SXM, H100 PCIe, and a small part (cap < 512 on all three)


def _emulate(x, sms, gamma, beta, n_real, drop_last_strided=False):
    """The kernel's statistics arithmetic on the host: fp32 thread sums relative to K, rn, d and the fused M2 as bn_stats_body
    has them, then a float64 combine.  drop_last_strided: every thread with two or more pixels skips its last one."""
    items, P, C = x.shape
    grid, b = B.stats_grid(P, C, sms), B.ppb(C)
    K, n, a1, a2 = B.thread_sums(x, grid, b)
    if drop_last_strided:
        S = grid * b
        T = K.shape[1]
        last = ((n - 1) * S + np.arange(T))
        drop = n >= 2
        xl = x[:, last] - K
        a1 = a1 - np.where(drop[None, :, None], xl, 0)
        a2 = a2 - np.where(drop[None, :, None], xl.astype(np.int64) ** 2, 0)
        n = n - drop
    rn = B.f32(1.0 / n.astype(np.float32))[None, :, None]
    d = B.f32(a1.astype(np.float32) * rn)
    m2 = np.maximum(B.fma32(-a1.astype(np.float32), d, a2.astype(np.float32)), 0).astype(np.float64)
    nn = n[None, :, None].astype(np.float64)
    mt = K + d.astype(np.float64)
    mu = (nn * mt).sum(1) / P
    v = (m2 + nn * (mt - mu[:, None]) ** 2).sum(1) / P
    inv = 1.0 / np.sqrt(v + float(np.float32(B.EPS)))
    gm = np.zeros(C); gm[:n_real] = gamma
    bt = np.zeros(C); bt[:n_real] = beta
    sc = gm * inv
    return {"mean": B.f32(mu), "var": B.f32(v), "uvar": B.f32(v * P / (P - 1)), "inv_std": B.f32(inv), "scale": B.f32(sc),
            "shift": B.f32(np.where(np.arange(C) < n_real, bt - mu * sc, 0.0))}


@pytest.mark.parametrize("sms", SMS_LIST)
def test_every_case_sums_exactly_in_fp32(sms):
    for case in B.stats_cases(sms):
        x = B.stats_operands(case)[0]
        assert np.abs(x).max() <= 256 and np.abs(x[:, :, case.n_real:]).max(initial=0) == 0, case
        a2, a1 = B.sums_precondition(case, x, sms)
        assert a2 < B.EXACT_LIMIT and a1 < B.EXACT_LIMIT, (case, a2, a1)


@pytest.mark.parametrize("sms", SMS_LIST)
def test_case_lists_reach_every_edge(sms):
    seen = set().union(*(B.stats_classes(c, sms) for c in B.stats_cases(sms)))
    missing = B.required_classes(sms) - seen
    assert not missing, missing
    for C in B.BN_CS:                                   # each C at each pixel-count edge
        per_c = set().union(*(B.stats_classes(c, sms) for c in B.stats_cases(sms) if c.C == C))
        assert {"P=2", "P=3", "P=ppb-1", "P=ppb", "P=ppb+1", "blocks=cap-1", "blocks=cap", "blocks=cap+1"} <= per_c, C
    seen_a = set().union(*(B.apply_classes(c, sms) for c in B.apply_cases(sms)))
    assert {f"C={C}" for C in B.BN_CS} | {"grid-stride", "cap<1", "per item", "one item"} <= seen_a


def test_padded_channel_and_special_channels():
    case = B.Case(True, 3, 500, 64, 56, seed=7)
    x = B.stats_operands(case)[0]
    mu, v, _ = B.exact_stats(x)
    assert (v[:, 0] == 0).all() and (mu[:, 56:] == 0).all() and (v[:, 56:] == 0).all()
    assert (np.abs(mu[:, 1]) > 190).all() and (v[:, 1] <= 1).all()         # a mean far above its spread
    assert (v[:, 2:56] == 0).any() and (v[:, 2:56] > 100).any()


@pytest.mark.parametrize("sms", [132])
def test_bounds_are_a_quarter_of_every_planted_defect(sms):
    for case in B.stats_cases(sms):
        x, gamma, beta, _, _ = B.stats_operands(case)
        bnd = B.stats_bounds(x, sms, gamma, beta, case.n_real)
        ratios = B.defect_ratios(x, bnd, gamma, case.n_real)
        assert set(ratios) >= {"drop", "double", "p-1"} and ("neighbour" in ratios) == (case.items > 1), case
        assert min(ratios.values()) >= B.DEFECT_MARGIN, (case, ratios)


@pytest.mark.parametrize("case", [B.Case(False, 1, 3 * 264 * 128 + 999, 16, 3, seed=1), B.Case(True, 3, 1000, 64, 56, seed=2),
                                  B.Case(True, 2, 2 * 264 * 8 + 3, 256, 248, seed=3), B.Case(False, 1, 23, 192, seed=4)],
                         ids=lambda c: c.id)
def test_emulated_kernel_passes_and_each_defect_fails(case):
    sms = 132
    x, gamma, beta, _, _ = B.stats_operands(case)
    bnd = B.stats_bounds(x, sms, gamma, beta, case.n_real)
    keys = ["mean", "var", "uvar", "inv_std", "scale", "shift"]
    got = _emulate(x, sms, gamma, beta, case.n_real)
    worst = B.check_stats(got, bnd, "emulated", keys)
    assert max(worst.values()) <= 1.0
    P = case.P
    planted = {"drop": x[:, :-1], "double": np.concatenate([x, x[:, -1:]], 1)}
    if case.items > 1:
        y = x.copy(); y[0, -1] = x[1, -1]
        planted["neighbour"] = y
    for name, y in planted.items():
        with pytest.raises(AssertionError):
            B.check_stats(_emulate(y, sms, gamma, beta, case.n_real), bnd, name, keys)
    bad = dict(got, var=B.f32(got["var"].astype(np.float64) * P / (P - 1)))
    with pytest.raises(AssertionError):
        B.check_stats(bad, bnd, "P - 1", ["var"])
    if B.cdiv(P, B.stats_grid(P, case.C, sms) * B.ppb(case.C)) >= 2:
        with pytest.raises(AssertionError):
            B.check_stats(_emulate(x, sms, gamma, beta, case.n_real, drop_last_strided=True), bnd, "last strided", keys)


def test_running_replay_rejects_reverse_item_order():
    rng = np.random.default_rng(3)
    mean, uvar = B.f32(rng.standard_normal((5, 40)) * 50), B.f32(rng.random((5, 40)) * 900)
    rm, rv = B.f32(rng.standard_normal(40)), B.f32(rng.random(40) + 0.5)
    fwd = B.running_items_replay(rm, rv, mean, uvar, 0.1)
    rev = B.running_items_replay(rm, rv, mean[::-1], uvar[::-1], 0.1)
    assert (fwd[0] != rev[0]).any() and (fwd[1] != rev[1]).any()
    # momentum 0 keeps, 1 takes the last item's value
    assert (B.running_items_replay(rm, rv, mean, uvar, 0.0)[0] == rm).all()
    assert (B.running_items_replay(rm, rv, mean, uvar, 1.0)[1] == uvar[-1]).all()
    # the call-wide form is the one-item case; its candidates bracket the single-rounding value
    c = B.running_call_candidates(rv, uvar[0].astype(np.float64) * 9 / 10, 10, 0.1)
    assert (c[0] <= c[1]).all() and (c[1] <= c[2]).all()


def test_fma32_is_single_rounding():
    a, b, c = B.f32([3.0, 1 + 2 ** -23]), B.f32([1 / 3, 1 - 2 ** -23]), B.f32([-1.0, -1.0])
    want = [float(B.round32(B.Fraction(float(x)) * B.Fraction(float(y)) + B.Fraction(float(z)))) for x, y, z in zip(a, b, c)]
    assert B.fma32(a, b, c).tolist() == want
    assert B.fma32(a, b, c)[1] == np.float32(-2.0 ** -46) and (a * b + c)[1] == 0     # the fused form keeps what fl() loses


@pytest.mark.parametrize("i", range(len(B.apply_cases(132))))
def test_apply_operands_expose_a_contracted_fma(i):
    items, P, C = B.apply_cases(132)[i]
    for k, residual in enumerate((False, True)):
        g, scale, shift, r = B.apply_operands(items, P, C, residual, seed=i * 2 + k)
        assert np.abs(g).max() <= 256 and (r is None or np.abs(r).max() <= 256)
        want = B.apply_replay(g, scale, shift, r)
        fused = B.apply_replay(g, scale, shift, r, fused=True)
        share = float((want != fused).mean())
        assert share >= 0.10, (items, P, C, residual, share)
        with pytest.raises(AssertionError):
            assert_exact(torch.from_numpy(fused), torch.from_numpy(want), "contracted apply")
        # each item its own scale / shift row: the first item's row applied to every item changes the result
        if items > 1:
            one = B.apply_replay(g, np.repeat(scale[:1], items, 0), np.repeat(shift[:1], items, 0), r)
            assert (one != want).any()


def test_bf16_bits_round_to_nearest_even():
    v = B.f32([1.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8, 1 + 2 ** -8 + 2 ** -20, -2.5, 3.0e-39])
    got = B.bf16_bits(v)
    want = torch.from_numpy(v).bfloat16().view(torch.int16).numpy()
    assert (got == want).all()
