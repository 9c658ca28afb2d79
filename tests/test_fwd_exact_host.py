"""Without a GPU: the references of test_gpu_fwd_exact.py agree with torch, every case keeps its partial sums exact in fp32,
the RAW cases need bf16 rounding often enough, the checks reject the defects a kernel could have, and the case lists cover the
kernels' edge classes and every layer class the engine plans."""
import zlib

import pytest
import torch
import torch.nn.functional as F

import bwd_exact_util as U
import fwd_exact_util as X


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _rejects(check, *args, **kw):
    with pytest.raises(AssertionError) as e:
        check(*args, **kw)
    print(f"\nrejected: {str(e.value)[:200]}")


# ------------------------------------------------------------------ references
@pytest.mark.parametrize("f", [2, 4, 8])
def test_nearest_matches_f_interpolate(f):
    x = U.int_tensor((2, 3, 8 * 3, 8 * 5), 9, _gen("nearest", f)).double()
    assert torch.equal(X.nearest(x, "down", f), F.interpolate(x, scale_factor=1.0 / f))
    assert torch.equal(X.nearest(x, "up", f), F.interpolate(x, scale_factor=f))


@pytest.mark.parametrize("h", X.BIL_HW)
@pytest.mark.parametrize("w", X.BIL_HW)
def test_bilinear4_of_small_integers_is_dyadic_and_exact_in_bf16(h, w):
    """align_corners=False x4: the taps are multiples of 1/8, so blends of integers |x| <= 3 are multiples of 1/64 below 3, exact
    in bf16 (and in fp32, whatever the order of the kernel's lerps)."""
    x = U.int_tensor((2, 4, h, w), X.A_BIL, _gen("bil", h, w), zero_frac=0.0)
    y = X.bilinear4(x)
    assert torch.equal(y * 64, (y * 64).round()), "not a multiple of 1/64"
    assert float(y.abs().max()) <= X.A_BIL
    assert torch.equal(y.float().bfloat16().double(), y), "not exact in bf16"
    # the separable form of read_upsample_bilinear4 (vertical then horizontal lerp, fp32) gives the same values
    yv = F.interpolate(x.float(), size=(4 * h, w), mode="bilinear", align_corners=False)
    assert torch.equal(F.interpolate(yv, size=(4 * h, 4 * w), mode="bilinear", align_corners=False).double(), y)


def test_pinned_gate_emulation_matches_an_fp32_epilogue():
    """ref()'s gate-pinned values are what an fp32 epilogue computes: fmaf(f * 1.0, scale, shift) + residual, then bf16."""
    c = X.Case("emulation", "tma", ((32, "id", 1),), 32, 3, 1, 2, 9, 7, residual=True)
    o = X.make(c, _gen("emu"))
    r = X.ref(c, o)
    F_ = (o["accf"] + o["bf"].double()).float()
    sig = torch.sigmoid(torch.full_like(F_, X.PIN_BIAS_M))
    assert bool((sig == 1.0).all())
    y = torch.addcmul(o["shift"].expand_as(F_), F_ * sig, o["scale"].expand_as(F_))     # one rounding: exact products here
    y = (y.double() + o["res"].double()).float().bfloat16().double()
    p = o["pinned"].expand_as(F_)
    assert torch.equal(y[p], r["y_pin"][p])


# ------------------------------------------------------------------ exactness precondition and test strength
def test_every_case_keeps_its_partial_sums_below_2_24():
    worst = {}
    for c in X.EXACT_CASES:
        m = X.precondition(c)
        worst[c.impl] = max(worst.get(c.impl, 0), m)
        if c.addin:
            assert c.cout <= 64, c.id                                  # the add-in is in concat order only for one n-tile
    print("\nworst-case partial sums (units):", {k: f"{v} (2^{v.bit_length() - 1})" for k, v in worst.items()})


def test_precondition_refuses_a_case_beyond_2_24(monkeypatch):
    monkeypatch.setattr(X, "AW", 256)
    monkeypatch.setattr(X, "A", 256)
    _rejects(X.precondition, X.Case("too wide", "tma", ((256, "id", 1),), 128, 4, 2, 1, 4, 4))


@pytest.mark.parametrize("case", [c for c in X.EXACT_CASES if c.out == "raw"], ids=lambda c: c.id)
def test_raw_cases_need_rounding_often(case):
    o = X.make(case, _gen(case))
    frac = U.bf16_nonrepresentable_fraction(X.ref(case, o)["raw"] / o["unit"])
    print(f"\n{case.id}: s = {o['s']}, {frac:.2f} of the exact sums are not bf16 values")
    assert frac >= 0.1


@pytest.mark.parametrize("case", [c for c in X.EXACT_CASES if c.out != "raw"][::4], ids=lambda c: c.id)
def test_gated_cases_pin_half_the_channels_and_spread_the_gate(case):
    o = X.make(case, _gen(case))
    r = X.ref(case, o)
    m = (o["accm"] + o["bm"].double())[..., ~o["pinned"]]
    print(f"\n{case.id}: s = {o['s']}, exact share {float(r['exact'].double().mean()):.2f}, |m| median {float(m.abs().median()):.2f}")
    assert float(r["exact"].double().mean()) >= 0.2
    assert bool((torch.sigmoid(m) > 0.05).any() and (torch.sigmoid(m) < 0.95).any()), "the ordinary gates all saturate"


# ------------------------------------------------------------------ the checks reject a defective kernel
def _raw_case():
    c = X.Case("mut", "tma", ((128, "id", 1),), 32, 3, 1, 2, 17, 9, out="raw")
    o = X.make(c, _gen("mut"))
    return c, o, X.ref(c, o)


def test_raw_check_rejects_a_skipped_last_k_chunk():
    c, o, r = _raw_case()
    U.assert_bf16_rn(r["raw_rn"], r["raw"], "unmodified")
    x = o["srcs"][0].clone()
    x[..., 64:] = 0                                                 # the last 64-channel K chunk never accumulated
    xd = x.double().permute(0, 3, 1, 2)
    bad = U.to_raw(torch.cat([F.conv2d(xd, w.double(), padding=1) for w in (o["wf"], o["wm"])], 1).permute(0, 2, 3, 1))
    _rejects(U.assert_bf16_rn, bad.float().bfloat16(), r["raw"], "skipped chunk")


def test_raw_check_rejects_truncation():
    c, o, r = _raw_case()
    trunc = (r["raw"].float().view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
    _rejects(U.assert_bf16_rn, trunc, r["raw"], "truncation")


def test_gated_checks_reject_swapped_channels_and_a_dropped_residual_row():
    c = X.Case("mut", "tma", ((32, "id", 1),), 32, 3, 1, 2, 17, 9, residual=True)
    o = X.make(c, _gen("mut gated"))
    r = X.ref(c, o)
    good = r["y_pin"].clone()
    good[~r["exact"]] = r["y64"][~r["exact"]].float().bfloat16().double()
    b = X.bound(c, o, r, X.TAU_FAST)
    U.assert_exact(good[r["exact"]], r["y_pin"][r["exact"]], "unmodified")
    U.assert_bound(good[~r["exact"]], r["y64"][~r["exact"]], b[~r["exact"]], 1.0, "unmodified")
    swap = good.clone()
    swap[..., [4, 5]] = good[..., [5, 4]]                           # one epilogue channel pair exchanged
    _rejects(U.assert_exact, swap[r["exact"]], r["y_pin"][r["exact"]], "swap")
    norow = good.clone()
    norow[:, -1] = (good[:, -1] - r["res"][:, -1]).float().bfloat16().double()     # the residual of the last row missing
    _rejects(U.assert_exact, norow[r["exact"]], r["y_pin"][r["exact"]], "residual row")
    ulps = good.float().bfloat16()
    e = (~r["exact"]).nonzero()[0].tolist()
    bits = ulps.view(torch.int16)
    bits[tuple(e)] += 3                                             # an ordinary channel three bf16 ulps off
    _rejects(U.assert_bound, ulps.double()[~r["exact"]], r["y64"][~r["exact"]], b[~r["exact"]], 1.0, "3 ulp")


# ------------------------------------------------------------------ coverage
def test_tma_cases_cover_every_edge_class():
    cls = set().union(*(X.tma_classes(c) for c in X.TMA_CASES))
    print(f"\nTMA kernel: {sorted(cls)}")
    need = {"K chunk 16", "K chunk 32", "K chunk 64", "1 n-tiles", "2 n-tiles", "resident weights", "streamed weights",
            "resident weights of exactly 144 KB", "1 CTAs per SM", "2 CTAs per SM", "several K chunks", "B==1", "B==3"}
    need |= {f"W%8=={w % 8}" for w in (1, 7, 8, 9, 17)} | {f"H%16=={h % 16}" for h in (1, 15, 16, 17, 33)}
    assert need <= cls, sorted(need - cls)
    outs = {c.wout for c in X.TMA_CASES} | {c.hout for c in X.TMA_CASES}
    assert {1, 7, 8, 9, 17} <= {c.wout for c in X.TMA_CASES} and {1, 15, 16, 17, 33} <= {c.hout for c in X.TMA_CASES}, outs
    geo = {(c.k, c.stride, c.out, len(c.srcs) > 1, c.residual, c.addin) for c in X.TMA_CASES}
    for g in [(3, 1, "raw", False, True, False), (3, 1, "raw", False, False, False), (3, 2, "raw", False, False, False),
              (4, 2, "raw", False, False, False), (1, 1, "raw", True, False, True), (1, 1, "raw", True, False, False),
              (1, 1, "nhwc", True, False, True), (3, 1, "nhwc", False, True, False), (3, 1, "nchw", False, False, False)]:
        assert g in geo, g
    assert {16, 32, 64} <= {c.cout for c in X.TMA_CASES if c.out == "raw" and c.k == 1}
    assert {2, 4, 8} <= {f for c in X.TMA_CASES for _, m, f in c.srcs if m == "down"}
    assert {8, 16, 32, 64, 128, 256} <= {c.cin for c in X.TMA_CASES}
    assert {16, 32, 64, 128, 256} <= {c.cout for c in X.TMA_CASES}
    assert all(c.H == 2 * c.hout and c.W == 2 * c.wout for c in X.TMA_CASES if c.stride == 2)


def test_gather_and_generic_cases_cover_their_edges():
    g = X.GATHER_CASES
    modes = {(m, f) for c in g for _, m, f in c.srcs}
    assert {("up", 2), ("up", 4), ("up", 8), ("down", 2), ("down", 4), ("bil4", 4)} <= modes, modes
    assert any(c.stride == 2 and c.H % 2 and c.W % 2 for c in g), "stride 2 on odd shapes"
    assert any(c.cout == 248 for c in g) and any(c.out == "nchw" for c in g)
    assert any(c.residual and c.out2 for c in g)
    assert 480 in {c.cin for c in g}
    assert {c.wout % X.G_TW for c in g} >= {1, 4, 9} and {c.hout % X.G_TH for c in g} >= {0, 1, 7}
    gen = X.GENERIC_CASES
    assert {"bf16", "f32"} == {c.act for c in gen}
    assert any(c.mul for c in gen if c.act == "bf16") and any(c.mul for c in gen if c.act == "f32")


def test_every_engine_layer_class_has_an_exact_case():
    covered = {X.case_class(c) for c in X.EXACT_CASES}
    for key, census in X.ENGINE_CENSUS.items():
        print(f"\n{key}: {len(census)} classes")
        assert census <= covered, (key, sorted(census - covered))
    assert len({c.id for c in X.EXACT_CASES}) == len(X.EXACT_CASES), "case ids must be unique"
