"""Without a GPU: the census of tests/vgg_exact_util.py is current and every class in it has an exact case, every case keeps its
partial sums exact in fp32, the float32 replays of csrc/vgg.cu agree with torch's own operators where torch has the same one,
and the checks of test_gpu_vgg_exact.py reject the defects a kernel could have."""
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import bwd_exact_util as U
import fwd_exact_util as X
import vgg_exact_util as E
from read_b200 import vgg_loss as V


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _rejects(check, *args, **kw):
    with pytest.raises(AssertionError) as e:
        check(*args, **kw)
    print(f"\nrejected: {str(e.value)[:200]}")


# ------------------------------------------------------------------ census and coverage
def test_census_is_current():
    d = E.derived_census()
    assert d["walks"] == E.WALKS, "vgg_loss's layer walks changed: update WALKS, the classes and their exact cases"
    assert d["fwd"] == E.FWD_CLASSES, sorted(d["fwd"] ^ E.FWD_CLASSES)
    assert d["dgrad"] == E.DGRAD_CLASSES, sorted(d["dgrad"] ^ E.DGRAD_CLASSES)
    assert d["cin8"] == E.CIN8_CS
    assert d["split"] == E.SPLIT_BLOCKS, d["split"]


def test_every_census_class_has_exact_cases():
    fwd = {(c.cin, c.cout) for c in E.VGG_FWD_CASES}
    assert fwd == E.FWD_CLASSES, sorted(fwd ^ E.FWD_CLASSES)
    dg = {E.dgrad_class(c) for c in E.VGG_DGRAD_CASES}
    assert dg == E.DGRAD_CLASSES, sorted(dg ^ E.DGRAD_CLASSES)
    assert all(c.out == "raw" and not c.residual and c.k == 3 and c.stride == 1 and c.impl == "tma" for c in E.VGG_FWD_CASES)
    assert len({c.id for c in E.VGG_FWD_CASES}) == len(E.VGG_FWD_CASES), "case ids must be unique"
    assert len(set(E.VGG_DGRAD_CASES)) == len(E.VGG_DGRAD_CASES)


def test_cases_reach_the_edges_and_the_training_sizes():
    # forward: ragged tiles, H = 1 and W = 1, even batches (the loss runs 2n images), every class at its 256^2-crop size
    fwd = E.VGG_FWD_CASES
    assert all(c.B % 2 == 0 for c in fwd)
    assert any(c.H == 1 for c in fwd) and any(c.W == 1 for c in fwd)
    assert {c.W % X.TC_TW for c in fwd} >= {1, 7} and {c.H % X.TC_TH for c in fwd} >= {1, 15}
    crop = {(64, 32): 256, (8, 32): 256, (64, 64): 128, (128, 64): 128, (128, 128): 64, (256, 128): 64, (256, 256): 32,
            (512, 256): 32}
    for (cin, cout), hw in crop.items():
        assert any((c.cin, c.cout, c.H, c.W) == (cin, cout, hw, hw) for c in fwd), (cin, cout, hw)
    assert any((c.cin, c.H, c.W) == (512, 16, 16) for c in fwd), "conv5_x at 16 x 16"
    # input gradient: every class at H and W of 1, a multiple of the tile and a ragged size, and at its crop size
    for cls in E.DGRAD_CLASSES:
        cs = [c for c in E.VGG_DGRAD_CASES if E.dgrad_class(c) == cls]
        hs, ws = {c[3] for c in cs}, {c[4] for c in cs}
        assert 1 in hs | ws and any(h % 8 == 0 for h in hs | ws) and any(h % 8 for h in hs | ws if h > 1), (cls, hs, ws)
        assert any(c[3] >= 16 and c[3] == c[4] for c in cs), cls


def test_64_to_64_raw_plan_streams_its_weights():
    """conv2_1 (64 -> 2 x 64 RAW): its packed weights are exactly the 144 KB resident limit, but with the RAW epilogue ring (two
    stages of 128 pixels x 128 bf16 columns) and two halo stages they need 254 KB of the 224 KB a CTA may have: tc_plan_create's
    rule streams them through the B ring, one CTA per SM."""
    for c in E.VGG_FWD_CASES:
        cin_blk, kchunks, n_tile, n_tiles, total_b, resident, ctas = X.tma_geom(c)
        if (c.cin, c.cout) == (64, 64):
            assert (cin_blk, kchunks, n_tile, n_tiles, total_b) == (64, 1, 128, 1, X.TC_RESIDENT_MAX)
            assert not resident and ctas == 1
        if c.cin == 512:
            assert (n_tiles, kchunks, resident) == (4, 8, False), "conv4_x / conv5_x: four n-tiles, eight K chunks, streamed"


# ------------------------------------------------------------------ exactness preconditions and test strength
def test_every_case_keeps_its_partial_sums_below_2_24():
    worst = max(X.precondition(c) for c in E.VGG_FWD_CASES)
    worst_dg = max(E.dgrad_max_partial(c) for c in E.VGG_DGRAD_CASES)
    worst_path = max(E.path_max_partial(max(s.cin, 8)) for s in V.layer_walk(V.LAYERS_OPTIMIZED))
    print(f"\nworst partial sums (units): forward {worst}, input gradient {worst_dg}, VGG path {worst_path}")
    assert worst_dg < U.EXACT_LIMIT and worst_path < U.EXACT_LIMIT


@pytest.mark.parametrize("case", [c for c in E.VGG_FWD_CASES if c.H * c.W <= 64 * 64], ids=lambda c: c.id)
def test_forward_cases_need_rounding_often(case):
    o = X.make(case, _gen(case))
    frac = U.bf16_nonrepresentable_fraction(X.ref(case, o)["raw"] / o["unit"])
    print(f"\n{case.id}: {frac:.2f} of the exact sums are not bf16 values")
    assert frac >= 0.1


def test_glue_operands_need_rounding_and_reach_every_code():
    g = _gen("glue operands")
    n, H, W, C = 2, 9, 7, 64
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    y = E.post_values(raw, bias, n)
    assert U.bf16_nonrepresentable_fraction(y) >= 0.1
    assert U.bf16_nonrepresentable_fraction(E.pool_replay(y)) >= 0.1
    codes = E.post_codes(y, n, True)
    assert set(codes.unique().tolist()) == {0, 1, 2, 3}
    # the loss term: integer |d|, so the kernel's fp32 per-thread sums and its double combines are all exact
    assert torch.equal(y, y.round())
    assert E.term_sum(y, n, False) == E.term_exact_sum(y, n)
    mask = E.glue_mask(n, H, W, g, "holes")
    yp = E.post_values(raw, bias, n, mask)
    diff = E.post_values(raw, bias, n, mask, fused=False) != yp
    print(f"\npartial post: the fused and the unfused raw * ratio + bias differ on {int(diff.sum())} of {diff.numel()} elements")
    assert bool(diff.any()), "the partial operands do not tell the fused rounding from the unfused one"


# ------------------------------------------------------------------ the replays agree with torch
def test_post_replay_matches_relu_and_avg_pool():
    g = _gen("relu pool")
    n, H, W, C = 2, 9, 7, 64
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    y = E.post_values(raw, bias, n)
    assert torch.equal(y, F.relu(raw.float() + bias))
    # AvgPool2d(2, 2) on exactly representable data (integer sums below 2^24, then a quarter): the same values, odd rows and
    # columns dropped
    want = F.avg_pool2d(y.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(E.pool_replay(y), want)


def test_ratio_is_reciprocal_times_nine():
    c = torch.arange(0, 10)
    r = E.vg_ratio(c)
    assert r[0] == 0
    for k in range(1, 10):
        assert r[k].item() == (torch.tensor(1.0) / torch.tensor(float(k)) * torch.tensor(9.0)).item()
    correctly_rounded = torch.tensor([9.0 / k for k in range(1, 10)], dtype=torch.float64).float()
    differ = [k for k in range(1, 10) if r[k] != correctly_rounded[k - 1]]
    assert differ == [5, 7], differ


def test_partial_replay_matches_partial_conv2d():
    """The unfused replay of vgg_post_partial is vgg_loss.PartialConv2d's fp32 arithmetic: a partial conv whose conv is the
    identity (centre tap 1) over the RAW values, masked as the kernel's input is, then ReLU."""
    g = _gen("partial conv")
    n, H, W, C = 2, 9, 7, 16
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    for kind in ("holes", "valid", "invalid"):
        mask = E.glue_mask(n, H, W, g, kind)
        m = torch.cat([mask, mask])[:, None].float()
        conv = nn.Conv2d(C, C, 3, padding=1)
        with torch.no_grad():
            conv.weight.zero_()
            conv.weight[torch.arange(C), torch.arange(C), 1, 1] = 1.0
            conv.bias.copy_(bias)
        pc = V.PartialConv2d.from_conv(conv)
        raw_m = (raw.float() * m.permute(0, 2, 3, 1)).bfloat16()            # the conv output of the masked input
        want = F.relu(pc(raw_m.float().permute(0, 3, 1, 2), m)).permute(0, 2, 3, 1)
        got = E.post_values(raw_m, bias, n, mask, fused=False)
        assert torch.equal(got, want), kind


# ------------------------------------------------------------------ the checks reject a defective kernel
def _post_case():
    g = _gen("defects")
    n, H, W, C = 2, 9, 7, 64
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    return n, H, W, C, raw, bias, E.post_values(raw, bias, n)


def test_checks_reject_a_truncated_bf16_store():
    n, H, W, C, raw, bias, y = _post_case()
    want = E.post_out(y, False)
    E.assert_same_bits(want, want, "unmodified")
    trunc = (y.view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
    _rejects(E.assert_same_bits, trunc, want, "truncated store")


def test_checks_reject_a_pool_that_keeps_the_odd_row():
    n, H, W, C, raw, bias, y = _post_case()
    want = E.post_out(y, True)
    keeps = E.post_out(y[:, 1:], True)                               # rows (1, 2), (3, 4), ..., (7, 8): row 8 kept, row 0 lost
    assert keeps.shape == want.shape
    _rejects(E.assert_same_bits, keeps, want, "pool keeping the odd row")


def test_checks_reject_a_flipped_code_sign():
    n, H, W, C, raw, bias, y = _post_case()
    want = E.post_codes(y, n, True)
    flipped = torch.where(want != 0, 4 - want, want)
    _rejects(E.assert_same_bits, flipped, want, "code sign flipped")


def test_checks_reject_an_input_gradient_with_two_channels_swapped():
    g = _gen("swap")
    dy = U.int_tensor((2, 9, 7, 64), E.PATH_AMP, g)
    w = U.int_tensor((64, 32, 3, 3), E.PATH_AMP, g)
    want = E.conv_input_grad_ref(dy, w)
    got = want.float().bfloat16()
    U.assert_bf16_rn(got, want, "unmodified")
    _rejects(U.assert_bf16_rn, got[..., [1, 0] + list(range(2, 32))], want, "channels 0 and 1 swapped")


def test_checks_reject_a_write_past_the_pooled_output():
    n, H, W, C, raw, bias, y = _post_case()
    want = E.post_out(y, True)
    out = U.Guarded(want.numel(), torch.bfloat16, "cpu")
    out.out.copy_(want.reshape(-1))
    out.check("unmodified")
    out.buf[out.guard + out.n] = want.reshape(-1)[-1]                 # one element past the end
    _rejects(out.check, "write past the pooled output")


def test_checks_reject_a_term_off_by_the_unfused_rounding():
    """The term check is an equality: prefill + s * scale rounded twice instead of once is caught where the two differ."""
    prefill, scale = 1.0 / 3.0, 1.0 / (2 * 64 * 9 * 7)
    s = next(v for v in range(1, 10 ** 6) if prefill + v * scale != E.fused_term(prefill, float(v), scale))
    E.assert_term(E.fused_term(prefill, float(s), scale), E.fused_term(prefill, float(s), scale), "unmodified")
    _rejects(E.assert_term, prefill + s * scale, E.fused_term(prefill, float(s), scale), "unfused term")
