"""-m gpu: fused gated-conv kernels vs a plain PyTorch fp32 reference of the same op (BasicConv, unet.py:22-53)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import _lib as L

pytestmark = pytest.mark.gpu


def ref_gated(x, wf, bf, wm, bm, scale, shift, k, stride, elu, residual=None):
    p = int((k - 1) / 2)
    f = F.conv2d(x, wf, bf, stride=stride, padding=p)
    if elu:
        f = F.elu(f)
    y = f * torch.sigmoid(F.conv2d(x, wm, bm, stride=stride, padding=p))
    y = y * scale[None, :, None, None] + shift[None, :, None, None]
    return y if residual is None else y + residual


def resample(t, mode, f):
    if mode == "id":
        return t
    if mode == "down":
        return F.interpolate(t, scale_factor=1.0 / f)
    if mode == "up":
        return F.interpolate(t, scale_factor=f)
    return F.interpolate(t, scale_factor=4, mode="bilinear", align_corners=False)


def run_conv(srcs, cout, k, stride, elu, act_bf16, impl, residual=False, out2=False, final=False, mul=False, seed=0,
             reversed_order=False):
    """srcs: list of (C, h, w, mode, factor) describing NCHW fp32 source tensors.  Returns (got, want[, got2, want2])."""
    lib = L.load()
    d = dev()
    g = torch.Generator().manual_seed(seed)
    adt = torch.bfloat16 if act_bf16 else torch.float32
    B = 2
    xs = [torch.rand((B, c, h, w), generator=g) * 2 - 1 for (c, h, w, _, _) in srcs]
    if act_bf16:
        xs = [x.to(torch.bfloat16).float() for x in xs]
    logical = torch.cat([resample(x, m, f) for x, (_, _, _, m, f) in zip(xs, srcs)], 1)
    cin, hin, win = logical.shape[1:]
    bound = 1.0 / (cin * k * k) ** 0.5
    wf = (torch.rand((cout, cin, k, k), generator=g) * 2 - 1) * bound
    wm = (torch.rand((cout, cin, k, k), generator=g) * 2 - 1) * bound
    bf = (torch.rand(cout, generator=g) * 2 - 1) * bound
    bm = (torch.rand(cout, generator=g) * 2 - 1) * bound
    scale = torch.rand(cout, generator=g) + 0.5
    shift = torch.randn(cout, generator=g) * 0.1
    pad = int((k - 1) / 2)
    hout, wout = (hin + 2 * pad - k) // stride + 1, (win + 2 * pad - k) // stride + 1
    res = m2 = mulx = None
    if residual:
        res = torch.rand((B, cout, hout, wout), generator=g)
        res = res.to(adt).float()
    if out2:
        m2 = torch.rand((B, cout, hout, wout), generator=g).to(adt).float()
    if mul:
        mulx = torch.rand((B, cin, hin, win), generator=g).to(adt).float()
    tc = impl in (L.CONV_TCGEN05, L.CONV_TCGEN05_GATHER)
    wf_r, wm_r = (wf.to(torch.bfloat16).float(), wm.to(torch.bfloat16).float()) if tc else (wf, wm)
    want = ref_gated(logical * mulx if mul else logical, wf_r, bf, wm_r, bm, scale, shift, k, stride, elu, res)

    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(d, adt)
    dsc = L.ReadConvDesc()
    dsc.act_dtype = L.ACT_BF16 if act_bf16 else L.ACT_F32
    dsc.n_src = len(srcs)
    keep = []
    modes = {"id": L.SRC_IDENTITY, "down": L.SRC_NEAREST_DOWN, "up": L.SRC_NEAREST_UP, "bil4": L.SRC_BILINEAR_UP4}
    for i, (x, (c, h, w, m, f)) in enumerate(zip(xs, srcs)):
        t = nhwc(x)
        keep.append(t)
        dsc.src[i].ptr, dsc.src[i].C, dsc.src[i].H, dsc.src[i].W = t.data_ptr(), c, h, w
        dsc.src[i].mode, dsc.src[i].factor = modes[m], f
    dsc.B, dsc.Hin, dsc.Win, dsc.Cin = B, hin, win, cin
    dsc.Hout, dsc.Wout, dsc.Cout = hout, wout, cout
    dsc.k, dsc.stride, dsc.pad, dsc.elu = k, stride, pad, int(elu)
    dv = [t.to(d).contiguous() for t in (wf, wm, bf, bm, scale, shift)]
    keep += dv
    dsc.bias_f, dsc.bias_m, dsc.bn_scale, dsc.bn_shift = (t.data_ptr() for t in dv[2:])
    stream = L.stream_ptr()
    if impl == L.CONV_TCGEN05:
        wt = torch.empty(lib.read_tc_weight_elems(cout, cin, k), dtype=torch.bfloat16, device=d)
        L.check(lib.read_pack_weights_tc_for(ctypes.byref(dsc), dv[0].data_ptr(), dv[1].data_ptr(), wt.data_ptr(), stream))
        dsc.w_tc = wt.data_ptr()
        keep.append(wt)
    elif impl == L.CONV_TCGEN05_GATHER:
        wt = torch.empty(lib.read_tcg_weight_elems(cout, cin, k), dtype=torch.bfloat16, device=d)
        L.check(lib.read_pack_weights_tcg(dv[0].data_ptr(), dv[1].data_ptr(), cout, cin, k, wt.data_ptr(), stream))
        dsc.w_tc = wt.data_ptr()
        keep.append(wt)
    else:
        npad, kpad = lib.read_generic_npad(cout), ((k * k * cin + 15) // 16) * 16
        wg = torch.empty(npad * kpad, dtype=torch.float32, device=d)
        L.check(lib.read_pack_weights_generic(dv[0].data_ptr(), dv[1].data_ptr(), cout, cin, k, wg.data_ptr(), stream))
        dsc.w_generic = wg.data_ptr()
        keep.append(wg)
    dsc.impl = impl
    if final:
        out = torch.full((B, cout, hout, wout), float("nan"), dtype=torch.float32, device=d)
        dsc.out_mode = L.OUT_NCHW_F32
    else:
        out = torch.full((B, hout, wout, cout), float("nan"), dtype=adt, device=d)
        dsc.out_mode = L.OUT_NHWC
    dsc.out = out.data_ptr()
    if residual:
        r = nhwc(res); keep.append(r); dsc.residual = r.data_ptr()
    o2 = None
    if out2:
        mm = nhwc(m2); keep.append(mm)
        o2 = torch.full_like(out, float("nan"))
        dsc.out2, dsc.out2_mul = o2.data_ptr(), mm.data_ptr()
    if mul:
        mx = nhwc(mulx); keep.append(mx); dsc.mul = mx.data_ptr()
    plan = L.c_vp()
    L.check(lib.read_conv_plan_create(ctypes.byref(dsc), ctypes.byref(plan)))
    assert lib.read_conv_plan_impl(plan) == impl
    if reversed_order:
        L.check(lib.read_conv_plan_set_tile_order(plan, 1))
    L.check(lib.read_conv_plan_launch(plan, stream))
    torch.cuda.synchronize()
    lib.read_conv_plan_destroy(plan)
    got = out.float().cpu() if final else out.float().permute(0, 3, 1, 2).cpu()
    if out2:
        return got, want, o2.float().permute(0, 3, 1, 2).cpu(), want.to(adt).float() * m2
    return got, want


GEN = L.CONV_GENERIC
TC = L.CONV_TCGEN05

# every distinct layer kind of the net (SURVEY.md §8a census), at small spatial sizes incl. ragged tiles
GENERIC_CASES = [
    ("3x3 8->32 first conv", [(8, 20, 28, "id", 1)], 32, 3, 1, True, {}),
    ("3x3 32->32 ELU", [(32, 17, 23, "id", 1)], 32, 3, 1, True, {}),
    ("3x3 64->64 noact + residual", [(64, 16, 16, "id", 1)], 64, 3, 1, False, {"residual": True}),
    ("3x3 s2 32->64 + FAM product output", [(32, 16, 24, "id", 1)], 64, 3, 2, True, {"out2": True}),
    ("4x4 s2 64->32", [(64, 16, 16, "id", 1)], 32, 4, 2, True, {}),
    ("1x1 16->32", [(16, 9, 13, "id", 1)], 32, 1, 1, True, {}),
    ("1x1 32->56 ragged Cout", [(32, 8, 8, "id", 1)], 56, 1, 1, True, {}),
    ("SCM concat 8+56 -> 64 1x1", [(8, 10, 12, "id", 1), (56, 10, 12, "id", 1)], 64, 1, 1, False, {}),
    ("AFF0 480->32: id, up2, up4, up8", [(32, 16, 16, "id", 1), (64, 8, 8, "up", 2), (128, 4, 4, "up", 4), (256, 2, 2, "up", 8)], 32, 1, 1, True, {}),
    ("AFF2 480->128: down4, down2, id, up2", [(32, 16, 16, "down", 4), (64, 8, 8, "down", 2), (128, 4, 4, "id", 1), (256, 2, 2, "up", 2)], 128, 1, 1, True, {}),
    ("decoder merge: bilinear x4 + id, 256->128", [(128, 3, 5, "bil4", 4), (128, 12, 20, "id", 1)], 128, 1, 1, True, {}),
    ("final 32->3 NCHW f32", [(32, 16, 24, "id", 1)], 3, 3, 1, False, {"final": True}),
    ("FAM product on the input side", [(32, 9, 9, "id", 1)], 32, 3, 1, False, {"mul": True, "residual": True}),
]


@pytest.mark.parametrize("case", GENERIC_CASES, ids=[c[0] for c in GENERIC_CASES])
def test_generic_fp32_matches_torch(case):
    _, srcs, cout, k, stride, elu, kw = case
    r = run_conv(srcs, cout, k, stride, elu, False, GEN, **kw)
    err = float((r[0] - r[1]).abs().max())
    assert err < 2e-5, err                                 # fp32 math, only summation order differs
    if kw.get("out2"):
        assert float((r[2] - r[3]).abs().max()) < 2e-5


@pytest.mark.parametrize("case", GENERIC_CASES[:6], ids=[c[0] for c in GENERIC_CASES[:6]])
def test_generic_bf16_activations(case):
    _, srcs, cout, k, stride, elu, kw = case
    r = run_conv(srcs, cout, k, stride, elu, True, GEN, **kw)
    # inputs are bf16-exact, math fp32: the only error is the final bf16 rounding of the output (2^-9 relative)
    tol = 2 ** -8 * float(r[1].abs().max()) + 1e-3
    assert float((r[0] - r[1]).abs().max()) < tol


TC_CASES = [
    ("C32 16x32 exact tiles", [(32, 16, 32, "id", 1)], 32, 3, True, {}),
    ("C32 ragged 19x23", [(32, 19, 23, "id", 1)], 32, 3, False, {"residual": True}),
    ("C64 24x40", [(64, 24, 40, "id", 1)], 64, 3, True, {}),
    ("C64 ragged + residual", [(64, 9, 17, "id", 1)], 64, 3, False, {"residual": True}),
    ("C128 two k-chunks", [(128, 16, 16, "id", 1)], 128, 3, True, {}),
    ("C256 two n-tiles, four k-chunks", [(256, 10, 18, "id", 1)], 256, 3, False, {"residual": True}),
    ("C64 1x1", [(64, 8, 16, "id", 1)], 64, 1, True, {}),
    ("C32 -> 64 channels, FAM product output", [(32, 16, 16, "id", 1)], 64, 3, True, {"out2": True}),
    ("many tiles per CTA (persistence, phases wrap)", [(32, 200, 208, "id", 1)], 32, 3, True, {"residual": True}),
    ("persistent C32, 2560 tiles (17 per CTA)", [(32, 512, 640, "id", 1)], 32, 3, True, {}),
    ("persistent C64 + residual, 1280 tiles", [(64, 256, 640, "id", 1)], 64, 3, False, {"residual": True}),
    ("final layer 32->3, NCHW f32 output", [(32, 24, 40, "id", 1)], 3, 3, False, {"final": True}),
    # 8- / 16-channel inputs: one 16-channel K step (SWIZZLE_32B rows); an 8-channel tensor is read with a 16-channel TMA box whose
    # out-of-range half is zero-filled
    ("first conv 8->32 (feat_extract.0), ragged", [(8, 20, 28, "id", 1)], 32, 3, True, {}),
    ("SCM main.0 8->16", [(8, 33, 17, "id", 1)], 16, 3, True, {}),
    ("SCM main.0 8->64 + residual-free no-act", [(8, 16, 24, "id", 1)], 64, 3, False, {}),
    ("3x3 16->32", [(16, 19, 23, "id", 1)], 32, 3, True, {"residual": True}),
    ("1x1 16->32 (SCM2.main.1)", [(16, 24, 40, "id", 1)], 32, 1, True, {}),
    ("persistent 8->32, 2560 tiles", [(8, 512, 640, "id", 1)], 32, 3, True, {}),
    # the C3 shapes of the streamed-weight instances (B = 2): the B ring and the accumulator ring wrap many times per CTA
    ("persistent C128 @272x480 + residual (Encoder.2 at C3), 14 tiles per CTA", [(128, 272, 480, "id", 1)], 128, 3, False, {"residual": True}),
    ("persistent C128 @272x480 ELU", [(128, 272, 480, "id", 1)], 128, 3, True, {}),
    ("persistent C256 @136x240 + residual (Encoder.3 at C3), two n-tiles", [(256, 136, 240, "id", 1)], 256, 3, False, {"residual": True}),
    ("persistent C256 @136x240 ELU", [(256, 136, 240, "id", 1)], 256, 3, True, {}),
    # stride 2 on the TMA path: four phase tiles per stage (even / odd input columns x rows), traversal-stride-2 TMA loads
    ("3x3 s2 32->64 + FAM product output (feat_extract.1)", [(32, 32, 48, "id", 1)], 64, 3, True, {"stride": 2, "out2": True}),
    ("3x3 s2 64->128 ragged tiles (feat_extract.2)", [(64, 38, 26, "id", 1)], 128, 3, True, {"stride": 2, "out2": True}),
    ("3x3 s2 128->256, two n-tiles, four k-chunks (feat_extract.6)", [(128, 32, 32, "id", 1)], 256, 3, True, {"stride": 2}),
    ("4x4 s2 256->128 (feat_extract.7)", [(256, 32, 16, "id", 1)], 128, 4, True, {"stride": 2}),
    ("4x4 s2 64->32 (feat_extract.4)", [(64, 64, 48, "id", 1)], 32, 4, True, {"stride": 2}),
    ("3x3 s2 persistent, 1200 tiles", [(32, 640, 960, "id", 1)], 64, 3, True, {"stride": 2}),
    # virtual concat on the TMA path (1x1): identity + nearest-down sources, one tensor map per source
    ("decoder merge 32+32 -> 32 (Convs.2: 32-channel K chunks)", [(32, 40, 56, "id", 1), (32, 40, 56, "id", 1)], 32, 1, True, {}),
    ("decoder merge 128+128 -> 128 (Convs.0)", [(128, 24, 24, "id", 1), (128, 24, 24, "id", 1)], 128, 1, True, {}),
    ("concat down4 + down2 + id (AFF2 without its upsampled source)", [(32, 64, 96, "down", 4), (64, 32, 48, "down", 2), (128, 16, 24, "id", 1)], 64, 1, True, {}),
    ("persistent concat 64+64 -> 64, 1280 tiles", [(64, 256, 640, "id", 1), (64, 256, 640, "id", 1)], 64, 1, False, {"residual": True}),
]


@pytest.mark.parametrize("case", TC_CASES, ids=[c[0] for c in TC_CASES])
def test_tcgen05_matches_torch(case):
    _, srcs, cout, k, elu, kw = case
    kw = dict(kw)
    r = run_conv(srcs, cout, k, kw.pop("stride", 1), elu, True, TC, **kw)
    got, want = r[0], r[1]
    assert torch.isfinite(got).all(), "TMA kernel left outputs unwritten (NaN sentinel)"
    # bf16 operands are exact in the reference (weights/inputs pre-rounded), accumulation fp32 on both sides:
    # error = output bf16 rounding + approx ex2/tanh (~1e-3 abs)
    tol = 2 ** -8 * float(want.abs().max()) + 4e-3
    err = float((got - want).abs().max())
    assert err < tol, (err, tol)
    if kw.get("out2"):
        assert float((r[2] - r[3]).abs().max()) < tol


GATHER = L.CONV_TCGEN05_GATHER
GATHER_CASES = [c for c in GENERIC_CASES if not c[6].get("mul")] + [
    ("3x3 C64 stride 1 (also a TMA shape)", [(64, 24, 40, "id", 1)], 64, 3, 1, True, {"residual": True}),
    ("SCM0 tail 128->248 (Cout padded to 256, two n-tiles)", [(128, 9, 11, "id", 1)], 248, 1, 1, True, {}),
    ("3x3 s2 128->256", [(128, 16, 16, "id", 1)], 256, 3, 2, True, {"out2": True}),
    ("4x4 s2 256->128", [(256, 16, 16, "id", 1)], 128, 4, 2, True, {}),
    ("many tiles (phases wrap), s2", [(32, 256, 320, "id", 1)], 64, 3, 2, True, {}),
    # persistence: 17+ tiles per CTA so every ring (A stages, streamed weight stages, barrier phases) wraps several times
    ("persistent 1x1 32->32 + residual, 2560 tiles", [(32, 512, 640, "id", 1)], 32, 1, 1, True, {"residual": True}),
    ("persistent 3x3 8->32, 2 k-blocks per tile, 2560 tiles", [(8, 512, 640, "id", 1)], 32, 3, 1, True, {}),
    ("persistent concat 32+32 -> 64 1x1, 2560 tiles", [(32, 512, 640, "id", 1), (32, 256, 320, "up", 2)], 64, 1, 1, False, {}),
]


@pytest.mark.parametrize("case", GATHER_CASES, ids=[c[0] for c in GATHER_CASES])
def test_tcgen05_gather_matches_torch(case):
    _, srcs, cout, k, stride, elu, kw = case
    r = run_conv(srcs, cout, k, stride, elu, True, GATHER, **kw)
    got, want = r[0], r[1]
    assert torch.isfinite(got).all(), "gather kernel left outputs unwritten (NaN sentinel)"
    # bilinear sources are blended in fp32 then rounded to bf16 before the MMA (the reference blends in fp32): + 2^-8
    tol = 2 ** -7 * float(want.abs().max()) + 4e-3
    err = float((got - want).abs().max())
    assert err < tol, (err, tol)
    if kw.get("out2"):
        assert float((r[2] - r[3]).abs().max()) < tol


def test_tc_supported_predicate():
    lib = L.load()
    d = L.ReadConvDesc()
    d.act_dtype, d.n_src = L.ACT_BF16, 1
    d.src[0].mode = L.SRC_IDENTITY
    d.k, d.stride, d.pad, d.out_mode = 3, 1, 1, L.OUT_NHWC
    d.Hin = d.Hout = 8
    d.Win = d.Wout = 8
    for cin, cout, ok in [(32, 32, 1), (64, 64, 1), (128, 128, 1), (256, 256, 1), (8, 32, 1), (16, 32, 1), (8, 128, 0), (32, 3, 0), (56, 64, 0), (480, 32, 1), (64, 32, 1)]:   # (32,3) needs NCHW f32 output, see below
        d.Cin, d.Cout = cin, cout
        assert lib.read_conv_tc_supported(ctypes.byref(d)) == ok, (cin, cout)
    d.Cin, d.Cout, d.out_mode = 32, 3, L.OUT_NCHW_F32
    assert lib.read_conv_tc_supported(ctypes.byref(d)) == 1            # final layer shape
    d.Cin = d.Cout = 32
    d.out_mode = L.OUT_NHWC
    d.act_dtype = L.ACT_F32
    assert lib.read_conv_tc_supported(ctypes.byref(d)) == 0


@pytest.mark.parametrize("bf16", [False, True])
def test_upsample_bilinear4_matches_torch(bf16):
    lib = L.load()
    g = torch.Generator().manual_seed(4)
    x = torch.rand((2, 16, 5, 7), generator=g)
    dt = torch.bfloat16 if bf16 else torch.float32
    if bf16:
        x = x.to(dt).float()
    want = F.interpolate(x, scale_factor=4, mode="bilinear", align_corners=False)
    xin = x.permute(0, 2, 3, 1).contiguous().to(dev(), dt)
    out = torch.empty((2, 20, 28, 16), dtype=dt, device=dev())
    L.check(lib.read_upsample_bilinear4(xin.data_ptr(), L.ACT_BF16 if bf16 else L.ACT_F32, 2, 5, 7, 16, out.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    err = float((out.float().permute(0, 3, 1, 2).cpu() - want).abs().max())
    assert err < (2 ** -8 if bf16 else 1e-6), err


# ---------------------------------------------------------------- RAW terms + add-in (the AFF heads split by linearity)
def _pack_tc(lib, dsc, wf, wm, d):
    wt = torch.empty(lib.read_tc_weight_elems(dsc.Cout, dsc.Cin, dsc.k), dtype=torch.bfloat16, device=d)
    L.check(lib.read_pack_weights_tc_for(ctypes.byref(dsc), wf.data_ptr(), wm.data_ptr(), wt.data_ptr(), L.stream_ptr()))
    return wt


def _run_1x1(srcs_nchw, modes, cout, elu, raw, addin_nchw, seed):
    """1x1 gated conv on the TMA-fed wgmma kernel with RAW output and/or an add-in; returns (got NCHW, want NCHW)."""
    lib, d = L.load(), dev()
    g = torch.Generator().manual_seed(seed)
    xs = [x.to(torch.bfloat16).float() for x in srcs_nchw]
    logical = torch.cat([resample(x, m, f) for x, (m, f) in zip(xs, modes)], 1)
    B, cin, h, w = logical.shape
    bound = 1.0 / cin ** 0.5
    wf = ((torch.rand((cout, cin, 1, 1), generator=g) * 2 - 1) * bound).to(torch.bfloat16).float()
    wm = ((torch.rand((cout, cin, 1, 1), generator=g) * 2 - 1) * bound).to(torch.bfloat16).float()
    bf, bm = (torch.rand(cout, generator=g) * 2 - 1) * bound, (torch.rand(cout, generator=g) * 2 - 1) * bound
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g) * 0.1
    f = F.conv2d(logical, wf)
    m = F.conv2d(logical, wm)
    if addin_nchw is not None:
        up = F.interpolate(addin_nchw.to(torch.bfloat16).float(), scale_factor=2)[:, :, :h, :w]
        f, m = f + up[:, :cout], m + up[:, cout:]
    if raw:
        want = torch.cat([f, m], 1)
    else:
        f, m = f + bf[None, :, None, None], m + bm[None, :, None, None]
        want = (F.elu(f) if elu else f) * torch.sigmoid(m) * scale[None, :, None, None] + shift[None, :, None, None]
    nhwc = lambda t: t.permute(0, 2, 3, 1).contiguous().to(d, torch.bfloat16)
    dsc = L.ReadConvDesc()
    dsc.act_dtype, dsc.n_src = L.ACT_BF16, len(xs)
    keep = []
    mm = {"id": L.SRC_IDENTITY, "down": L.SRC_NEAREST_DOWN}
    for i, (x, (mo, fa)) in enumerate(zip(xs, modes)):
        t = nhwc(x); keep.append(t)
        dsc.src[i].ptr, dsc.src[i].C, dsc.src[i].H, dsc.src[i].W = t.data_ptr(), x.shape[1], x.shape[2], x.shape[3]
        dsc.src[i].mode, dsc.src[i].factor = mm[mo], fa
    dsc.B, dsc.Hin, dsc.Win, dsc.Cin, dsc.Hout, dsc.Wout, dsc.Cout = B, h, w, cin, h, w, cout
    dsc.k, dsc.stride, dsc.pad, dsc.elu = 1, 1, 0, int(elu)
    dv = [t.to(d).contiguous() for t in (wf, wm, bf, bm, scale, shift)]
    dsc.bias_f, dsc.bias_m, dsc.bn_scale, dsc.bn_shift = (t.data_ptr() for t in dv[2:])
    dsc.impl = L.CONV_TCGEN05
    oc = 2 * cout if raw else cout
    out = torch.full((B, h, w, oc), float("nan"), dtype=torch.bfloat16, device=d)
    dsc.out, dsc.out_mode = out.data_ptr(), (L.OUT_RAW_NHWC if raw else L.OUT_NHWC)
    if addin_nchw is not None:
        ad = nhwc(addin_nchw); keep.append(ad)
        dsc.addin, dsc.addin_H, dsc.addin_W = ad.data_ptr(), ad.shape[1], ad.shape[2]
    assert lib.read_conv_tc_supported(ctypes.byref(dsc)) == 1
    wt = _pack_tc(lib, dsc, dv[0], dv[1], d)
    dsc.w_tc = wt.data_ptr()
    plan = L.c_vp()
    L.check(lib.read_conv_plan_create(ctypes.byref(dsc), ctypes.byref(plan)))
    L.check(lib.read_conv_plan_launch(plan, L.stream_ptr()))
    torch.cuda.synchronize()
    lib.read_conv_plan_destroy(plan)
    return out.float().permute(0, 3, 1, 2).cpu(), want


@pytest.mark.parametrize("cout,cin,h,w,with_addin", [(32, 256, 17, 30, False), (32, 128, 34, 60, True), (64, 128, 33, 23, True),
                                                      (32, 64, 256, 320, True)])
def test_tcgen05_raw_term_matches_torch(cout, cin, h, w, with_addin):
    g = torch.Generator().manual_seed(3)
    x = torch.rand((2, cin, h, w), generator=g) * 2 - 1
    addin = (torch.rand((2, 2 * cout, (h + 1) // 2, (w + 1) // 2), generator=g) * 2 - 1) if with_addin else None
    got, want = _run_1x1([x], [("id", 1)], cout, False, True, addin, seed=1)
    assert torch.isfinite(got).all(), "outputs left unwritten"
    tol = 2 ** -8 * float(want.abs().max()) + 1e-3           # fp32 accumulate + add, one bf16 rounding
    assert float((got - want).abs().max()) < tol


@pytest.mark.parametrize("cout", [32, 64])
def test_tcgen05_addin_gated_matches_torch(cout):
    """Final term of an AFF head: two TMA sources (one nearest-down) + the coarse terms as add-in, then the gate."""
    g = torch.Generator().manual_seed(4)
    h, w = 40, 56
    a = torch.rand((2, 32, 2 * h, 2 * w), generator=g) * 2 - 1        # read with traversal stride 2
    b = torch.rand((2, 64, h, w), generator=g) * 2 - 1
    addin = torch.rand((2, 2 * cout, h // 2, w // 2), generator=g) * 2 - 1
    got, want = _run_1x1([a, b], [("down", 2), ("id", 1)], cout, True, False, addin, seed=2)
    assert torch.isfinite(got).all(), "outputs left unwritten"
    tol = 2 ** -8 * float(want.abs().max()) + 4e-3
    assert float((got - want).abs().max()) < tol


# ---------------------------------------------------------------- TMA kernel: small-channel, wide and persistent shapes
PAIR_CASES = [
    ("C32 16x32 exact tiles (2 pairs)", [(32, 16, 32, "id", 1)], 32, 3, True, {}),
    ("C32 ragged 19x23, odd tile count", [(32, 19, 23, "id", 1)], 32, 3, False, {"residual": True}),
    ("C32 one tile per image (a pair spans two images)", [(32, 16, 8, "id", 1)], 32, 3, True, {}),
    ("C64 24x40", [(64, 24, 40, "id", 1)], 64, 3, True, {}),
    ("C64 ragged + residual", [(64, 9, 17, "id", 1)], 64, 3, False, {"residual": True}),
    ("C32 -> 16 channels", [(32, 33, 20, "id", 1)], 16, 3, True, {}),
    ("C64 -> 32 channels, no activation", [(64, 20, 24, "id", 1)], 32, 3, False, {}),
    ("persistent C32, 2560 tiles (17 pairs per cluster: rings wrap)", [(32, 512, 640, "id", 1)], 32, 3, True, {"residual": True}),
    ("persistent C64 + residual, 1280 tiles", [(64, 256, 640, "id", 1)], 64, 3, False, {"residual": True}),
    # streamed weights: K chunks of 64 channels, several n tiles
    ("wide C128 24x40 (2 K chunks)", [(128, 24, 40, "id", 1)], 128, 3, True, {}),
    ("wide C128 ragged, odd tile count + residual", [(128, 19, 23, "id", 1)], 128, 3, False, {"residual": True}),
    ("wide C256 (4 K chunks, 2 n tiles)", [(256, 17, 24, "id", 1)], 256, 3, True, {}),
    ("wide C256 + residual, one tile per image", [(256, 16, 8, "id", 1)], 256, 3, False, {"residual": True}),
    ("wide C128 -> 256", [(128, 16, 16, "id", 1)], 256, 3, True, {}),
    ("wide C256 -> 128", [(256, 16, 24, "id", 1)], 128, 3, True, {}),
    ("persistent wide C128, 1360 tiles (rings wrap many times)", [(128, 272, 640, "id", 1)], 128, 3, False, {"residual": True}),
    ("persistent wide C256, 680 tiles x 2 n tiles", [(256, 136, 640, "id", 1)], 256, 3, True, {}),
]


@pytest.mark.parametrize("case", PAIR_CASES, ids=[c[0] for c in PAIR_CASES])
def test_tcgen05_cta_pair_matches_torch_and_the_single_cta_kernel(case):
    """The shapes the CTA-pair kernels of the Blackwell build served (ragged tiles, tiles spanning images, resident and streamed
    weights, several n tiles, persistent grids whose rings wrap many times) now run on the TMA kernel: same tolerance against torch
    as the other TMA-kernel cases, and within one bf16 ulp of the gather kernel on the same inputs (the two kernels accumulate
    the K dimension in different orders)."""
    _, srcs, cout, k, elu, kw = case
    got, want = run_conv(srcs, cout, k, 1, elu, True, TC, **kw)[:2]
    other = run_conv(srcs, cout, k, 1, elu, True, GATHER, **kw)[0]
    assert torch.isfinite(got).all(), "kernel left outputs unwritten (NaN sentinel)"
    tol = 2 ** -8 * float(want.abs().max()) + 4e-3
    assert float((got - want).abs().max()) < tol
    assert float((got - other).abs().max()) <= 2 ** -7 * float(want.abs().max())


ORDER_CASES = [c for c in TC_CASES if not c[0].startswith("persistent C")][:24] + PAIR_CASES


@pytest.mark.parametrize("case", ORDER_CASES, ids=[f"{i}: {c[0]}" for i, c in enumerate(ORDER_CASES)])
def test_reversed_tile_order_is_bit_identical(case):
    """read_conv_plan_set_tile_order(plan, 1) walks the tiles bottom-up (the engine alternates the direction between consecutive
    layers for L2 reuse): same output bit for bit on the TMA kernel, resident and streamed weights alike."""
    _, srcs, cout, k, elu, kw = case
    kw = dict(kw)
    stride = kw.pop("stride", 1)
    fwd = run_conv(srcs, cout, k, stride, elu, True, TC, **kw)
    rev = run_conv(srcs, cout, k, stride, elu, True, TC, reversed_order=True, **kw)
    assert torch.isfinite(rev[0]).all(), "outputs left unwritten (NaN sentinel)"
    assert torch.equal(fwd[0], rev[0])
    if kw.get("out2"):
        assert torch.equal(fwd[2], rev[2])
