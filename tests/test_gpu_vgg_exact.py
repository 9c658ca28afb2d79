"""Exact checks of the VGG perceptual loss's kernels (tests/vgg_exact_util.py states the method):

* census: VGGLoss forward + backward, both layer sets, with and without partialconv, launches exactly the RAW plan classes and
  the dgrad_cin8 C the census lists, so a new layer or packing fails here until it has exact cases;
* every forward RAW 3x3 class (fwd_exact_util's method, through test_gpu_fwd_exact._run_case) and every input-gradient class
  (test_gpu_bwd_exact's RAW 3x3 method) at ragged tiles, image edges and the sizes a 256^2 training crop gives each layer;
* the VGG path itself: the filters VGGLoss.filters packs from integer torchvision-layout features, launched as _forward and
  backward launch them, give the natural-order float64 conv and its input gradient, rounded to bf16;
* the glue kernels of csrc/vgg.cu bit for bit against their float32 replays, every output inside a guard band.
"""
import pytest
import torch

import bwd_exact_util as U
import fwd_exact_util as X
import vgg_exact_util as E
import vgg_partial_util
import vgg_util
from gpu_util import dev
from read_b200 import _lib as L, blocks, vgg_loss
from read_b200.vgg_loss import VGGLoss
from test_gpu_fwd_exact import _gen, _run_case, gate_pinned  # noqa: F401  (gate_pinned is a module fixture)

pytestmark = pytest.mark.gpu
NHWC = ["b", "y", "x", "c"]


# ------------------------------------------------------------------ 1. the census of what VGGLoss launches
@pytest.mark.parametrize("partialconv", [False, True])
@pytest.mark.parametrize("optimized", [False, True])
def test_vgg_loss_launches_exactly_the_census(optimized, partialconv, monkeypatch):
    feats = vgg_util.seeded_features()
    crit = VGGLoss(optimized=optimized, partialconv=partialconv,
                   features=vgg_loss.partial_features(feats) if partialconv else feats).to(dev())
    pk = crit.filters(dev())
    packing = {p["w_tc"].data_ptr(): "tc" for p in pk}
    packing.update({p["w_dgrad"].data_ptr(): "tc_dgrad" for p in pk if p["w_dgrad"] is not None})
    modes = {L.OUT_RAW_NHWC: "raw", L.OUT_NHWC: "nhwc", L.OUT_NCHW_F32: "nchw"}
    seen, cin8 = [], []
    launch, lib = blocks._launch, L.load()
    dgrad_cin8 = lib.read_conv3x3_dgrad_cin8

    def rec(lib_, src, cout, w_tc, par, elu, out_mode, out, residual=None, k=3, stride=1):
        seen.append((packing.get(w_tc.data_ptr(), "other"), src.shape[3], cout, k, stride, modes[out_mode], residual is not None))
        return launch(lib_, src, cout, w_tc, par, elu, out_mode, out, residual, k, stride)

    def rec8(dy, wf, wm, n, h, w, C, out, st):
        cin8.append(C)
        return dgrad_cin8(dy, wf, wm, n, h, w, C, out, st)

    monkeypatch.setattr(blocks, "_launch", rec)
    monkeypatch.setattr(lib, "read_conv3x3_dgrad_cin8", rec8)
    x, t = (v.to(dev()) for v in vgg_partial_util.masked_pair("holes" if partialconv else "dense", 1, 48, 40, 3))
    xx = x.clone().requires_grad_(True)
    crit(xx, t).backward()
    torch.cuda.synchronize()
    steps = crit.steps()
    assert len(seen) == 2 * len(steps) - 1 and len(cin8) == 1, (len(seen), len(cin8))
    assert set(seen) == E.launch_census(), (f"new {sorted(set(seen) - E.launch_census())}, "
                                            f"gone {sorted(E.launch_census() - set(seen))}")
    assert set(cin8) == E.CIN8_CS


# ------------------------------------------------------------------ 2. forward RAW plans
@pytest.mark.parametrize("case", E.VGG_FWD_CASES, ids=lambda c: c.id)
def test_vgg_forward_raw_plan_is_exact(case, gate_pinned):  # noqa: F811
    if (case.cin, case.cout) == (64, 64):
        assert not X.tma_geom(case)[5], "64 -> 2 x 64 RAW: 144 KB of weights, streamed (test_vgg_exact_host)"
    _run_case(case, gate_pinned)


# ------------------------------------------------------------------ 3. input-gradient RAW plans
@pytest.mark.parametrize("case", E.VGG_DGRAD_CASES, ids=lambda c: "cin{}-C{}-B{}-{}x{}".format(*c))
def test_vgg_dgrad_raw_plan_is_exact(case):
    cin, C, B, H, W = case
    lib, st = L.load(), L.stream_ptr()
    g = _gen("vgg dgrad", case)
    dcat = U.int_tensor((B, H, W, 2 * C), E.DGRAD_AMP, g).to(dev())
    wcat = U.int_tensor((2 * C, cin, 3, 3), E.DGRAD_AMP, g).to(dev())
    wf, wm = wcat[:C].contiguous(), wcat[C:].contiguous()
    w_dgrad = torch.empty(lib.read_tc_weight_elems(cin // 2, 2 * C, 3), dtype=torch.bfloat16, device=dev())
    L.check(lib.read_pack_weights_tc_dgrad(wf.data_ptr(), wm.data_ptr(), C, cin, w_dgrad.data_ptr(), st))
    dfm = U.to_raw(dcat).bfloat16().contiguous()
    want = U.dgrad_ref(dcat, wcat, H, W, 1)
    frac = U.bf16_nonrepresentable_fraction(want)
    assert frac >= 0.1, f"only {frac:.2f} of the exact sums need rounding"
    out = U.Guarded(B * H * W * cin, torch.bfloat16, dev())
    zeros = torch.zeros(cin, dtype=torch.float32, device=dev())
    blocks._launch(lib, dfm, cin // 2, w_dgrad, (zeros,) * 4, False, L.OUT_RAW_NHWC, out.out)
    torch.cuda.synchronize()
    what = f"VGG RAW 3x3 dgrad {case}"
    out.check(what)
    U.assert_bf16_rn(out.out.view(B, H, W, cin), want, what, NHWC)


# ------------------------------------------------------------------ 4. the VGG path: split, packing and channel order
def test_vgg_filters_give_the_natural_channel_order():
    """Every conv of the walk (LAYERS_OPTIMIZED runs all 16): VGGLoss.filters from integer features, the forward plan launched as
    _forward launches it, the input gradient as backward does (dgrad_cin8 for conv1_1): natural channel order, exact sums."""
    lib, st = L.load(), L.stream_ptr()
    g = _gen("vgg path")
    crit = VGGLoss(optimized=True, features=E.int_features(g)).to(dev())
    pk = crit.filters(dev())
    zeros = torch.zeros(256, dtype=torch.float32, device=dev())
    n2, h, w = E.PATH_SHAPE
    n = n2 // 2
    for i, s in enumerate(crit.steps()):
        conv = crit.vgg19[s.conv]
        wt = conv.weight.detach().double()
        cin = max(s.cin, 8)
        x = E.nz(U.int_tensor((n2, h, w, cin), E.PATH_AMP, g)).to(dev())
        want = E.conv_ref(x[..., :s.cin], wt)
        raw = U.Guarded(n2 * h * w * s.cout, torch.bfloat16, dev())
        blocks._launch(lib, x.bfloat16().contiguous(), s.cout // 2, pk[i]["w_tc"], (zeros,) * 4, False, L.OUT_RAW_NHWC, raw.out)
        torch.cuda.synchronize()
        what = f"conv {s.conv} ({s.cin}->{s.cout}) forward"
        raw.check(what)
        U.assert_bf16_rn(raw.out.view(n2, h, w, s.cout), want, what, NHWC)
        dy = E.nz(U.int_tensor((n, h, w, s.cout), E.PATH_AMP, g)).to(dev())
        dyb = dy.bfloat16().contiguous()
        want = E.conv_input_grad_ref(dy, wt)
        up = U.Guarded(n * h * w * cin, torch.bfloat16, dev())
        if i == 0:
            L.check(lib.read_conv3x3_dgrad_cin8(dyb.data_ptr(), pk[0]["wf"].data_ptr(), pk[0]["wm"].data_ptr(), n, h, w,
                                                s.cout // 2, up.out.data_ptr(), st))
            want = torch.cat([want, torch.zeros((n, h, w, cin - s.cin), dtype=want.dtype, device=want.device)], -1)
        else:
            blocks._launch(lib, dyb, s.cin // 2, pk[i]["w_dgrad"], (zeros,) * 4, False, L.OUT_RAW_NHWC, up.out)
        torch.cuda.synchronize()
        what = f"conv {s.conv} ({s.cin}->{s.cout}) input gradient"
        up.check(what)
        U.assert_bf16_rn(up.out.view(n, h, w, cin), want, what, NHWC)


# ------------------------------------------------------------------ 5. the glue kernels, bit for bit
# (n, H, W, C): odd and even sizes at every VGG width; 2 x 256^2 x 64 runs 4 grid-stride steps per thread at pool 0, and
# 2 x 259 x 257 x 64 at pool 1 more than 1024 x 256 units: the 1024 CTAs' partials are combined
POST_SHAPES = [(2, 9, 7, 64), (1, 8, 6, 128), (2, 5, 3, 256), (1, 4, 2, 512), (2, 3, 1, 512), (1, 1, 1, 64), (2, 256, 256, 64),
               (2, 259, 257, 64)]


def _term_buf(prefill):
    """[sentinel, prefill, sentinel] float64: *term is element 1, its neighbours must stay put."""
    return torch.tensor([-7.25, prefill, 13.5], dtype=torch.float64, device=dev())


def _check_term_buf(buf, want, what):
    got = buf.cpu().tolist()
    assert got[0] == -7.25 and got[2] == 13.5, f"{what}: written next to the term: {got}"
    E.assert_term(got[1], want, what)


@pytest.mark.parametrize("pool", [0, 1])
@pytest.mark.parametrize("shape", POST_SHAPES, ids=lambda s: "n{}-{}x{}x{}".format(*s))
def test_post_is_bit_exact(shape, pool):
    n, H, W, C = shape
    lib, st = L.load(), L.stream_ptr()
    g = _gen("post", shape, pool)
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    y = E.post_values(raw, bias, n)
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    scale = 1.0 / (2 * n * H * W * C)
    prefill = 0.3 + n / 7.0
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev())
    rawd, biasd = raw.to(dev()), bias.to(dev())
    for loss in (False, True):
        what = f"vgg_post pool={pool} loss={loss} {shape}"
        out = U.Guarded(2 * n * Ho * Wo * C, torch.bfloat16, dev())
        code = U.Guarded(n * H * W * C, torch.int8, dev())
        term = _term_buf(prefill)
        L.check(lib.read_vgg_post(rawd.data_ptr(), n, H, W, C, biasd.data_ptr(), pool, out.out.data_ptr(), code.out.data_ptr(),
                                  term[1:].data_ptr() if loss else None, scale, ws.data_ptr(), st))
        torch.cuda.synchronize()
        out.check(what + " out")
        code.check(what + " code")
        if Ho and Wo:
            E.assert_same_bits(out.out.view(2 * n, Ho, Wo, C), E.post_out(y, pool), what + " out", NHWC)
        E.assert_same_bits(code.out.view(n, H, W, C), E.post_codes(y, n, loss), what + " code", NHWC)
        s = E.term_sum(y, n, pool)
        assert s == E.term_exact_sum(y, n)                         # integer operands: every partial sum exact
        _check_term_buf(term, E.fused_term(prefill, s, scale) if loss else prefill, what + " term")


@pytest.mark.parametrize("shape", [(2, 9, 7, 64), (1, 4, 3, 512), (2, 256, 256, 64)], ids=lambda s: "n{}-{}x{}x{}".format(*s))
def test_post_in_place_is_bit_exact(shape):
    """out == raw (pool 0), as _forward runs the layers no pool follows."""
    n, H, W, C = shape
    lib, st = L.load(), L.stream_ptr()
    g = _gen("post in place", shape)
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    y = E.post_values(raw, bias, n)
    buf = U.Guarded(raw.numel(), torch.bfloat16, dev(), raw.to(dev()))
    code = U.Guarded(n * H * W * C, torch.int8, dev())
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev())
    term, scale = _term_buf(0.5), 1.0 / (2 * n * H * W * C)
    biasd = bias.to(dev())
    L.check(lib.read_vgg_post(buf.out.data_ptr(), n, H, W, C, biasd.data_ptr(), 0, buf.out.data_ptr(), code.out.data_ptr(),
                              term[1:].data_ptr(), scale, ws.data_ptr(), st))
    torch.cuda.synchronize()
    what = f"vgg_post in place {shape}"
    buf.check(what)
    code.check(what + " code")
    E.assert_same_bits(buf.out.view(2 * n, H, W, C), E.post_out(y, 0), what, NHWC)
    E.assert_same_bits(code.out.view(n, H, W, C), E.post_codes(y, n, True), what + " code", NHWC)
    _check_term_buf(term, E.fused_term(0.5, E.term_sum(y, n, 0), scale), what + " term")


@pytest.mark.parametrize("pool", [0, 1])
@pytest.mark.parametrize("shape", [(2, 9, 7, 128), (1, 8, 6, 64), (2, 5, 3, 512), (2, 256, 256, 64)],
                         ids=lambda s: "n{}-{}x{}x{}".format(*s))
def test_dgrad_in_is_bit_exact(shape, pool):
    n, H, W, C = shape
    lib, st = L.load(), L.stream_ptr()
    gen = _gen("dgrad_in", shape, pool)
    Hu, Wu = (H // 2, W // 2) if pool else (H, W)
    up = E.nz(torch.randn((n, Hu, Wu, C), generator=gen) * 3).bfloat16()
    code = torch.randint(0, 4, (n, H, W, C), generator=gen, dtype=torch.int8)
    coefs = [(0.75, 1.0 / (2 * n * H * W * C)), (-1.5, 1e-1), (0.75, 0.0)]     # a loss layer's coef, a large one, non-loss layers
    upd, coded = up.to(dev()), code.to(dev())
    for has_up in (True, False):                                  # up = NULL: the last layer
        for gv, coef in coefs:
            what = f"vgg_dgrad_in pool={pool} up={has_up} g={gv} coef={coef} {shape}"
            gt = torch.tensor([gv], dtype=torch.float32, device=dev())
            dy = U.Guarded(n * H * W * C, torch.bfloat16, dev())
            L.check(lib.read_vgg_dgrad_in(upd.data_ptr() if has_up else None, pool, coded.data_ptr(), n, H, W, C, gt.data_ptr(),
                                          coef, dy.out.data_ptr(), st))
            torch.cuda.synchronize()
            dy.check(what)
            E.assert_same_bits(dy.out.view(n, H, W, C), E.dgrad_in_replay(up if has_up else None, code, H, W, pool, gv, coef),
                               what, NHWC)


@pytest.mark.parametrize("kind", ["holes", "valid", "invalid"])
@pytest.mark.parametrize("shape", [(2, 9, 7, 64), (1, 1, 5, 64), (2, 256, 256, 64)], ids=lambda s: "n{}-{}x{}x{}".format(*s))
def test_partial_kernels_are_bit_exact(shape, kind):
    """vgg_post_partial (raw * ratio + bias fused, as compiled: the replay rounds it once) and vgg_dgrad_in_partial."""
    n, H, W, C = shape
    lib, st = L.load(), L.stream_ptr()
    g = _gen("partial", shape, kind)
    raw, bias = E.glue_raw(n, H, W, C, g), E.glue_bias(C, g)
    mask = E.glue_mask(n, H, W, g, kind)
    y = E.post_values(raw, bias, n, mask)
    maskd = mask.to(dev())
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev())
    rawd, biasd = raw.to(dev()), bias.to(dev())
    scale = 1.0 / (2 * n * H * W * C)
    for loss in (False, True):
        what = f"vgg_post_partial {kind} loss={loss} {shape}"
        out = U.Guarded(raw.numel(), torch.bfloat16, dev())
        code = U.Guarded(n * H * W * C, torch.int8, dev())
        term = _term_buf(0.25)
        L.check(lib.read_vgg_post_partial(rawd.data_ptr(), maskd.data_ptr(), n, H, W, C, biasd.data_ptr(), out.out.data_ptr(),
                                          code.out.data_ptr(), term[1:].data_ptr() if loss else None, scale, ws.data_ptr(), st))
        torch.cuda.synchronize()
        out.check(what)
        code.check(what + " code")
        E.assert_same_bits(out.out.view(2 * n, H, W, C), E.post_out(y, 0), what, NHWC)
        E.assert_same_bits(code.out.view(n, H, W, C), E.post_codes(y, n, loss), what + " code", NHWC)
        _check_term_buf(term, E.fused_term(0.25, E.term_sum(y, n, 0), scale) if loss else 0.25, what + " term")
    up = E.nz(torch.randn((n, H, W, C), generator=g) * 3).bfloat16()
    code = torch.randint(0, 4, (n, H, W, C), generator=g, dtype=torch.int8)
    upd, coded = up.to(dev()), code.to(dev())
    for has_up, gv, coef in ((True, 0.75, scale), (True, -1.5, 0.0), (False, 0.75, 0.1)):
        what = f"vgg_dgrad_in_partial {kind} up={has_up} g={gv} coef={coef} {shape}"
        gt = torch.tensor([gv], dtype=torch.float32, device=dev())
        dy = U.Guarded(n * H * W * C, torch.bfloat16, dev())
        L.check(lib.read_vgg_dgrad_in_partial(upd.data_ptr() if has_up else None, maskd.data_ptr(), coded.data_ptr(), n, H, W, C,
                                              gt.data_ptr(), coef, dy.out.data_ptr(), st))
        torch.cuda.synchronize()
        dy.check(what)
        want = E.dgrad_in_replay(up if has_up else None, code, H, W, False, gv, coef, mask)
        E.assert_same_bits(dy.out.view(n, H, W, C), want, what, NHWC)


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("net", ["caffe", "pytorch"])
def test_normalize_and_image_grad_are_bit_exact(net, masked):
    lib, st = L.load(), L.stream_ptr()
    mean, std = vgg_loss.normalization(net)
    md, sd = mean.reshape(3).contiguous().to(dev()), std.reshape(3).contiguous().to(dev())
    for n, H, W in ((3, 13, 11), (1, 1, 1), (2, 256, 256)):
        g = _gen("normalize", net, masked, n, H, W)
        x, t = vgg_partial_util.masked_pair("holes", n, H, W, 5)
        xd, td = x.to(dev()), t.to(dev())
        what = f"{net} masked={masked} {n}x{H}x{W}"
        out = U.Guarded(2 * n * H * W * 8, torch.bfloat16, dev())
        mask = None
        if masked:
            mg = U.Guarded(n * H * W, torch.uint8, dev())
            L.check(lib.read_vgg_normalize_masked(xd.data_ptr(), td.data_ptr(), n, H, W, md.data_ptr(), sd.data_ptr(),
                                                  out.out.data_ptr(), mg.out.data_ptr(), st))
            torch.cuda.synchronize()
            mg.check("vgg_normalize_masked mask " + what)
            mask = vgg_loss.target_mask(t)[:, 0].to(torch.uint8)
            E.assert_same_bits(mg.out.view(n, H, W), mask, "vgg_normalize_masked mask " + what)
        else:
            L.check(lib.read_vgg_normalize(xd.data_ptr(), td.data_ptr(), n, H, W, md.data_ptr(), sd.data_ptr(), out.out.data_ptr(),
                                           st))
            torch.cuda.synchronize()
        out.check("vgg_normalize " + what)
        E.assert_same_bits(out.out.view(2 * n, H, W, 8), E.normalize_replay(x, t, mean, std, mask), "vgg_normalize " + what, NHWC)
        dx = (torch.randn((n, H, W, 8), generator=g) * 2).bfloat16()
        dxd = dx.to(dev())
        gr = U.Guarded(n * 3 * H * W, torch.float32, dev())
        if masked:
            L.check(lib.read_vgg_image_grad_masked(dxd.data_ptr(), mask.to(dev()).data_ptr(), n, H, W, sd.data_ptr(),
                                                   gr.out.data_ptr(), st))
        else:
            L.check(lib.read_vgg_image_grad(dxd.data_ptr(), n, H, W, sd.data_ptr(), gr.out.data_ptr(), st))
        torch.cuda.synchronize()
        gr.check("vgg_image_grad " + what)
        E.assert_same_bits(gr.out.view(n, 3, H, W), E.image_grad_replay(dx, std, mask), "vgg_image_grad " + what)
