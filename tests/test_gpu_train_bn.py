"""-m gpu: bf16 training of the gated convs with train-mode BatchNorm (batch statistics; read_b200/blocks.py batch_stats=True,
csrc/bn_train.cu and the batch-statistics gate backward of csrc/conv_bwd.cu) against float64 torch in train mode.

* each new kernel alone on the same bf16 operands: the statistics within relative error 1e-5 of float64 and bit-identical run to
  run (padded channels and a channel whose mean is far above its spread included), the apply within 1 bf16 ulp of the fp32
  formula, the backward reduction plus the corrected gate backward within relative L2 1e-3 of float64;
* every stack C, every single 3x3 conv (FAM both ways) and every 1x1 / stride-2 conv on ragged B = 2 shapes against float64
  autograd of the same modules in train mode: output, every gradient and the running statistics within relative L2 2e-2 and
  cosine 0.999, num_batches_tracked equal; a stack of alternating train / eval convs; a frozen conv; an in-place update;
* the whole net at 2 x 256 x 256 in train(), 'bf16' and 'bf16_all' against 'fp32': loss, gradients (looser bounds, see the
  test), 20 Adam steps, the first running-statistics update, and eval-mode inference afterwards bit-identical to a fresh net loaded from the trained state_dict;
* the packed-filter cache hands out exactly the filters a fresh pack makes and re-packs after an optimizer step.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import _lib as L, blocks
from read_b200.unet import UNet, GatedConv

pytestmark = pytest.mark.gpu


def _init(m, cout, g, k=3, cin=None):
    cin = cin or m.block["conv_f"].weight.shape[1]
    bound = 1.0 / (k * k * cin) ** 0.5
    with torch.no_grad():
        for name in ("conv_f", "conv_m"):
            conv = m.block[name]
            conv.weight.copy_((torch.rand(conv.weight.shape, generator=g) * 2 - 1) * bound)
            conv.bias.copy_((torch.rand(conv.bias.shape, generator=g) * 2 - 1) * bound)
        n = m.block["norm"]
        n.weight.copy_(torch.rand(cout, generator=g) + 0.5)
        n.bias.copy_(torch.randn(cout, generator=g) * 0.1)
        n.running_mean.copy_(torch.randn(cout, generator=g) * 0.1)
        n.running_var.copy_(torch.rand(cout, generator=g) + 0.5)
    return m


def _conv(cin, cout, k, stride, elu, seed):
    return _init(GatedConv(cin, cout, k, stride, elu), cout, torch.Generator().manual_seed(seed), k).train()


def _rel_cos(got, want):
    got, want = got.detach().double().flatten().cpu(), want.detach().double().flatten().cpu()
    rel = float((got - want).norm() / want.norm())
    cos = float(torch.dot(got, want) / (got.norm() * want.norm()))
    return rel, cos


def _check(rows, what):
    worst_rel = max(rows, key=lambda r: r[1])
    worst_cos = min(rows, key=lambda r: r[2])
    print(f"\n{what}: worst rel L2 {worst_rel[1]:.3e} ({worst_rel[0]}), worst cosine {worst_cos[2]:.6f} ({worst_cos[0]})")
    for name, rel, cos in rows:
        assert rel <= 2e-2 and cos >= 0.999, (name, rel, cos)


def _rows(ours, ref, prefix=""):
    """Parameter gradients and running statistics of the module lists ``ours`` / ``ref``; num_batches_tracked must agree."""
    rows = []
    for i, (mo, mr) in enumerate(zip(ours, ref)):
        for (pn, po), pr in zip(mo.named_parameters(), mr.parameters()):
            if po.grad is not None or pr.grad is not None:
                rows.append((f"{prefix}{i}.{pn}",) + _rel_cos(po.grad, pr.grad))
        no, nr = mo.block["norm"], mr.block["norm"]
        assert int(no.num_batches_tracked) == int(nr.num_batches_tracked), (i, no.num_batches_tracked, nr.num_batches_tracked)
        rows.append((f"{prefix}{i}.running_mean",) + _rel_cos(no.running_mean, nr.running_mean))
        rows.append((f"{prefix}{i}.running_var",) + _rel_cos(no.running_var, nr.running_var))
    return rows


# ------------------------------------------------------------------ the kernels alone
def _stats(lib, gd, C, n_real, gamma, beta, rm, rv, eps=1e-5, momentum=0.1):
    P = gd.numel() // C
    out = torch.zeros((5, C), dtype=torch.float32, device=dev())           # mean, inv_std, var, scale, shift
    ws = torch.empty(lib.read_bn_workspace_bytes(C), dtype=torch.uint8, device=dev())
    L.check(lib.read_bn_batch_stats(gd.data_ptr(), P, C, n_real, gamma.data_ptr(), beta.data_ptr(), eps, momentum, rm.data_ptr(),
                                    rv.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(),
                                    out[4].data_ptr(), ws.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("C,n_real,P,outlier", [(16, 3, 2 * 83 * 131, False), (64, 56, 2 * 45 * 67, False),
                                                (192, 192, 2 * 21 * 27, False), (256, 248, 2 * 13 * 19, False),
                                                (32, 32, 2, False), (64, 64, 2 * 45 * 67, True), (256, 256, 2 * 13 * 19, True)])
def test_batch_stats_kernel_matches_fp64_and_is_deterministic(C, n_real, P, outlier):
    lib = L.load()
    g = torch.Generator().manual_seed(C + P)
    offs = torch.rand(C, generator=g) * 2 + 2.0
    std = torch.rand(C, generator=g) + 0.1
    g_ = torch.randn((P, C), generator=g) * std + offs
    g_[:, 0] = 32.0 + 0.5 * torch.randn(P, generator=g)                     # mean far above the spread
    if outlier:                                                             # pixel 0 (the first a thread reads) far off the mean
        g_[0, 1:] += 300.0 * std[1:]
    g_[:, n_real:] = 0.0                                                    # padded channels
    gb = g_.bfloat16()
    gd = gb.to(dev())
    gamma, beta = torch.rand(n_real, generator=g) + 0.5, torch.randn(n_real, generator=g) * 0.1
    rm0, rv0 = torch.randn(n_real, generator=g) * 0.1, torch.rand(n_real, generator=g) + 0.5
    runs = []
    for _ in range(2):
        rm, rv = rm0.to(dev()), rv0.to(dev())
        out = _stats(lib, gd, C, n_real, gamma.to(dev()), beta.to(dev()), rm, rv)
        runs.append((out, rm.cpu(), rv.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1])), "two runs differ"
    out, rm, rv = runs[0]
    x = gb.double()
    mu, var = x.mean(0), x.var(0, unbiased=False)
    r = slice(0, n_real)
    err_mu = float(((out[0, r].double() - mu[r]).abs() / mu[r].abs()).max())
    zero = var[r] == 0                                                      # P = 2 and both values equal: exactly 0
    assert torch.equal(out[2, r][zero], torch.zeros(int(zero.sum())))
    err_var = float(((out[2, r].double() - var[r]).abs() / var[r])[~zero].max())
    print(f"\nbn_stats C={C} P={P} outlier={outlier}: worst relative error mean {err_mu:.2e}, variance {err_var:.2e}")
    assert err_mu <= 1e-5 and err_var <= 1e-5, (err_mu, err_var)
    inv = 1.0 / torch.sqrt(var + 1e-5)
    assert torch.allclose(out[1, r].double(), inv[r], rtol=1e-5)
    assert torch.allclose(out[3, r].double(), gamma.double() * inv[r], rtol=1e-5)
    assert torch.allclose(out[4, r].double(), beta.double() - mu[r] * gamma.double() * inv[r], rtol=1e-4, atol=1e-5)
    want_rm = 0.9 * rm0.double() + 0.1 * mu[r]
    want_rv = 0.9 * rv0.double() + 0.1 * var[r] * P / (P - 1)
    assert torch.allclose(rm.double(), want_rm, rtol=1e-5, atol=1e-6) and torch.allclose(rv.double(), want_rv, rtol=1e-5, atol=1e-6)
    if n_real < C:                                                          # padding: output 0, no NaN
        pad = out[:, n_real:]
        assert torch.equal(pad[0], torch.zeros(C - n_real)) and torch.equal(pad[2], torch.zeros(C - n_real))
        assert torch.equal(pad[3], torch.zeros(C - n_real)) and torch.equal(pad[4], torch.zeros(C - n_real))
        assert torch.allclose(pad[1].double(), torch.full((C - n_real,), 1e-5).double().rsqrt(), rtol=1e-6)


@pytest.mark.parametrize("C,residual", [(16, False), (64, True), (192, True), (256, False)])
def test_bn_apply_is_within_one_ulp_of_the_fp32_formula(C, residual):
    lib = L.load()
    P = 2 * 29 * 35
    g = torch.Generator().manual_seed(C)
    gb = (torch.randn((P, C), generator=g) * 3).bfloat16()
    scale, shift = torch.randn(C, generator=g), torch.randn(C, generator=g)
    rb = (torch.randn((P, C), generator=g)).bfloat16() if residual else None
    want = gb.float() * scale + shift + (rb.float() if residual else 0.0)
    want = want.bfloat16()
    for in_place in (False, True):
        gd = gb.to(dev())
        y = gd if in_place else torch.empty_like(gd)
        sd, hd, rd = scale.to(dev()), shift.to(dev()), rb.to(dev()) if residual else None
        L.check(lib.read_bn_apply(gd.data_ptr(), P, C, sd.data_ptr(), hd.data_ptr(), L.ptr(rd), y.data_ptr(), L.stream_ptr()))
        torch.cuda.synchronize()
        got = y.cpu().float()
        mag = torch.maximum(got.abs(), want.float().abs())
        ulp = torch.ldexp(torch.ones_like(mag), torch.frexp(mag).exponent - 8)   # bf16: 8 significant bits
        worst = float(((got - want.float()).abs() / ulp).max())
        print(f"\nbn_apply C={C} residual={residual} in place={in_place}: worst {worst:.2f} ulp")
        assert worst <= 1.0, worst


@pytest.mark.parametrize("C,elu", [(16, True), (32, False), (64, True), (128, False), (256, True)])
def test_backward_reduce_and_corrected_gate_backward_match_fp64(C, elu):
    lib = L.load()
    P = 2 * 21 * 27
    g = torch.Generator().manual_seed(C + int(elu))
    fmcat = (torch.randn((P, 2 * C), generator=g)).bfloat16()
    dy = torch.randn((P, C), generator=g).bfloat16()
    bf, bm = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    f = fmcat[:, :C].double().requires_grad_(True)
    m = fmcat[:, C:].double().requires_grad_(True)
    bfd, bmd = bf.double().requires_grad_(True), bm.double().requires_grad_(True)
    gd_, bd_ = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    a = f + bfd
    gg = (F.elu(a) if elu else a) * torch.sigmoid(m + bmd)
    mu, var = gg.mean(0), gg.var(0, unbiased=False)
    inv = 1.0 / torch.sqrt(var + 1e-5)
    y = (gg - mu) * inv * gd_ + bd_
    y.backward(dy.double())
    mean32, inv32 = mu.detach().float(), inv.detach().float()
    dv = lambda t: t.contiguous().to(dev())
    fm = dv(fmcat[:, blocks.fm_columns(C)])
    red = torch.zeros((4, C), device=dev())
    dfm = torch.empty((P, 2 * C), dtype=torch.bfloat16, device=dev())
    scale = dv(gamma * inv32)
    dyd, bfd_, bmd_, mud, invd = dv(dy), dv(bf), dv(bm), dv(mean32), dv(inv32)
    st = L.stream_ptr()
    L.check(lib.read_bn_backward_reduce(dyd.data_ptr(), fm.data_ptr(), P, C, int(elu), bfd_.data_ptr(), bmd_.data_ptr(),
                                        mud.data_ptr(), invd.data_ptr(), red[3].data_ptr(), red[2].data_ptr(), st))
    L.check(lib.read_gate_backward_batch_stats(dyd.data_ptr(), fm.data_ptr(), P, C, int(elu), bfd_.data_ptr(), bmd_.data_ptr(),
                                               scale.data_ptr(), mud.data_ptr(), invd.data_ptr(), red[3].data_ptr(),
                                               red[2].data_ptr(), dfm.data_ptr(), red[0].data_ptr(), red[1].data_ptr(), st))
    torch.cuda.synchronize()
    dcat = torch.empty((P, 2 * C))
    dcat[:, blocks.fm_columns(C)] = dfm.float().cpu()
    bf16 = lambda t: t.float().bfloat16().double()                      # [df | dm] are stored in bf16
    rels = {"df": _rel_cos(dcat[:, :C], bf16(f.grad))[0], "dm": _rel_cos(dcat[:, C:], bf16(m.grad))[0],
            "dbias_f": _rel_cos(red[0], bfd.grad)[0], "dbias_m": _rel_cos(red[1], bmd.grad)[0],
            "dgamma": _rel_cos(red[2], gd_.grad)[0], "dbeta": _rel_cos(red[3], bd_.grad)[0]}
    print(f"\nbatch-statistics gate backward C={C} elu={elu}: " + ", ".join(f"{k} {v:.2e}" for k, v in rels.items()))
    for k, v in rels.items():
        assert v <= 1e-3, (k, v)


# ------------------------------------------------------------------ the Functions against float64 autograd in train mode
STACKS = [(32, 2, 37, 45), (64, 2, 29, 35), (128, 2, 21, 27), (256, 2, 13, 19)]


def _stack(C, seed, modes=None):
    g = torch.Generator().manual_seed(seed)
    mods = torch.nn.ModuleList([_init(GatedConv(C, C, 3, 1, elu=(i % 2 == 0)), C, g) for i in range(8)]).train()
    for m, train in zip(mods, modes or [True] * 8):
        m.train(train)
    return mods


def _run_stack(mods, C, B, H, W, what):
    g = torch.Generator().manual_seed(H * W)
    x, gy = torch.randn((B, C, H, W), generator=g), torch.randn((B, C, H, W), generator=g)
    ref = copy.deepcopy(mods).double()
    xr = x.double().requires_grad_(True)
    t = xr
    for r in range(0, 8, 2):
        t = ref[r + 1](ref[r](t)) + t
    t.backward(gy.double())
    ours = mods.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    yo = blocks.stack_forward(list(ours), xo, batch_stats=True)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    _check([("out",) + _rel_cos(yo, t), ("dx",) + _rel_cos(xo.grad, xr.grad)] + _rows(ours, ref), what)


@pytest.mark.parametrize("C,B,H,W", STACKS)
def test_train_mode_stack_matches_fp64(C, B, H, W):
    _run_stack(_stack(C, seed=C + H), C, B, H, W, f"train-mode stack C={C} {B}x{H}x{W}")


def test_stack_of_alternating_train_and_eval_convs_matches_fp64():
    modes = [i % 2 == 0 for i in range(8)]
    _run_stack(_stack(64, seed=5, modes=modes), 64, 2, 29, 35, "stack C=64, train / eval alternating")


# (layer, cin, cout, elu, B, H, W)
SINGLE = [("feat_extract.0", 8, 32, True, 2, 83, 131), ("feat_extract.5", 32, 3, False, 2, 83, 131),
          ("SCM2.main.0", 8, 16, True, 2, 45, 67), ("SCM1.main.0", 8, 32, True, 2, 29, 35), ("SCM0.main.0", 8, 64, True, 2, 21, 27),
          ("SCM2.main.2", 32, 32, True, 2, 45, 67), ("SCM1.main.2", 64, 64, True, 2, 29, 35), ("SCM0.main.2", 128, 128, True, 2, 13, 19),
          ("AFFs.0.conv.1", 32, 32, False, 2, 37, 45), ("AFFs.1.conv.1", 64, 64, False, 2, 29, 35),
          ("AFFs.2.conv.1", 128, 128, False, 2, 21, 27)]


@pytest.mark.parametrize("name,cin,cout,elu,B,H,W", SINGLE, ids=[c[0] for c in SINGLE])
def test_train_mode_single_conv_matches_fp64(name, cin, cout, elu, B, H, W):
    m = _conv(cin, cout, 3, 1, elu, seed=cin + cout + H)
    g = torch.Generator().manual_seed(H * W + cout)
    x, gy = torch.randn((B, cin, H, W), generator=g), torch.randn((B, cout, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    xr = x.double().requires_grad_(True)
    yr = ref(xr)
    yr.backward(gy.double())
    ours = m.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    yo = blocks.gated_conv(ours, xo, batch_stats=True, name=name)
    assert yo.shape == (B, cout, H, W)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    _check([("out",) + _rel_cos(yo, yr), ("dx",) + _rel_cos(xo.grad, xr.grad)] + _rows([ours], [ref]),
           f"train-mode {name} {cin}->{cout} {B}x{H}x{W}")


@pytest.mark.parametrize("C,B,H,W", [(64, 2, 45, 67), (128, 2, 29, 35), (256, 2, 13, 19)])
@pytest.mark.parametrize("fused", [False, True], ids=["torch_sum", "residual"])
def test_train_mode_fam_merge_matches_fp64(C, B, H, W, fused):
    m = _conv(C, C, 3, 1, False, seed=C + H)
    g = torch.Generator().manual_seed(C * H)
    a, b = torch.randn((B, C, H, W), generator=g), torch.rand((B, C, H, W), generator=g)
    gy = torch.randn((B, C, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    ar, br = a.double().requires_grad_(True), b.double().requires_grad_(True)
    yr = ar + ref(ar * br)
    yr.backward(gy.double())
    ours = m.to(dev())
    ao, bo = a.to(dev()).requires_grad_(True), b.to(dev()).requires_grad_(True)
    if fused:
        yo = blocks.gated_conv(ours, ao * bo, residual=ao, batch_stats=True)
    else:
        yo = ao + blocks.gated_conv(ours, ao * bo, batch_stats=True)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr), ("da",) + _rel_cos(ao.grad, ar.grad), ("db",) + _rel_cos(bo.grad, br.grad)]
    _check(rows + _rows([ours], [ref]), f"train-mode FAM merge C={C} ({'residual' if fused else 'torch sum'})")


# (layer, sources' channels, Cout, k, stride, ELU, B, H, W of the input)
MULTI = [("feat_extract.1", [32], 64, 3, 2, True, 2, 86, 134), ("feat_extract.2", [64], 128, 3, 2, True, 2, 46, 70),
         ("feat_extract.6", [128], 256, 3, 2, True, 2, 26, 38),
         ("feat_extract.4", [64], 32, 4, 2, True, 2, 86, 134), ("feat_extract.3", [128], 64, 4, 2, True, 2, 46, 70),
         ("feat_extract.7", [256], 128, 4, 2, True, 2, 26, 38),
         ("AFFs.0.conv.0", [32, 64, 128, 256], 32, 1, 1, True, 2, 37, 45),
         ("AFFs.1.conv.0", [32, 64, 128, 256], 64, 1, 1, True, 2, 29, 35),
         ("AFFs.2.conv.0", [32, 64, 128, 256], 128, 1, 1, True, 2, 21, 27),
         ("Convs.0", [128, 128], 128, 1, 1, True, 2, 21, 27), ("Convs.1", [64, 64], 64, 1, 1, True, 2, 29, 35),
         ("Convs.2", [32, 32], 32, 1, 1, True, 2, 37, 45),
         ("SCM2.main.1", [16], 32, 1, 1, True, 2, 45, 67), ("SCM1.main.1", [32], 64, 1, 1, True, 2, 29, 35),
         ("SCM0.main.1", [64], 128, 1, 1, True, 2, 13, 19),
         ("SCM2.main.3", [32], 56, 1, 1, True, 2, 45, 67), ("SCM1.main.3", [64], 120, 1, 1, True, 2, 29, 35),
         ("SCM0.main.3", [128], 248, 1, 1, True, 2, 13, 19),
         ("SCM2.conv", [64], 64, 1, 1, False, 2, 45, 67), ("SCM1.conv", [128], 128, 1, 1, False, 2, 29, 35),
         ("SCM0.conv", [256], 256, 1, 1, False, 2, 13, 19)]


@pytest.mark.parametrize("name,srcs,cout,k,stride,elu,B,H,W", MULTI, ids=[c[0] for c in MULTI])
def test_train_mode_1x1_and_stride2_conv_matches_fp64(name, srcs, cout, k, stride, elu, B, H, W):
    m = _conv(sum(srcs), cout, k, stride, elu, seed=sum(srcs) * 7 + cout + H)
    g = torch.Generator().manual_seed(H * W + cout)
    xs = [torch.randn((B, c, H, W), generator=g) for c in srcs]
    Ho, Wo = H // stride, W // stride
    gy = torch.randn((B, cout, Ho, Wo), generator=g)
    ref = copy.deepcopy(m).double()
    xr = [x.double().requires_grad_(True) for x in xs]
    yr = ref(torch.cat(xr, 1) if len(xr) > 1 else xr[0])
    yr.backward(gy.double())
    ours = m.to(dev())
    xo = [x.to(dev()).requires_grad_(True) for x in xs]
    yo = blocks.gated_conv_srcs(ours, xo, name, batch_stats=True)
    assert yo.shape == (B, cout, Ho, Wo)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr)] + [(f"dx{i}",) + _rel_cos(a.grad, b.grad) for i, (a, b) in enumerate(zip(xo, xr))]
    _check(rows + _rows([ours], [ref]), f"train-mode {name} {srcs}->{cout} k={k} s={stride} {B}x{H}x{W}")


def test_frozen_train_mode_conv_gives_input_gradients_and_updates_running_stats():
    m = _conv(64, 128, 4, 2, True, seed=11)
    m.requires_grad_(False)
    ref = copy.deepcopy(m).double()
    g = torch.Generator().manual_seed(12)
    x, gy = torch.randn((2, 64, 38, 46), generator=g), torch.randn((2, 128, 19, 23), generator=g)
    xr = x.double().requires_grad_(True)
    ref(xr).backward(gy.double())
    ours = m.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    blocks.gated_conv_srcs(ours, [xo], batch_stats=True).backward(gy.to(dev()))
    torch.cuda.synchronize()
    assert all(p.grad is None for p in ours.parameters())
    _check([("dx",) + _rel_cos(xo.grad, xr.grad)] + _rows([ours], [ref]), "frozen train-mode conv 64->128 k=4 s=2")


def test_in_place_parameter_update_before_backward_raises():
    m = _conv(32, 32, 3, 1, True, seed=9).to(dev())
    x = torch.randn((1, 32, 20, 24), device=dev(), requires_grad=True)
    y = blocks.gated_conv(m, x, batch_stats=True)
    with torch.no_grad():
        m.block["norm"].weight.mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


# ------------------------------------------------------------------ the whole net
def _net(sd, tp):
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.to(dev())
    net.train_precision = tp
    return net


def _norms(net):
    return [m for m in net.modules() if isinstance(m, torch.nn.BatchNorm2d)]


def test_full_net_train_mode_bf16_tracks_fp32(synth_sd):
    g = torch.Generator().manual_seed(3)
    xs = [torch.rand((2, 8, 256 >> l, 256 >> l), generator=g).to(dev()) for l in range(4)]
    target = torch.rand((2, 3, 256, 256), generator=g).to(dev())
    nets = {tp: _net(synth_sd, tp) for tp in ("fp32", "bf16", "bf16_all")}
    # float64 reference: torch's operators in double, train mode, the same batch
    ref = _net(synth_sd, "fp32").double().train()
    xr = [x.double().requires_grad_(True) for x in xs]
    F.l1_loss(ref(*xr), target.double()).backward()
    ref_grads = {n: p.grad for n, p in ref.named_parameters() if p.grad is not None}
    ref_dx = [x.grad for x in xr]
    del ref
    with torch.no_grad():                                    # an inference engine built before training, to be invalidated
        nets["bf16_all"].eval()(*xs)
    loss, dxs = {}, {}
    rs0 = [(n.running_mean.clone(), n.running_var.clone()) for n in _norms(nets["fp32"])]
    for tp, net in nets.items():
        net.train()
        xi = [x.clone().requires_grad_(True) for x in xs]
        lv = F.l1_loss(net(*xi), target)
        lv.backward()
        loss[tp], dxs[tp] = lv.detach(), [x.grad for x in xi]
    torch.cuda.synchronize()
    # distance of every precision's gradients from float64 (the fp32 path runs torch's defaults: cuDNN convolutions in TF32)
    to64 = {}
    for tp, net in nets.items():
        pairs = [(p.grad, ref_grads[n]) for n, p in net.named_parameters() if p.grad is not None]
        worst64 = min(_rel_cos(a, b)[1] for a, b in pairs)
        total64 = _rel_cos(torch.cat([a.flatten() for a, _ in pairs]), torch.cat([b.flatten() for _, b in pairs]))[1]
        d64 = min(_rel_cos(dxs[tp][l], ref_dx[l])[1] for l in range(4))
        to64[tp] = (worst64, total64, d64)
        print(f"\n{tp} against float64: worst parameter cosine {worst64:.5f}, all parameters together {total64:.6f}, "
              f"worst descriptor level {d64:.5f}")
    for tp in ("bf16", "bf16_all"):
        # bf16 keeps 8 significant bits where TF32 keeps 11: rounding errors 8x larger, 1 - cosine about 64x larger.  Bound
        # bf16's loss of cosine against float64 by 64x the fp32 path's (its own bound 0.99 per parameter)
        for i, what in enumerate(("worst parameter", "all parameters", "worst descriptor level")):
            assert 1.0 - to64[tp][i] <= 64.0 * (1.0 - to64["fp32"][i]) + 1e-4, (tp, what, to64[tp][i], to64["fp32"][i])
        assert to64["fp32"][0] >= 0.99, to64["fp32"]
        rel = abs(float(loss[tp]) - float(loss["fp32"])) / float(loss["fp32"])
        worst, coss, flat_a, flat_b = (1.0, None), [], [], []
        for (name, pa), pb in zip(nets["fp32"].named_parameters(), nets[tp].parameters()):
            assert (pa.grad is None) == (pb.grad is None), name
            if pa.grad is None:
                continue
            cos = _rel_cos(pb.grad, pa.grad)[1]
            worst = min(worst, (cos, name))
            coss.append(cos)
            flat_a.append(pa.grad.flatten())
            flat_b.append(pb.grad.flatten())
        total = _rel_cos(torch.cat(flat_b), torch.cat(flat_a))[1]
        dcos = [_rel_cos(dxs[tp][l], dxs["fp32"][l])[1] for l in range(4)]
        print(f"\ntrain mode 2x256x256 {tp}: loss fp32 {float(loss['fp32']):.6f} {tp} {float(loss[tp]):.6f} (rel {rel:.2e}), "
              f"worst grad cosine {worst[0]:.5f} ({worst[1]}), {sum(c < 0.99 for c in coss)} of {len(coss)} below 0.99, "
              f"all parameters together {total:.6f}, descriptor cosines {[round(c, 5) for c in dcos]}")
        # the first batch's running-statistics updates (the same weights in every precision): the change of every norm's
        # running mean / variance against fp32's
        worst_rs = 1.0
        for (m0, v0), a, b in zip(rs0, _norms(nets["fp32"]), _norms(nets[tp])):
            if int(a.num_batches_tracked) == 0:                      # ConvsOut.*: unused by forward
                continue
            worst_rs = min(worst_rs, _rel_cos(b.running_mean - m0, a.running_mean - m0)[1],
                           _rel_cos(b.running_var - v0, a.running_var - v0)[1])
        print(f"{tp}: worst cosine of the first running-statistics update against fp32 {worst_rs:.6f}")
        assert worst_rs >= 0.999, (tp, worst_rs)
        assert rel <= 1e-2, (tp, rel)
        # Batch statistics amplify rounding through the 99 layers; the per-parameter distance is bounded against float64 above
        # (the worst single parameter against fp32 moves run to run with the order of the backward's atomics).  Against fp32:
        # 0.95 for all parameters together and per descriptor level.  Each conv alone matches float64 within the limits of the
        # tests above, and the 20 Adam steps below track fp32 within 5 %.
        assert total >= 0.95 and min(dcos) >= 0.95, (tp, worst, total, dcos)

    final = {}
    for tp, net in nets.items():
        net.zero_grad(set_to_none=True)
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        for _ in range(20):
            opt.zero_grad(set_to_none=True)
            lv = F.l1_loss(net(*xs), target)
            lv.backward()
            opt.step()
        with torch.no_grad():
            final[tp] = float(F.l1_loss(net(*xs), target))            # still train(): one more batch-statistics forward
    descent = {tp: float(loss[tp]) - final[tp] for tp in final}
    print(f"after 20 Adam steps: final {final}, descent {descent}")
    for tp in ("bf16", "bf16_all"):
        assert descent["fp32"] > 0 and descent[tp] > 0, descent
        assert abs(final[tp] - final["fp32"]) <= 0.05 * final["fp32"], final
        assert abs(descent[tp] - descent["fp32"]) <= 0.05 * descent["fp32"], descent
        nf, nb = _norms(nets["fp32"]), _norms(nets[tp])
        assert len(nb) == 101
        worst = 1.0
        for a, b in zip(nf, nb):
            if int(a.num_batches_tracked) == 0:                      # ConvsOut.*: unused by forward
                assert int(b.num_batches_tracked) == 0
                continue
            assert int(a.num_batches_tracked) == int(b.num_batches_tracked) == 22
            worst = min(worst, _rel_cos(b.running_mean, a.running_mean)[1], _rel_cos(b.running_var, a.running_var)[1])
        # after 20 steps the weights differ between precisions (the trajectories are within 5 %, above), and so do the statistics
        print(f"{tp}: after 20 steps, worst running-statistics cosine against fp32 {worst:.6f} (not bounded)")

    net = nets["bf16_all"].eval()
    fresh = UNet()
    fresh.load_state_dict(net.state_dict(), strict=True)
    fresh.to(dev()).eval()
    with torch.no_grad():
        a, b = net(*xs).clone(), fresh(*xs).clone()
    torch.cuda.synchronize()
    assert torch.equal(a, b), "inference after training does not match a net loaded from the trained state_dict"


def test_filter_cache_changes_no_result(synth_sd):
    """The cache hands out the same filters a fresh pack makes: every cached filter tensor (the forward's, and the backward's
    packed with them) equals a re-pack of the live weights bit for bit, after a forward and after an optimizer step (which must
    re-pack); and the whole net's training forward is bit-identical with the cache and without it.  Gradients are not compared
    bit for bit: the backward accumulates bias and weight gradients with fp32 atomics, whose order varies run to run."""
    g = torch.Generator().manual_seed(5)
    xs = [torch.rand((2, 8, 128 >> l, 128 >> l), generator=g).to(dev()) for l in range(4)]
    outs = []
    for cached in (True, False):
        blocks.clear_filter_cache()
        blocks.cache_filters = cached
        try:
            net = _net(synth_sd, 'bf16_all').eval()
            for _ in range(2):                                       # the second call runs on the cached filters
                out = net(*xs)                                       # parameters need grad: the training (autograd) path
            outs.append(out.detach().clone())
        finally:
            blocks.cache_filters = True
    assert torch.equal(outs[0], outs[1])

    # cached filters against a fresh pack, before and after an optimizer step
    net = _net(synth_sd, 'bf16_all').eval()
    opt = torch.optim.SGD(net.parameters(), lr=1e-3)
    blocks.clear_filter_cache()
    for step in range(2):                                           # step 1 runs after an optimizer step: every conv re-packs
        net.zero_grad(set_to_none=True)
        net(*xs).square().mean().backward()
        n_checked = 0
        for mod, (key, pk) in list(blocks._FILTERS.items()):
            wf, wm = mod.block["conv_f"].weight, mod.block["conv_m"].weight
            srcs = None if key[8] is None else [torch.empty((2, 16, 16, c), dtype=torch.bfloat16, device=dev()) for c in key[8]]
            assert key == blocks.filter_key(mod, wf, wm, key[6], srcs), "a cached entry for stale weights"
            blocks.cache_filters = False
            try:
                fresh = blocks._packed(mod, wf, wm, key[6], srcs)
            finally:
                blocks.cache_filters = True
            assert set(pk) == set(fresh), (set(pk), set(fresh))
            for name, t in pk.items():
                f = fresh[name]
                ts, fs = (t, f) if isinstance(t, list) else ([t], [f])
                assert len(ts) == len(fs) and all((a is None and b is None) or torch.equal(a, b) for a, b in zip(ts, fs)), name
            n_checked += 1
        assert n_checked == 99
        opt.step()


def test_running_statistics_updates_alone_rebuild_the_inference_engine(synth_sd):
    """A train-mode forward without any optimizer step changes only the running statistics (and num_batches_tracked); the cached
    inference engine must see them: eval() output afterwards equals a fresh net loaded from the state_dict, and differs from the
    output before."""
    g = torch.Generator().manual_seed(8)
    xs = [torch.rand((1, 8, 128 >> l, 128 >> l), generator=g).to(dev()) for l in range(4)]
    net = _net(synth_sd, "bf16_all").eval()
    with torch.no_grad():
        before = net(*xs).clone()                                    # builds and caches the engine
        params = [p.clone() for p in net.parameters()]
        net.train()
        net(*xs)                                                     # batch statistics: running-statistics updates only
        net.eval()
        after = net(*xs).clone()
    assert all(torch.equal(a, b) for a, b in zip(params, net.parameters()))
    assert sorted(int(n.num_batches_tracked) for n in _norms(net)) == [0, 0] + [1] * 99     # ConvsOut.*: unused
    fresh = UNet()
    fresh.load_state_dict(net.state_dict(), strict=True)
    fresh.to(dev()).eval()
    with torch.no_grad():
        want = fresh(*xs).clone()
    torch.cuda.synchronize()
    assert not torch.equal(before, after), "the running-statistics update did not reach the inference engine"
    assert torch.equal(after, want)
