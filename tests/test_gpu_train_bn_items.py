"""-m gpu: per-item train-mode BatchNorm (UNet.train_batchnorm = 'per_item'; blocks.py per_item=True, the *_items kernels of
csrc/bn_train.cu and csrc/conv_bwd.cu): each batch item normalised with its own statistics, the running statistics updated once per
item in item order.

* the statistics kernel: item i's mean / inv_std / scale / shift bit-identical to read_bn_batch_stats on item i's rows alone, the
  running statistics bit-identical to B such calls in a row, two runs bit-identical (300-sigma outliers included); the apply
  bit-identical to one call per item; the backward reduction and the corrected gate backward against float64 per item;
* every conv kind on B = 3 ragged shapes against a float64 per-item loop of the same modules;
* the whole net under 'bf16_all' in train(): the batched call bit-identical to the per-item loop of the same net (output and every
  running statistic), its gradients against float64 no worse than the loop's, 20 Adam steps, the inference engine rebuilt after a
  train-mode forward alone, and B = 1 bit-identical to 'batch'.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import _lib as L, blocks
from read_b200.unet import UNet, GatedConv
from test_gpu_train_bn import MULTI, SINGLE, STACKS, _check, _conv, _init, _net, _norms, _rel_cos, _rows, _stats

pytestmark = pytest.mark.gpu
ITEMS = 3


# ------------------------------------------------------------------ the kernels alone
def _stats_items(lib, gd, items, C, n_real, gamma, beta, rm, rv, eps=1e-5, momentum=0.1):
    P = gd.numel() // (C * items)
    out = torch.zeros((4, items, C), dtype=torch.float32, device=dev())    # mean, inv_std, scale, shift
    ws = torch.empty(lib.read_bn_workspace_bytes_items(items, C), dtype=torch.uint8, device=dev())
    L.check(lib.read_bn_batch_stats_items(gd.data_ptr(), items, P, C, n_real, gamma.data_ptr(), beta.data_ptr(), eps, momentum,
                                          rm.data_ptr(), rv.data_ptr(), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                                          out[3].data_ptr(), ws.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    return out.cpu()


@pytest.mark.parametrize("C,n_real,P,outlier", [(16, 3, 83 * 131, False), (64, 56, 45 * 67, False), (192, 192, 21 * 27, False),
                                                (256, 248, 13 * 19, False), (32, 32, 2, False), (64, 64, 45 * 67, True),
                                                (256, 256, 13 * 19, True)])
def test_per_item_stats_are_bit_identical_to_single_item_calls(C, n_real, P, outlier):
    lib = L.load()
    g = torch.Generator().manual_seed(C + P)
    items = []
    for i in range(ITEMS):                                                  # each item its own offsets and spread
        offs, std = torch.rand(C, generator=g) * 2 + 2.0 + i, torch.rand(C, generator=g) + 0.1
        x = torch.randn((P, C), generator=g) * std + offs
        x[:, 0] = 32.0 + 0.5 * torch.randn(P, generator=g)
        if outlier:
            x[i % P, 1:] += 300.0 * std[1:]
        x[:, n_real:] = 0.0
        items.append(x)
    gd = torch.cat(items).bfloat16().to(dev())
    gamma, beta = (torch.rand(n_real, generator=g) + 0.5).to(dev()), (torch.randn(n_real, generator=g) * 0.1).to(dev())
    rm0, rv0 = (torch.randn(n_real, generator=g) * 0.1).to(dev()), (torch.rand(n_real, generator=g) + 0.5).to(dev())
    runs = []
    for _ in range(2):
        rm, rv = rm0.clone(), rv0.clone()
        runs.append((_stats_items(lib, gd, ITEMS, C, n_real, gamma, beta, rm, rv), rm.cpu(), rv.cpu()))
    assert all(torch.equal(a, b) for a, b in zip(runs[0], runs[1])), "two runs differ"
    out, rm, rv = runs[0]
    rm_s, rv_s = rm0.clone(), rv0.clone()
    for i in range(ITEMS):                                                  # one call per item, in item order
        one = _stats(lib, gd[i * P:(i + 1) * P].contiguous(), C, n_real, gamma, beta, rm_s, rv_s)
        for j, k in enumerate((0, 1, 3, 4)):                                # mean, inv_std, scale, shift
            assert torch.equal(out[j, i], one[k]), (i, j)
    assert torch.equal(rm, rm_s.cpu()) and torch.equal(rv, rv_s.cpu())


@pytest.mark.parametrize("C,residual", [(16, False), (64, True), (192, True), (256, False)])
def test_per_item_apply_is_bit_identical_to_one_call_per_item(C, residual):
    lib = L.load()
    P = 29 * 35
    g = torch.Generator().manual_seed(C)
    gd = (torch.randn((ITEMS * P, C), generator=g) * 3).bfloat16().to(dev())
    scale, shift = torch.randn((ITEMS, C), generator=g).to(dev()), torch.randn((ITEMS, C), generator=g).to(dev())
    rd = torch.randn((ITEMS * P, C), generator=g).bfloat16().to(dev()) if residual else None
    y = torch.empty_like(gd)
    L.check(lib.read_bn_apply_items(gd.data_ptr(), ITEMS, P, C, scale.data_ptr(), shift.data_ptr(), L.ptr(rd), y.data_ptr(),
                                    L.stream_ptr()))
    want = torch.empty_like(gd)
    for i in range(ITEMS):
        r = slice(i * P, (i + 1) * P)
        L.check(lib.read_bn_apply(gd[r].data_ptr(), P, C, scale[i].data_ptr(), shift[i].data_ptr(),
                                  L.ptr(rd[r] if residual else None), want[r].data_ptr(), L.stream_ptr()))
    in_place = gd.clone()
    L.check(lib.read_bn_apply_items(in_place.data_ptr(), ITEMS, P, C, scale.data_ptr(), shift.data_ptr(), L.ptr(rd),
                                    in_place.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.equal(y, want) and torch.equal(in_place, want)


@pytest.mark.parametrize("C,elu", [(16, True), (32, False), (64, True), (128, False), (256, True)])
def test_per_item_backward_reduce_and_gate_backward_match_fp64(C, elu):
    lib = L.load()
    P = 21 * 27
    g = torch.Generator().manual_seed(C + int(elu))
    fmcat = torch.randn((ITEMS * P, 2 * C), generator=g)
    fmcat[P:2 * P] = fmcat[P:2 * P] * 2 + 0.5                               # items with different statistics
    fmcat = fmcat.bfloat16()
    dy = torch.randn((ITEMS * P, C), generator=g).bfloat16()
    bf, bm = torch.randn(C, generator=g) * 0.1, torch.randn(C, generator=g) * 0.1
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    f = fmcat[:, :C].double().requires_grad_(True)
    m = fmcat[:, C:].double().requires_grad_(True)
    bfd, bmd = bf.double().requires_grad_(True), bm.double().requires_grad_(True)
    gd_, bd_ = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    a = f + bfd
    gg = ((F.elu(a) if elu else a) * torch.sigmoid(m + bmd)).view(ITEMS, P, C)
    mu, var = gg.mean(1, keepdim=True), gg.var(1, unbiased=False, keepdim=True)
    inv = 1.0 / torch.sqrt(var + 1e-5)
    xhat = (gg - mu) * inv
    y = xhat * gd_ + bd_
    dyv = dy.double().view(ITEMS, P, C)
    want_sdy, want_sdx = dyv.sum(1), (dyv * xhat.detach()).sum(1)
    y.backward(dyv)
    mean32, inv32 = mu.detach().float().view(ITEMS, C), inv.detach().float().view(ITEMS, C)
    dv = lambda t: t.contiguous().to(dev())
    fm = dv(fmcat[:, blocks.fm_columns(C)])
    sums = torch.zeros((2, ITEMS, C), device=dev())
    red = torch.zeros((2, C), device=dev())
    dfm = torch.empty((ITEMS * P, 2 * C), dtype=torch.bfloat16, device=dev())
    scale = dv(gamma * inv32)
    dyd, bfd_, bmd_, mud, invd = dv(dy), dv(bf), dv(bm), dv(mean32), dv(inv32)
    st = L.stream_ptr()
    L.check(lib.read_bn_backward_reduce_items(dyd.data_ptr(), fm.data_ptr(), ITEMS, P, C, int(elu), bfd_.data_ptr(),
                                              bmd_.data_ptr(), mud.data_ptr(), invd.data_ptr(), sums[0].data_ptr(),
                                              sums[1].data_ptr(), st))
    L.check(lib.read_gate_backward_batch_stats_items(dyd.data_ptr(), fm.data_ptr(), ITEMS, P, C, int(elu), bfd_.data_ptr(),
                                                     bmd_.data_ptr(), scale.data_ptr(), mud.data_ptr(), invd.data_ptr(),
                                                     sums[0].data_ptr(), sums[1].data_ptr(), dfm.data_ptr(), red[0].data_ptr(),
                                                     red[1].data_ptr(), st))
    torch.cuda.synchronize()
    dcat = torch.empty((ITEMS * P, 2 * C))
    dcat[:, blocks.fm_columns(C)] = dfm.float().cpu()
    bf16 = lambda t: t.float().bfloat16().double()                      # [df | dm] are stored in bf16
    want_dfm = torch.cat([bf16(f.grad), bf16(m.grad)], 1)
    rels = {"[df|dm]": _rel_cos(dcat, want_dfm)[0], "sum_dy": _rel_cos(sums[0], want_sdy)[0],
            "sum_dy_xhat": _rel_cos(sums[1], want_sdx)[0], "dbias_f": _rel_cos(red[0], bfd.grad)[0],
            "dbias_m": _rel_cos(red[1], bmd.grad)[0], "dgamma": _rel_cos(sums[1].sum(0), gd_.grad)[0],
            "dbeta": _rel_cos(sums[0].sum(0), bd_.grad)[0]}
    print(f"\nper-item gate backward C={C} elu={elu}: " + ", ".join(f"{k} {v:.2e}" for k, v in rels.items()))
    assert rels["[df|dm]"] <= 2.7e-5, rels
    for k in ("sum_dy", "sum_dy_xhat", "dgamma", "dbeta"):
        assert rels[k] <= 9e-7, (k, rels)
    for k in ("dbias_f", "dbias_m"):
        assert rels[k] <= 1e-5, (k, rels)


# ------------------------------------------------------------------ the Functions against a float64 per-item loop
def _loop(ref, *xs):
    """The float64 reference: ``ref`` (a callable of NCHW tensors) on one item at a time, in item order."""
    return torch.cat([ref(*[x[i:i + 1] for x in xs]) for i in range(xs[0].shape[0])])


def _stack(C, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.nn.ModuleList([_init(GatedConv(C, C, 3, 1, elu=(i % 2 == 0)), C, g) for i in range(8)]).train()


@pytest.mark.parametrize("C,B,H,W", [(C, ITEMS, H, W) for C, _, H, W in STACKS])
def test_per_item_stack_matches_fp64_loop(C, B, H, W):
    mods = _stack(C, seed=C + H)
    g = torch.Generator().manual_seed(H * W)
    x, gy = torch.randn((B, C, H, W), generator=g), torch.randn((B, C, H, W), generator=g)
    ref = copy.deepcopy(mods).double()

    def stack(t):
        for r in range(0, 8, 2):
            t = ref[r + 1](ref[r](t)) + t
        return t
    xr = x.double().requires_grad_(True)
    t = _loop(stack, xr)
    t.backward(gy.double())
    ours = mods.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    yo = blocks.stack_forward(list(ours), xo, batch_stats=True, per_item=True)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    _check([("out",) + _rel_cos(yo, t), ("dx",) + _rel_cos(xo.grad, xr.grad)] + _rows(ours, ref), f"per-item stack C={C}")


@pytest.mark.parametrize("name,cin,cout,elu,B,H,W", SINGLE, ids=[c[0] for c in SINGLE])
def test_per_item_single_conv_matches_fp64_loop(name, cin, cout, elu, B, H, W):
    B = ITEMS
    m = _conv(cin, cout, 3, 1, elu, seed=cin + cout + H)
    g = torch.Generator().manual_seed(H * W + cout)
    x, gy = torch.randn((B, cin, H, W), generator=g), torch.randn((B, cout, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    xr = x.double().requires_grad_(True)
    yr = _loop(ref, xr)
    yr.backward(gy.double())
    ours = m.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    yo = blocks.gated_conv(ours, xo, batch_stats=True, name=name, per_item=True)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    _check([("out",) + _rel_cos(yo, yr), ("dx",) + _rel_cos(xo.grad, xr.grad)] + _rows([ours], [ref]), f"per-item {name}")


@pytest.mark.parametrize("C,H,W", [(64, 45, 67), (128, 29, 35), (256, 13, 19)])
@pytest.mark.parametrize("fused", [False, True], ids=["torch_sum", "residual"])
def test_per_item_fam_merge_matches_fp64_loop(C, H, W, fused):
    B = ITEMS
    m = _conv(C, C, 3, 1, False, seed=C + H)
    g = torch.Generator().manual_seed(C * H)
    a, b = torch.randn((B, C, H, W), generator=g), torch.rand((B, C, H, W), generator=g)
    gy = torch.randn((B, C, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    ar, br = a.double().requires_grad_(True), b.double().requires_grad_(True)
    yr = _loop(lambda p, q: p + ref(p * q), ar, br)
    yr.backward(gy.double())
    ours = m.to(dev())
    ao, bo = a.to(dev()).requires_grad_(True), b.to(dev()).requires_grad_(True)
    if fused:
        yo = blocks.gated_conv(ours, ao * bo, residual=ao, batch_stats=True, per_item=True)
    else:
        yo = ao + blocks.gated_conv(ours, ao * bo, batch_stats=True, per_item=True)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr), ("da",) + _rel_cos(ao.grad, ar.grad), ("db",) + _rel_cos(bo.grad, br.grad)]
    _check(rows + _rows([ours], [ref]), f"per-item FAM merge C={C} ({'residual' if fused else 'torch sum'})")


@pytest.mark.parametrize("name,srcs,cout,k,stride,elu,B,H,W", MULTI, ids=[c[0] for c in MULTI])
def test_per_item_1x1_and_stride2_conv_matches_fp64_loop(name, srcs, cout, k, stride, elu, B, H, W):
    B = ITEMS
    m = _conv(sum(srcs), cout, k, stride, elu, seed=sum(srcs) * 7 + cout + H)
    g = torch.Generator().manual_seed(H * W + cout)
    xs = [torch.randn((B, c, H, W), generator=g) for c in srcs]
    gy = torch.randn((B, cout, H // stride, W // stride), generator=g)
    ref = copy.deepcopy(m).double()
    xr = [x.double().requires_grad_(True) for x in xs]
    yr = _loop(lambda *ts: ref(torch.cat(ts, 1) if len(ts) > 1 else ts[0]), *xr)
    yr.backward(gy.double())
    ours = m.to(dev())
    xo = [x.to(dev()).requires_grad_(True) for x in xs]
    yo = blocks.gated_conv_srcs(ours, xo, name, batch_stats=True, per_item=True)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr)] + [(f"dx{i}",) + _rel_cos(a.grad, b.grad) for i, (a, b) in enumerate(zip(xo, xr))]
    _check(rows + _rows([ours], [ref]), f"per-item {name}")


# ------------------------------------------------------------------ the whole net
def _per_item_net(sd, tp):
    net = _net(sd, tp).train()
    net.train_batchnorm = 'per_item'
    return net


def _running(net):
    return [t.clone() for n in _norms(net) for t in (n.running_mean, n.running_var, n.num_batches_tracked)]


def test_full_net_batched_per_item_call_equals_the_loop(synth_sd):
    B, S = 4, 128
    g = torch.Generator().manual_seed(4)
    xs = [torch.rand((B, 8, S >> l, S >> l), generator=g).to(dev()) for l in range(4)]
    target = torch.rand((B, 3, S, S), generator=g).to(dev())
    batched = _per_item_net(synth_sd, 'bf16_all')
    loop = copy.deepcopy(batched)
    loop.train_batchnorm = 'batch'                               # the per-item loop as NetAndTexture runs it without the option
    loss_of = lambda out: F.l1_loss(out, target)

    def loop_out(net, xi):
        return torch.cat([net(*[x[i:i + 1] for x in xi]) for i in range(B)])

    # float64 reference: the per-item loop on torch's operators in double
    ref = _per_item_net(synth_sd, 'fp32').double()
    xr = [x.double().requires_grad_(True) for x in xs]
    F.l1_loss(loop_out(ref, xr), target.double()).backward()
    ref_grads = {n: p.grad for n, p in ref.named_parameters() if p.grad is not None}
    del ref

    res = {}
    for what, net, run in (("batched", batched, lambda n, xi: n(*xi)), ("loop", loop, loop_out)):
        xi = [x.clone().requires_grad_(True) for x in xs]
        out = run(net, xi)
        lv = loss_of(out)
        lv.backward()
        torch.cuda.synchronize()
        res[what] = (out.detach(), float(lv), [x.grad for x in xi], _running(net))
    assert torch.equal(res["batched"][0], res["loop"][0]), "the batched per-item output differs from the loop's"
    assert all(torch.equal(a, b) for a, b in zip(res["batched"][3], res["loop"][3])), "running statistics differ"

    def to64(net, dxs):
        pairs = [(p.grad, ref_grads[n]) for n, p in net.named_parameters() if p.grad is not None]
        total = _rel_cos(torch.cat([a.flatten() for a, _ in pairs]), torch.cat([b.flatten() for _, b in pairs]))[1]
        return [total] + [_rel_cos(dxs[l], xr[l].grad)[1] for l in range(4)]
    cb, cl = to64(batched, res["batched"][2]), to64(loop, res["loop"][2])
    print(f"\nagainst float64 (all parameters, descriptor levels 0-3): batched {[round(c, 6) for c in cb]}, "
          f"loop {[round(c, 6) for c in cl]}")
    for a, b in zip(cb, cl):
        assert 1.0 - a <= 2.0 * (1.0 - b) + 1e-4, (cb, cl)

    final, first = {}, {"batched": res["batched"][1], "loop": res["loop"][1]}
    for what, net, run in (("batched", batched, lambda n, xi: n(*xi)), ("loop", loop, loop_out)):
        net.zero_grad(set_to_none=True)
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        for _ in range(20):
            opt.zero_grad(set_to_none=True)
            loss_of(run(net, xs)).backward()
            opt.step()
        with torch.no_grad():
            final[what] = float(loss_of(run(net, xs)))
    descent = {k: first[k] - final[k] for k in final}
    print(f"after 20 Adam steps: final {final}, descent {descent}")
    assert descent["loop"] > 0 and descent["batched"] > 0, descent
    assert abs(final["batched"] - final["loop"]) <= 0.02 * final["loop"], final
    assert abs(descent["batched"] - descent["loop"]) <= 0.02 * descent["loop"], descent


@pytest.mark.parametrize("tp", ["fp32", "bf16", "bf16_all"])
def test_one_item_per_item_equals_batch(synth_sd, tp):
    g = torch.Generator().manual_seed(6)
    xs = [torch.rand((1, 8, 64 >> l, 64 >> l), generator=g).to(dev()) for l in range(4)]
    a, b = _per_item_net(synth_sd, tp), _net(synth_sd, tp).train()
    with torch.no_grad():
        ya, yb = a(*xs), b(*xs)
    torch.cuda.synchronize()
    assert torch.equal(ya, yb)
    assert all(torch.equal(p, q) for p, q in zip(_running(a), _running(b)))


def test_per_item_forward_alone_rebuilds_the_inference_engine(synth_sd):
    g = torch.Generator().manual_seed(8)
    xs = [torch.rand((2, 8, 128 >> l, 128 >> l), generator=g).to(dev()) for l in range(4)]
    net = _net(synth_sd, "bf16_all").eval()
    net.train_batchnorm = 'per_item'
    with torch.no_grad():
        before = net(*xs).clone()
        net.train()
        net(*xs)
        net.eval()
        after = net(*xs).clone()
    assert sorted(int(n.num_batches_tracked) for n in _norms(net)) == [0, 0] + [2] * 99     # ConvsOut.*: unused
    fresh = UNet()
    fresh.load_state_dict(net.state_dict(), strict=True)
    fresh.to(dev()).eval()
    with torch.no_grad():
        want = fresh(*xs).clone()
    torch.cuda.synchronize()
    assert not torch.equal(before, after) and torch.equal(after, want)


def test_per_item_one_pixel_per_item_raises_naming_the_layer(synth_sd):
    """At 16x16 feat_extract.7's output is 1 pixel per item: 'batch' accepts B = 2, 'per_item' raises where the loop raises."""
    xs = [torch.rand((2, 8, 16 >> l, 16 >> l)).to(dev()) for l in range(4)]
    _net(synth_sd, "bf16_all").train()(*xs)
    with pytest.raises(ValueError, match="feat_extract.7.*per item"):
        _per_item_net(synth_sd, "bf16_all")(*xs)
