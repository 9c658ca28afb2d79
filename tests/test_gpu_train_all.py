"""-m gpu: bf16 training of the 21 gated 1x1 and stride-2 convs under train_precision='bf16_all' (read_b200/blocks.py:
gated_conv_srcs, csrc/conv_bwd.cu) against torch autograd.

Tolerances as for the block stacks (tests/test_gpu_train_blocks.py):
* one conv of every row (every C) of the 1x1 / stride-2 convs, on ragged B = 2 shapes (stride 2 at even H, W that are not
  multiples of 16 or 32, 1x1 at odd H, W), against float64 autograd of the same module with the same torch-side concat and slice:
  the output and every gradient (each source, conv_f / conv_m weight and bias, BatchNorm weight and bias) within relative L2 error
  2e-2 and cosine >= 0.999;
* each new kernel alone on the same bf16 operands within relative L2 1e-3: the weight-gradient instances against
  torch.nn.grad.conv2d_weight, the stride-2 and 1x1 input gradients against conv2d_input;
* the whole net at 2 x 256 x 256, 'bf16_all' against 'fp32': loss within 1e-2, every parameter gradient and each descriptor level's
  gradient at cosine >= 0.99, and 20 Adam steps that lower both losses alike (final loss and descent within 5 %).
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import _lib as L, blocks, ops
from read_b200.unet import UNet, GatedConv

pytestmark = pytest.mark.gpu


def _conv(cin, cout, k, stride, elu, seed):
    g = torch.Generator().manual_seed(seed)
    m = GatedConv(cin, cout, k, stride, elu)
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
    return m.eval()


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


# (layer, sources' channels, Cout, k, stride, ELU, B, H, W of the input)
CONVS = [("feat_extract.1", [32], 64, 3, 2, True, 2, 86, 134), ("feat_extract.2", [64], 128, 3, 2, True, 2, 46, 70),
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


@pytest.mark.parametrize("name,srcs,cout,k,stride,elu,B,H,W", CONVS, ids=[c[0] for c in CONVS])
def test_conv_forward_and_grads_match_fp64_autograd(name, srcs, cout, k, stride, elu, B, H, W):
    m = _conv(sum(srcs), cout, k, stride, elu, seed=sum(srcs) * 7 + cout + H)
    g = torch.Generator().manual_seed(H * W + cout)
    xs = [torch.randn((B, c, H, W), generator=g) for c in srcs]
    Ho, Wo = (H // 2, W // 2) if stride == 2 else (H, W)
    gy = torch.randn((B, cout, Ho, Wo), generator=g)
    ref = copy.deepcopy(m).double()
    xr = [x.double().requires_grad_(True) for x in xs]
    yr = ref(torch.cat(xr, 1) if len(xr) > 1 else xr[0])
    yr.backward(gy.double())
    ours = m.to(dev())
    xo = [x.to(dev()).requires_grad_(True) for x in xs]
    yo = blocks.gated_conv_srcs(ours, xo, name)
    assert yo.shape == (B, cout, Ho, Wo)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr)] + [(f"dx{i}",) + _rel_cos(a.grad, b.grad) for i, (a, b) in enumerate(zip(xo, xr))]
    for (pn, po), pr in zip(ours.named_parameters(), ref.parameters()):
        assert po.grad.shape == po.shape, pn
        rows.append((pn,) + _rel_cos(po.grad, pr.grad))
    _check(rows, f"{name} {srcs}->{cout} k={k} s={stride} {B}x{H}x{W}")


def _operands(C, Ho, Wo, B, seed):
    """[df | dm] in channel order (bf16, NHWC) and the kernels' RAW column order of it on the device."""
    g = torch.Generator().manual_seed(seed)
    dcat = torch.randn((B, Ho, Wo, 2 * C), generator=g).bfloat16()
    return dcat, dcat[..., blocks.fm_columns(C)].contiguous().to(dev())


def _rel(got, want):
    return float((got.double() - want).norm() / want.norm())


@pytest.mark.parametrize("cin,C,k,stride,B,H,W", [(16, 32, 1, 1, 2, 37, 45), (64, 128, 1, 1, 2, 21, 27), (32, 64, 3, 2, 2, 86, 70),
                                                  (128, 256, 3, 2, 2, 26, 38), (64, 32, 4, 2, 2, 86, 70), (256, 128, 4, 2, 2, 26, 38)])
def test_wgrad_matches_conv2d_weight_on_bf16_operands(cin, C, k, stride, B, H, W):
    lib = L.load()
    Ho, Wo = H // stride, W // stride
    dcat, dfm = _operands(C, Ho, Wo, B, seed=C + k)
    x = torch.randn((B, H, W, cin), generator=torch.Generator().manual_seed(cin)).bfloat16()
    dwf = torch.zeros((C, cin, k, k), device=dev())
    dwm = torch.zeros_like(dwf)
    xd = x.to(dev())
    L.check(lib.read_conv_wgrad(dfm.data_ptr(), xd.data_ptr(), B, H, W, Ho, Wo, C, cin, k, stride, dwf.data_ptr(), dwm.data_ptr(),
                                L.stream_ptr()))
    want = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (2 * C, cin, k, k), dcat.double().permute(0, 3, 1, 2),
                                       stride=stride, padding=(k - 1) // 2)
    rel = _rel(torch.cat([dwf, dwm], 0).cpu(), want)
    print(f"\nwgrad k={k} s={stride} {cin}->{C}: rel L2 {rel:.3e}")
    assert rel <= 1e-3, rel


@pytest.mark.parametrize("cin,C,k,B,H,W", [(32, 64, 3, 2, 86, 134), (64, 128, 3, 2, 46, 70), (128, 256, 3, 2, 26, 38),
                                           (64, 32, 4, 2, 86, 134), (128, 64, 4, 2, 46, 70), (256, 128, 4, 2, 26, 38)])
def test_stride2_dgrad_matches_conv2d_input_on_bf16_operands(cin, C, k, B, H, W):
    m = _conv(cin, C, k, 2, True, seed=C + k).to(dev())
    xs = [torch.zeros((B, H, W, cin), dtype=torch.bfloat16, device=dev())]
    fc = blocks.FoldedConv(m, *blocks.stack_params([m]), srcs=xs)
    dcat, dfm = _operands(C, H // 2, W // 2, B, seed=cin)
    dx = torch.empty((B, H, W, cin), dtype=torch.bfloat16, device=dev())
    L.check(L.load().read_conv_dgrad_s2(dfm.data_ptr(), blocks.dgrad_s2_filters(fc).data_ptr(), B, H // 2, W // 2, C, cin, k,
                                        dx.data_ptr(), L.stream_ptr()))
    w = torch.cat([m.block["conv_f"].weight, m.block["conv_m"].weight], 0).detach().cpu().bfloat16().double()
    want = torch.nn.grad.conv2d_input((B, cin, H, W), w, dcat.double().permute(0, 3, 1, 2), stride=2, padding=1)
    want = want.permute(0, 2, 3, 1).float().bfloat16().double()
    rel = _rel(dx.float().cpu(), want)
    print(f"\ndgrad stride 2 k={k} {cin}->{C}: rel L2 {rel:.3e}")
    assert rel <= 1e-3, rel


@pytest.mark.parametrize("srcs,C", [([32, 64, 128, 256], 128), ([16], 32), ([256], 256), ([64], 64), ([128, 128], 128)])
def test_1x1_dgrad_matches_conv2d_input_on_bf16_operands(srcs, C):
    B, H, W = 2, 21, 27
    m = _conv(sum(srcs), C, 1, 1, True, seed=C).to(dev())
    xs = [torch.zeros((B, H, W, c), dtype=torch.bfloat16, device=dev()) for c in srcs]
    fc = blocks.FoldedConv(m, *blocks.stack_params([m]), srcs=xs)
    dcat, dfm = _operands(C, H, W, B, seed=sum(srcs))
    w = torch.cat([m.block["conv_f"].weight, m.block["conv_m"].weight], 0).detach().cpu().bfloat16().double()
    want = torch.nn.grad.conv2d_input((B, sum(srcs), H, W), w, dcat.double().permute(0, 3, 1, 2))
    want = want.permute(0, 2, 3, 1).float().bfloat16().double()
    c0 = 0
    for cs in srcs:
        got = blocks.dgrad_1x1(dfm, fc, c0, cs)
        assert got.shape == (B, H, W, cs)
        rel = _rel(got.float().cpu(), want[..., c0:c0 + cs])
        print(f"\ndgrad 1x1 {srcs}->{C}, source {c0}:{c0 + cs}: rel L2 {rel:.3e}")
        assert rel <= 1e-3, rel
        c0 += cs


@pytest.mark.parametrize("srcs,cout,k,stride", [([32, 64, 128, 256], 32, 1, 1), ([128], 64, 4, 2)])
def test_frozen_conv_gives_input_gradients_only_and_skips_the_weight_gradient(srcs, cout, k, stride):
    B, H, W = 2, 38, 46
    m = _conv(sum(srcs), cout, k, stride, True, seed=3).to(dev())
    g = torch.Generator().manual_seed(4)
    xs = [torch.randn((B, c, H, W), generator=g).to(dev()) for c in srcs]
    gy = torch.randn((B, cout, H // stride, W // stride), generator=g).to(dev())

    def run(frozen):
        m.zero_grad(set_to_none=True)
        m.requires_grad_(not frozen)
        xi = [x.clone().requires_grad_(i != 1) for i, x in enumerate(xs)]      # source 1 (when there is one) needs no gradient
        y = blocks.gated_conv_srcs(m, xi)
        torch.cuda.synchronize()
        n0 = ops.launch_count()
        y.backward(gy)
        torch.cuda.synchronize()
        return ops.launch_count() - n0, [x.grad for x in xi]

    n_train, dx_train = run(False)
    assert all(p.grad is not None for p in m.parameters())
    n_frozen, dx_frozen = run(True)
    assert all(p.grad is None for p in m.parameters())
    assert n_train - n_frozen == len(srcs)                                     # one weight-gradient launch per source
    for i, (a, b) in enumerate(zip(dx_train, dx_frozen)):
        if i == 1:
            assert a is None and b is None
        else:
            assert torch.equal(a, b)


def test_in_place_parameter_update_before_backward_raises():
    m = _conv(64, 32, 4, 2, True, seed=9).to(dev())
    x = torch.randn((1, 64, 20, 24), device=dev(), requires_grad=True)
    y = blocks.gated_conv_srcs(m, [x])
    with torch.no_grad():
        m.block["conv_m"].weight.mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


def test_odd_stride2_input_raises():
    m = _conv(32, 64, 3, 2, True, seed=1).to(dev())
    with pytest.raises(ValueError, match="feat_extract.1.*even"):
        blocks.gated_conv_srcs(m, [torch.randn((1, 32, 21, 24), device=dev())], "feat_extract.1")


def _net(sd, tp):
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.to(dev()).eval()
    net.train_precision = tp
    return net


def test_full_net_bf16_all_tracks_fp32_training(synth_sd):
    g = torch.Generator().manual_seed(3)
    xs = [torch.rand((2, 8, 256 >> l, 256 >> l), generator=g).to(dev()) for l in range(4)]
    target = torch.rand((2, 3, 256, 256), generator=g).to(dev())
    nets = {tp: _net(synth_sd, tp) for tp in ("fp32", "bf16_all")}
    loss, dxs = {}, {}
    for tp, net in nets.items():
        xi = [x.clone().requires_grad_(True) for x in xs]
        lv = F.l1_loss(net(*xi), target)
        lv.backward()
        loss[tp], dxs[tp] = lv.detach(), [x.grad for x in xi]
    torch.cuda.synchronize()
    rel = abs(float(loss["bf16_all"]) - float(loss["fp32"])) / float(loss["fp32"])
    worst = (1.0, None)
    for (name, pa), pb in zip(nets["fp32"].named_parameters(), nets["bf16_all"].parameters()):
        assert (pa.grad is None) == (pb.grad is None), name
        if pa.grad is None:
            continue
        cos = _rel_cos(pb.grad, pa.grad)[1]
        worst = min(worst, (cos, name))
        assert cos >= 0.99, (name, cos)
    for l in range(4):
        cos = _rel_cos(dxs["bf16_all"][l], dxs["fp32"][l])[1]
        print(f"\ndescriptor level {l}: gradient cosine bf16_all vs fp32 {cos:.5f}")
        assert cos >= 0.99, (l, cos)
    print(f"\nfull net 2x256x256: loss fp32 {float(loss['fp32']):.6f} bf16_all {float(loss['bf16_all']):.6f} (rel {rel:.2e}), "
          f"worst grad cosine {worst[0]:.5f} ({worst[1]})")
    assert rel <= 1e-2, rel

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
            final[tp] = float(F.l1_loss(net._forward_torch(xs), target))
    descent = {tp: float(loss[tp]) - final[tp] for tp in final}
    print(f"after 20 Adam steps: fp32 {final['fp32']:.6f}, bf16_all {final['bf16_all']:.6f}; descent fp32 "
          f"{descent['fp32']:.6f}, bf16_all {descent['bf16_all']:.6f}")
    assert descent["fp32"] > 0 and descent["bf16_all"] > 0, descent
    assert abs(final["bf16_all"] - final["fp32"]) <= 0.05 * final["fp32"], final
    assert abs(descent["bf16_all"] - descent["fp32"]) <= 0.05 * descent["fp32"], descent
