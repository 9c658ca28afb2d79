"""-m gpu: bf16 training of the residual block stacks (read_b200/blocks.py, csrc/conv_bwd.cu) against torch autograd.

Parity definition (DESIGN.md §7), tolerances set once on an H100 and frozen:
* one stack (4 ResBlocks, 8 gated 3x3 convs) against float64 autograd of the same modules on the same parameters: the output and
  every gradient tensor (input, conv_f / conv_m weight and bias, BatchNorm weight and bias of each conv) within relative L2 error
  2e-2 and cosine similarity >= 0.999;
* the input-gradient launch alone (flipped / transposed filter packing, RAW epilogue with residual) against
  torch.nn.grad.conv2d_input on the same bf16 operands, accumulated in float64 and rounded to bf16 like the kernel's output:
  relative L2 error <= 1e-3;
* the whole net, train_precision 'bf16' against 'fp32' at 256x256, B = 2: loss within 1e-2 (relative), every parameter gradient
  cosine >= 0.99, and 20 Adam steps on a fixed target end within 5 % of the fp32 run's loss.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import blocks, synth
from read_b200.unet import UNet, GatedConv

pytestmark = pytest.mark.gpu


def _stack(C, seed):
    """The 8 GatedConvs of one stack (ELU on the first conv of every ResBlock), weights ~ U(+-1/sqrt(fan_in)), eval-mode BatchNorm
    with random affine and running statistics."""
    g = torch.Generator().manual_seed(seed)
    mods = torch.nn.ModuleList([GatedConv(C, C, 3, 1, elu=(i % 2 == 0)) for i in range(8)])
    bound = 1.0 / (9 * C) ** 0.5
    with torch.no_grad():
        for m in mods:
            for name in ("conv_f", "conv_m"):
                conv = m.block[name]
                conv.weight.copy_((torch.rand(conv.weight.shape, generator=g) * 2 - 1) * bound)
                conv.bias.copy_((torch.rand(conv.bias.shape, generator=g) * 2 - 1) * bound)
            n = m.block["norm"]
            n.weight.copy_(torch.rand(C, generator=g) + 0.5)
            n.bias.copy_(torch.randn(C, generator=g) * 0.1)
            n.running_mean.copy_(torch.randn(C, generator=g) * 0.1)
            n.running_var.copy_(torch.rand(C, generator=g) + 0.5)
    return mods.eval()


def _ref_stack(mods, x):
    t = x
    for r in range(0, len(mods), 2):
        t = mods[r + 1](mods[r](t)) + t
    return t


def _rel_cos(got, want):
    got, want = got.detach().double().flatten().cpu(), want.detach().double().flatten().cpu()
    rel = float((got - want).norm() / want.norm())
    cos = float(torch.dot(got, want) / (got.norm() * want.norm()))
    return rel, cos


# (C, B, H, W): H, W not multiples of the 16 x 8 tile; the second C = 32 shape spans many tiles and many 32-pixel row segments
SHAPES = [(32, 2, 37, 45), (32, 2, 83, 131), (64, 2, 29, 35), (128, 2, 21, 27), (256, 2, 13, 19)]


@pytest.mark.parametrize("C,B,H,W", SHAPES)
def test_stack_forward_and_grads_match_fp64_autograd(C, B, H, W):
    mods = _stack(C, seed=C + H)
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn((B, C, H, W), generator=g)
    gy = torch.randn((B, C, H, W), generator=g)

    ref = copy.deepcopy(mods).double()
    xr = x.double().requires_grad_(True)
    yr = _ref_stack(ref, xr)
    yr.backward(gy.double())

    ours = mods.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    yo = blocks.stack_forward(list(ours), xo)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()

    rows = [("out",) + _rel_cos(yo, yr), ("dx",) + _rel_cos(xo.grad, xr.grad)]
    for i, (mo, mr) in enumerate(zip(ours, ref)):
        for (name, po), pr in zip(mo.named_parameters(), mr.parameters()):
            rows.append((f"{i}.{name}",) + _rel_cos(po.grad, pr.grad))
    worst_rel = max(rows, key=lambda r: r[1])
    worst_cos = min(rows, key=lambda r: r[2])
    print(f"\nstack C={C} {B}x{H}x{W}: worst rel L2 {worst_rel[1]:.3e} ({worst_rel[0]}), worst cosine {worst_cos[2]:.6f} ({worst_cos[0]})")
    for name, rel, cos in rows:
        assert rel <= 2e-2 and cos >= 0.999, (name, rel, cos)


def test_frozen_stack_gives_the_input_gradient_only():
    """A frozen net (parameters without requires_grad, descriptors trained through it) skips the weight gradients and still
    back-propagates to the input."""
    C, B, H, W = 64, 2, 29, 35
    mods = _stack(C, seed=5)
    g = torch.Generator().manual_seed(11)
    x = torch.randn((B, C, H, W), generator=g)
    gy = torch.randn((B, C, H, W), generator=g)
    ref = copy.deepcopy(mods).double()
    xr = x.double().requires_grad_(True)
    _ref_stack(ref, xr).backward(gy.double())
    ours = mods.to(dev()).requires_grad_(False)
    xo = x.to(dev()).requires_grad_(True)
    blocks.stack_forward(list(ours), xo).backward(gy.to(dev()))
    rel, cos = _rel_cos(xo.grad, xr.grad)
    assert rel <= 2e-2 and cos >= 0.999, (rel, cos)
    assert all(p.grad is None for p in ours.parameters())


def test_in_place_parameter_update_before_backward_raises():
    mods = _stack(32, seed=9).to(dev())
    x = torch.randn((1, 32, 20, 24), device=dev(), requires_grad=True)
    y = blocks.stack_forward(list(mods), x)
    with torch.no_grad():
        mods[3].block["conv_f"].bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


@pytest.mark.parametrize("C,B,H,W", [(32, 2, 37, 45), (64, 2, 29, 35), (128, 2, 21, 27), (256, 2, 13, 19)])
def test_dgrad_matches_conv2d_input_on_bf16_operands(C, B, H, W):
    m = _stack(C, seed=7)[0].to(dev())
    fc = blocks.FoldedConv(m, *blocks.stack_params([m]))
    g = torch.Generator().manual_seed(C)
    dcat = torch.randn((B, H, W, 2 * C), generator=g).bfloat16()            # [df | dm] in channel order
    res = torch.randn((B, H, W, C), generator=g).bfloat16()
    dfm = dcat[..., blocks.fm_columns(C)].contiguous().to(dev())              # the kernels' column order
    got = blocks.dgrad(dfm, fc, residual=res.to(dev())).float().cpu()
    w = torch.cat([m.block["conv_f"].weight, m.block["conv_m"].weight], 0).detach().cpu().bfloat16().double()
    want = torch.nn.grad.conv2d_input((B, C, H, W), w, dcat.double().permute(0, 3, 1, 2), padding=1)
    want = (want.permute(0, 2, 3, 1) + res.double()).float().bfloat16().double()
    rel = float((got.double() - want).norm() / want.norm())
    print(f"\ndgrad C={C}: rel L2 {rel:.3e}")
    assert rel <= 1e-3, rel


def _net(sd, tp):
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.to(dev()).eval()
    net.train_precision = tp
    return net


def test_full_net_bf16_blocks_track_fp32_training(synth_sd):
    g = torch.Generator().manual_seed(3)
    xs = [torch.rand((2, 8, 256 >> l, 256 >> l), generator=g).to(dev()) for l in range(4)]
    target = torch.rand((2, 3, 256, 256), generator=g).to(dev())
    nets = {tp: _net(synth_sd, tp) for tp in ("fp32", "bf16")}
    loss = {}
    for tp, net in nets.items():
        lv = F.l1_loss(net(*xs), target)
        lv.backward()
        loss[tp] = lv.detach()
    torch.cuda.synchronize()
    rel = abs(float(loss["bf16"]) - float(loss["fp32"])) / float(loss["fp32"])
    worst = (1.0, None)
    for (name, pa), pb in zip(nets["fp32"].named_parameters(), nets["bf16"].parameters()):
        assert (pa.grad is None) == (pb.grad is None), name
        if pa.grad is None:
            continue
        cos = _rel_cos(pb.grad, pa.grad)[1]
        worst = min(worst, (cos, name))
        assert cos >= 0.99, (name, cos)
    print(f"\nfull net 2x256x256: loss fp32 {float(loss['fp32']):.6f} bf16 {float(loss['bf16']):.6f} (rel {rel:.2e}), "
          f"worst grad cosine {worst[0]:.5f} ({worst[1]})")
    assert rel <= 1e-2, rel

    final = {}
    for tp, net in nets.items():
        net.zero_grad(set_to_none=True)
        # the net's training rate (bench.py c5); at 1e-3 this random-weight net spikes to a loss of ~30 within three steps at
        # either precision and the runs part ways
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        for _ in range(20):
            opt.zero_grad(set_to_none=True)
            lv = F.l1_loss(net(*xs), target)
            lv.backward()
            opt.step()
        with torch.no_grad():
            final[tp] = float(F.l1_loss(net._forward_torch(xs), target))
    print(f"after 20 Adam steps: fp32 {final['fp32']:.6f}, bf16 {final['bf16']:.6f} (start {float(loss['fp32']):.6f})")
    descent = {tp: float(loss[tp]) - final[tp] for tp in final}
    print(f"descent over 20 steps: fp32 {descent['fp32']:.6f}, bf16 {descent['bf16']:.6f}")
    assert descent["fp32"] > 0 and descent["bf16"] > 0, descent             # both runs trained
    assert abs(final["bf16"] - final["fp32"]) <= 0.05 * final["fp32"], final
    assert abs(descent["bf16"] - descent["fp32"]) <= 0.05 * descent["fp32"], descent
