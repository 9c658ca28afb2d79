"""-m gpu: bf16 training of the 14 gated 3x3 stride-1 convs outside the residual blocks (read_b200/blocks.py: gated_conv,
csrc/conv_bwd.cu) against torch autograd.

Tolerances as for the block stacks (tests/test_gpu_train_blocks.py):
* one conv of every row of unet.layer_table that trains through gated_conv, at every C it has, on ragged B = 2 shapes, against
  float64 autograd of the same module: the output and every gradient (input, conv_f / conv_m weight and bias, BatchNorm weight
  and bias) within relative L2 error 2e-2 and cosine >= 0.999; FAM as a + merge(a * b), the gradients of a and b included;
* the 8-channel input-gradient kernel alone against torch.nn.grad.conv2d_input on the same bf16 operands: relative L2 <= 1e-3;
* the whole net at 2 x 256 x 256: each of the four descriptor-pyramid levels' gradient under 'bf16' has cosine >= 0.99 against
  'fp32'.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import blocks
from read_b200.unet import UNet, GatedConv

pytestmark = pytest.mark.gpu


def _conv(cin, cout, elu, seed):
    g = torch.Generator().manual_seed(seed)
    m = GatedConv(cin, cout, 3, 1, elu)
    bound = 1.0 / (9 * cin) ** 0.5
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


# (layer, Cin, Cout, ELU, B, H, W): every row of the table at every C; H, W not multiples of the 16 x 8 tile, the 32-pixel
# weight-gradient segment or the 64-pixel segment of the 8-channel input gradient
CONVS = [("feat_extract.0", 8, 32, True, 2, 83, 131), ("feat_extract.5", 32, 3, False, 2, 83, 131),
         ("SCM2.main.0", 8, 16, True, 2, 45, 67), ("SCM1.main.0", 8, 32, True, 2, 29, 35), ("SCM0.main.0", 8, 64, True, 2, 21, 27),
         ("SCM2.main.2", 32, 32, True, 2, 45, 67), ("SCM1.main.2", 64, 64, True, 2, 29, 35),
         ("SCM0.main.2", 128, 128, True, 2, 13, 19),
         ("AFFs.0.conv.1", 32, 32, False, 2, 37, 45), ("AFFs.1.conv.1", 64, 64, False, 2, 29, 35),
         ("AFFs.2.conv.1", 128, 128, False, 2, 21, 27)]


@pytest.mark.parametrize("name,cin,cout,elu,B,H,W", CONVS, ids=[c[0] for c in CONVS])
def test_conv_forward_and_grads_match_fp64_autograd(name, cin, cout, elu, B, H, W):
    m = _conv(cin, cout, elu, seed=cin * 7 + cout + H)
    g = torch.Generator().manual_seed(H * W + cout)
    x = torch.rand((B, cin, H, W), generator=g) if cin == 8 else torch.randn((B, cin, H, W), generator=g)
    gy = torch.randn((B, cout, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    xr = x.double().requires_grad_(True)
    yr = ref(xr)
    yr.backward(gy.double())
    ours = m.to(dev())
    xo = x.to(dev()).requires_grad_(True)
    yo = blocks.gated_conv(ours, xo)
    assert yo.shape == (B, cout, H, W)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr), ("dx",) + _rel_cos(xo.grad, xr.grad)]
    for (pn, po), pr in zip(ours.named_parameters(), ref.parameters()):
        assert po.grad.shape == po.shape, pn
        rows.append((pn,) + _rel_cos(po.grad, pr.grad))
    _check(rows, f"{name} {cin}->{cout} {B}x{H}x{W}")


@pytest.mark.parametrize("C,B,H,W", [(64, 2, 45, 67), (128, 2, 29, 35), (256, 2, 13, 19)])
@pytest.mark.parametrize("fused", [False, True], ids=["torch_sum", "residual"])
def test_fam_merge_matches_fp64_autograd(C, B, H, W, fused):
    """a + merge(a * b): with the sum on torch (the net's routing) and through gated_conv's residual operand."""
    m = _conv(C, C, False, seed=C + H)
    g = torch.Generator().manual_seed(C * H)
    a, b = torch.randn((B, C, H, W), generator=g), torch.rand((B, C, H, W), generator=g)
    gy = torch.randn((B, C, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    ar, br = a.double().requires_grad_(True), b.double().requires_grad_(True)
    yr = ar + ref(ar * br)
    yr.backward(gy.double())
    ours = m.to(dev())
    ao, bo = a.to(dev()).requires_grad_(True), b.to(dev()).requires_grad_(True)
    yo = blocks.gated_conv(ours, ao * bo, residual=ao) if fused else ao + blocks.gated_conv(ours, ao * bo)
    yo.backward(gy.to(dev()))
    torch.cuda.synchronize()
    rows = [("out",) + _rel_cos(yo, yr), ("da",) + _rel_cos(ao.grad, ar.grad), ("db",) + _rel_cos(bo.grad, br.grad)]
    for (pn, po), pr in zip(ours.named_parameters(), ref.parameters()):
        rows.append((pn,) + _rel_cos(po.grad, pr.grad))
    _check(rows, f"FAM merge C={C} ({'residual' if fused else 'torch sum'})")


@pytest.mark.parametrize("C,B,H,W", [(16, 2, 45, 67), (32, 2, 83, 131), (64, 2, 21, 27)])
def test_cin8_dgrad_matches_conv2d_input_on_bf16_operands(C, B, H, W):
    m = _conv(8, C, True, seed=C).to(dev())
    fc = blocks.FoldedConv(m, *blocks.stack_params([m]))
    assert fc.w_dgrad is None
    g = torch.Generator().manual_seed(C)
    dcat = torch.randn((B, H, W, 2 * C), generator=g).bfloat16()            # [df | dm] in channel order
    dfm = dcat[..., blocks.fm_columns(C)].contiguous().to(dev())              # the kernels' column order
    got = blocks.dgrad(dfm, fc).float().cpu()
    w = torch.cat([m.block["conv_f"].weight, m.block["conv_m"].weight], 0).detach().cpu().bfloat16().double()
    want = torch.nn.grad.conv2d_input((B, 8, H, W), w, dcat.double().permute(0, 3, 1, 2), padding=1)
    want = want.permute(0, 2, 3, 1).float().bfloat16().double()
    rel = float((got.double() - want).norm() / want.norm())
    print(f"\ndgrad Cin=8 C={C}: rel L2 {rel:.3e}")
    assert rel <= 1e-3, rel


@pytest.mark.parametrize("cin,cout", [(8, 32), (32, 3)])
def test_frozen_conv_gives_the_input_gradient_only(cin, cout):
    B, H, W = 2, 37, 45
    m = _conv(cin, cout, cout > 3, seed=3)
    g = torch.Generator().manual_seed(4)
    x, gy = torch.rand((B, cin, H, W), generator=g), torch.randn((B, cout, H, W), generator=g)
    ref = copy.deepcopy(m).double()
    xr = x.double().requires_grad_(True)
    ref(xr).backward(gy.double())
    ours = m.to(dev()).requires_grad_(False)
    xo = x.to(dev()).requires_grad_(True)
    blocks.gated_conv(ours, xo).backward(gy.to(dev()))
    rel, cos = _rel_cos(xo.grad, xr.grad)
    assert rel <= 2e-2 and cos >= 0.999, (rel, cos)
    assert all(p.grad is None for p in ours.parameters())


def test_in_place_parameter_update_before_backward_raises():
    m = _conv(8, 32, True, seed=9).to(dev())
    x = torch.rand((1, 8, 20, 24), device=dev(), requires_grad=True)
    y = blocks.gated_conv(m, x)
    with torch.no_grad():
        m.block["norm"].weight.mul_(2.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


def test_full_net_descriptor_gradients_track_fp32(synth_sd):
    """Every descriptor-pyramid level gets its gradient from the bf16 kernels (feat_extract.0 and the three SCM*.main.0)."""
    g = torch.Generator().manual_seed(5)
    xs = [torch.rand((2, 8, 256 >> l, 256 >> l), generator=g) for l in range(4)]
    target = torch.rand((2, 3, 256, 256), generator=g).to(dev())
    grads = {}
    for tp in ("fp32", "bf16"):
        net = UNet()
        net.load_state_dict(synth_sd, strict=True)
        net.to(dev()).eval()
        net.train_precision = tp
        xi = [x.to(dev()).requires_grad_(True) for x in xs]
        F.l1_loss(net(*xi), target).backward()
        grads[tp] = [x.grad for x in xi]
    torch.cuda.synchronize()
    for l in range(4):
        cos = _rel_cos(grads["bf16"][l], grads["fp32"][l])[1]
        print(f"\ndescriptor level {l}: gradient cosine bf16 vs fp32 {cos:.5f}")
        assert cos >= 0.99, (l, cos)
