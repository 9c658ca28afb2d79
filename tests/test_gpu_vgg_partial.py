"""-m gpu: the masked VGG loss (VGGLoss(partialconv=True), csrc/vgg.cu's partial kernels) and VGGLossMix on our kernels, seeded
weights (tests/vgg_util.py) and the target kinds of tests/vgg_partial_util.py.

* each new kernel on the same operands: the masked normalise, its byte mask and the masked image gradient bit-exact against
  torch's fp32 arithmetic; the partial post-conv pass and the partial dgrad_in against float64;
* the loss and the input gradient against the float64 restatement (vgg_loss.reference_loss) at 2 x 70 x 46, for both nets, both
  layer sets and every target kind, within the VGG loss bounds of tests/test_gpu_vgg_loss.py; the gradient exactly 0 where the
  mask is 0, and loss and gradient 0 for an all-zero target;
* the loss bit-identical under no_grad, and (gradient too) when forced into one image pair per chunk;
* no torch convolution in a forward + backward; VGGLossMix against its two halves;
* 20 Adam steps of the bf16_all net in train() with per-item BatchNorm under ModelAndLoss(use_mask=True) and the masked loss track
  the fp32 net trained with the torch masked loss.
"""
import copy
import os
import sys

import pytest
import torch

from read_b200 import _lib as L, vgg_loss
from read_b200.compose import ModelAndLoss
from read_b200.unet import UNet
from read_b200.vgg_loss import VGGLoss, VGGLossMix

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vgg_partial_util  # noqa: E402
import vgg_util  # noqa: E402
from gpu_util import dev  # noqa: E402

pytestmark = pytest.mark.gpu

# the VGG loss bounds frozen in DESIGN.md (section 7, VGG loss) for independent images
LOSS_REL = 1e-2
GRAD_REL = 1e-1
GRAD_COS = 0.995
# Whole net, 20 Adam steps of the bf16_all net with the masked loss on our kernels, against the same net with the torch masked loss
# (the loss's own share) and the fp32 net with the torch masked loss.  Measured over three runs: descents within 0.24 %, final losses
# within 1.8 %.  The final loss is the residual after an 88 % descent, and the same net with the same torch loss moved up to 1.7 %
# between runs.
TRAIN_DESCENT_REL = 0.01
TRAIN_FINAL_REL = 0.03


def _crit(net="caffe", optimized=False):
    return VGGLoss(net=net, partialconv=True, optimized=optimized,
                   features=vgg_loss.partial_features(vgg_util.seeded_features())).to(dev())


def _rel_cos(got, want):
    g, w = got.double().flatten(), want.double().flatten()
    return float((g - w).norm() / w.norm()), float(g @ w / (g.norm() * w.norm()))


def _bf16(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(torch.bfloat16).to(dev())


def _mask(n, H, W, g):
    """A byte mask [n, H, W] with empty, full and mixed 3x3 windows."""
    m = (torch.rand((n, H, W), generator=g) < 0.7).to(torch.uint8)
    m[0, :4, :5] = 0
    m[-1, -3:, :] = 1
    return m.to(dev())


def _ratio_upd(m):
    """ratio and upd [n, H, W, 1] in float64 of a byte mask [n, H, W]."""
    cnt = torch.nn.functional.conv2d(m.double()[:, None], torch.ones((1, 1, 3, 3), dtype=torch.float64, device=m.device), padding=1)
    upd = cnt.clamp(0, 1)
    return (9 / cnt.clamp_min(1) * upd).permute(0, 2, 3, 1), upd.permute(0, 2, 3, 1)


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("net", ["caffe", "pytorch"])
def test_normalize_masked_kernel_is_bit_exact(net):
    lib = L.load()
    n, H, W = 3, 13, 11
    x, t = vgg_partial_util.masked_pair("holes", n, H, W, 1)
    t[1, :, 5, 5] = torch.tensor([1e-10, 0.0, 0.0])                     # sums below the threshold count as masked out
    mean, std = vgg_loss.normalization(net)
    xd, td, md, sd = x.to(dev()), t.to(dev()), mean.reshape(3).to(dev()), std.reshape(3).to(dev())
    out = torch.empty((2 * n, H, W, 8), dtype=torch.bfloat16, device=dev())
    mask = torch.empty((n, H, W), dtype=torch.uint8, device=dev())
    L.check(lib.read_vgg_normalize_masked(xd.data_ptr(), td.data_ptr(), n, H, W, md.data_ptr(), sd.data_ptr(), out.data_ptr(),
                                          mask.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    m = vgg_loss.target_mask(t)                                           # torch's fp32 arithmetic on the CPU
    want = ((torch.cat([x, t]) - mean) / std * torch.cat([m, m])).permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(mask.cpu(), m[:, 0].to(torch.uint8))
    assert int(mask[1, 5, 5]) == 0 and 0 < int(mask.sum()) < n * H * W
    assert torch.equal(out[..., :3].cpu(), want)
    assert torch.equal(out[..., 3:], torch.zeros_like(out[..., 3:]))


@pytest.mark.parametrize("loss", [False, True])
def test_post_partial_kernel(loss):
    lib, g = L.load(), torch.Generator().manual_seed(21)
    n, H, W, C = 2, 9, 7, 64
    raw = _bf16((2 * n, H, W, C), g, 3.0)
    bias = torch.randn(C, generator=g).to(dev())
    mask = _mask(n, H, W, g)
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev())
    out = torch.empty((2 * n, H, W, C), dtype=torch.bfloat16, device=dev())
    code = torch.empty((n, H, W, C), dtype=torch.int8, device=dev())
    term = torch.zeros(1, dtype=torch.float64, device=dev())
    L.check(lib.read_vgg_post_partial(raw.data_ptr(), mask.data_ptr(), n, H, W, C, bias.data_ptr(), out.data_ptr(), code.data_ptr(),
                                      term.data_ptr() if loss else None, 0.5, ws.data_ptr(), L.stream_ptr()))
    ratio, upd = _ratio_upd(mask)
    ratio, upd = torch.cat([ratio, ratio]), torch.cat([upd, upd])
    y = ((raw.double() * ratio + bias.double()) * upd).clamp_min(0)
    yi, yt = y[:n], y[n:]
    d = yi - yt
    want_code = torch.where(yi > 0, 2 + (torch.sign(d) if loss else 0), torch.zeros_like(d))
    close = (yi.abs() < 1e-5) | (d.abs() < 1e-5)                         # fp32 rounding of raw * ratio + bias
    assert torch.equal(code.double()[~close], want_code[~close])
    assert not code[upd[:n].expand_as(yi) == 0].any()                    # an empty window: both halves 0, code 0
    if loss:
        s = 0.5 * float(d.abs().sum())
        assert abs(float(term) - s) <= 1e-6 * s
    assert torch.allclose(out.double(), y, rtol=2 ** -8, atol=1e-6)


def test_dgrad_in_partial_kernel():
    lib, g = L.load(), torch.Generator().manual_seed(22)
    n, H, W, C = 2, 9, 7, 64
    up = _bf16((n, H, W, C), g)
    code = torch.randint(0, 4, (n, H, W, C), generator=g, dtype=torch.int8).to(dev())
    mask = _mask(n, H, W, g)
    gout, coef = torch.tensor([0.75], device=dev()), 1e-1
    dy = torch.empty((n, H, W, C), dtype=torch.bfloat16, device=dev())
    L.check(lib.read_vgg_dgrad_in_partial(up.data_ptr(), mask.data_ptr(), code.data_ptr(), n, H, W, C, gout.data_ptr(), coef,
                                          dy.data_ptr(), L.stream_ptr()))
    c = code.double()
    ratio, _ = _ratio_upd(mask)
    want = torch.where(c != 0, up.double() + (c - 2) * 0.75 * coef, torch.zeros_like(c)) * ratio
    assert torch.allclose(dy.double(), want, rtol=2 ** -8, atol=1e-6)


def test_image_grad_masked_kernel_is_bit_exact():
    lib, g = L.load(), torch.Generator().manual_seed(23)
    n, H, W = 3, 10, 6
    dx = _bf16((n, H, W, 8), g)
    mask = _mask(n, H, W, g)
    std = vgg_loss.normalization("pytorch")[1]
    sd = std.reshape(3).to(dev())
    out = torch.empty((n, 3, H, W), device=dev())
    L.check(lib.read_vgg_image_grad_masked(dx.data_ptr(), mask.data_ptr(), n, H, W, sd.data_ptr(), out.data_ptr(), L.stream_ptr()))
    want = dx[..., :3].cpu().float().permute(0, 3, 1, 2) * mask.cpu()[:, None].float() / std
    assert torch.equal(out.cpu(), want)


# ------------------------------------------------------------------ the whole loss
def _f64(crit, x, t):
    xx = x.detach().double().requires_grad_(True)
    loss = vgg_loss.reference_loss(copy.deepcopy(crit.vgg19).double(), crit.mean_.double(), crit.std_.double(), crit.layers, xx,
                                   t.double())
    loss.backward()
    return float(loss.detach()), xx.grad


def _ours(crit, x, t):
    xx = x.clone().requires_grad_(True)
    loss = crit(xx, t)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), xx.grad


@pytest.mark.parametrize("kind", vgg_partial_util.KINDS)
@pytest.mark.parametrize("net", ["caffe", "pytorch"])
@pytest.mark.parametrize("optimized", [False, True])
def test_partial_loss_and_gradient_match_float64(kind, net, optimized):
    crit = _crit(net, optimized)
    x, t = (v.to(dev()) for v in vgg_partial_util.masked_pair(kind, 2, 70, 46, 7))
    loss, grad = _ours(crit, x, t)
    masked_out = vgg_loss.target_mask(t).expand_as(x) == 0
    assert not grad[masked_out].any()                                    # exactly 0 wherever the mask is 0
    if kind == "zero":
        assert float(loss) == 0 and not grad.any()
        return
    want_loss, want_grad = _f64(crit, x, t)
    rel_loss = abs(float(loss) - want_loss) / want_loss
    rel, cos = _rel_cos(grad, want_grad)
    print(f"\n{kind} {net} optimized={optimized}: loss rel {rel_loss:.2e}, grad rel L2 {rel:.3e} cos {cos:.6f}")
    assert rel_loss <= LOSS_REL
    assert rel <= GRAD_REL and cos >= GRAD_COS, (rel, cos)


def test_partial_no_grad_and_chunks_agree(monkeypatch):
    crit = _crit()
    x, t = (v.to(dev()) for v in vgg_partial_util.masked_pair("holes", 3, 70, 46, 9))
    l1, g1 = _ours(crit, x, t)
    with torch.no_grad():
        l2 = crit(x, t)
    assert torch.equal(l1, l2)
    steps = vgg_loss.layer_walk(crit.layers)
    monkeypatch.setattr(vgg_loss, "RAW_LIMIT", 2 * 70 * 46 * 64 + 1)    # one image pair per chunk, each with its own mask
    assert vgg_loss.chunk_pairs(steps, 70, 46) == 1
    l3, g3 = _ours(crit, x, t)
    assert torch.equal(g1, g3)
    assert abs(float(l3) - float(l1)) <= 1e-6 * float(l1)


def test_no_torch_convolution_in_the_partial_loss():
    crit = _crit()
    x, t = (v.to(dev()) for v in vgg_partial_util.masked_pair("holes", 2, 64, 64, 11))
    _ours(crit, x, t)
    xx = x.clone().requires_grad_(True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU]) as prof:
        crit(xx, t).backward()
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    assert not [n for n in names if "conv" in n.lower() or "cudnn" in n.lower()], names


def test_mix_is_the_weighted_sum_of_its_halves():
    w = 0.3
    features = vgg_util.seeded_features()
    mix = VGGLossMix(weight=w, features=features).to(dev())
    a, b = VGGLoss(features=features).to(dev()), VGGLoss(net='caffe', features=features).to(dev())
    x, t = (v.to(dev()) for v in vgg_partial_util.masked_pair("holes", 2, 48, 40, 13))
    lm, gm = _ours(mix, x, t)
    (la, ga), (lb, gb) = _ours(a, x, t), _ours(b, x, t)
    assert torch.equal(lm, la * w + lb * (1 - w))
    rel, cos = _rel_cos(gm, w * ga + (1 - w) * gb)                       # bf16 rounds w * g differently from g
    assert rel <= 1e-2 and cos >= 0.9999, (rel, cos)


def test_full_net_bf16_all_with_masked_loss_tracks_fp32(synth_sd):
    g = torch.Generator().manual_seed(5)
    xs = [torch.rand((2, 8, 256 >> l, 256 >> l), generator=g).to(dev()) for l in range(4)]
    mask = torch.ones((2, 1, 256, 256))
    mask[0, :, 40:120, 60:200] = 0
    mask[1, :, 150:, :90] = 0
    mask = mask.to(dev())
    target = torch.rand((2, 3, 256, 256), generator=g).to(dev()) * mask          # as the reference's train loop masks it
    crit = _crit()
    torch_loss = lambda out, t: vgg_loss.reference_loss(crit.vgg19, crit.mean_, crit.std_, crit.layers, out, t)
    arms = {"fp32": ("fp32", torch_loss), "bf16_all": ("bf16_all", crit), "bf16_all torch loss": ("bf16_all", torch_loss)}
    first, final = {}, {}
    for arm, (tp, lossf) in arms.items():
        net = UNet()
        net.load_state_dict(synth_sd, strict=True)
        net.to(dev()).train()
        net.train_precision = tp
        net.train_batchnorm = 'per_item'
        model = ModelAndLoss(net, lossf, use_mask=True)
        opt = torch.optim.Adam(net.parameters(), lr=1e-4)
        for s in range(20):
            opt.zero_grad(set_to_none=True)
            out, loss = model(*xs, target, mask=mask)
            if s == 0:
                with torch.no_grad():
                    first[arm] = float(torch_loss(out * mask, target))
            loss.backward()
            opt.step()
        with torch.no_grad():
            final[arm] = float(torch_loss(net(*xs) * mask, target))
    descent = {k: first[k] - final[k] for k in final}
    print(f"\nmasked VGG loss, 20 Adam steps: first {first}, final {final}, descent {descent}")
    assert all(d > 0 for d in descent.values()), descent
    for other in ("bf16_all torch loss", "fp32"):
        assert abs(descent["bf16_all"] - descent[other]) <= TRAIN_DESCENT_REL * descent[other], descent
        assert abs(final["bf16_all"] - final[other]) <= TRAIN_FINAL_REL * final[other], final
