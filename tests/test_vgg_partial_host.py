"""The masked VGG loss (VGGLoss(partialconv=True)) and VGGLossMix without a GPU: the float64 restatement against the reference's
own classes (tests/golden/ref_vgg_loss_partial.npz), the partial conv's ratio against torch's fp32 arithmetic, the module layout
and the rejections."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from read_b200 import vgg_loss
from read_b200.vgg_loss import PartialConv2d, VGGLoss, VGGLossMix

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vgg_partial_util  # noqa: E402
import vgg_util  # noqa: E402
from conftest import load_golden  # noqa: E402

SHAPE = (2, 36, 52)          # as tests/golden/make_ref_vgg_partial_golden.py
IMAGE_SEED = 12
MIX_WEIGHT = 0.3
# The golden gradients are the reference's fp32 ones.  On the 'dense' targets they are up to 1.5e-3 (relative L2) from float64,
# on the 'holes' targets 2e-7; the restatement evaluated in fp32 gives the reference's 'caffe' gradients bit for bit.
GRAD_REL = 3e-3


@pytest.fixture
def features():
    return vgg_util.seeded_features()          # per test: .double() converts the modules in place


@pytest.fixture(scope="module")
def golden():
    return load_golden("ref_vgg_loss_partial")


def _f64_loss_grad(crit, x, t):
    x = x.double().requires_grad_(True)
    loss = vgg_loss.reference_loss(crit.vgg19, crit.mean_, crit.std_, crit.layers, x, t.double())
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize("kind", vgg_partial_util.KINDS)
@pytest.mark.parametrize("net", ["caffe", "pytorch"])
@pytest.mark.parametrize("optimized", [False, True])
def test_float64_partial_restatement_reproduces_reference(features, golden, kind, net, optimized):
    """reference_loss over a PartialConv2d in float64 against the reference's VGGLoss(partialconv=True) in float32."""
    crit = VGGLoss(net=net, partialconv=True, optimized=optimized, features=vgg_loss.partial_features(features)).double()
    x, t = vgg_partial_util.masked_pair(kind, *SHAPE, IMAGE_SEED)
    loss, grad = _f64_loss_grad(crit, x, t)
    tag = f"{kind}_{net}_{'opt' if optimized else 'all'}"
    want_loss, want = float(golden[f"loss_{tag}"]), torch.from_numpy(golden[f"grad_{tag}"]).double()
    if kind == "zero":
        # an empty mask: both images are 0 after conv1_1, so every term and the whole gradient vanish
        assert want_loss == 0 and not want.any()
        assert loss.item() == 0 and not grad.any()
        return
    assert abs(loss.item() - want_loss) <= 1e-5 * abs(loss.item())
    assert float((grad - want).norm() / want.norm()) <= GRAD_REL
    mask = vgg_loss.target_mask(t).expand_as(x)
    assert not grad[mask == 0].any()                                     # nothing reaches a masked-out pixel


def test_partial_differs_from_plain_even_without_holes(features):
    """The zero padding makes the border windows' count < 9, so they are rescaled even when the mask is all ones."""
    x, t = vgg_partial_util.masked_pair("dense", *SHAPE, IMAGE_SEED)
    assert bool((vgg_loss.target_mask(t) == 1).all())
    lp, _ = _f64_loss_grad(VGGLoss(partialconv=True, features=vgg_loss.partial_features(features)).double(), x, t)
    lf, _ = _f64_loss_grad(VGGLoss(features=features).double(), x, t)
    assert lp.item() != lf.item()


def test_mix_reproduces_reference(features, golden):
    mix = VGGLossMix(weight=MIX_WEIGHT, features=features).double()
    x, t = vgg_partial_util.masked_pair("holes", *SHAPE, IMAGE_SEED)
    x = x.double().requires_grad_(True)
    loss = sum(w * vgg_loss.reference_loss(c.vgg19, c.mean_, c.std_, c.layers, x, t.double())
               for w, c in ((MIX_WEIGHT, mix.l1), (1 - MIX_WEIGHT, mix.l2)))
    loss.backward()
    assert abs(loss.item() - float(golden["loss_mix"])) <= 1e-5 * abs(loss.item())
    want = torch.from_numpy(golden["grad_mix"]).double()
    assert float((x.grad - want).norm() / want.norm()) <= 1e-4


def test_ratio_matches_torch_fp32_bit_for_bit():
    """What vg_ratio in csrc/vgg.cu computes, reciprocal(c) * 9 rounded twice in fp32 (0 at c = 0), against torch's fp32
    9 / (c + 1e-8) * clamp(c, 0, 1) for every count of a 3x3 window."""
    c = torch.arange(10, dtype=torch.float32)
    want = 9 / (c + 1e-8) * torch.clamp(c, 0, 1)
    f32 = np.float32
    got = np.array([0.0 if k == 0 else f32(f32(1) / f32(k)) * f32(9) for k in range(10)], dtype=np.float32)
    assert np.array_equal(got.view(np.int32), want.numpy().view(np.int32))
    # a correctly rounded 9 / c is not what torch computes: it is one ulp off at c = 5 and 7
    exact = np.array([0.0] + [9.0 / k for k in range(1, 10)], dtype=np.float32)
    assert [k for k in range(10) if exact[k] != got[k]] == [5, 7]


def test_partial_conv_module(features):
    conv = features[0]
    p = PartialConv2d.from_conv(conv)
    assert p.weight is conv.weight and p.bias is conv.bias
    assert set(p.state_dict()) == {'weight', 'bias'}
    g = torch.Generator().manual_seed(3)
    x = torch.randn((2, 3, 9, 7), generator=g, dtype=torch.float64)
    p64 = PartialConv2d.from_conv(nn.Conv2d(3, 64, 3, padding=1).double())
    ones = torch.ones((2, 1, 9, 7), dtype=torch.float64)
    out = p64(x, ones)
    plain = nn.functional.conv2d(x, p64.weight, p64.bias, padding=1)
    # an all-ones mask leaves the interior as the plain conv's (up to the 1e-8 in the ratio's denominator) and rescales the
    # border by 9 / count
    assert torch.allclose(out[..., 1:-1, 1:-1], plain[..., 1:-1, 1:-1], rtol=0, atol=1e-8)
    b = p64.bias.view(1, -1, 1, 1)
    assert torch.allclose(out[..., 0, 0], ((plain - b) * 9 / 4 + b)[..., 0, 0], rtol=1e-7)
    m = torch.zeros_like(ones)
    assert not p64(x, m).any()                                           # an empty window gives 0, not the bias


def test_layout_and_state_dict_keys(features, golden, tmp_path):
    # from the weights file, as the reference builds it: the plain first conv is wrapped, sharing its Parameters
    torch.save(features, tmp_path / vgg_loss.CAFFE_FILE)
    crit = VGGLoss(partialconv=True, save_dir=str(tmp_path))
    assert crit.partialconv is True and VGGLoss(save_dir=str(tmp_path)).partialconv is False
    assert type(crit.vgg19[0]) is PartialConv2d
    assert torch.equal(crit.vgg19[0].weight, features[0].weight) and torch.equal(crit.vgg19[0].bias, features[0].bias)
    assert not any(p.requires_grad for p in crit.parameters())
    vgg_loss.check_layout(crit.vgg19)
    assert sorted(crit.state_dict()) == list(golden["keys_partial"])
    mix = VGGLossMix(save_dir=str(tmp_path))
    assert sorted(mix.state_dict()) == list(golden["keys_mix"])
    assert mix.weight == 0.5 and isinstance(mix.l1, VGGLoss) and isinstance(mix.l2, VGGLoss)
    assert torch.equal(mix.l1.std_, mix.l2.std_)                        # both halves are 'caffe', as in the reference
    # partial_features: a new Sequential whose first conv is a PartialConv2d on the same Parameters, the input untouched
    pf = vgg_loss.partial_features(features)
    assert type(pf[0]) is PartialConv2d and type(features[0]) is nn.Conv2d
    assert pf[0].weight is features[0].weight and pf[0].bias is features[0].bias
    assert all(a is b for a, b in zip(list(pf)[1:], list(features)[1:]))
    crit = VGGLoss(partialconv=True, features=pf)
    assert crit.vgg19[0] is pf[0] and sorted(crit.state_dict()) == list(golden["keys_partial"])
    # a PartialConv2d is accepted at index 0 only
    mods = list(pf)
    mods[2] = PartialConv2d.from_conv(mods[2])
    with pytest.raises(ValueError, match=r"features\[2\]"):
        vgg_loss.check_layout(nn.Sequential(*mods))


def test_features_are_used_as_given(features, tmp_path):
    """features= is never rewritten: its first conv must be a PartialConv2d exactly when partialconv=True."""
    with pytest.raises(ValueError, match="partialconv=True"):
        VGGLoss(partialconv=True, features=features)
    with pytest.raises(ValueError, match="partialconv=False"):
        VGGLoss(features=vgg_loss.partial_features(features))
    with pytest.raises(ValueError, match="net"):
        VGGLoss(net='vgg', partialconv=True, features=vgg_loss.partial_features(features))
    with pytest.raises(FileNotFoundError, match=str(tmp_path / vgg_loss.CAFFE_FILE)):
        VGGLoss(partialconv=True, save_dir=str(tmp_path))
    with pytest.raises(FileNotFoundError, match=str(tmp_path / vgg_loss.CAFFE_FILE)):
        VGGLossMix(save_dir=str(tmp_path))


def test_partial_forward_rejections(features):
    crit = VGGLoss(partialconv=True, features=vgg_loss.partial_features(features))
    x, t = vgg_partial_util.masked_pair("holes", 1, 32, 32, 1)
    with pytest.raises(ValueError, match="target"):
        crit(x, t.clone().requires_grad_(True))
    crit.vgg19[0].weight.requires_grad_(True)
    with pytest.raises(ValueError, match="frozen"):
        crit(x, t)
    crit.vgg19[0].weight.requires_grad_(False)
    with pytest.raises(ValueError, match="shape"):
        crit(x, t[:, :, :16])
    with pytest.raises(RuntimeError, match="CUDA"):
        crit(x, t)


def test_partial_replica_evaluates_through_torch(features):
    crit = VGGLoss(partialconv=True, features=vgg_loss.partial_features(features))
    x, t = vgg_partial_util.masked_pair("holes", 1, 32, 32, 2)
    crit._is_replica = True
    want = vgg_loss.reference_loss(crit.vgg19, crit.mean_, crit.std_, crit.layers, x, t)
    assert torch.equal(crit(x, t), want)
    plain = VGGLoss(features=features)
    assert not torch.equal(vgg_loss.reference_loss(plain.vgg19, plain.mean_, plain.std_, plain.layers, x, t), want)
