"""VGG loss host logic, no GPU: the layer walk, the filter split, the chunking rule, every rejection, and the float64 restatement
against the reference's own VGGLoss (tests/golden/ref_vgg_loss.npz)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from read_b200 import blocks, vgg_loss
from read_b200.vgg_loss import VGGLoss

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import vgg_util  # noqa: E402
from conftest import load_golden  # noqa: E402


@pytest.fixture(scope="module")
def features():
    return vgg_util.seeded_features()


def test_layer_walk(features):
    vgg_loss.check_layout(features)
    kinds = vgg_loss.vgg19_modules()
    assert len(kinds) == len(features) == 37
    for i, m in enumerate(features):
        want = {'relu': nn.ReLU, 'pool': nn.MaxPool2d}.get(kinds[i], nn.Conv2d)
        assert isinstance(m, want), i
    steps = vgg_loss.layer_walk(vgg_loss.LAYERS)
    assert [s.conv for s in steps] == [0, 2, 5, 7, 10, 12, 14, 16, 19, 21, 23, 25, 28]
    assert [s.relu for s in steps] == list(vgg_loss.LAYERS)
    assert all(s.loss for s in steps)
    assert [s.conv for s in steps if s.pool] == [2, 7, 16, 25]          # pools 4, 9, 18, 27
    assert [(s.cin, s.cout) for s in steps][:3] == [(3, 64), (64, 64), (64, 128)]
    steps = vgg_loss.layer_walk(vgg_loss.LAYERS_OPTIMIZED)
    assert steps[-1].relu == 35 and len(steps) == 16                    # the last pool (36) is not run
    assert [s.relu for s in steps if s.loss] == list(vgg_loss.LAYERS_OPTIMIZED)
    assert [s.conv for s in steps if s.pool] == [2, 7, 16, 25]
    assert vgg_loss.layer_sizes(steps, 70, 46)[-1] == (4, 2)             # 70 -> 35 -> 17 -> 8 -> 4, 46 -> 23 -> 11 -> 5 -> 2
    with pytest.raises(ValueError, match="ReLU outputs"):
        vgg_loss.layer_walk([1, 4])


def _conv(cin, cout, **kw):
    return nn.Conv2d(cin, cout, kernel_size=kw.pop('k', 3), padding=kw.pop('padding', 1), **kw)


@pytest.mark.parametrize("case", ["vgg16", "vgg19_bn", "channels", "stride", "no_bias", "linear", "pool3", "list"])
def test_rejects_non_vgg19_layouts(features, case):
    from torchvision.models import vgg
    if case == "vgg16":
        f = vgg.make_layers(vgg.cfgs['D'])
    elif case == "vgg19_bn":
        f = vgg.make_layers(vgg.cfgs['E'], batch_norm=True)
    elif case == "list":
        f = list(features)
    else:
        mods = list(features)
        if case == "channels":
            mods[2] = _conv(64, 32)
        elif case == "stride":
            mods[2] = _conv(64, 64, stride=2)
        elif case == "no_bias":
            mods[2] = _conv(64, 64, bias=False)
        elif case == "linear":
            mods[2] = nn.Linear(64, 64)
        else:
            mods[4] = nn.MaxPool2d(3, 2)
        f = nn.Sequential(*mods)
    with pytest.raises(ValueError):
        vgg_loss.check_layout(f)
    with pytest.raises(ValueError):
        VGGLoss(features=f)


@pytest.mark.parametrize("c", [64, 128, 256, 512])
def test_filter_split_gives_natural_raw_order(c):
    w = torch.randn(c, 16, 3, 3)
    wf, wm = vgg_loss.split_filters(w)
    assert wf.shape == wm.shape == (c // 2, 16, 3, 3)
    # RAW column j of the gated pair holds channel fm_columns(c/2)[j] of [f | m]: it must be plain output channel j
    assert torch.equal(torch.cat([wf, wm])[blocks.fm_columns(c // 2)], w)


def test_chunking_rule(monkeypatch):
    steps = vgg_loss.layer_walk(vgg_loss.LAYERS)
    # the widest RAW output is conv1_x: 2n x H x W x 64 elements, below 2^31
    assert vgg_loss.chunk_pairs(steps, 256, 256) == (2 ** 31 - 1) // (2 * 256 * 256 * 64)
    assert vgg_loss.chunk_pairs(steps, 70, 46, limit=2 * 70 * 46 * 64 + 1) == 1
    assert vgg_loss.chunk_pairs(steps, 70, 46, limit=3 * 2 * 70 * 46 * 64) == 2
    with pytest.raises(ValueError, match="RAW output limit"):
        vgg_loss.chunk_pairs(steps, 70, 46, limit=2 * 70 * 46 * 64)
    monkeypatch.setattr(vgg_loss, "RAW_LIMIT", 2 * 70 * 46 * 64 + 1)
    assert vgg_loss.chunk_pairs(steps, 70, 46) == 1


def test_constructor_rejections(features, tmp_path, monkeypatch):
    with pytest.raises(ValueError, match="partialconv"):
        VGGLoss(partialconv=True, features=features)
    with pytest.raises(ValueError, match="net"):
        VGGLoss(net='vgg', features=features)
    with pytest.raises(FileNotFoundError, match=str(tmp_path / vgg_loss.CAFFE_FILE)):
        VGGLoss(save_dir=str(tmp_path))
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "hub"))
    with pytest.raises(FileNotFoundError, match=vgg_loss.TORCHVISION_FILE):
        VGGLoss(net='pytorch')


def test_caffe_file_and_dropin_layout(features, tmp_path):
    torch.save(features, tmp_path / vgg_loss.CAFFE_FILE)
    crit = VGGLoss(save_dir=str(tmp_path))
    convs = [i for i, k in enumerate(vgg_loss.vgg19_modules()) if isinstance(k, tuple)]
    assert set(crit.state_dict()) == {'mean_', 'std_'} | {f"vgg19.{i}.{p}" for i in convs for p in ('weight', 'bias')}
    assert all(isinstance(crit.vgg19[i], nn.AvgPool2d) for i, k in enumerate(vgg_loss.vgg19_modules()) if k == 'pool')
    assert not any(p.requires_grad for p in crit.parameters())
    for i in convs:
        assert torch.equal(crit.vgg19[i].weight, features[i].weight)
    assert crit.layers == list(vgg_loss.LAYERS)
    assert VGGLoss(optimized=True, save_dir=str(tmp_path)).layers == list(vgg_loss.LAYERS_OPTIMIZED)
    assert torch.equal(crit.std_, torch.full((1, 3, 1, 1), 1. / 255))


def test_forward_rejections(features):
    crit = VGGLoss(features=features)
    x, t = vgg_util.seeded_images(1, 32, 32, 1)
    with pytest.raises(ValueError, match="target"):
        crit(x, t.clone().requires_grad_(True))
    crit.vgg19[0].weight.requires_grad_(True)
    with pytest.raises(ValueError, match="frozen"):
        crit(x, t)
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA"):     # without autograd a trainable weight is allowed
        crit(x, t)
    crit.vgg19[0].weight.requires_grad_(False)
    with pytest.raises(ValueError, match="shape"):
        crit(x, t[:, :, :16])
    with pytest.raises(ValueError, match="shape"):
        crit(x[:, :2], t[:, :2])
    with pytest.raises(RuntimeError, match="CUDA"):
        crit(x, t)


def test_replica_evaluates_through_torch(features):
    crit = VGGLoss(features=features)
    x, t = vgg_util.seeded_images(1, 32, 32, 2)
    crit._is_replica = True
    want = vgg_loss.reference_loss(crit.vgg19, crit.mean_, crit.std_, crit.layers, x, t)
    assert torch.equal(crit(x, t), want)


@pytest.mark.parametrize("net", ["caffe", "pytorch"])
@pytest.mark.parametrize("optimized", [False, True])
def test_float64_restatement_reproduces_reference(features, net, optimized):
    """The restatement the GPU tests use as ground truth, in float64, against the reference's VGGLoss in float32."""
    g = load_golden("ref_vgg_loss")
    tag = f"{net}_{'opt' if optimized else 'all'}"
    crit = VGGLoss(net=net, optimized=optimized, features=features).double()
    x, t = vgg_util.seeded_images(2, 48, 64, 5)
    x = x.double().requires_grad_(True)
    loss = vgg_loss.reference_loss(crit.vgg19, crit.mean_, crit.std_, crit.layers, x, t.double())
    loss.backward()
    assert abs(loss.item() - float(g[f"loss_{tag}"])) <= 1e-5 * abs(loss.item())
    want = torch.from_numpy(g[f"grad_{tag}"]).double()
    assert float((x.grad - want).norm() / want.norm()) <= 1e-4
