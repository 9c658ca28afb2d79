"""-m gpu: the reference's headless trainer (src/train.py --headless) on read_b200.headless, with its step restated in
tests/headless_util.py (MyRender.render -> to_device -> ModelAndLoss -> vgg + 1e4 * huber (+ the mask terms) -> backward -> Adam and
the pipeline's descriptor optimizer) on a synthetic scene, the pipeline built by headless.TexturePipeline.create through a stand-in
for READ.datasets.dynamic, the scene's texture warm-started from its checkpoint and VGG19 weights seeded (tests/vgg_util.py).

* eval mode: headless.NetAndTexture's 'im_out' bit-identical to compose.NetAndTexture's output, for both net.precision values and
  the example config's five 'uv' keys;
* 20 steps at 2 x 256^2: bf16_all with VGGLoss on our kernels against fp32 with the torch VGG loss, both descending, the descent and
  the final loss within bounds frozen per configuration: in eval mode (eval_in_train), with use_mask and VGGLoss(partialconv=True),
  and in train() with per-item BatchNorm;
* the step under nn.DataParallel with one device gives the loss it gives without.
"""
import os
import sys

import pytest
import torch

from read_b200 import compose, headless, pipeline, synth, vgg_loss
from read_b200.myrender import MyRender
from read_b200.texture import PointTexture
from read_b200.unet import UNet
from read_b200.vgg_loss import VGGLoss

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import headless_util as hu  # noqa: E402
import vgg_util  # noqa: E402
from gpu_util import dev  # noqa: E402

pytestmark = pytest.mark.gpu

W = H = 256
N_POINTS = 300_000
CAMERAS = [3, 11]
STEPS = 20
# 20 steps of bf16_all + VGGLoss against fp32 + the torch VGG loss, (descent, final loss) bounds measured on an H100 80GB HBM3 and
# frozen.  Eval mode, three runs: the arms' descents within 0.7 %, final losses within 1.4 %; with the mask, one run: 0.2 % / 0.4 %.
# train() per item, three runs of each arm: descents within 4.5 %, final losses within 5.4 %.  There the fp32 arm alone moved by
# 3.0 % (descent) and 7.2 % (final) between runs: batch statistics and the descriptors' RMSprop (lr 0.1, whose first steps are
# about +-lr * 10 whatever the gradient's size) amplify rounding differences, cuDNN's among them.
BOUNDS = {"eval": (0.015, 0.03), "use_mask": (0.015, 0.03), "train_per_item": (0.10, 0.10)}


def _rand_texture(n, seed=synth.SEED):
    tex = PointTexture(8, n)
    with torch.no_grad():
        tex.texture_.copy_(torch.rand((1, 8, n), generator=torch.Generator().manual_seed(seed)))
    return tex


@pytest.fixture(scope="module")
def scene():
    return hu.scene(N_POINTS, W, H)


@pytest.fixture(scope="module")
def texture_ckpt(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("headless") / "PointTexture_synthetic.pth")
    pipeline.save_model(path, _rand_texture(N_POINTS))
    return path


def _renderer(scene):
    r = MyRender()
    r.update_ds([scene])
    return r


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_eval_im_out_is_bit_identical_to_compose(scene, precision, synth_sd):
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    net.precision = precision
    tex = _rand_texture(N_POINTS)
    ours = headless.NetAndTexture(net, {0: tex})
    base = compose.NetAndTexture(net, {0: tex})
    for m in (ours, base):
        m.load_textures([0])
        m.to(dev()).eval()
    inputs, _ = _renderer(scene).render(hu.batch(W, H, CAMERAS))
    assert len(inputs) == 6                                               # five 'uv' keys and 'id'
    maps = hu.to_device(inputs, dev())
    with torch.no_grad():
        want, want_input = base(dict(maps), return_input=True)
        got = ours(dict(maps), label=None, mask=None)
        got_r, got_input = ours(dict(maps), return_input=True)
    torch.cuda.synchronize()
    assert set(got) == {'im_out'} and got['im_out'].shape == (2, 3, H, W)
    assert torch.equal(got['im_out'], want) and torch.equal(got_r['im_out'], want)
    assert all(torch.equal(a, b) for a, b in zip(got_input, want_input))


def _pipeline(monkeypatch, scene, texture_ckpt, synth_sd, precision, batchnorm, criterion):
    mod = hu.datasets_module([scene], [texture_ckpt])
    for name in ("READ", "READ.datasets", "READ.datasets.dynamic"):
        monkeypatch.setitem(sys.modules, name, mod)
    crit_cls, crit_args = criterion
    p = headless.TexturePipeline()
    p.create(hu.pipeline_args(net_train_precision=precision, net_train_batchnorm=batchnorm, criterion_module=crit_cls,
                              criterion_args=crit_args))
    p.net.load_state_dict(synth_sd, strict=True)
    return p


def _features(partial):
    f = vgg_util.seeded_features()
    return vgg_loss.partial_features(f) if partial else f


def _target_and_mask(use_mask):
    target = torch.rand((2, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev())
    if not use_mask:
        return target, None
    mask = torch.ones((2, 1, H, W))
    mask[0, :, 40:120, 60:200] = 0
    mask[1, :, 150:, :90] = 0
    mask = mask.to(dev())
    return target * mask, mask                                           # src/train.py:176-187


def _run(p, scene, train_mode, use_mask, eval_crit):
    """The trainer's epoch set-up (src/train.py:145-166, 313-320, 330-352) and STEPS steps; returns (first, final) losses measured
    with ``eval_crit`` on the arm's own net path."""
    renderer = _renderer(scene)
    model = hu.ModelAndLoss(p.model, p.criterion, use_mask=use_mask)
    measure = hu.ModelAndLoss(p.model, eval_crit, use_mask=use_mask)
    p.model.train(train_mode)
    p.dataset_load([scene])
    extra = p.extra_optimizer([scene])
    p.model.cuda()
    data = hu.batch(W, H, CAMERAS)
    target, mask = _target_and_mask(use_mask)

    def loss_of(m):
        return float(hu.forward_loss(renderer, m, data, target, mask, dev(), p.model.reg_loss).detach())

    first = loss_of(measure)
    for _ in range(STEPS):
        hu.train_step(renderer, model, data, target, mask, dev(), p, extra)
    final = loss_of(measure)
    p.dataset_unload([scene])
    return first, final


CONFIGS = {
    "eval": dict(train_mode=False, batchnorm='batch', use_mask=False),
    "use_mask": dict(train_mode=False, batchnorm='batch', use_mask=True),
    "train_per_item": dict(train_mode=True, batchnorm='per_item', use_mask=False),
}


@pytest.mark.parametrize("config", list(CONFIGS))
def test_bf16_all_with_vgg_loss_tracks_fp32_with_the_torch_loss(monkeypatch, scene, texture_ckpt, synth_sd, config):
    c = CONFIGS[config]
    partial = c['use_mask']
    eval_crit = hu.TorchVGG(partialconv=partial, features=_features(partial)).to(dev())
    arms = {"fp32": ("fp32", (hu.TorchVGG, {'partialconv': partial, 'features': _features(partial)})),
            "bf16_all": ("bf16_all", (VGGLoss, {'partialconv': partial, 'features': _features(partial)}))}
    first, final = {}, {}
    for arm, (precision, criterion) in arms.items():
        p = _pipeline(monkeypatch, scene, texture_ckpt, synth_sd, precision, c['batchnorm'], criterion)
        assert isinstance(p.criterion, criterion[0])
        first[arm], final[arm] = _run(p, scene, c['train_mode'], c['use_mask'], eval_crit)
    descent = {k: first[k] - final[k] for k in final}
    print(f"\nheadless step {config}, {STEPS} steps: first {first}, final {final}, descent {descent}")
    assert all(d > 0 for d in descent.values()), descent
    descent_rel, final_rel = BOUNDS[config]
    assert abs(descent["bf16_all"] - descent["fp32"]) <= descent_rel * descent["fp32"], descent
    assert abs(final["bf16_all"] - final["fp32"]) <= final_rel * final["fp32"], final


def test_data_parallel_with_one_device_gives_the_same_loss(monkeypatch, scene, texture_ckpt, synth_sd):
    p = _pipeline(monkeypatch, scene, texture_ckpt, synth_sd, "bf16_all", "batch", (VGGLoss, {'features': _features(False)}))
    renderer = _renderer(scene)
    model = hu.ModelAndLoss(p.model, p.criterion)
    p.model.eval()
    p.dataset_load([scene])
    p.model.cuda()
    data = hu.batch(W, H, CAMERAS)
    target, _ = _target_and_mask(False)
    plain = hu.forward_loss(renderer, model, data, target, None, dev(), p.model.reg_loss)
    wrapped = hu.forward_loss(renderer, torch.nn.DataParallel(model, device_ids=[0]), data, target, None, dev(), p.model.reg_loss)
    torch.cuda.synchronize()
    print(f"\nloss {float(plain)} plain, {float(wrapped)} under DataParallel")
    assert torch.equal(plain, wrapped)
    p.dataset_unload([scene])
