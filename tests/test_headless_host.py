"""read_b200.headless without a GPU: the restated src ModelAndLoss (tests/headless_util.py) against the reference's own, recorded in
tests/golden/ref_headless.npz; NetAndTexture's {'im_out'} contract; TexturePipeline.create's per-scene texture checkpoints, net, model
and --model check; and the reference's save_pipeline / load_pipeline (src/READ/pipelines/pipeline.py:34-74, restated) on it."""
import os
import pydoc
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

from read_b200 import compose, headless, pipeline, synth
from read_b200.unet import UNet

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import headless_util as hu  # noqa: E402
from conftest import load_golden  # noqa: E402


@pytest.fixture(scope="module")
def gold():
    return load_golden("ref_headless")


class _Fixed(nn.Module):
    def __init__(self, im_out):
        super().__init__()
        self.im_out = im_out

    def forward(self, *inputs, **kwargs):
        return {'im_out': self.im_out}


@pytest.mark.parametrize("tag,use_mask,with_mask", [("plain", False, False), ("mask", True, True), ("mask_none", True, False)])
def test_model_and_loss_restatement_matches_the_reference_bit_for_bit(gold, tag, use_mask, with_mask):
    im_out, target, mask = (torch.from_numpy(gold[k]) for k in ("im_out_operand", "target_operand", "mask_operand"))
    mal = hu.ModelAndLoss(_Fixed(im_out), nn.L1Loss(), use_mask=use_mask)
    output, loss = mal({'id': torch.zeros(2)}, target, label=None, mask=mask if with_mask else None)
    assert output['im_out'] is im_out
    assert list(loss) == list(gold[f"loss_keys_{tag}"])
    for k, v in loss.items():
        assert np.array_equal(v.detach().numpy(), gold[f"loss_{tag}_{k}"]), (k, float(v))


def test_unet_matches_the_src_unet(gold, synth_sd):
    """The src UNet returns {'im_out'}; ours returns the tensor NetAndTexture wraps: same keys, same values (torch path, fp32)."""
    assert list(gold["net_out_keys"]) == ['im_out']
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    net.eval()
    assert sorted(net.state_dict()) == sorted(gold["net_state_dict_keys"])
    out = net(*[torch.from_numpy(gold[f"net_input_{l}"]) for l in range(4)])      # grad enabled: the torch path on the CPU
    want = torch.from_numpy(gold["net_im_out"])
    assert float((out.detach() - want).abs().max()) <= 1e-5 * float(want.abs().max())


class _CountingNet(nn.Module):
    def __init__(self):
        super().__init__()
        self.calls, self.kwargs, self.outputs = 0, [], []

    def forward(self, *inputs, **kwargs):
        self.calls += 1
        self.kwargs.append(dict(kwargs))
        out = inputs[0][:, :3] * 2
        self.outputs.append(out)
        return out


class _StubTexture(nn.Module):
    """An 8-channel 'texture' of index maps on the CPU (PointTexture samples on the GPU only)."""

    def forward(self, ids):
        return ids.expand(-1, 8, -1, -1) * torch.arange(1., 9.)[None, :, None, None]


def _maps(B, S, n, gen):
    keys = [k.strip() for k in hu.INPUT_FORMAT.split(',')]
    maps = {k: torch.randint(0, n, (B, 1, S >> l, S >> l), generator=gen).float() for l, k in enumerate(keys)}
    maps['id'] = torch.zeros(B, dtype=torch.long)
    return maps


def test_net_and_texture_returns_im_out_and_passes_return_input_through():
    gen = torch.Generator().manual_seed(3)
    tex = _StubTexture()
    net = _CountingNet()
    model = headless.NetAndTexture(net, {0: tex}).eval()
    model.load_textures([0])
    maps = _maps(2, 16, 50, gen)
    out = model(maps, label=None, mask=None)
    assert set(out) == {'im_out'} and net.calls == 1                  # eval mode, one texture: one batched net call
    assert out['im_out'] is net.outputs[-1]
    assert net.kwargs[-1] == {'label': None, 'mask': None}
    res, net_input = model(maps, return_input=True)
    assert set(res) == {'im_out'} and res['im_out'] is net.outputs[-1]
    assert net.kwargs[-1] == {'return_input': True}
    base = compose.NetAndTexture(net, {0: tex}).eval()
    base.load_textures([0])
    want, want_input = base(maps, return_input=True)
    assert torch.equal(res['im_out'], want)
    assert len(net_input) == 5 and all(torch.equal(a, b) for a, b in zip(net_input, want_input))


def _two_scenes(tmp_path, monkeypatch, **kw):
    """Two scenes through a stubbed READ.datasets.dynamic; scene 0 warm-starts from a checkpoint, scene 1 has none."""
    scenes = [hu.scene(300, 32, 32, name="a", ds_id=0, seed=1), hu.scene(200, 32, 32, name="b/c", ds_id=1, seed=2)]
    ckpt_tex = pipeline.PointTexture(8, 300, init_method='rand')
    path = str(tmp_path / "PointTexture_a.pth")
    pipeline.save_model(path, ckpt_tex)
    mod = hu.datasets_module(scenes, [path, None])
    for name in ("READ", "READ.datasets", "READ.datasets.dynamic"):
        monkeypatch.setitem(sys.modules, name, mod)
    args = hu.pipeline_args(**kw)
    p = headless.TexturePipeline()
    p.create(args)
    return p, args, ckpt_tex


def test_create_loads_each_scene_texture_from_its_own_checkpoint(tmp_path, monkeypatch, gold):
    p, args, ckpt_tex = _two_scenes(tmp_path, monkeypatch, net_train_precision='bf16_all', net_train_batchnorm='per_item')
    assert torch.equal(p.textures[0].texture_.detach(), ckpt_tex.texture_.detach())
    assert p.textures[1].texture_.shape == (1, 8, 200) and not p.textures[1].texture_.detach().any()     # fresh: zeros
    assert args.input_channels == args.descriptor_size == 8
    assert isinstance(p.model, headless.NetAndTexture) and p.model.net is p.net is p.get_net()
    assert sorted(p.net.state_dict()) == sorted(gold["net_state_dict_keys"])
    assert (p.net.train_precision, p.net.train_batchnorm) == ('bf16_all', 'per_item')
    assert p._extra_optimizer is None and isinstance(p.optimizer, torch.optim.Adam)
    assert set(p.state_objects()) == {'net', 'a', 'b/c'}


def test_create_keeps_given_input_channels_and_needs_the_unet(tmp_path, monkeypatch):
    p, args, _ = _two_scenes(tmp_path, monkeypatch, input_channels=[8, 8])
    assert args.input_channels == [8, 8]
    with pytest.raises(ValueError, match="'other'"):
        headless.TexturePipeline().create(hu.pipeline_args(model='other'))


def test_inference_create_gives_a_fresh_texture():
    p = headless.TexturePipeline()
    p.create(hu.pipeline_args(inference=True, n_points=77))
    assert p.textures[0].texture_.shape == (1, 8, 77) and isinstance(p.model, headless.NetAndTexture)


def _save_pipeline(p, save_dir, epoch, args):
    """src/READ/pipelines/pipeline.py:58-74 with save_model of src/READ/utils/train.py:68-82."""
    for name, obj in p.state_objects().items():
        if name == 'net' and args.freeze_net:
            continue
        filename = f'{obj.__class__.__name__}_latest_{epoch}_{name.replace("/", "_")}'
        torch.save({'state_dict': obj.state_dict(), 'args': _deval_args(args)}, os.path.join(save_dir, filename + '.pth'))


def _deval_args(args):
    """The args as the reference's deval_args leaves them: modules named by their dotted path (src/READ/utils/arguments.py)."""
    return {k: f'{v.__module__}.{v.__qualname__}' if isinstance(v, type) else v for k, v in vars(args).items()}


def _load_pipeline(checkpoint, args_to_update):
    """src/READ/pipelines/pipeline.py:34-55 (munch.munchify replaced by a namespace)."""
    ckpt = torch.load(checkpoint, map_location='cpu')
    ckpt['args'].update(args_to_update)
    args = hu.pipeline_args(**ckpt['args'])
    p = pydoc.locate(args.pipeline)()
    p.create(args)
    p.get_net().load_state_dict(ckpt['state_dict'])
    return p, args


@pytest.mark.parametrize("freeze_net", [False, True])
def test_reference_save_and_load_pipeline(tmp_path, monkeypatch, freeze_net):
    p, args, _ = _two_scenes(tmp_path, monkeypatch, pipeline='read_b200.headless.TexturePipeline', freeze_net=freeze_net)
    with torch.no_grad():
        p.net.load_state_dict(synth.synth_state_dict(5))
        p.textures[1].texture_.add_(0.25)
    out = tmp_path / "ckpt"
    out.mkdir()
    _save_pipeline(p, str(out), 3, args)
    want = {'PointTexture_latest_3_a.pth', 'PointTexture_latest_3_b_c.pth'} | (set() if freeze_net else {'UNet_latest_3_net.pth'})
    assert set(os.listdir(out)) == want
    tex = pipeline.load_model_checkpoint(str(out / 'PointTexture_latest_3_b_c.pth'), pipeline.PointTexture(8, 200))
    assert torch.equal(tex.texture_, p.textures[1].texture_)
    if freeze_net:
        return
    q, _ = _load_pipeline(str(out / 'UNet_latest_3_net.pth'), {'inference': True, 'n_points': 300})
    assert isinstance(q, headless.TexturePipeline) and isinstance(q.model, headless.NetAndTexture)
    sd = q.net.state_dict()
    assert all(torch.equal(sd[k], v) for k, v in p.net.state_dict().items())
