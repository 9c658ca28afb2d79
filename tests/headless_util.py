"""The training step of the reference's headless trainer (src/train.py:161-266), restated for the tests and
scripts/bench_headless_step.py (the reference is not importable there), and a synthetic one-scene dataset for it.

One step: ``MyRender.render`` -> ``to_device`` -> ``ModelAndLoss`` (src/READ/models/compose.py:14-42) -> ``vgg + 1e4 * huber``,
with a mask divided by its mean and the background term added -> ``+ reg_loss`` -> ``backward`` -> the net's optimizer and the
pipeline's descriptor optimizer.  tests/test_headless_host.py pins ModelAndLoss to the reference through tests/golden/ref_headless.npz.
"""
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from read_b200 import synth, vgg_loss

HUBER_RATIO = 1e4            # src/train.py:572
BKG_WEIGHT = 500             # src/train.py:234
INPUT_FORMAT = "uv_1d_p1, uv_1d_p1_ds1, uv_1d_p1_ds2, uv_1d_p1_ds3, uv_1d_p1_ds4"     # src/configs/train_example.yaml


class ModelAndLoss(nn.Module):
    """src/READ/models/compose.py:14-42: the model's {'im_out'} and {'vgg_loss', 'huber_loss'[, 'seg_loss']}."""

    def __init__(self, model, loss, use_mask=False):
        super().__init__()
        self.model, self.loss, self.use_mask = model, loss, use_mask

    def forward(self, *args, **kwargs):
        output = self.model(*args[:-1], **kwargs)
        im_out, target, mask = output['im_out'], args[-1], kwargs.get('mask')
        x = im_out * mask if self.use_mask and mask is not None else im_out
        loss = {'vgg_loss': self.loss(x, target), 'huber_loss': F.huber_loss(x, target)}
        if 'seg_out' in output and kwargs.get('label') is not None:
            loss['seg_loss'] = F.cross_entropy(output['seg_out'], kwargs['label'], ignore_index=0)
        return output, loss


def to_device(data, device):
    """src/READ/utils/train.py:40-53."""
    if isinstance(data, torch.Tensor):
        return data.to(device, non_blocking=True)
    if isinstance(data, dict):
        for k in data:
            data[k] = to_device(data[k], device)
    return data


def step_loss(output, loss_dict, mask, reg_loss):
    """src/train.py:226-253: the scalar the trainer backpropagates."""
    im_out = output['im_out']
    loss = loss_dict['vgg_loss'] + loss_dict['huber_loss'] * HUBER_RATIO
    if mask is not None:
        loss = loss / (mask.mean() + 1e-6)
        n_mask = 1 - mask
        bkg = torch.zeros((1, 3, 1, 1), device=loss.device) * n_mask
        loss = loss + BKG_WEIGHT * torch.abs(im_out * n_mask - bkg).mean() / (n_mask.mean() + 1e-6)
    return loss + reg_loss


def forward_loss(renderer, model, data, target, mask, device, reg_loss):
    """Render, move to the device, run ``model`` (a ModelAndLoss, possibly under nn.DataParallel) -> the step's loss."""
    inputs, _depths = renderer.render(data)
    data_input = to_device(inputs, device)
    output, loss_dict = model(data_input, target, label=None, mask=mask)
    return step_loss(output, loss_dict, mask, reg_loss())


def train_step(renderer, model, data, target, mask, device, pipeline, extra_optimizer):
    loss = forward_loss(renderer, model, data, target, mask, device, pipeline.model.reg_loss)
    loss.backward()
    pipeline.optimizer.step()
    pipeline.optimizer.zero_grad()
    if extra_optimizer is not None:
        extra_optimizer.step()
        extra_optimizer.zero_grad()
    return loss


class TorchVGG(nn.Module):
    """The reference's VGG loss loop on torch operators (vgg_loss.reference_loss) over the layers of a VGGLoss."""

    def __init__(self, **kwargs):
        super().__init__()
        self.crit = vgg_loss.VGGLoss(**kwargs)

    def forward(self, input, target):
        c = self.crit
        return vgg_loss.reference_loss(c.vgg19, c.mean_, c.std_, c.layers, input, target)


def scene(n_points, W, H, name="synthetic", ds_id=0, seed=synth.SEED, depth=60.0):
    """One dataset as the pipeline and MyRender see it: id, name, tgt_sh, input_format and the point cloud; load / unload are no-ops."""
    return types.SimpleNamespace(id=ds_id, name=name, tgt_sh=(W, H), input_format=INPUT_FORMAT,
                                 scene_data={'pointcloud': {'xyz': synth.street_scene(n_points, depth=depth, seed=seed)}},
                                 load=lambda: None, unload=lambda: None)


def batch(W, H, ts, ds_id=0, seed=synth.SEED):
    """The DataLoader fields MyRender.render reads: input ids and per-crop projection / view matrices (CPU)."""
    proj, view = synth.crop_cameras(W, H, ts, np.random.default_rng(seed))
    return {'input': {'id': torch.full((len(ts),), ds_id, dtype=torch.long)},
            'proj_matrix': torch.from_numpy(proj), 'view_matrix': torch.from_numpy(view)}


def pipeline_args(**kw):
    """The parsed flags src/train.py hands to TexturePipeline.create for one synthetic scene."""
    a = dict(descriptor_size=8, texture_activation='none', texture_lr=1e-1, lr=1e-4, n_points=0, inference=False,
             use_mesh=False, model='unet', input_channels=None, supersampling=1, net_train_precision='fp32',
             net_train_batchnorm='batch', criterion_module=nn.L1Loss, criterion_args={})
    a.update(kw)
    return types.SimpleNamespace(**a)


def datasets_module(datasets, texture_ckpts):
    """A stand-in for READ.datasets.dynamic whose get_datasets returns ``(datasets, datasets, texture_ckpts)``."""
    return types.SimpleNamespace(get_datasets=lambda args: (list(datasets), list(datasets), list(texture_ckpts)))
