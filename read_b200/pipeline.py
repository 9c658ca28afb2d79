"""Drop-in for ``READ.pipelines.ogl.TexturePipeline`` (READ/pipelines/ogl.py:58-154) over the H100 kernels.

Use ``--pipeline read_b200.pipeline.TexturePipeline`` with the reference's train.py (the plugin is located by dotted path,
READ/utils/train.py:148-154), or shadow ``READ.pipelines.ogl`` (INTEGRATION.md).  The plugin contract train.py / viewer.py rely
on, restated here rather than lifted:

* CLI: ``--descriptor_size --texture_size --texture_ckpt --texture_lr --texture_activation --n_points`` (ogl.py:59-65);
* after ``create(args)``: ``model`` (NetAndTexture), ``net``, ``textures`` {dataset id -> PointTexture}, ``args`` and - in training
  mode - ``ds_train``, ``ds_val``, ``optimizer`` (Adam over the net), ``criterion`` (train.py:509-510);
* ``state_objects()`` -> what gets checkpointed: the net under 'net', each texture under its dataset's name (ogl.py:114-120);
* ``dataset_load / dataset_unload`` bracket every train / eval epoch, ``extra_optimizer(datasets)`` returns the RMSprop over the
  descriptors whose learning rate follows the net's schedule (ogl.py:129-144);
* checkpoints are ``{'state_dict': ..., 'args': ...}`` (READ/utils/train.py:42-65).

Dataset construction (``get_datasets``) and the loss stay the reference's own code: they are outside the render hot path
(SURVEY.md §8) and are imported lazily from ``READ`` only in training mode.
"""
from pathlib import Path

import torch
from torch import optim

from .texture import PointTexture
from .unet import UNet
from .compose import NetAndTexture

TextureOptimizerClass = optim.RMSprop        # the descriptor optimizer the reference uses (ogl.py:16)


def _texture_optimizer(args, textures, lr):
    """The reference's dense RMSprop, or (default) read_b200.train.SparseRMSprop: same update, applied only to the points a batch
    touched, fed by the sparse gather backward (``--dense_texture_optimizer`` keeps torch's)."""
    if getattr(args, 'dense_texture_optimizer', False):
        return TextureOptimizerClass([{'params': t.parameters()} for t in textures], lr=lr)
    from .train import SparseRMSprop
    return SparseRMSprop(list(textures), lr=lr)

# (flag, kwargs, registered through parser.add - the reference's "also store in the yaml config" alias - or add_argument)
_CLI = (
    ('--descriptor_size', dict(type=int, default=8), False),
    ('--texture_size', dict(type=int), False),
    ('--texture_ckpt', dict(type=Path), False),
    ('--texture_lr', dict(type=float, default=1e-1), True),
    ('--texture_activation', dict(type=str, default='none'), True),
    ('--n_points', dict(type=int, default=0, help='this is for inference'), True),
    ('--dense_texture_optimizer', dict(action='store_true', help='torch.optim.RMSprop over all points instead of the sparse kernel'), False),
    ('--net_train_precision', dict(type=str, default='fp32', choices=['fp32', 'bf16', 'bf16_all'],
                                   help="bf16: train the net's 3x3 stride-1 convs on the wgmma kernels; bf16_all: every conv "
                                        "(UNet.train_precision)"), False),
    ('--net_train_batchnorm', dict(type=str, default='batch', choices=['batch', 'per_item'],
                                   help="train-mode BatchNorm statistics over the whole net call (batch) or per crop (per_item: "
                                        "the training batch runs as one net call, with the statistics of the per-crop loop; "
                                        "UNet.train_batchnorm)"), False),
)


class Pipeline:
    """The plugin protocol of READ/pipelines/pipeline.py:10-31: a pipeline must be able to register its flags, build itself from
    the parsed args and hand out its net; the dataset hooks and the extra optimizer are optional."""

    def _abstract(self, what):
        raise NotImplementedError(f"{type(self).__name__} must implement {what}()")

    def export_args(self, parser):
        self._abstract('export_args')

    def create(self, args):
        self._abstract('create')

    def get_net(self):
        self._abstract('get_net')

    def dataset_load(self, *args, **kwargs):
        return None

    def dataset_unload(self, *args, **kwargs):
        return None

    def extra_optimizer(self, *args):
        return None


def load_model_checkpoint(path, model):
    """Counterpart of READ/utils/train.py:60-65: restore ``model`` from a ``{'state_dict': ...}`` file."""
    state = torch.load(path, map_location='cpu')['state_dict']
    model.load_state_dict(state)
    return model


def save_model(save_path, model, args=None):
    """Counterpart of READ/utils/train.py:42-57: ``{'state_dict': ..., 'args': ...}``; a DataParallel wrapper is looked through."""
    payload = {'state_dict': getattr(model, 'module', model).state_dict()}
    if args is not None:
        payload['args'] = dict(vars(args)) if hasattr(args, '__dict__') else dict(args)
    torch.save(payload, save_path)


def get_net(input_channels, args):
    """The refinement net of the texture pipeline (ogl.py:19-27): 8 descriptor channels in, RGB out, 4 residual blocks per stage."""
    return UNet(num_input_channels=8, num_output_channels=3, feature_scale=4, num_res=4)


def get_texture(num_channels, size, args):
    """One descriptor set (ogl.py:30-43); ``args.texture_ckpt`` warm-starts it.  Mesh textures are not on the point-cloud path."""
    if getattr(args, 'use_mesh', False):
        raise NotImplementedError("read_b200: mesh textures (MeshTexture) are outside the point-cloud hot path")
    if not hasattr(args, 'reg_weight'):
        args.reg_weight = 0.
    texture = PointTexture(num_channels, size, activation=args.texture_activation, reg_weight=args.reg_weight)
    ckpt = getattr(args, 'texture_ckpt', None)
    return load_model_checkpoint(ckpt, texture) if ckpt else texture


class TexturePipeline(Pipeline):
    def export_args(self, parser):
        for flag, kw, via_add in _CLI:
            (getattr(parser, 'add', parser.add_argument) if via_add else parser.add_argument)(flag, **kw)

    # -------------------------------------------------------------------------------------------- construction
    def create(self, args):
        if not getattr(args, 'input_channels', None):                      # older configs do not carry it (ogl.py:46-47,71-72)
            args.input_channels = [args.descriptor_size] * getattr(args, 'num_mipmap', 5)
        self.args = args
        self.net = get_net(args.input_channels, args)
        self.net.train_precision = getattr(args, 'net_train_precision', 'fp32')
        self.net.train_batchnorm = getattr(args, 'net_train_batchnorm', 'batch')
        if getattr(args, 'inference', False):
            self.textures = {0: get_texture(args.descriptor_size, args.n_points, args)}
        else:
            self.textures = self._create_training_state(args)
        self.model = NetAndTexture(self.net, self.textures, getattr(args, 'supersampling', 1))

    def _create_training_state(self, args):
        """Datasets, one texture per scene, both optimizers and the criterion (ogl.py:84-102)."""
        from READ.datasets.dynamic import get_datasets          # the reference's data path, out of scope here
        self.ds_train, self.ds_val = get_datasets(args)
        textures = {}
        for ds in self.ds_train:
            cloud = ds.scene_data['pointcloud']
            assert cloud is not None, 'set pointcloud'
            textures[ds.id] = get_texture(args.descriptor_size, cloud['xyz'].shape[0], args)
        self.optimizer = optim.Adam(self.net.parameters(), lr=args.lr)
        # a single scene keeps ONE descriptor optimizer alive so that its running averages survive across epochs
        self._extra_optimizer = _texture_optimizer(args, [textures[0]], args.texture_lr) if len(textures) == 1 else None
        self.criterion = args.criterion_module(**args.criterion_args).cuda()
        return textures

    # -------------------------------------------------------------------------------------------- train.py hooks
    def state_objects(self):
        objs = {ds.name: self.textures[ds.id] for ds in self.ds_train}
        objs['net'] = self.net
        return objs

    def dataset_load(self, dataset):
        self.model.load_textures([ds.id for ds in dataset])
        for ds in dataset:
            ds.load()

    def dataset_unload(self, dataset):
        self.model.unload_textures()
        for ds in dataset:
            ds.unload()
            self.textures[ds.id].null_grad()

    def _texture_lr(self):
        """texture_lr scaled by however far the net's schedule has dropped its own rate (ogl.py:131-132,142)."""
        return self.args.texture_lr * self.optimizer.param_groups[0]['lr'] / self.args.lr

    def extra_optimizer(self, dataset):
        lr = self._texture_lr()
        if self._extra_optimizer is None:
            return _texture_optimizer(self.args, [self.textures[ds.id] for ds in dataset], lr)
        self._extra_optimizer.param_groups[0]['lr'] = lr
        return self._extra_optimizer

    def get_net(self):
        return self.net
