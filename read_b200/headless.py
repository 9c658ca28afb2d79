"""The model contract of the reference's headless trainer (``src/train.py --headless``) over read_b200's classes.

The reference ships two trainers. The top-level one renders with OpenGL and needs a display; ``src/train.py --headless`` renders
with ``pcpr`` / ``MyRender`` in the training loop, so it is the one a GPU server without a screen runs. Its ``src/READ`` package
keeps a different model contract from the top-level one that ``read_b200.compose`` / ``read_b200.pipeline`` restate:

* ``NetAndTexture.forward`` returns ``{'im_out': [B,3,H,W]}`` (src/READ/models/compose.py:133-192), and ``(dict, net_input)``
  with ``return_input=True``; the ``ModelAndLoss`` of ``src/`` reads ``output['im_out']``;
* the pipeline (src/READ/pipelines/ogl.py:64-120) unpacks ``(train, val, texture_ckpts)`` from ``get_datasets`` and warm-starts
  each scene's descriptors from its own checkpoint, takes the net from ``READ.models.{args.model}`` and sets
  ``args.input_channels = args.descriptor_size``.

Use ``--pipeline read_b200.headless.TexturePipeline`` (INTEGRATION.md, "Headless trainer"). Everything else - texture residency,
one-call batching, the direct-to-engine inference shortcut, ``render()``, the CLI flags, the sparse descriptor optimizer and the
train.py hooks - is inherited from ``read_b200.compose`` / ``read_b200.pipeline``.
"""
from torch import optim

from . import compose, pipeline
from .texture import PointTexture

MODELS = ('unet',)          # the model files of src/READ/models that --model may name


class NetAndTexture(compose.NetAndTexture):
    """``compose.NetAndTexture`` returning the headless trainer's ``{'im_out': out}``; ``out`` is the same tensor, not a copy.
    Keyword arguments (``label``, ``mask``, ``return_input``) reach the net as in the reference, which ignores them."""

    def forward(self, inputs, **kwargs):
        res = super().forward(inputs, **kwargs)
        if kwargs.get('return_input'):
            out, net_input = res
            return {'im_out': out}, net_input
        return {'im_out': res}


def get_texture(num_channels, size, args, texture_ckpt=None):
    """One descriptor set, warm-started from ``texture_ckpt`` when it is not None (src/READ/pipelines/ogl.py:38-48)."""
    if getattr(args, 'use_mesh', False):
        raise NotImplementedError("read_b200: mesh textures (MeshTexture) are outside the point-cloud hot path")
    if not hasattr(args, 'reg_weight'):
        args.reg_weight = 0.
    texture = PointTexture(num_channels, size, activation=args.texture_activation, reg_weight=args.reg_weight)
    return pipeline.load_model_checkpoint(texture_ckpt, texture) if texture_ckpt is not None else texture


class TexturePipeline(pipeline.TexturePipeline):
    """``pipeline.TexturePipeline`` with the construction of src/READ/pipelines/ogl.py:73-120."""

    def create(self, args):
        model = getattr(args, 'model', 'unet')
        if model not in MODELS:
            raise ValueError(f"read_b200.headless: --model {model!r} is not available; the net is read_b200.unet.UNet "
                             f"(--model {' / '.join(MODELS)})")
        if not getattr(args, 'input_channels', None):
            args.input_channels = args.descriptor_size
        self.args = args
        self.net = pipeline.get_net(args.input_channels, args)
        self.net.train_precision = getattr(args, 'net_train_precision', 'fp32')
        self.net.train_batchnorm = getattr(args, 'net_train_batchnorm', 'batch')
        if getattr(args, 'inference', False):
            self.textures = {0: get_texture(args.descriptor_size, args.n_points, args)}
        else:
            self.textures = self._create_training_state(args)
        self.model = NetAndTexture(self.net, self.textures, getattr(args, 'supersampling', 1))

    def _create_training_state(self, args):
        """Datasets, one texture per scene from its own checkpoint (None: fresh), both optimizers and the criterion."""
        from READ.datasets.dynamic import get_datasets          # the reference's data path, out of scope here
        self.ds_train, self.ds_val, self.texture_ckpts = get_datasets(args)
        textures = {}
        for ds in self.ds_train:
            cloud = ds.scene_data['pointcloud']
            assert cloud is not None, 'set pointcloud'
            textures[ds.id] = get_texture(args.descriptor_size, cloud['xyz'].shape[0], args, self.texture_ckpts[ds.id])
        self.optimizer = optim.Adam(self.net.parameters(), lr=args.lr)
        # a single scene keeps ONE descriptor optimizer alive so that its running averages survive across epochs
        self._extra_optimizer = pipeline._texture_optimizer(args, [textures[0]], args.texture_lr) if len(textures) == 1 else None
        self.criterion = args.criterion_module(**args.criterion_args).cuda()
        return textures
