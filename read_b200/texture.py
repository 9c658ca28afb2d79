"""Drop-in for ``READ.models.texture.PointTexture`` (READ/models/texture.py:14-70).

Same constructor, same parameter (``texture_`` [1,C,N] f32, so checkpoints load unchanged), same forward
contract (ids [B,1|3,h,w] float -> [B,C,h,w] f32; int32 maps, which clouds of more than 2^24 + 1 points get, pass unconverted).  The gather and its backward (scatter-add into
``texture_.grad``) are hand-written CUDA kernels reading a point-major [N,C] shadow of the parameter.
"""
import torch
import torch.nn as nn

from . import ops
from . import _lib as L


class Texture(nn.Module):
    """Interface of the reference's texture modules (READ/models/texture.py:6-11): a regulariser that defaults to zero and a
    ``null_grad`` every concrete texture must provide (train.py calls it when a dataset is unloaded)."""

    def null_grad(self):
        raise NotImplementedError(f"{type(self).__name__} does not implement null_grad()")

    def reg_loss(self):
        return 0.


class _Gather(torch.autograd.Function):
    @staticmethod
    def forward(ctx, texture_, ids):
        tex_nd = ops.texture_to_point_major(texture_)
        ctx.save_for_backward(ids)
        ctx.n = texture_.shape[-1]
        return ops.gather_from_index(tex_nd, ids, L.FEAT_NCHW_F32)

    @staticmethod
    def backward(ctx, grad_out):
        (ids,) = ctx.saved_tensors
        g_nd = ops.gather_backward(grad_out, ids, ctx.n)        # [N,C]
        return ops.texture_to_channel_major(g_nd), None         # [1,C,N]


class _GatherItems(torch.autograd.Function):
    """_Gather / train._GatherSparse for a batch whose item b samples ``textures[slots[b]]``: one gather and one scatter per call.
    Sparse: every slot's accumulator receives its items' gradient and the Function returns None; dense: one [1, 8, N] gradient per
    texture.  A texture whose parameter does not require grad gets None and its accumulator is left alone."""

    @staticmethod
    def forward(ctx, ids, slots, textures, sparse, *params):
        ctx.save_for_backward(ids)
        ctx.slots, ctx.textures, ctx.sparse = slots, textures, sparse
        return ops.gather_from_index_items([t.point_major() for t in textures], slots, ids, L.FEAT_NCHW_F32)

    @staticmethod
    def backward(ctx, grad_out):
        (ids,) = ctx.saved_tensors
        need = ctx.needs_input_grad[4:]
        g = grad_out if grad_out.dtype == torch.float32 else grad_out.float()
        N = [t.texture_.shape[-1] for t in ctx.textures]
        if ctx.sparse:
            st = [t._sparse if n else None for t, n in zip(ctx.textures, need)]
            ops.gather_backward_items(g, ids, ctx.slots, N, [None if s is None else s.grad for s in st],
                                      [None if s is None else s.touched for s in st])
            return (None,) * (4 + len(N))
        grads = [torch.zeros((n, 8), dtype=torch.float32, device=g.device) if r else None for n, r in zip(N, need)]
        ops.gather_backward_items(g, ids, ctx.slots, N, grads)
        return (None,) * 4 + tuple(None if gd is None else ops.texture_to_channel_major(gd) for gd in grads)


def sample_items(textures, slots, inputs):
    """``PointTexture.forward`` for a batch whose item b samples ``textures[slots[b]]``, in one gather launch (and one scatter in the
    backward).  The textures are PointTextures with 8 channels, one activation and one gradient mode (read_b200.compose checks)."""
    ids = inputs[:, 0]
    for t in textures:
        if not t.texture_.is_cuda:
            raise RuntimeError("read_b200.PointTexture: texture must be on a CUDA device (no CPU fallback)")
    ids = ops.index_map(ids, textures[0].texture_.device)
    act = textures[0].activation
    params = [t.texture_ for t in textures]
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        sparse = getattr(textures[0], '_sparse_requested', False)
        if sparse:
            from . import train
            for t in textures:
                train.enable_sparse_grad(t)
        sample = _GatherItems.apply(ids, tuple(slots), tuple(textures), sparse, *params)
        if act == 'sigmoid':
            return torch.sigmoid(sample)
        if act == 'tanh':
            return torch.tanh(sample)
        return sample
    return ops.gather_from_index_items([t.point_major() for t in textures], slots, ids, L.FEAT_NCHW_F32, act)


_INITIALISERS = {'zeros': torch.zeros, 'rand': torch.rand}


class PointTexture(Texture):
    """Per-point descriptors.  Constructor contract of READ/models/texture.py:14-35: ``texture_`` is a float32 Parameter of shape
    [1, num_channels, size] (channel-major, the checkpoint layout), filled by ``init_method`` ('zeros' | 'rand'), or taken from a
    pickled ``{'texture': module}`` checkpoint; ``activation`` in {'none', 'sigmoid', 'tanh'} is applied to the samples."""

    def __init__(self, num_channels, size, activation='none', checkpoint=None, init_method='zeros', reg_weight=0.):
        super().__init__()
        assert isinstance(size, int), 'size must be int'
        if checkpoint:
            descriptors = torch.load(checkpoint, map_location='cpu')['texture'].texture_
        else:
            make = _INITIALISERS.get(init_method)
            if make is None:
                raise ValueError(init_method)
            descriptors = nn.Parameter(make((1, num_channels, size), dtype=torch.float32))
        self.texture_ = descriptors
        self.activation, self.reg_weight = activation, reg_weight
        self._shadow = self._shadow_key = None          # point-major copy for the gather kernels, see point_major()
        self._sparse, self._sparse_requested = None, False     # read_b200.train: sparse gradient accumulator

    def null_grad(self):
        self.texture_.grad = None
        sp = getattr(self, '_sparse', None)
        if sp is not None:                             # the pending regulariser's gradient goes with it, as texture_.grad does
            sp.reg_coef = None

    def reg_loss(self):
        """L2 regulariser of texture.py:40-41: reg_weight * mean(texture^2).  A CUDA texture in sparse mode (SparseRMSprop) that
        needs a gradient takes train._RegLoss: the value from our reduction kernel, and a backward that leaves the gradient as one
        scalar for the optimizer step instead of a dense texture_.grad.  Otherwise (reg_weight 0 included) the torch expression."""
        t = self.texture_
        if (self.reg_weight != 0 and getattr(self, '_sparse_requested', False) and t.is_cuda and torch.is_grad_enabled()
                and t.requires_grad):
            from . import train
            return train._RegLoss.apply(t, self)
        return self.reg_weight * t.square().mean()

    def point_major(self):
        """[N,C] shadow of ``texture_`` on its device, refreshed whenever the parameter changes."""
        t = self.texture_
        key = (t.data_ptr(), t._version, t.device)
        if self._shadow_key != key:
            self._shadow = ops.texture_to_point_major(t.detach())
            self._shadow_key = key
        return self._shadow

    def forward(self, inputs):
        if isinstance(inputs, dict):
            ids = None
            for f, x in inputs.items():
                if 'uv' in f:
                    ids = x[:, 0]
            assert ids is not None, 'Input format does not have uv'
        else:
            ids = inputs[:, 0]                                   # BxHxW
        if not self.texture_.is_cuda:
            raise RuntimeError("read_b200.PointTexture: texture must be on a CUDA device (no CPU fallback)")
        ids = ops.index_map(ids, self.texture_.device)
        if torch.is_grad_enabled() and self.texture_.requires_grad:
            if getattr(self, '_sparse_requested', False):
                # training with read_b200.train.SparseRMSprop: the backward scatter-adds into a persistent point-major accumulator
                # and flags the touched points; texture_.grad is never materialised
                from . import train
                train.enable_sparse_grad(self)
                sample = train._GatherSparse.apply(self.texture_, ids, self)
            else:
                sample = _Gather.apply(self.texture_, ids)
            if self.activation == 'sigmoid':
                return torch.sigmoid(sample)
            if self.activation == 'tanh':
                return torch.tanh(sample)
            return sample
        return ops.gather_from_index(self.point_major(), ids, L.FEAT_NCHW_F32, self.activation)
