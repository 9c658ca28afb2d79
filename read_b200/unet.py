"""Drop-in for ``READ.models.unet.UNet`` (READ/models/unet.py:121-285).

``state_dict()`` keys and shapes are identical to the reference (909 entries such as
``Encoder.0.layers.0.main.0.block.conv_f.weight`` / ``...block.norm.running_mean``), so ``load_state_dict`` of a
reference checkpoint works with ``strict=True``.  The module tree is generated from a layer table instead of
hand-written block classes; it only HOLDS parameters.

Inference (``torch.no_grad()`` + ``.eval()`` on a CUDA device) runs on ``engine.UNetEngine``: 99 fused
gated-conv kernel launches (wgmma tensor-core kernels for the dominant 3x3 layers) replayed as one CUDA graph.
There is no CPU path: inference on a CPU tensor raises.

Training (autograd enabled) is routed through torch's own conv/batch-norm operators on the same parameters —
a LIBRARY path (cuDNN), kept so that the reference's train.py keeps working.  ``train_precision = 'bf16'`` moves the 78
gated 3x3 stride-1 convs onto the wgmma kernels, forward and backward (read_b200/blocks.py): the 8 residual block stacks
(64 convs) and the 14 single convs feat_extract.0 / .5, SCM*.main.0 / .2, AFFs.*.conv.1 and FAM*.merge.  The other 21
convs (the 1x1 convs and the stride-2 3x3 / 4x4 convs), FAM's product and sum, the interpolations and the concats stay on
torch.  ``'bf16_all'`` also moves those 21 convs onto the wgmma kernels (blocks.gated_conv_srcs), so every conv of the net trains
there; FAM's product and sum, the interpolations, the concats that include an 8-channel source, the loss and the optimizers stay
on torch.  The default ``'fp32'`` keeps every layer on torch.
"""
import threading

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import blocks
from .engine import UNetEngine

TRAIN_PRECISIONS = ('fp32', 'bf16', 'bf16_all')


def layer_table(base=32, num_res=4):
    """(dotted prefix, cin, cout, k, stride, elu) for every BasicConv created by UNet.__init__ (unet.py:130-200)."""
    c = base
    t = []
    for e, ch in enumerate([c, 2 * c, 4 * c, 8 * c]):
        for r in range(num_res):
            t += [(f"Encoder.{e}.layers.{r}.main.0", ch, ch, 3, 1, True), (f"Encoder.{e}.layers.{r}.main.1", ch, ch, 3, 1, False)]
    t += [("feat_extract.0", 8, c, 3, 1, True), ("feat_extract.1", c, 2 * c, 3, 2, True),
          ("feat_extract.2", 2 * c, 4 * c, 3, 2, True), ("feat_extract.3", 4 * c, 2 * c, 4, 2, True),
          ("feat_extract.4", 2 * c, c, 4, 2, True), ("feat_extract.5", c, 3, 3, 1, False),
          ("feat_extract.6", 4 * c, 8 * c, 3, 2, True), ("feat_extract.7", 8 * c, 4 * c, 4, 2, True)]
    for d, ch in enumerate([8 * c, 4 * c, 2 * c, c]):
        for r in range(num_res):
            t += [(f"Decoder.{d}.layers.{r}.main.0", ch, ch, 3, 1, True), (f"Decoder.{d}.layers.{r}.main.1", ch, ch, 3, 1, False)]
    t += [("Convs.0", 8 * c, 4 * c, 1, 1, True), ("Convs.1", 4 * c, 2 * c, 1, 1, True), ("Convs.2", 2 * c, c, 1, 1, True)]
    t += [("ConvsOut.0", 4 * c, 3, 3, 1, False), ("ConvsOut.1", 2 * c, 3, 3, 1, False)]      # unused by forward (unet.py:181-186)
    for a, ch in enumerate([c, 2 * c, 4 * c]):
        t += [(f"AFFs.{a}.conv.0", 15 * c, ch, 1, 1, True), (f"AFFs.{a}.conv.1", ch, ch, 3, 1, False)]
    for name, ch in [("FAM1", 4 * c), ("SCM1", 4 * c), ("FAM2", 2 * c), ("SCM2", 2 * c), ("FAM0", 8 * c), ("SCM0", 8 * c)]:
        if name.startswith("FAM"):
            t += [(f"{name}.merge", ch, ch, 3, 1, False)]
        else:
            t += [(f"{name}.main.0", 8, ch // 4, 3, 1, True), (f"{name}.main.1", ch // 4, ch // 2, 1, 1, True),
                  (f"{name}.main.2", ch // 2, ch // 2, 3, 1, True), (f"{name}.main.3", ch // 2, ch - 8, 1, 1, True),
                  (f"{name}.conv", ch, ch, 1, 1, False)]
    return t


class _Group(nn.Module):
    """Parameter container node (stands in for ModuleList / Sequential / the block classes)."""


class GatedConv(nn.Module):
    """Parameters of one BasicConv (unet.py:22-53): ``block.{conv_f,conv_m,norm}``."""

    def __init__(self, cin, cout, k, stride, elu):
        super().__init__()
        p = int((k - 1) / 2)
        self.k, self.stride, self.elu = k, stride, elu
        self.block = nn.ModuleDict({
            'conv_f': nn.Conv2d(cin, cout, k, stride=stride, padding=p),
            'conv_m': nn.Conv2d(cin, cout, k, stride=stride, padding=p),
            'norm': nn.BatchNorm2d(cout),
        })

    def forward(self, x):   # torch library path (training only)
        f = self.block['conv_f'](x)
        if self.elu:
            f = F.elu(f)
        return self.block['norm'](f * torch.sigmoid(self.block['conv_m'](x)))


def _attach(root, dotted, module):
    node = root
    parts = dotted.split('.')
    for p in parts[:-1]:
        if p not in node._modules:
            node.add_module(p, _Group())
        node = node._modules[p]
    node.add_module(parts[-1], module)


class UNet(nn.Module):
    r"""Rendering network, multi-scale input (same signature as the reference)."""

    def __init__(self, num_input_channels=8, num_output_channels=3, feature_scale=4, num_res=4):
        super().__init__()
        self.feature_scale = feature_scale
        self.num_res = num_res
        self.base = 32
        for prefix, cin, cout, k, stride, elu in layer_table(self.base, num_res):
            m = GatedConv(cin, cout, k, stride, elu)
            _attach(self, prefix, m)
        self.precision = 'bf16'          # 'bf16' (tensor cores) | 'fp32' (CUDA-core parity mode)
        # training (autograd) path: 'fp32' = torch operators everywhere | 'bf16' = the 78 gated 3x3 stride-1 convs on the wgmma kernels
        # | 'bf16_all' = all 99 convs on the wgmma kernels
        self.train_precision = 'fp32'
        self.conv_impl = 'auto'
        self.use_graph = True
        self._engines = {}
        self._engine_lock = threading.Lock()

    # engines hold CUDA graphs and the lock is not picklable: copies / pickles of the module start with an empty cache
    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop('_engine_lock', None)
        state.pop('_vt', None)
        state['_engines'] = {}
        return state

    def __setstate__(self, state):
        super().__setstate__(state)
        self._engines = {}
        self._engine_lock = threading.Lock()

    # ------------------------------------------------------------------ engine management
    def _weights_version(self):
        """Sum of the in-place version counters of every parameter and buffer: changes on load_state_dict, optimizer steps and
        BatchNorm running-stat updates.  The tensor list is cached (909 entries; rebuilt when the module is moved / cast, which
        re-creates the tensors)."""
        vt = self.__dict__.get('_vt')
        if vt is None:
            vt = self.__dict__['_vt'] = list(self.parameters()) + list(self.buffers())
        return sum(t._version for t in vt)

    def _apply(self, fn, *a, **kw):
        self.__dict__.pop('_vt', None)
        return super()._apply(fn, *a, **kw)

    def load_state_dict(self, *a, **kw):
        self.__dict__.pop('_vt', None)
        return super().load_state_dict(*a, **kw)

    def engine(self, B, H, W, device):
        """The static-shape executor for this (batch, size, device, mode), rebuilt when the weights changed.  The cache dict is
        mutated in place under a lock: nn.DataParallel replicas share it with the source module (they are shallow copies)."""
        key = (B, H, W, str(device), self.precision, self.conv_impl, self.use_graph)
        ver = self._weights_version()
        with self._engine_lock:
            ent = self._engines.get(key)
            if ent is not None and ent[0] == ver:
                return ent[1]
            for k in [k for k, v in self._engines.items() if v[0] != ver]:     # drop stale engines
                del self._engines[k]
            with torch.cuda.device(device):
                eng = UNetEngine(self.state_dict(), B, H, W, device, precision=self.precision, conv_impl=self.conv_impl,
                                 use_graph=self.use_graph, base=self.base, num_res=self.num_res)
            self._engines[key] = (ver, eng)
            return eng

    # ------------------------------------------------------------------ forward
    def forward(self, *inputs, **kwargs):
        inputs = list(inputs)
        x = inputs[0]
        needs_autograd = torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters())
                                                      or any(t.requires_grad for t in inputs[:4]))
        # nn.DataParallel replicas (the reference's legacy multi-GPU eval, train.py:138-139) get freshly broadcast parameter
        # copies every call: an engine cached for them could not see weight updates, and concurrent CUDA-graph captures from the
        # replica threads would collide - replicas evaluate through torch's operators (library path, like training).
        # read_b200's own multi-GPU path is read_b200.dist (one process per GPU).
        if needs_autograd or self.training or getattr(self, '_is_replica', False):
            return self._forward_torch(inputs)
        if not x.is_cuda:
            raise RuntimeError("read_b200.UNet: inference needs CUDA tensors on an H100 (no CPU fallback)")
        B, _, H, W = x.shape
        eng = self.engine(B, H, W, x.device)
        eng.set_inputs_nchw(inputs[:4])
        return eng.run().clone()

    def _c(self, name, x):
        return self.get_submodule(name)(x)

    def _forward_torch(self, inputs):
        """Library (cuDNN/autograd) evaluation of unet.py:202-285 on the same parameters; training only."""
        c = self._c
        x, x_2, x_4, x_8 = inputs[:4]
        tp = getattr(self, 'train_precision', 'fp32')       # modules pickled before the attribute existed
        if tp not in TRAIN_PRECISIONS:
            raise ValueError(f"read_b200.UNet: train_precision must be one of {TRAIN_PRECISIONS}, got {tp!r}")

        bf16 = tp in ('bf16', 'bf16_all')
        # a conv whose BatchNorm is in train mode (the net in train()) normalises with batch statistics on our kernels, like
        # torch's BatchNorm2d; the keyword is passed only when some norm trains, so an eval-mode net calls res_stack as before
        bs = {'batch_stats': True} if bf16 and any(m.training for m in self.modules() if isinstance(m, nn.BatchNorm2d)) else {}

        def c3(name, t):
            # the gated 3x3 stride-1 convs outside the blocks: feat_extract.0 / .5, SCM*.main.0 / .2, AFFs.*.conv.1, FAM*.merge
            if bf16:
                return blocks.gated_conv(self.get_submodule(name), t, name=name, **bs)
            return c(name, t)

        def c1(name, *ts):
            # the 1x1 and stride-2 convs; a 1x1 conv's sources are concatenated along channels (virtually under 'bf16_all')
            if tp == 'bf16_all':
                return blocks.gated_conv_srcs(self.get_submodule(name), ts, name, **bs)
            return c(name, ts[0] if len(ts) == 1 else torch.cat(ts, 1))

        def res(p, t):
            return c(p + ".main.1", c(p + ".main.0", t)) + t

        def blk(p, t):
            if bf16:
                return blocks.res_stack(self, p, t, **bs)
            for i in range(self.num_res):
                t = res(f"{p}.layers.{i}", t)
            return t

        def scm(p, t):
            y = c1(p + ".main.3", c3(p + ".main.2", c1(p + ".main.1", c3(p + ".main.0", t))))
            return c1(p + ".conv", torch.cat([t, y], 1))      # torch's concat: the 8-channel source is not 32-channel granular

        def fam(p, a, b):
            return a + c3(p + ".merge", a * b)

        def aff(i, *xs):
            return c3(f"AFFs.{i}.conv.1", c1(f"AFFs.{i}.conv.0", *xs))

        up4 = lambda t: F.interpolate(t, scale_factor=4, mode='bilinear', align_corners=False)
        nn_ = lambda t, s: F.interpolate(t, scale_factor=s)
        z2, z4, z8 = scm("SCM2", x_2), scm("SCM1", x_4), scm("SCM0", x_8)
        res1 = blk("Encoder.0", c3("feat_extract.0", x))
        res2 = blk("Encoder.1", fam("FAM2", c1("feat_extract.1", res1), z2))
        res3 = blk("Encoder.2", fam("FAM1", c1("feat_extract.2", res2), z4))
        z = blk("Encoder.3", fam("FAM0", c1("feat_extract.6", res3), z8))
        r1 = aff(0, res1, nn_(res2, 2), nn_(res3, 4), nn_(z, 8))
        r2 = aff(1, nn_(res1, 0.5), res2, nn_(res3, 2), nn_(z, 4))
        r3 = aff(2, nn_(res1, 0.25), nn_(res2, 0.5), res3, nn_(z, 2))
        z = blk("Decoder.0", z)
        z = blk("Decoder.1", c1("Convs.0", up4(c1("feat_extract.7", z)), r3))
        z = blk("Decoder.2", c1("Convs.1", up4(c1("feat_extract.3", z)), r2))
        z = blk("Decoder.3", c1("Convs.2", up4(c1("feat_extract.4", z)), r1))
        return c3("feat_extract.5", z)
