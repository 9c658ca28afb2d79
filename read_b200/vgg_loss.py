"""The reference's VGG19 perceptual loss (READ/criterions/vgg_loss.py:20-111) on our kernels: ``VGGLoss`` is a drop-in for
``READ.criterions.vgg_loss.VGGLoss`` (``--criterion_module read_b200.vgg_loss.VGGLoss``).

loss = sum over the loss layers i of F.l1_loss(f_i(input), f_i(target)), f_i the output of module i of torchvision's
``vgg19().features`` with every MaxPool2d replaced by AvgPool2d(2, 2), over inputs normalised as (x - mean) / std.  The weights are
frozen, so backward computes the input gradient of ``input`` only.

One autograd Function (_VGGLossFn).  Forward: input and target go through the net as ONE NHWC bf16 batch of 2B images (8 channels,
3 real), so every conv is one launch over both.  A plain conv of c filters is run as the gated pair (wf, wm) of c/2 filters each
whose RAW [f | m] column order (blocks.fm_columns) is the natural channel order (split_filters): the RAW 3x3 plan of the TMA wgmma
kernel computes it with the existing packing, and csrc/vgg.cu adds bias and ReLU, sums the L1 term, records what backward needs (one
int8 code per element of the output half: the ReLU mask and the sign of f_in - f_tgt) and writes the next conv's input, pooled
when a pool follows.  Backward, last conv to first: dY = mask * (upstream + sign * g / numel) (the pool's backward folded into the
read of the upstream gradient), then the conv's input gradient: a RAW plan with read_pack_weights_tc_dgrad filters, or for the
image (conv1_1, 3 channels run as 8) read_conv3x3_dgrad_cin8.  The packed filters are cached per module and device.

partialconv=True is the mask-aware form: conv1_1 becomes a partial convolution (PartialConv2d) over the validity mask of the target
(M = [sum of the target's channels > 1e-9], from the raw target, the same M for both images).  The forward then normalises with
read_vgg_normalize_masked (both images times M, M saved as one byte per pixel) and runs conv1_1's post-conv pass as
read_vgg_post_partial; backward multiplies conv1_1's dY by the partial conv's ratio (read_vgg_dgrad_in_partial) and the image
gradient by M (read_vgg_image_grad_masked).  Nothing flows through the mask: it depends on the target only.
"""
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib as L
from . import blocks

CAFFE_FILE = 'vgg_caffe_features.pth'            # what the reference writes into save_dir
TORCHVISION_FILE = 'vgg19-dcbb9e9d.pth'          # torchvision's pretrained VGG19 in torch.hub's checkpoint directory
VGG19_CFG = (64, 64, 'P', 128, 128, 'P', 256, 256, 256, 256, 'P', 512, 512, 512, 512, 'P', 512, 512, 512, 512, 'P')
LAYERS = (1, 3, 6, 8, 11, 13, 15, 17, 20, 22, 24, 26, 29)     # every ReLU output up to relu5_1
LAYERS_OPTIMIZED = (3, 8, 17, 26, 35)
# A RAW plan's output holds fewer elements than this (conv_tc.cu, tc_supported); a batch whose widest RAW output would reach it
# runs in chunks of image pairs.  Module level so that a test can lower it.
RAW_LIMIT = 1 << 31


def vgg19_modules():
    """The module kinds of torchvision's vgg19().features, index by index: ('conv', cin, cout), 'relu' or 'pool'."""
    out, cin = [], 3
    for v in VGG19_CFG:
        if v == 'P':
            out.append('pool')
        else:
            out += [('conv', cin, v), 'relu']
            cin = v
    return out


MASK_EPS = 1e-9                                  # a target pixel is valid where its channel sum exceeds this


class PartialConv2d(nn.Conv2d):
    """VGG's first conv as partialconv=True runs it: a partial convolution with one mask channel shared by all input channels
    (Liu et al., "Image Inpainting for Irregular Holes Using Partial Convolutions", 2018).  With cnt the number of valid pixels
    in each window of ``mask_in`` [B, 1, H, W] (zero padding), upd = clamp(cnt, 0, 1) and ratio = window size / (cnt + 1e-8) * upd:
    out = (conv(input * mask_in) * ratio + bias) * upd.  The parameters are those of the plain conv it replaces (state_dict keys
    ``weight`` / ``bias``); the mask gets no gradient.  Built with from_conv, so that the weights are shared, not copied."""

    @classmethod
    def from_conv(cls, conv):
        p = cls(conv.in_channels, conv.out_channels, conv.kernel_size, stride=conv.stride, padding=conv.padding,
                dilation=conv.dilation, groups=conv.groups, bias=conv.bias is not None, device='meta')
        p.weight, p.bias = conv.weight, conv.bias
        return p

    def forward(self, input, mask_in):
        with torch.no_grad():
            ones = torch.ones((1, 1, *self.kernel_size), dtype=mask_in.dtype, device=mask_in.device)
            cnt = F.conv2d(mask_in, ones, stride=self.stride, padding=self.padding, dilation=self.dilation)
            upd = cnt.clamp(0, 1)
            ratio = self.kernel_size[0] * self.kernel_size[1] / (cnt + 1e-8) * upd
        out = F.conv2d(input * mask_in, self.weight, None, self.stride, self.padding, self.dilation, self.groups) * ratio
        if self.bias is not None:
            out = out + self.bias.view(1, -1, 1, 1)
        return out * upd


def partial_features(features):
    """A new nn.Sequential of ``features``' modules with the first conv replaced by a PartialConv2d sharing its weight and bias:
    the layout VGGLoss(partialconv=True, features=...) takes.  ``features`` itself is not modified."""
    mods = list(features)
    mods[0] = PartialConv2d.from_conv(mods[0])
    return nn.Sequential(*mods)


def target_mask(target):
    """partialconv=True's validity mask [B, 1, H, W] of the raw target: 1 where the channels sum above MASK_EPS, else 0."""
    return (target.sum(1, keepdim=True) > MASK_EPS).to(target.dtype)


def check_layout(features):
    """Raise a ValueError unless ``features`` is an nn.Sequential in the layout of torchvision's vgg19().features: 37 modules,
    3x3 stride-1 pad-1 convs with bias at the VGG19 channel counts, ReLUs, and 2x2 pools (MaxPool2d, or the reference's
    AvgPool2d(2, 2)) where the pools are.  The first conv may be a PartialConv2d (partialconv=True)."""
    if not isinstance(features, nn.Sequential):
        raise ValueError(f"read_b200.VGGLoss: features must be an nn.Sequential (got {type(features).__name__})")
    mods, want = list(features), vgg19_modules()
    if len(mods) != len(want):
        raise ValueError(f"read_b200.VGGLoss: features has {len(mods)} modules, VGG19's have {len(want)}")
    for i, (m, w) in enumerate(zip(mods, want)):
        if w == 'relu':
            ok = isinstance(m, nn.ReLU)
        elif w == 'pool':
            ok = (isinstance(m, (nn.MaxPool2d, nn.AvgPool2d)) and _pair(m.kernel_size) == (2, 2) and _pair(m.stride) == (2, 2)
                  and _pair(m.padding) == (0, 0) and not m.ceil_mode)
        else:
            ok = (type(m) in ((nn.Conv2d, PartialConv2d) if i == 0 else (nn.Conv2d,)) and (m.in_channels, m.out_channels) == w[1:]
                  and m.kernel_size == (3, 3) and m.stride == (1, 1) and m.padding == (1, 1) and m.dilation == (1, 1)
                  and m.groups == 1 and m.bias is not None and m.padding_mode == 'zeros')
        if not ok:
            raise ValueError(f"read_b200.VGGLoss: features[{i}] is {m}, VGG19 has a {w if isinstance(w, str) else 'conv %d -> %d' % w[1:]}"
                             " there")


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


class Step:
    """One conv of the walk: module indices of the conv and its ReLU, channels, whether the ReLU output is a loss term and whether
    a pool follows before the next conv."""

    def __init__(self, conv, cin, cout, loss):
        self.conv, self.relu, self.cin, self.cout, self.loss, self.pool = conv, conv + 1, cin, cout, loss, False

    def __repr__(self):
        return f"Step(conv={self.conv}, {self.cin}->{self.cout}, loss={self.loss}, pool={self.pool})"


def layer_walk(layers):
    """The convs to run for the loss terms ``layers`` (ReLU indices): up to the ReLU of the last one; modules after it do not
    change the value."""
    kinds = vgg19_modules()
    last = max(layers)
    bad = [i for i in layers if not (0 <= i < len(kinds) and kinds[i] == 'relu')]
    if bad:
        raise ValueError(f"read_b200.VGGLoss: loss layers must be ReLU outputs of VGG19's features (got {bad})")
    steps = []
    for i, k in enumerate(kinds[:last + 1]):
        if k == 'pool':
            steps[-1].pool = True
        elif k != 'relu':
            steps.append(Step(i, k[1], k[2], i + 1 in layers))
    return steps


def layer_sizes(steps, H, W):
    """(h, w) of each step's conv; AvgPool2d floors odd sizes."""
    out = []
    for s in steps:
        out.append((H, W))
        if s.pool:
            H, W = H // 2, W // 2
    return out


def chunk_pairs(steps, H, W, limit=None):
    """Image pairs per chunk: the most for which every RAW output of the forward ([2n, h, w, cout]) stays below ``limit``
    (RAW_LIMIT) elements.  The backward's RAW outputs ([n, h, w, cin]) are smaller."""
    limit = RAW_LIMIT if limit is None else limit
    widest = max(2 * h * w * s.cout for s, (h, w) in zip(steps, layer_sizes(steps, H, W)))
    n = (limit - 1) // widest
    if n < 1:
        raise ValueError(f"read_b200.VGGLoss: a {H}x{W} image pair exceeds the conv kernel's RAW output limit")
    return n


def split_filters(w):
    """The gated pair (wf, wm) of c/2 filters each of the plain conv filters ``w`` [c, cin, 3, 3] whose RAW [f | m] columns are
    the c output channels in order: blocks of 2h columns (h = min(c/2, 64)), f half first, so block b's f half is channels
    2hb .. 2hb + h - 1 and its m half the next h."""
    c = w.shape[0]
    h = min(c // 2, 64)
    v = w.reshape(c // (2 * h), 2, h, *w.shape[1:])
    return v[:, 0].reshape(c // 2, *w.shape[1:]).contiguous(), v[:, 1].reshape(c // 2, *w.shape[1:]).contiguous()


def load_features(net, save_dir):
    """VGG19's features for ``net`` from the files the reference uses.  Nothing is downloaded: a missing file raises."""
    if net == 'caffe':
        path = os.path.join(save_dir, CAFFE_FILE)
        if not os.path.exists(path):
            raise FileNotFoundError(f"read_b200.VGGLoss: {path} not found; read_b200 does not download weights (the reference's "
                                    "VGGLoss writes this file, or pass features=)")
        return torch.load(path, map_location='cpu', weights_only=False)     # the reference pickles the whole nn.Sequential
    path = os.path.join(torch.hub.get_dir(), 'checkpoints', TORCHVISION_FILE)
    if not os.path.exists(path):
        raise FileNotFoundError(f"read_b200.VGGLoss: {path} not found; read_b200 does not download weights (torchvision's "
                                "pretrained VGG19 goes there, or pass features=)")
    import torchvision
    model = torchvision.models.vgg19()
    model.load_state_dict(torch.load(path, map_location='cpu'))
    return model.features


def normalization(net):
    """(mean, std) [1, 3, 1, 1] f32 as the reference builds them."""
    if net == 'caffe':
        return (torch.FloatTensor([103.939, 116.779, 123.680])[None, :, None, None] / 255.,
                torch.FloatTensor([1. / 255, 1. / 255, 1. / 255])[None, :, None, None])
    return (torch.FloatTensor([0.485, 0.456, 0.406])[None, :, None, None],
            torch.FloatTensor([0.229, 0.224, 0.225])[None, :, None, None])


def reference_loss(vgg19, mean, std, layers, input, target):
    """The reference's loop (vgg_loss.py:100-111) in torch, stopped after the last loss layer: DataParallel replicas, the float64
    restatement of the tests and the torch arm of the benchmark.  A PartialConv2d runs over target_mask(target) for both images."""
    mask = target_mask(target) if any(isinstance(m, PartialConv2d) for m in vgg19) else None
    x, y = (input - mean) / std, (target - mean) / std
    loss = 0
    for i, layer in enumerate(vgg19):
        if i > max(layers):
            break
        if isinstance(layer, PartialConv2d):
            x, y = layer(x, mask), layer(y, mask)
        else:
            x, y = layer(x), layer(y)
        if i in layers:
            loss = loss + F.l1_loss(x, y)
    return loss


class VGGLoss(nn.Module):
    """Drop-in for READ.criterions.vgg_loss.VGGLoss: same constructor, buffers (mean_, std_), module list (vgg19, pools as
    AvgPool2d(2, 2)) and forward(input, target) -> scalar.  ``features``: VGG19's features (torchvision layout) to use instead of
    the file ``net`` names.  partialconv=True runs vgg19[0] as a PartialConv2d over the target's validity mask: loaded from the
    file, the plain conv is wrapped as the reference does (same weight and bias Parameters).  ``features`` is used exactly as
    given, never rewritten: its first conv must already be a PartialConv2d when partialconv=True (partial_features(features)
    builds that layout) and a plain Conv2d otherwise."""

    def __init__(self, net='caffe', partialconv=False, optimized=False, save_dir='.cache/torch/models', features=None):
        super().__init__()
        if net not in ('caffe', 'pytorch'):
            raise ValueError(f"read_b200.VGGLoss: net must be 'caffe' or 'pytorch' (got {net!r})")
        self.partialconv = bool(partialconv)
        loaded = features is None
        if loaded:
            features = load_features(net, save_dir)
        check_layout(features)
        if loaded and self.partialconv:
            features = partial_features(features)
        if self.partialconv != (type(features[0]) is PartialConv2d):
            raise ValueError(f"read_b200.VGGLoss: partialconv={self.partialconv} but features[0] is a {type(features[0]).__name__}; "
                             "features= is used as given, so pass vgg_loss.partial_features(features) with partialconv=True "
                             "and a plain first conv without it")
        mean, std = normalization(net)
        self.register_buffer('mean_', mean)
        self.register_buffer('std_', std)
        for p in features.parameters():
            p.requires_grad = False
        self.vgg19 = nn.Sequential(*[nn.AvgPool2d(kernel_size=2, stride=2, padding=0) if isinstance(m, nn.MaxPool2d) else m
                                     for m in features])
        self.layers = list(LAYERS_OPTIMIZED if optimized else LAYERS)
        self._packed = {}

    def steps(self):
        return layer_walk(self.layers)

    def filters(self, device):
        """Per conv of the walk: the pair split fp32 (wf, wm), the bf16 forward filters, the bf16 input-gradient filters (None for
        conv1_1, whose kernel reads wf / wm) and the bias, packed once per device and weight version."""
        steps = self.steps()
        convs = [self.vgg19[s.conv] for s in steps]
        key = tuple(blocks.filter_key(c, c.weight, c.bias, s.cout) for c, s in zip(convs, steps))
        ent = self._packed.get(str(device))
        if ent is not None and ent[0] == key:
            return ent[1]
        lib, st = L.load(), L.stream_ptr()
        out = []
        for c, s in zip(convs, steps):
            w = c.weight.detach().float()
            if s.cin == 3:
                w = F.pad(w, (0, 0, 0, 0, 0, 5))             # the image runs as 8 channels, the 5 padded ones zero
            wf, wm = split_filters(w)
            h, cin = s.cout // 2, w.shape[1]
            w_tc = torch.empty(lib.read_tc_weight_elems(h, cin, 3), dtype=torch.bfloat16, device=device)
            L.check(lib.read_pack_weights_tc(wf.data_ptr(), wm.data_ptr(), h, cin, 3, w_tc.data_ptr(), st))
            w_dg = None
            if cin != 8:
                w_dg = torch.empty(lib.read_tc_weight_elems(cin // 2, 2 * h, 3), dtype=torch.bfloat16, device=device)
                L.check(lib.read_pack_weights_tc_dgrad(wf.data_ptr(), wm.data_ptr(), h, cin, w_dg.data_ptr(), st))
            out.append({'wf': wf, 'wm': wm, 'w_tc': w_tc, 'w_dgrad': w_dg, 'bias': c.bias.detach().float().contiguous()})
        self._packed[str(device)] = (key, out)
        return out

    def forward(self, input, target):
        if getattr(self, '_is_replica', False):
            # nn.DataParallel replicas get freshly broadcast weight copies every call, which a filter cache could not follow:
            # they evaluate through torch's operators, as UNet.forward does
            return reference_loss(self.vgg19, self.mean_, self.std_, self.layers, input, target)
        if target.requires_grad:
            raise ValueError("read_b200.VGGLoss: the target must not require grad (only the input gradient is computed)")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.vgg19.parameters()):
            raise ValueError("read_b200.VGGLoss: the VGG weights are frozen (requires_grad=False); there is no weight gradient")
        if input.dim() != 4 or input.shape[1] != 3 or input.shape != target.shape:
            raise ValueError(f"read_b200.VGGLoss: input and target must be [B, 3, H, W] of one shape (got {tuple(input.shape)} "
                             f"and {tuple(target.shape)})")
        if not (input.is_cuda and target.is_cuda):
            raise RuntimeError("read_b200.VGGLoss runs on the H100 kernels and needs CUDA tensors (no CPU fallback)")
        L.require_device(input.device.index)
        if self.mean_.device != input.device or self.vgg19[0].weight.device != input.device:
            raise ValueError(f"read_b200.VGGLoss: the module is on {self.mean_.device}, the input on {input.device}")
        steps = self.steps()
        h, w = layer_sizes(steps, input.shape[2], input.shape[3])[-1]
        if h < 1 or w < 1:
            raise ValueError(f"read_b200.VGGLoss: a {input.shape[2]}x{input.shape[3]} image pools to nothing before layer "
                             f"{steps[-1].relu}")
        pk = self.filters(input.device)
        if torch.is_grad_enabled() and input.requires_grad:
            return _VGGLossFn.apply(input, target, self, pk)
        return _forward(self, pk, input, target, None)


def _forward(mod, pk, input, target, chunks):
    """The loss (f32 scalar) of input against target.  ``chunks`` (a list) receives, per chunk of image pairs, (b0, n, codes,
    mask) for backward, mask the chunk's byte mask [n, H, W] (None unless partialconv); None saves nothing."""
    lib, st = L.load(), L.stream_ptr()
    steps = mod.steps()
    B, _, H, W = input.shape
    sizes = layer_sizes(steps, H, W)
    dev = input.device
    inp, tgt = input.detach().float().contiguous(), target.detach().float().contiguous()
    mean, std = mod.mean_.float().contiguous(), mod.std_.float().contiguous()
    n_loss = sum(s.loss for s in steps)
    terms = torch.zeros(n_loss, dtype=torch.float64, device=dev)
    ws = torch.empty(lib.read_vgg_workspace_bytes(), dtype=torch.uint8, device=dev)
    zeros = torch.zeros(256, dtype=torch.float32, device=dev)             # a RAW launch reads no epilogue parameters
    per = chunk_pairs(steps, H, W)
    for b0 in range(0, B, per):
        n = min(per, B - b0)
        x = torch.empty((2 * n, H, W, 8), dtype=torch.bfloat16, device=dev)
        mask = None
        if mod.partialconv:
            mask = torch.empty((n, H, W), dtype=torch.uint8, device=dev)
            L.check(lib.read_vgg_normalize_masked(inp[b0].data_ptr(), tgt[b0].data_ptr(), n, H, W, mean.data_ptr(), std.data_ptr(),
                                                  x.data_ptr(), mask.data_ptr(), st))
        else:
            L.check(lib.read_vgg_normalize(inp[b0].data_ptr(), tgt[b0].data_ptr(), n, H, W, mean.data_ptr(), std.data_ptr(),
                                           x.data_ptr(), st))
        codes, k = [], 0
        for i, (s, (h, w)) in enumerate(zip(steps, sizes)):
            raw = torch.empty((2 * n, h, w, s.cout), dtype=torch.bfloat16, device=dev)
            blocks._launch(lib, x, s.cout // 2, pk[i]['w_tc'], (zeros,) * 4, False, L.OUT_RAW_NHWC, raw)
            if i == len(steps) - 1:
                x = None                                                  # nothing reads the last layer's activations
            elif s.pool:
                x = torch.empty((2 * n, h // 2, w // 2, s.cout), dtype=torch.bfloat16, device=dev)
            else:
                x = raw                                                   # in place
            code = torch.empty((n, h, w, s.cout), dtype=torch.int8, device=dev) if chunks is not None else None
            term = terms[k].data_ptr() if s.loss else None
            if i == 0 and mask is not None:
                L.check(lib.read_vgg_post_partial(raw.data_ptr(), mask.data_ptr(), n, h, w, s.cout, pk[i]['bias'].data_ptr(),
                                                  L.ptr(x), L.ptr(code), term, 1.0 / (B * s.cout * h * w), ws.data_ptr(), st))
            else:
                L.check(lib.read_vgg_post(raw.data_ptr(), n, h, w, s.cout, pk[i]['bias'].data_ptr(), int(s.pool), L.ptr(x),
                                          L.ptr(code), term, 1.0 / (B * s.cout * h * w), ws.data_ptr(), st))
            k += s.loss
            codes.append(code)
        if chunks is not None:
            chunks.append((b0, n, codes, mask))
    return terms.sum().float()


class _VGGLossFn(torch.autograd.Function):
    """VGGLoss's loss of ``input`` (differentiable) against ``target`` (not)."""

    @staticmethod
    def forward(ctx, input, target, mod, pk):
        chunks = []
        loss = _forward(mod, pk, input, target, chunks)
        ctx.mod, ctx.pk, ctx.chunks, ctx.shape = mod, pk, chunks, tuple(input.shape)
        ctx.std = mod.std_.float().contiguous()
        return loss

    @staticmethod
    def backward(ctx, gout):
        lib, st = L.load(), L.stream_ptr()
        mod, pk = ctx.mod, ctx.pk
        steps = mod.steps()
        B, _, H, W = ctx.shape
        sizes = layer_sizes(steps, H, W)
        dev = gout.device
        g = gout.detach().float().reshape(1).contiguous()
        zeros = torch.zeros(256, dtype=torch.float32, device=dev)
        grad = torch.empty(ctx.shape, dtype=torch.float32, device=dev)
        for b0, n, codes, mask in ctx.chunks:
            up = None
            for i in reversed(range(len(steps))):
                s, (h, w) = steps[i], sizes[i]
                dy = torch.empty((n, h, w, s.cout), dtype=torch.bfloat16, device=dev)
                coef = 1.0 / (B * s.cout * h * w) if s.loss else 0.0
                if i == 0 and mask is not None:
                    L.check(lib.read_vgg_dgrad_in_partial(L.ptr(up), mask.data_ptr(), codes[i].data_ptr(), n, h, w, s.cout,
                                                          g.data_ptr(), coef, dy.data_ptr(), st))
                else:
                    L.check(lib.read_vgg_dgrad_in(L.ptr(up), int(s.pool), codes[i].data_ptr(), n, h, w, s.cout, g.data_ptr(),
                                                  coef, dy.data_ptr(), st))
                codes[i] = None
                if i == 0:
                    up = torch.empty((n, h, w, 8), dtype=torch.bfloat16, device=dev)
                    L.check(lib.read_conv3x3_dgrad_cin8(dy.data_ptr(), pk[0]['wf'].data_ptr(), pk[0]['wm'].data_ptr(), n, h, w,
                                                        s.cout // 2, up.data_ptr(), st))
                else:
                    up = torch.empty((n, h, w, s.cin), dtype=torch.bfloat16, device=dev)
                    blocks._launch(lib, dy, s.cin // 2, pk[i]['w_dgrad'], (zeros,) * 4, False, L.OUT_RAW_NHWC, up)
            if mask is not None:
                L.check(lib.read_vgg_image_grad_masked(up.data_ptr(), mask.data_ptr(), n, H, W, ctx.std.data_ptr(),
                                                       grad[b0].data_ptr(), st))
            else:
                L.check(lib.read_vgg_image_grad(up.data_ptr(), n, H, W, ctx.std.data_ptr(), grad[b0].data_ptr(), st))
        ctx.chunks = None
        return grad, None, None, None


class VGGLossMix(nn.Module):
    """Drop-in for READ.criterions.vgg_loss.VGGLossMix: weight * l1(input, target) + (1 - weight) * l2(input, target), l1 and l2
    VGGLoss() and VGGLoss(net='caffe') as the reference builds them (both 'caffe').  ``kwargs`` (save_dir, features) go to both."""

    def __init__(self, weight=0.5, **kwargs):
        super().__init__()
        self.l1 = VGGLoss(**kwargs)
        self.l2 = VGGLoss(net='caffe', **kwargs)
        self.weight = weight

    def forward(self, input, target):
        return self.l1(input, target) * self.weight + self.l2(input, target) * (1 - self.weight)
