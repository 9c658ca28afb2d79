"""bf16 training of the gated 3x3 stride-1 convs (READ/models/unet.py:22-53) on the wgmma kernels.

``UNet.train_precision = 'bf16'`` sends 78 of the net's 99 convs here; the other 21 (the 1x1 and stride-2 convs), the
interpolations, concats and FAM products / sums stay on torch operators in the same autograd graph.  ``'bf16_all'`` also sends
those 21 convs here (``MultiSourceConvFn``, at the end of this file).
* ``ResStackFn``: each of the 8 residual block stacks (Encoder.0-3, Decoder.0-3: 4 ResBlocks = 8 convs at constant C, 64 convs).
* ``GatedConvFn``: one conv with an optional residual, for the 14 single convs feat_extract.0 (8 -> 32), feat_extract.5 (32 -> 3,
  the RGB output, run padded to C = 16), SCM*.main.0 (8 -> 16 / 32 / 64), SCM*.main.2, AFFs.*.conv.1 and FAM*.merge.

Forward: NCHW f32 -> NHWC bf16 once, launches of the TMA wgmma kernel (in a stack the second conv of each ResBlock adds the skip in
its epilogue), NHWC bf16 -> NCHW f32 once.  Saved for backward: the input of every conv (bf16, Cin channels per pixel), which the
weight gradient needs anyway.  The pre-activation [f | m] (2C channels per pixel) is NOT saved: backward recomputes it per conv
with a RAW launch of the same kernel.  That costs one extra forward conv per conv and keeps the saved activations at a third of
what saving [f | m] as well would take (C5, 8 crops of 256^2: about 1 GB instead of 3 GB across the 8 stacks, and 147 MB for the
14 single convs).

Backward, per conv, last to first (csrc/conv_bwd.cu): recompute [f | m]; gate backward -> [df | dm] and the bias / BatchNorm-affine
gradients; weight gradient (tensor-core kernel, fp32 atomics into the torch-layout gradients; skipped when no weight needs one);
input gradient = RAW launch of the TMA kernel over [df | dm] with flipped, transposed filters, the ResBlock skip added through its
residual operand, or for an 8-channel input (the descriptor pyramid) the dedicated dgrad_cin8 kernel.

BatchNorm is per conv, from the mode of that conv's norm at forward time:
* eval mode (running statistics, as the reference trains with eval_in_train): folded into scale / shift like the inference engine,
  the residual added in the conv's epilogue;
* train mode (the reference's default training, the net in train()), with ``batch_stats=True``: torch.nn.BatchNorm2d's train-mode
  semantics.  The conv launch writes g = A(f + b_f) * sigmoid(m + b_m) with an identity epilogue; csrc/bn_train.cu computes the
  batch mean / variance over the B * H_out * W_out pixels, the folded scale / shift and the in-place running-statistics update on the
  device, then y = g * scale + shift [+ residual].  Backward adds the terms through the statistics (read_bn_backward_reduce, then
  read_gate_backward_batch_stats).  Without ``batch_stats`` a train-mode norm raises, as before.
  With ``per_item`` as well (UNet.train_batchnorm = 'per_item'), each batch item is normalised with the statistics of its own
  H_out * W_out pixels, and the running statistics are updated once per item in item order: one batched call computes what B
  calls of one item each would.  The statistics are [items, C] and the *_items entry points take them.
The packed bf16 filters are cached per module and weight version (_packed): an optimizer step re-packs them, repeated calls with
the same weights (the per-item loop of training in train()) do not.
"""
import ctypes
import weakref

import torch

from . import _lib as L
from . import ops


def _pad_rows(t, n):
    """``t`` with zero rows appended along dim 0 up to ``n`` rows."""
    return torch.cat([t, t.new_zeros((n - t.shape[0],) + tuple(t.shape[1:]))]) if n > t.shape[0] else t


def fm_columns(C):
    """Channel of the concatenation [f (0..C-1) | m (C..2C-1)] held by each column of a RAW [f | m] row: blocks of 2*min(C, 64)
    columns, the conv_f half of each block first (the column order of the TMA kernel's RAW output)."""
    half = min(C, 64)
    j = torch.arange(2 * C)
    blk, r = j // (2 * half), j % (2 * half)
    return torch.where(r < half, blk * half + r, C + blk * half + r - half)


def _desc(srcs, cout, k=3, stride=1):
    """Descriptor of a k x k conv (pad (k - 1) // 2) over the NHWC bf16 tensors ``srcs`` (a virtual concat when there are several)."""
    B, H, W, _ = srcs[0].shape
    d = L.ReadConvDesc()
    d.act_dtype, d.n_src = L.ACT_BF16, len(srcs)
    for i, s in enumerate(srcs):
        d.src[i].ptr = s.data_ptr()
        d.src[i].C, d.src[i].H, d.src[i].W = s.shape[3], H, W
        d.src[i].mode, d.src[i].factor = L.SRC_IDENTITY, 1
    pad = (k - 1) // 2
    d.B, d.Hin, d.Win, d.Cin = B, H, W, sum(s.shape[3] for s in srcs)
    d.Hout, d.Wout, d.Cout = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, cout
    d.k, d.stride, d.pad = k, stride, pad
    return d


def _launch(lib, src, cout, w_tc, par, elu, out_mode, out, residual=None, k=3, stride=1):
    """One launch of the TMA wgmma kernel over the NHWC bf16 tensor ``src`` (or a list of them: a 1x1 conv's virtual concat), a
    3x3 stride-1 conv unless ``k`` / ``stride`` say otherwise; par = (bias_f, bias_m, scale, shift)."""
    d = _desc(src if isinstance(src, (list, tuple)) else [src], cout, k, stride)
    d.elu = int(elu)
    d.bias_f, d.bias_m, d.bn_scale, d.bn_shift = (t.data_ptr() for t in par)
    d.w_tc, d.impl = w_tc.data_ptr(), L.CONV_TCGEN05
    d.out, d.out_mode = out.data_ptr(), out_mode
    if residual is not None:
        d.residual = residual.data_ptr()
    plan = L.c_vp()
    L.check(lib.read_conv_plan_create(ctypes.byref(d), ctypes.byref(plan)))
    try:
        L.check(lib.read_conv_plan_launch(plan, L.stream_ptr()))
    finally:
        lib.read_conv_plan_destroy(plan)


# packed filters per GatedConv: module -> (key, dict of filters); see _packed
_FILTERS = weakref.WeakKeyDictionary()
cache_filters = True        # False: pack on every call (measurement of the cache, scripts/bench_train_bf16.py)


def clear_filter_cache():
    _FILTERS.clear()


def filter_key(mod, wf, wm, C, srcs=None):
    """What the packed filters of ``mod`` depend on: the identity, storage and in-place version of both weights (an optimizer step
    bumps the version), the padded channel count and a concat's source channel split."""
    return (id(wf), wf.data_ptr(), wf._version, id(wm), wm.data_ptr(), wm._version, C, str(wf.device),
            None if srcs is None else tuple(s.shape[3] for s in srcs))


def _packed(mod, wf, wm, C, srcs):
    """The fp32 filters padded to C channels and the bf16 forward (and 3x3 input-gradient) filters of ``mod``, from the cache when
    the weights are unchanged.  The dict also holds the filters backward packs lazily (dgrad_s2_filters, recompute_fm,
    dgrad_1x1); entries are only ever added, and a new weight version starts a new dict, so a FoldedConv of an earlier forward
    keeps the filters it was built with.  Writes that bypass the version counter (through ``.data``) are not seen."""
    key = filter_key(mod, wf, wm, C, srcs)
    ent = _FILTERS.get(mod) if cache_filters else None
    if ent is not None and ent[0] == key:
        return ent[1]
    lib, st = L.load(), L.stream_ptr()
    cin = wf.shape[1]
    pad = lambda t: _pad_rows(t.detach().float(), C).contiguous()
    pk = {'wf': pad(wf), 'wm': pad(wm), 'w_dgrad': None}       # an 8-channel input's gradient kernel reads wf / wm itself
    pk['w_tc'] = torch.empty(lib.read_tc_weight_elems(C, cin, mod.k), dtype=torch.bfloat16, device=wf.device)
    if (mod.k, mod.stride) != (3, 1):
        L.check(lib.read_pack_weights_tc_for(ctypes.byref(_desc(srcs, C, mod.k, mod.stride)), pk['wf'].data_ptr(),
                                             pk['wm'].data_ptr(), pk['w_tc'].data_ptr(), st))
    else:
        L.check(lib.read_pack_weights_tc(pk['wf'].data_ptr(), pk['wm'].data_ptr(), C, cin, 3, pk['w_tc'].data_ptr(), st))
        if cin != 8:
            pk['w_dgrad'] = torch.empty(lib.read_tc_weight_elems(cin // 2, 2 * C, 3), dtype=torch.bfloat16, device=wf.device)
            L.check(lib.read_pack_weights_tc_dgrad(pk['wf'].data_ptr(), pk['wm'].data_ptr(), C, cin, pk['w_dgrad'].data_ptr(), st))
    if (mod.k, mod.stride) != (3, 1):
        # the backward's filters too, so that a backward packs nothing (its launches are the same on every call)
        c = _Filters(pk, C, mod.k, mod.stride)
        if mod.stride == 2:
            dgrad_s2_filters(c)
        else:
            if C > 64:
                _fm64_filters(lib, srcs, c)
            c0 = 0
            for s in srcs:
                for a in range(c0, c0 + s.shape[3], 128):
                    _dgrad1x1_filters(lib, c, a, min(128, c0 + s.shape[3] - a), wf.device)
                c0 += s.shape[3]
    if cache_filters:
        _FILTERS[mod] = (key, pk)
    return pk


class _Filters:
    """The attributes of a FoldedConv the filter packers read."""

    def __init__(self, pk, C, k, stride):
        self.pk, self.wf, self.wm, self.C, self.k, self.stride = pk, pk['wf'], pk['wm'], C, k, stride


class FoldedConv:
    """One GatedConv's live parameters for this step: its BatchNorm and the bf16 filters of the forward conv (also used for the RAW
    recompute) and of the input gradient.  ``cout`` > the conv's C pads it with zero filters, biases and BatchNorm scale / shift
    (the RGB output conv, C = 3, runs as C = 16; SCM*.main.3, C = 56 / 120 / 248, as 64 / 128 / 256): the padded channels compute
    0 and get 0 gradients.  A 1x1 or stride-2 conv (k in {1, 3, 4}, stride in {1, 2}) packs its forward filters for the launch
    over ``srcs`` (the NHWC sources, whose channel counts set a concat's K chunks); its input-gradient filters are packed in
    backward (dgrad_s2_filters, dgrad_1x1).
    An eval-mode norm is folded into scale / shift from its running statistics.  A train-mode norm (``batch``) runs the forward
    launch with the identity epilogue ``fwd_par``; mean / inv / scale / shift are then filled by bn_forward from the batch, per
    batch item ([items, C]) when ``items`` is given (per-item statistics), else per channel ([C])."""

    def __init__(self, mod, wf, bf, wm, bm, gamma, beta, cout=None, srcs=None, items=None):
        norm = mod.block['norm']
        C = cout or wf.shape[0]
        pad = lambda t: _pad_rows(t.detach().float(), C).contiguous()
        self.C, self.elu = C, bool(mod.elu)
        self.bf, self.bm = pad(bf), pad(bm)
        self.k, self.stride = mod.k, mod.stride
        self.batch = norm.training
        self.items = items if self.batch else None
        if self.batch:
            dev = wf.device
            self.norm, self.n_real = norm, wf.shape[0]
            self.gamma, self.beta = gamma.detach().float().contiguous(), beta.detach().float().contiguous()
            shape = (4, C) if items is None else (4, items, C)
            self.mean, self.inv, self.scale, self.shift = torch.empty(shape, dtype=torch.float32, device=dev).unbind(0)
            self.fwd_par = (self.bf, self.bm, torch.ones(C, device=dev), torch.zeros(C, device=dev))
        else:
            inv = torch.rsqrt(norm.running_var.detach().float() + norm.eps)
            scale = gamma.detach().float() * inv
            self.mean, self.inv = pad(norm.running_mean), pad(inv)
            self.scale, self.shift = pad(scale), pad(beta.detach().float() - norm.running_mean.detach().float() * scale)
            self.fwd_par = self.par
        self.pk = _packed(mod, wf, wm, C, srcs)
        self.wf, self.wm, self.w_tc, self.w_dgrad = self.pk['wf'], self.pk['wm'], self.pk['w_tc'], self.pk['w_dgrad']

    @property
    def par(self):
        return (self.bf, self.bm, self.scale, self.shift)


def bn_forward(lib, c, g, residual=None):
    """Train-mode BatchNorm of the FoldedConv ``c`` over its identity-epilogue output ``g`` (NHWC bf16, C channels), in place:
    batch statistics, running-statistics update and y = g * scale + shift [+ residual]."""
    st, n = L.stream_ptr(), c.norm
    if c.items is not None:
        _bn_forward_items(lib, c, g, residual)
        return
    P = g.numel() // c.C
    ws = torch.empty(lib.read_bn_workspace_bytes(c.C), dtype=torch.uint8, device=g.device)
    L.check(lib.read_bn_batch_stats(g.data_ptr(), P, c.C, c.n_real, c.gamma.data_ptr(), c.beta.data_ptr(), n.eps, n.momentum,
                                    n.running_mean.data_ptr(), n.running_var.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), None,
                                    c.scale.data_ptr(), c.shift.data_ptr(), ws.data_ptr(), st))
    n.num_batches_tracked.add_(1)              # torch's own op: bumps the version UNet._weights_version sums
    L.check(lib.read_bn_apply(g.data_ptr(), P, c.C, c.scale.data_ptr(), c.shift.data_ptr(), L.ptr(residual), g.data_ptr(), st))


def _bn_forward_items(lib, c, g, residual):
    """bn_forward with per-item statistics: item i of ``g`` ([items, H, W, C]) with its own; the running statistics are updated
    once per item, in item order, and num_batches_tracked advances by the number of items, as that many single-item calls would."""
    st, n = L.stream_ptr(), c.norm
    items, P = g.shape[0], g.shape[1] * g.shape[2]
    ws = torch.empty(lib.read_bn_workspace_bytes_items(items, c.C), dtype=torch.uint8, device=g.device)
    L.check(lib.read_bn_batch_stats_items(g.data_ptr(), items, P, c.C, c.n_real, c.gamma.data_ptr(), c.beta.data_ptr(), n.eps,
                                          n.momentum, n.running_mean.data_ptr(), n.running_var.data_ptr(), c.mean.data_ptr(),
                                          c.inv.data_ptr(), c.scale.data_ptr(), c.shift.data_ptr(), ws.data_ptr(), st))
    n.num_batches_tracked.add_(items)
    L.check(lib.read_bn_apply_items(g.data_ptr(), items, P, c.C, c.scale.data_ptr(), c.shift.data_ptr(), L.ptr(residual),
                                    g.data_ptr(), st))


def conv_forward(lib, src, c, out, residual=None):
    """Forward of the FoldedConv ``c`` over ``src`` into ``out`` (NHWC bf16): one launch with the folded BatchNorm and the residual
    in its epilogue, or for a train-mode norm the identity-epilogue launch followed by bn_forward."""
    if not c.batch:
        _launch(lib, src, c.C, c.w_tc, c.par, c.elu, L.OUT_NHWC, out, residual, k=c.k, stride=c.stride)
        return
    _launch(lib, src, c.C, c.w_tc, c.fwd_par, c.elu, L.OUT_NHWC, out, k=c.k, stride=c.stride)
    bn_forward(lib, c, out, residual)


def gate_backward(lib, g, fm, c, dfm):
    """[df | dm] (into ``dfm``, RAW column order) and [dbias_f, dbias_m, dgamma, dbeta] (fp32 [4, C]) of the FoldedConv ``c`` from
    its output gradient ``g`` and the recomputed [f | m]; a train-mode norm adds the terms through the batch statistics."""
    st = L.stream_ptr()
    P = g.numel() // c.C
    red = torch.zeros((4, c.C), dtype=torch.float32, device=g.device)  # dbias_f, dbias_m, dgamma, dbeta
    if torch.are_deterministic_algorithms_enabled():
        return _gate_backward_det(lib, g, fm, c, dfm, P, red, st)
    if c.items is not None:
        items, P = g.shape[0], g.shape[1] * g.shape[2]
        sums = torch.zeros((2, items, c.C), dtype=torch.float32, device=g.device)     # sum dy, sum dy * xhat per item
        L.check(lib.read_bn_backward_reduce_items(g.data_ptr(), fm.data_ptr(), items, P, c.C, int(c.elu), c.bf.data_ptr(),
                                                  c.bm.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), sums[0].data_ptr(),
                                                  sums[1].data_ptr(), st))
        L.check(lib.read_gate_backward_batch_stats_items(g.data_ptr(), fm.data_ptr(), items, P, c.C, int(c.elu), c.bf.data_ptr(),
                                                         c.bm.data_ptr(), c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(),
                                                         sums[0].data_ptr(), sums[1].data_ptr(), dfm.data_ptr(),
                                                         red[0].data_ptr(), red[1].data_ptr(), st))
        red[3], red[2] = sums[0].sum(0), sums[1].sum(0)
        return red
    if c.batch:
        L.check(lib.read_bn_backward_reduce(g.data_ptr(), fm.data_ptr(), P, c.C, int(c.elu), c.bf.data_ptr(), c.bm.data_ptr(),
                                            c.mean.data_ptr(), c.inv.data_ptr(), red[3].data_ptr(), red[2].data_ptr(), st))
        L.check(lib.read_gate_backward_batch_stats(g.data_ptr(), fm.data_ptr(), P, c.C, int(c.elu), c.bf.data_ptr(),
                                                   c.bm.data_ptr(), c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(),
                                                   red[3].data_ptr(), red[2].data_ptr(), dfm.data_ptr(), red[0].data_ptr(),
                                                   red[1].data_ptr(), st))
        return red
    L.check(lib.read_gate_backward(g.data_ptr(), fm.data_ptr(), P, c.C, int(c.elu), c.bf.data_ptr(), c.bm.data_ptr(),
                                   c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), dfm.data_ptr(),
                                   red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st))
    return red


def _gate_backward_det(lib, g, fm, c, dfm, P, red, st):
    """gate_backward under torch.use_deterministic_algorithms(True): the same passes through the *_det entry points, whose sums
    are combined in a fixed order."""
    items = g.shape[0] if c.items is not None else 1
    ws = ops.det_workspace(lib.read_gate_det_workspace_bytes(items, c.C), g.device, "gate backward")
    if c.items is not None:
        P = g.shape[1] * g.shape[2]
        sums = torch.zeros((2, items, c.C), dtype=torch.float32, device=g.device)
        L.check(lib.read_bn_backward_reduce_items_det(g.data_ptr(), fm.data_ptr(), items, P, c.C, int(c.elu), c.bf.data_ptr(),
                                                      c.bm.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), sums[0].data_ptr(),
                                                      sums[1].data_ptr(), ws.data_ptr(), st))
        L.check(lib.read_gate_backward_batch_stats_items_det(g.data_ptr(), fm.data_ptr(), items, P, c.C, int(c.elu),
                                                             c.bf.data_ptr(), c.bm.data_ptr(), c.scale.data_ptr(), c.mean.data_ptr(),
                                                             c.inv.data_ptr(), sums[0].data_ptr(), sums[1].data_ptr(),
                                                             dfm.data_ptr(), red[0].data_ptr(), red[1].data_ptr(), ws.data_ptr(),
                                                             st))
        red[3], red[2] = sums[0].sum(0), sums[1].sum(0)
        return red
    if c.batch:
        L.check(lib.read_bn_backward_reduce_det(g.data_ptr(), fm.data_ptr(), P, c.C, int(c.elu), c.bf.data_ptr(), c.bm.data_ptr(),
                                                c.mean.data_ptr(), c.inv.data_ptr(), red[3].data_ptr(), red[2].data_ptr(),
                                                ws.data_ptr(), st))
        L.check(lib.read_gate_backward_batch_stats_det(g.data_ptr(), fm.data_ptr(), P, c.C, int(c.elu), c.bf.data_ptr(),
                                                       c.bm.data_ptr(), c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(),
                                                       red[3].data_ptr(), red[2].data_ptr(), dfm.data_ptr(), red[0].data_ptr(),
                                                       red[1].data_ptr(), ws.data_ptr(), st))
        return red
    L.check(lib.read_gate_backward_det(g.data_ptr(), fm.data_ptr(), P, c.C, int(c.elu), c.bf.data_ptr(), c.bm.data_ptr(),
                                       c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), dfm.data_ptr(), red[0].data_ptr(),
                                       red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), ws.data_ptr(), st))
    return red


def conv_wgrad(lib, dfm, x, B, Hout, Wout, C, k, stride, dwf, dwm, st):
    """dwf / dwm [C][Cin][k][k] += the weight gradient of a gated conv from [df | dm] [B,Hout,Wout,2C] and its input x
    [B,stride*Hout,stride*Wout,Cin] (NHWC bf16); under torch.use_deterministic_algorithms(True) with the split-K partials added in
    a fixed order."""
    Hin, Win, Cin = x.shape[1], x.shape[2], x.shape[3]
    if torch.are_deterministic_algorithms_enabled():
        ws = ops.det_workspace(lib.read_conv_wgrad_det_workspace_bytes(B, Hout, Wout, C, Cin, k, stride), dfm.device, "conv wgrad")
        L.check(lib.read_conv_wgrad_det(dfm.data_ptr(), x.data_ptr(), B, Hin, Win, Hout, Wout, C, Cin, k, stride, dwf.data_ptr(),
                                        dwm.data_ptr(), ws.data_ptr(), st))
    elif k == 3 and stride == 1:
        L.check(lib.read_conv3x3_wgrad(dfm.data_ptr(), x.data_ptr(), B, Hout, Wout, C, Cin, dwf.data_ptr(), dwm.data_ptr(), st))
    else:
        L.check(lib.read_conv_wgrad(dfm.data_ptr(), x.data_ptr(), B, Hin, Win, Hout, Wout, C, Cin, k, stride, dwf.data_ptr(),
                                    dwm.data_ptr(), st))


def dgrad(dfm, conv, residual=None):
    """Input gradient [B,H,W,Cin] (bf16) of ``conv`` (a FoldedConv) from [df | dm] in RAW column order, plus ``residual``."""
    lib = L.load()
    B, H, W, _ = dfm.shape
    cin = conv.wf.shape[1]
    out = torch.empty((B, H, W, cin), dtype=torch.bfloat16, device=dfm.device)
    if cin == 8:                     # the descriptor pyramid: N = 8, below the TMA kernel's smallest N tile
        if residual is not None:
            raise ValueError("read_b200: the input gradient of an 8-channel input takes no residual")
        L.check(lib.read_conv3x3_dgrad_cin8(dfm.data_ptr(), conv.wf.data_ptr(), conv.wm.data_ptr(), B, H, W, conv.C,
                                            out.data_ptr(), L.stream_ptr()))
        return out
    zeros = torch.zeros(cin, dtype=torch.float32, device=dfm.device)      # a RAW launch reads no epilogue parameters
    _launch(lib, dfm, cin // 2, conv.w_dgrad, (zeros,) * 4, False, L.OUT_RAW_NHWC, out, residual)
    return out


def _check_cuda(x):
    if not x.is_cuda:
        raise RuntimeError("read_b200: train_precision='bf16' runs the gated 3x3 convs on the H100 kernels and needs CUDA tensors")
    L.require_device(x.device.index)


class ResStackFn(torch.autograd.Function):
    """x (NCHW f32) -> the 4-ResBlock stack; ``mods`` = the stack's 8 GatedConvs in order, ``params`` = per conv (conv_f.weight,
    conv_f.bias, conv_m.weight, conv_m.bias, norm.weight, norm.bias)."""

    @staticmethod
    def forward(ctx, x, mods, *params):
        return ResStackFn._forward(ctx, x, mods, params, None)

    @staticmethod
    def _forward(ctx, x, mods, params, items):
        _check_cuda(x)
        lib = L.load()
        convs = [FoldedConv(m, *params[6 * i: 6 * i + 6], items=items) for i, m in enumerate(mods)]   # packed before the first launch
        t = ops.nchw_to_nhwc(x.detach().float().contiguous(), True)
        C = t.shape[3]
        saved = []
        for r in range(0, len(convs), 2):
            h = torch.empty_like(t)
            conv_forward(lib, t, convs[r], h)
            y = torch.empty_like(t)
            conv_forward(lib, h, convs[r + 1], y, residual=t)
            saved += [t, h]
            t = y
        ctx.convs, ctx.n_inputs = convs, len(saved)
        # the parameters are saved too: the folded / packed copies in ctx.convs alias or derive from them, and saving them makes
        # autograd raise if one is modified in place between forward and backward
        ctx.save_for_backward(*saved, *params)
        return ops.nhwc_to_nchw(t)

    @staticmethod
    def backward(ctx, gout):
        lib, st = L.load(), L.stream_ptr()
        inputs, convs = ctx.saved_tensors[:ctx.n_inputs], ctx.convs
        B, H, W, C = inputs[0].shape
        dev = inputs[0].device
        g = ops.nchw_to_nhwc(gout.float().contiguous(), True)             # gradient of the stack's output, NHWC bf16
        fm = torch.empty((B, H, W, 2 * C), dtype=torch.bfloat16, device=dev)
        dfm = torch.empty_like(fm)
        grads = [None] * (6 * len(convs))
        g_block = g
        for i in reversed(range(len(convs))):
            c, x_in = convs[i], inputs[i]
            if i % 2 == 1:
                g_block = g                                               # gradient of this ResBlock's output
            _launch(lib, x_in, C, c.w_tc, c.par, c.elu, L.OUT_RAW_NHWC, fm)
            red = gate_backward(lib, g, fm, c, dfm)                       # dbias_f, dbias_m, dgamma, dbeta
            dwf = dwm = None
            if ctx.needs_input_grad[2 + 6 * i] or ctx.needs_input_grad[4 + 6 * i]:    # not for a frozen net
                dwf, dwm = torch.zeros_like(c.wf), torch.zeros_like(c.wm)
                conv_wgrad(lib, dfm, x_in, B, H, W, C, 3, 1, dwf, dwm, st)
            grads[6 * i: 6 * i + 6] = [dwf, red[0], dwm, red[1], red[2], red[3]]
            if i > 0 or ctx.needs_input_grad[0]:
                # the first conv of a ResBlock adds the gradient that reaches its input through the skip
                g = dgrad(dfm, c, residual=g_block if i % 2 == 0 else None)
        dx = ops.nhwc_to_nchw(g) if ctx.needs_input_grad[0] else None
        grads = [gr if ctx.needs_input_grad[2 + k] else None for k, gr in enumerate(grads)]
        return (dx, None, *grads)


class ResStackItemsFn(ResStackFn):
    """ResStackFn with per-item statistics for its train-mode norms (each batch item normalised with its own)."""

    @staticmethod
    def forward(ctx, x, mods, *params):
        return ResStackFn._forward(ctx, x, mods, params, x.shape[0])


def stack_convs(net, prefix):
    """The 8 GatedConvs of the stack ``prefix`` (e.g. 'Encoder.0') in forward order."""
    return [net.get_submodule(f"{prefix}.layers.{i}.main.{j}") for i in range(net.num_res) for j in (0, 1)]


def res_stack(net, prefix, x, batch_stats=False, per_item=False):
    """bf16 forward of one EBlock / DBlock of ``net`` on the wgmma kernels, differentiable through ResStackFn."""
    names = [f"{prefix}.layers.{i}.main.{j}" for i in range(net.num_res) for j in (0, 1)]
    if per_item:
        return stack_forward(stack_convs(net, prefix), x, batch_stats=batch_stats, names=names, per_item=True)
    return stack_forward(stack_convs(net, prefix), x, batch_stats=batch_stats, names=names)


def stack_params(mods):
    """ResStackFn's parameter list for the GatedConvs ``mods``."""
    params = []
    for m in mods:
        b = m.block
        params += [b['conv_f'].weight, b['conv_f'].bias, b['conv_m'].weight, b['conv_m'].bias, b['norm'].weight, b['norm'].bias]
    return params


def _check_eval(mods):
    if any(m.block['norm'].training for m in mods):
        raise RuntimeError("read_b200: train_precision='bf16' folds BatchNorm with its running statistics; put the net in eval() "
                           "mode (the reference trains with eval-mode BatchNorm)")


def _label(mod, name):
    return name or f"GatedConv(k={mod.k}, stride={mod.stride})"


def check_norms(mods, batch_stats, pixels, names=None, per_item=False):
    """Without ``batch_stats`` every norm must be in eval mode (RuntimeError).  With it, a train-mode norm must be one the batch
    statistics kernels implement (momentum set, running statistics tracked, affine) and the conv must have at least 2 output
    pixels (``pixels`` = B * H_out * W_out, or H_out * W_out per item with ``per_item``; torch raises for 1 too); otherwise a
    ValueError names the layer."""
    if not batch_stats:
        _check_eval(mods)
        return
    for i, m in enumerate(mods):
        n = m.block['norm']
        if not n.training:
            continue
        label = _label(m, names[i] if names else None)
        if n.momentum is None:
            raise ValueError(f"read_b200: {label}: train-mode BatchNorm with momentum=None (cumulative moving average) is not "
                             "supported on the bf16 path")
        if not n.track_running_stats or not n.affine:
            raise ValueError(f"read_b200: {label}: train-mode BatchNorm needs track_running_stats=True and affine=True on the "
                             f"bf16 path (got track_running_stats={n.track_running_stats}, affine={n.affine})")
        if pixels < 2:
            got = f"H * W = {pixels} per item" if per_item else f"B * H * W = {pixels}"
            raise ValueError(f"read_b200: {label}: train-mode BatchNorm needs more than 1 value per channel (got {got})")


def stack_forward(mods, x, batch_stats=False, names=None, per_item=False):
    """The ResBlocks t -> t + mods[2r+1](mods[2r](t)) applied to x in turn, bf16 on the wgmma kernels.  ``batch_stats``: a conv
    whose norm is in train mode normalises with batch statistics (else such a conv raises), each batch item with its own with
    ``per_item``; ``names`` label the convs in errors."""
    check_norms(mods, batch_stats, (1 if per_item else x.shape[0]) * x.shape[2] * x.shape[3], names, per_item)
    return (ResStackItemsFn if per_item else ResStackFn).apply(x, list(mods), *stack_params(mods))


class GatedConvFn(torch.autograd.Function):
    """x (NCHW f32) -> mod(x) [+ residual] for one gated 3x3 stride-1 conv ``mod``; ``params`` = (conv_f.weight, conv_f.bias,
    conv_m.weight, conv_m.bias, norm.weight, norm.bias).  A conv with C < 16 (the RGB output conv) runs padded to C = 16."""

    @staticmethod
    def forward(ctx, x, residual, mod, *params):
        return GatedConvFn._forward(ctx, x, residual, mod, params, None)

    @staticmethod
    def _forward(ctx, x, residual, mod, params, items):
        _check_cuda(x)
        lib = L.load()
        cout = params[0].shape[0]
        conv = FoldedConv(mod, *params, cout=max(cout, 16), items=items)
        if residual is not None and conv.C != cout:
            raise ValueError("read_b200: a residual needs C >= 16")
        t = ops.nchw_to_nhwc(x.detach().float().contiguous(), True)
        B, H, W, _ = t.shape
        r = None if residual is None else ops.nchw_to_nhwc(residual.detach().float().contiguous(), True)
        y = torch.empty((B, H, W, conv.C), dtype=torch.bfloat16, device=t.device)
        conv_forward(lib, t, conv, y, residual=r)
        ctx.conv, ctx.cout = conv, cout
        ctx.save_for_backward(t, *params)              # the parameters: an in-place update before backward raises
        y = ops.nhwc_to_nchw(y)
        return y if cout == conv.C else y[:, :cout].contiguous()

    @staticmethod
    def backward(ctx, gout):
        lib, st = L.load(), L.stream_ptr()
        x_in, c, cout = ctx.saved_tensors[0], ctx.conv, ctx.cout
        need = ctx.needs_input_grad
        B, H, W, _ = x_in.shape
        C, dev = c.C, x_in.device
        gp = gout.float()
        if cout < C:
            gp = torch.cat([gp, gp.new_zeros((B, C - cout, H, W))], 1)   # the padded channels' output gradient is 0
        g = ops.nchw_to_nhwc(gp.contiguous(), True)
        fm = torch.empty((B, H, W, 2 * C), dtype=torch.bfloat16, device=dev)
        dfm = torch.empty_like(fm)
        _launch(lib, x_in, C, c.w_tc, c.par, c.elu, L.OUT_RAW_NHWC, fm)
        red = gate_backward(lib, g, fm, c, dfm)                           # dbias_f, dbias_m, dgamma, dbeta
        dwf = dwm = None
        if need[3] or need[5]:                                            # not for a frozen net
            dwf, dwm = torch.zeros_like(c.wf), torch.zeros_like(c.wm)
            conv_wgrad(lib, dfm, x_in, B, H, W, C, 3, 1, dwf, dwm, st)
        dx = ops.nhwc_to_nchw(dgrad(dfm, c)) if need[0] else None
        grads = [dwf, red[0], dwm, red[1], red[2], red[3]]
        grads = [gr[:cout] if gr is not None and need[3 + k] else None for k, gr in enumerate(grads)]
        return (dx, gout if need[1] else None, None, *grads)


class GatedConvItemsFn(GatedConvFn):
    """GatedConvFn with per-item statistics for a train-mode norm (each batch item normalised with its own)."""

    @staticmethod
    def forward(ctx, x, residual, mod, *params):
        return GatedConvFn._forward(ctx, x, residual, mod, params, x.shape[0])


def gated_conv(mod, x, residual=None, batch_stats=False, name=None, per_item=False):
    """bf16 forward of the gated 3x3 stride-1 conv ``mod`` (a GatedConv) on the wgmma kernels, plus ``residual`` (NCHW, the
    output's shape) when given, differentiable through GatedConvFn.  ``batch_stats``: a train-mode norm normalises with batch
    statistics (else it raises), each batch item with its own with ``per_item``; ``name`` labels the layer in errors."""
    if mod.k != 3 or mod.stride != 1:
        raise ValueError(f"read_b200: gated_conv runs 3x3 stride-1 convs only (got k={mod.k}, stride={mod.stride})")
    check_norms([mod], batch_stats, (1 if per_item else x.shape[0]) * x.shape[2] * x.shape[3], [name], per_item)
    return (GatedConvItemsFn if per_item else GatedConvFn).apply(x, residual, mod, *stack_params([mod]))


# ------------------------------------------------------------------ the 1x1 and stride-2 convs ('bf16_all')
GEOMETRIES = ((1, 1), (3, 2), (4, 2))        # (k, stride) of the convs MultiSourceConvFn runs


def padded_channels(c):
    """The channel count a conv with C = c runs at: 16, 32, 64 or a multiple of 64 (the counts the gate backward, the weight
    gradient and the RAW 1x1 plans take)."""
    return 16 if c <= 16 else 32 if c <= 32 else 64 * ((c + 63) // 64)


def recompute_fm(lib, srcs, c):
    """[f | m] (RAW column order) of the FoldedConv ``c`` over the NHWC sources.  A RAW 1x1 plan takes at most 64 output channels
    (one N tile), so a wider 1x1 conv is recomputed per 64-channel block with that block's filters: block b of the RAW order is
    [f | m] of channels 64b .. 64b + 63."""
    d = _desc(srcs, c.C, c.k, c.stride)
    B, H, W = d.B, d.Hout, d.Wout
    zeros = torch.zeros(c.C, dtype=torch.float32, device=srcs[0].device)  # a RAW launch reads no epilogue parameters
    if c.k != 1 or c.C <= 64:
        fm = torch.empty((B, H, W, 2 * c.C), dtype=torch.bfloat16, device=srcs[0].device)
        _launch(lib, srcs, c.C, c.w_tc, (zeros,) * 4, False, L.OUT_RAW_NHWC, fm, k=c.k, stride=c.stride)
        return fm
    blocks_ = []
    for w in _fm64_filters(lib, srcs, c):
        out = torch.empty((B, H, W, 128), dtype=torch.bfloat16, device=srcs[0].device)
        _launch(lib, srcs, 64, w, (zeros,) * 4, False, L.OUT_RAW_NHWC, out, k=1)
        blocks_.append(out)
    return torch.cat(blocks_, -1)


def _fm64_filters(lib, srcs, c):
    """The forward filters of each 64-channel block of a 1x1 FoldedConv wider than 64 (recompute_fm), packed once per entry."""
    ws = c.pk.get('fm64')
    if ws is None:
        d64 = _desc(srcs, 64, 1, 1)
        ws = [torch.empty(lib.read_tc_weight_elems(64, d64.Cin, 1), dtype=torch.bfloat16, device=c.wf.device)
              for _ in range(c.C // 64)]
        for b, w in enumerate(ws):
            L.check(lib.read_pack_weights_tc_for(ctypes.byref(d64), c.wf[64 * b: 64 * b + 64].data_ptr(),
                                                 c.wm[64 * b: 64 * b + 64].data_ptr(), w.data_ptr(), L.stream_ptr()))
        c.pk['fm64'] = ws
    return ws


def _dgrad1x1_filters(lib, c, a, cn, device):
    """The transposed filters of the RAW 1x1 input-gradient plan for input channels a .. a + cn - 1 (dgrad_1x1)."""
    w = c.pk.get(('d1x1', a, cn))
    if w is None:
        n_out = max(cn, 32)
        w = torch.empty(lib.read_tc_weight_elems(n_out // 2, 2 * c.C, 1), dtype=torch.bfloat16, device=device)
        L.check(lib.read_pack_weights_tc_dgrad1x1(c.wf.data_ptr(), c.wm.data_ptr(), c.C, c.wf.shape[1], a, cn, w.data_ptr(),
                                                  L.stream_ptr()))
        c.pk[('d1x1', a, cn)] = w
    return w


def dgrad_s2_filters(c):
    """The flipped-by-phase filters [k*k][Cin][2C] (bf16) of the stride-2 input-gradient kernel for the FoldedConv ``c``."""
    w = c.pk.get('s2')
    if w is None:
        cin = c.wf.shape[1]
        w = torch.empty((c.k * c.k, cin, 2 * c.C), dtype=torch.bfloat16, device=c.wf.device)
        L.check(L.load().read_pack_weights_dgrad_s2(c.wf.data_ptr(), c.wm.data_ptr(), c.C, cin, c.k, w.data_ptr(), L.stream_ptr()))
        c.pk['s2'] = w
    return w


def dgrad_1x1(dfm, c, c0, cs):
    """Input gradient [B,H,W,cs] (bf16) of input channels c0 .. c0 + cs - 1 of the 1x1 FoldedConv ``c``: RAW 1x1 plans over
    [df | dm] with transposed filters, one per 128 channels (the plans' widest N tile); 16 channels run padded to 32."""
    lib = L.load()
    B, H, W, _ = dfm.shape
    parts = []
    for a in range(c0, c0 + cs, 128):
        cn = min(128, c0 + cs - a)
        n_out = max(cn, 32)
        w = _dgrad1x1_filters(lib, c, a, cn, dfm.device)
        out = torch.empty((B, H, W, n_out), dtype=torch.bfloat16, device=dfm.device)
        zeros = torch.zeros(n_out // 2, dtype=torch.float32, device=dfm.device)
        _launch(lib, dfm, n_out // 2, w, (zeros,) * 4, False, L.OUT_RAW_NHWC, out, k=1)
        parts.append(out if cn == n_out else out[..., :cn])
    return parts[0] if len(parts) == 1 else torch.cat(parts, -1)


class MultiSourceConvFn(torch.autograd.Function):
    """The gated 1x1 or stride-2 3x3 / 4x4 conv ``mod`` over the NCHW f32 tensors ``xs`` (a 1x1 conv reads several as a virtual
    concat along channels); ``params`` = (conv_f.weight, conv_f.bias, conv_m.weight, conv_m.bias, norm.weight, norm.bias).  A conv
    whose C is not 16, 32, 64 or a multiple of 64 runs padded (padded_channels)."""

    @staticmethod
    def forward(ctx, mod, n_src, *args):
        return MultiSourceConvFn._forward(ctx, mod, n_src, args, False)

    @staticmethod
    def _forward(ctx, mod, n_src, args, per_item):
        xs, params = args[:n_src], args[n_src:]
        _check_cuda(xs[0])
        lib = L.load()
        cout = params[0].shape[0]
        ts = [ops.nchw_to_nhwc(x.detach().float().contiguous(), True) for x in xs]
        conv = FoldedConv(mod, *params, cout=padded_channels(cout), srcs=ts, items=xs[0].shape[0] if per_item else None)
        d = _desc(ts, conv.C, mod.k, mod.stride)
        y = torch.empty((d.B, d.Hout, d.Wout, conv.C), dtype=torch.bfloat16, device=ts[0].device)
        conv_forward(lib, ts, conv, y)
        ctx.conv, ctx.cout, ctx.n_src = conv, cout, n_src
        ctx.save_for_backward(*ts, *params)            # the parameters: an in-place update before backward raises
        y = ops.nhwc_to_nchw(y)
        return y if cout == conv.C else y[:, :cout].contiguous()

    @staticmethod
    def backward(ctx, gout):
        lib, st = L.load(), L.stream_ptr()
        n_src, c, cout = ctx.n_src, ctx.conv, ctx.cout
        ts = ctx.saved_tensors[:n_src]
        need = ctx.needs_input_grad[2:]                                    # the sources, then the 6 parameters
        C, dev = c.C, ts[0].device
        B = ts[0].shape[0]
        gp = gout.float()
        if cout < C:
            gp = torch.cat([gp, gp.new_zeros((B, C - cout) + tuple(gp.shape[2:]))], 1)  # the padded channels' gradient is 0
        g = ops.nchw_to_nhwc(gp.contiguous(), True)
        Hout, Wout = g.shape[1], g.shape[2]
        fm = recompute_fm(lib, ts, c)
        dfm = torch.empty_like(fm)
        red = gate_backward(lib, g, fm, c, dfm)                            # dbias_f, dbias_m, dgamma, dbeta
        del fm
        dwf = dwm = None
        if need[n_src] or need[n_src + 2]:                                 # not for a frozen net
            kk = (c.k, c.k)
            dws = [(torch.zeros((C, t.shape[3]) + kk, device=dev), torch.zeros((C, t.shape[3]) + kk, device=dev)) for t in ts]
            for t, (wf_s, wm_s) in zip(ts, dws):
                conv_wgrad(lib, dfm, t, B, Hout, Wout, C, c.k, c.stride, wf_s, wm_s, st)
            dwf = torch.cat([w[0] for w in dws], 1) if n_src > 1 else dws[0][0]
            dwm = torch.cat([w[1] for w in dws], 1) if n_src > 1 else dws[0][1]
        dxs = [None] * n_src
        c0 = 0
        for i, t in enumerate(ts):
            cs = t.shape[3]
            if need[i]:
                if c.stride == 2:
                    dx = torch.empty_like(t)
                    L.check(lib.read_conv_dgrad_s2(dfm.data_ptr(), dgrad_s2_filters(c).data_ptr(), B, Hout, Wout, C, cs, c.k,
                                                   dx.data_ptr(), st))
                else:
                    dx = dgrad_1x1(dfm, c, c0, cs)
                dxs[i] = ops.nhwc_to_nchw(dx.contiguous())
            c0 += cs
        grads = [dwf, red[0], dwm, red[1], red[2], red[3]]
        grads = [gr[:cout] if gr is not None and need[n_src + j] else None for j, gr in enumerate(grads)]
        return (None, None, *dxs, *grads)


class MultiSourceConvItemsFn(MultiSourceConvFn):
    """MultiSourceConvFn with per-item statistics for a train-mode norm (each batch item normalised with its own)."""

    @staticmethod
    def forward(ctx, mod, n_src, *args):
        return MultiSourceConvFn._forward(ctx, mod, n_src, args, True)


def gated_conv_srcs(mod, xs, name=None, batch_stats=False, per_item=False):
    """bf16 forward of the gated 1x1 or stride-2 conv ``mod`` (a GatedConv) over the NCHW tensors ``xs`` on the wgmma kernels,
    differentiable through MultiSourceConvFn.  A 1x1 conv reads several sources as one concat (each a multiple of 32 channels);
    a stride-2 conv takes one source of even height and width.  ``name`` labels the layer in errors.  ``batch_stats``: a
    train-mode norm normalises with batch statistics (else it raises), each batch item with its own with ``per_item``."""
    label = name or f"GatedConv(k={mod.k}, stride={mod.stride})"
    xs = list(xs)
    if (mod.k, mod.stride) not in GEOMETRIES:
        raise ValueError(f"read_b200: {label}: gated_conv_srcs runs 1x1 and stride-2 3x3 / 4x4 convs (got k={mod.k}, "
                         f"stride={mod.stride}); a 3x3 stride-1 conv goes through gated_conv")
    if len(xs) > 1 and (mod.k != 1 or any(x.shape[1] % 32 for x in xs)):
        raise ValueError(f"read_b200: {label}: only a 1x1 conv reads several sources, each a multiple of 32 channels "
                         f"(got {[x.shape[1] for x in xs]})")
    if len(xs) > 4:
        raise ValueError(f"read_b200: {label}: at most 4 sources (got {len(xs)})")
    if mod.stride == 2 and (xs[0].shape[2] % 2 or xs[0].shape[3] % 2):
        raise ValueError(f"read_b200: {label}: a stride-2 conv needs an even input height and width (got "
                         f"{xs[0].shape[2]}x{xs[0].shape[3]})")
    pixels = (1 if per_item else xs[0].shape[0]) * (xs[0].shape[2] // mod.stride) * (xs[0].shape[3] // mod.stride)
    check_norms([mod], batch_stats, pixels, [label], per_item)
    return (MultiSourceConvItemsFn if per_item else MultiSourceConvFn).apply(mod, len(xs), *xs, *stack_params([mod]))
