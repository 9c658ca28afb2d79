"""bf16 training of the gated 3x3 stride-1 convs (READ/models/unet.py:22-53) on the wgmma kernels.

``UNet.train_precision = 'bf16'`` sends 78 of the net's 99 convs here; the other 21 (the 1x1 and stride-2 convs), the
interpolations, concats and FAM products / sums stay on torch operators in the same autograd graph.  ``'bf16_all'`` also sends
those 21 convs here (``gated_conv_srcs``).  One autograd Function, ``ConvChainFn``, runs every call:
* ``stack_forward``: each of the 8 residual block stacks (Encoder.0-3, Decoder.0-3: 4 ResBlocks = 8 convs at constant C, 64 convs).
* ``gated_conv``: one conv with an optional residual, for the 14 single convs feat_extract.0 (8 -> 32), feat_extract.5 (32 -> 3,
  the RGB output, run padded to C = 16), SCM*.main.0 (8 -> 16 / 32 / 64), SCM*.main.2, AFFs.*.conv.1 and FAM*.merge.

Forward: NCHW f32 -> NHWC bf16 once, launches of the TMA wgmma kernel (in a stack the second conv of each ResBlock adds the skip in
its epilogue), NHWC bf16 -> NCHW f32 once.  Saved for backward: the input of every conv (bf16, Cin channels per pixel), which the
weight gradient needs anyway.  The pre-activation [f | m] (2C channels per pixel) is NOT saved: backward recomputes it per conv
with a RAW launch of the same kernel.  That costs one extra forward conv per conv and keeps the saved activations at a third of
what saving [f | m] as well would take (C5, 8 crops of 256^2: about 1 GB instead of 3 GB across the 8 stacks, and 147 MB for the
14 single convs).

Backward, per conv, last to first (csrc/conv_bwd.cu, conv_backward): recompute [f | m]; gate backward -> [df | dm] and the bias /
BatchNorm-affine gradients; weight gradient (tensor-core kernel, fp32 atomics into the torch-layout gradients; skipped when no
weight needs one); input gradient (input_grad) = RAW launch of the TMA kernel over [df | dm] with flipped, transposed filters, the
ResBlock skip added through its residual operand, or for an 8-channel input (the descriptor pyramid) the dedicated dgrad_cin8
kernel; a stride-2 conv's has its own kernel, and a 1x1 conv's runs as RAW 1x1 plans per source.

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


def _launch_raw(lib, src, cout, w_tc, out, residual=None, k=3, stride=1):
    """A _launch with RAW output (the [f | m] accumulators, no epilogue): the kernel still stages ``cout`` epilogue parameters,
    which RAW output never uses, so they are zeros."""
    zeros = torch.zeros(cout, dtype=torch.float32, device=out.device)
    _launch(lib, src, cout, w_tc, (zeros,) * 4, False, L.OUT_RAW_NHWC, out, residual, k=k, stride=stride)


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
    """The fp32 filters padded to C channels and the bf16 forward and backward filters of ``mod``, from the cache when the weights
    are unchanged: for a 3x3 stride-1 conv the forward and input-gradient filters, for a 1x1 or stride-2 conv over ``srcs`` the
    forward filters and those its backward launches take (the stride-2 input-gradient filters, _fm64_filters,
    _dgrad1x1_filters), so that a backward packs nothing.  Entries are only ever added, and a new weight version starts a new
    dict, so a FoldedConv of an earlier forward keeps the filters it was built with.  Writes that bypass the version counter
    (through ``.data``) are not seen."""
    key = filter_key(mod, wf, wm, C, srcs)
    ent = _FILTERS.get(mod) if cache_filters else None
    if ent is not None and ent[0] == key:
        return ent[1]
    lib, st = L.load(), L.stream_ptr()
    cin = wf.shape[1]
    pad = lambda t: _pad_rows(t.detach().float(), C).contiguous()
    pk = {'wf': pad(wf), 'wm': pad(wm), 'w_dgrad': None}       # an 8-channel input's gradient kernel reads wf / wm itself
    pk['w_tc'] = torch.empty(lib.read_tc_weight_elems(C, cin, mod.k), dtype=torch.bfloat16, device=wf.device)
    if (mod.k, mod.stride) == (3, 1):
        L.check(lib.read_pack_weights_tc(pk['wf'].data_ptr(), pk['wm'].data_ptr(), C, cin, 3, pk['w_tc'].data_ptr(), st))
        if cin != 8:
            pk['w_dgrad'] = torch.empty(lib.read_tc_weight_elems(cin // 2, 2 * C, 3), dtype=torch.bfloat16, device=wf.device)
            L.check(lib.read_pack_weights_tc_dgrad(pk['wf'].data_ptr(), pk['wm'].data_ptr(), C, cin, pk['w_dgrad'].data_ptr(), st))
    else:
        L.check(lib.read_pack_weights_tc_for(ctypes.byref(_desc(srcs, C, mod.k, mod.stride)), pk['wf'].data_ptr(),
                                             pk['wm'].data_ptr(), pk['w_tc'].data_ptr(), st))
        if mod.stride == 2:             # the flipped-by-phase filters [k*k][Cin][2C] of the stride-2 input-gradient kernel
            pk['s2'] = torch.empty((mod.k * mod.k, cin, 2 * C), dtype=torch.bfloat16, device=wf.device)
            L.check(lib.read_pack_weights_dgrad_s2(pk['wf'].data_ptr(), pk['wm'].data_ptr(), C, cin, mod.k, pk['s2'].data_ptr(),
                                                   st))
        else:
            if C > 64:
                _fm64_filters(lib, pk, C, srcs)
            c0 = 0
            for s in srcs:
                _dgrad1x1_filters(lib, pk, C, c0, s.shape[3])
                c0 += s.shape[3]
    if cache_filters:
        _FILTERS[mod] = (key, pk)
    return pk


def _fm64_filters(lib, pk, C, srcs):
    """The forward filters of each 64-channel block of a 1x1 conv wider than 64 (recompute_fm) from its filters ``pk``
    (_packed) at C channels, packed once per entry."""
    ws = pk.get('fm64')
    if ws is None:
        wf, wm = pk['wf'], pk['wm']
        d64 = _desc(srcs, 64, 1, 1)
        ws = [torch.empty(lib.read_tc_weight_elems(64, d64.Cin, 1), dtype=torch.bfloat16, device=wf.device) for _ in range(C // 64)]
        for b, w in enumerate(ws):
            L.check(lib.read_pack_weights_tc_for(ctypes.byref(d64), wf[64 * b: 64 * b + 64].data_ptr(),
                                                 wm[64 * b: 64 * b + 64].data_ptr(), w.data_ptr(), L.stream_ptr()))
        pk['fm64'] = ws
    return ws


def _dgrad1x1_filters(lib, pk, C, c0, cs):
    """The transposed filters of the RAW 1x1 input-gradient plans (dgrad_1x1) of input channels c0 .. c0 + cs - 1 of a 1x1 conv
    with filters ``pk`` (_packed) at C channels, one plan per 128 channels: a list of (a, cn, filters of channels a .. a + cn - 1),
    each packed once per entry."""
    wf, wm = pk['wf'], pk['wm']
    plans = []
    for a in range(c0, c0 + cs, 128):
        cn = min(128, c0 + cs - a)
        w = pk.get(('d1x1', a, cn))
        if w is None:
            w = torch.empty(lib.read_tc_weight_elems(max(cn, 32) // 2, 2 * C, 1), dtype=torch.bfloat16, device=wf.device)
            L.check(lib.read_pack_weights_tc_dgrad1x1(wf.data_ptr(), wm.data_ptr(), C, wf.shape[1], a, cn, w.data_ptr(),
                                                      L.stream_ptr()))
            pk[('d1x1', a, cn)] = w
        plans.append((a, cn, w))
    return plans


def dgrad_s2_filters(c):
    """The flipped-by-phase filters [k*k][Cin][2C] (bf16) of the stride-2 input-gradient kernel for the stride-2 FoldedConv
    ``c``, packed with its forward filters (_packed)."""
    return c.pk['s2']


class FoldedConv:
    """One GatedConv's live parameters for this step: its BatchNorm and the bf16 filters of the forward conv (also used for the RAW
    recompute) and of the input gradient.  ``cout`` > the conv's C pads it with zero filters, biases and BatchNorm scale / shift
    (the RGB output conv, C = 3, runs as C = 16; SCM*.main.3, C = 56 / 120 / 248, as 64 / 128 / 256): the padded channels compute
    0 and get 0 gradients.  A 1x1 or stride-2 conv (k in {1, 3, 4}, stride in {1, 2}) packs its forward and backward filters
    for the launches over ``srcs`` (the NHWC sources, whose channel counts set a concat's K chunks).
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
    batch statistics, running-statistics update and y = g * scale + shift [+ residual].  With per-item statistics item i of ``g``
    ([items, H, W, C]) is normalised with its own; the running statistics are updated once per item, in item order, and
    num_batches_tracked advances by the number of items, as that many single-item calls would."""
    st, n, C = L.stream_ptr(), c.norm, c.C
    per_item = c.items is not None
    items = g.shape[0] if per_item else 1
    P, form = g.numel() // (items * C), "_items" if per_item else ""
    ws = torch.empty(lib.read_bn_workspace_bytes_items(items, C) if per_item else lib.read_bn_workspace_bytes(C), dtype=torch.uint8,
                     device=g.device)
    head = [g.data_ptr(), *([items] if per_item else []), P, C]
    L.check(getattr(lib, "read_bn_batch_stats" + form)(*head, c.n_real, c.gamma.data_ptr(), c.beta.data_ptr(), n.eps, n.momentum,
                                                       n.running_mean.data_ptr(), n.running_var.data_ptr(), c.mean.data_ptr(),
                                                       c.inv.data_ptr(), *([] if per_item else [None]), c.scale.data_ptr(),
                                                       c.shift.data_ptr(), ws.data_ptr(), st))
    n.num_batches_tracked.add_(items)          # torch's own op: bumps the version UNet._weights_version sums
    L.check(getattr(lib, "read_bn_apply" + form)(*head, c.scale.data_ptr(), c.shift.data_ptr(), L.ptr(residual), g.data_ptr(), st))


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
    its output gradient ``g`` and the recomputed [f | m]; a train-mode norm adds the terms through the batch statistics (per item
    with per-item statistics).  Under torch.use_deterministic_algorithms(True) the *_det entry points combine the sums in a fixed
    order."""
    st, C = L.stream_ptr(), c.C
    red = torch.zeros((4, C), dtype=torch.float32, device=g.device)    # dbias_f, dbias_m, dgamma, dbeta
    mode = "eval" if not c.batch else "batch" if c.items is None else "items"
    items = g.shape[0] if mode == "items" else 1
    P = g.numel() // (items * C)
    det = "_det" if torch.are_deterministic_algorithms_enabled() else ""
    ws = ops.det_workspace(lib.read_gate_det_workspace_bytes(items, C), g.device, "gate backward") if det else None
    tail = ([ws.data_ptr()] if det else []) + [st]
    head = [g.data_ptr(), fm.data_ptr(), *([items] if mode == "items" else []), P, C, int(c.elu), c.bf.data_ptr(),
            c.bm.data_ptr()]
    if mode == "eval":
        L.check(getattr(lib, "read_gate_backward" + det)(*head, c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(),
                                                         dfm.data_ptr(), *(r.data_ptr() for r in red), *tail))
        return red
    # sum dy, sum dy * xhat: dbeta and dgamma, per item ([items, C]) with per-item statistics
    sums = (red[3], red[2]) if mode == "batch" else torch.zeros((2, items, C), dtype=torch.float32, device=g.device)
    form = ("_items" if mode == "items" else "") + det
    L.check(getattr(lib, "read_bn_backward_reduce" + form)(*head, c.mean.data_ptr(), c.inv.data_ptr(), sums[0].data_ptr(),
                                                           sums[1].data_ptr(), *tail))
    L.check(getattr(lib, "read_gate_backward_batch_stats" + form)(*head, c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(),
                                                                  sums[0].data_ptr(), sums[1].data_ptr(), dfm.data_ptr(),
                                                                  red[0].data_ptr(), red[1].data_ptr(), *tail))
    if mode == "items":
        red[3], red[2] = sums[0].sum(0), sums[1].sum(0)
    return red


def conv_wgrad(lib, dfm, x, B, Hout, Wout, C, k, stride, dwf, dwm, st):
    """dwf / dwm [C][Cin][k][k] += the weight gradient of a gated conv from [df | dm] [B,Hout,Wout,2C] and its input x
    [B,stride*Hout,stride*Wout,Cin] (NHWC bf16); under torch.use_deterministic_algorithms(True) with the split-K partials added in
    a fixed order."""
    Hin, Win, Cin = x.shape[1], x.shape[2], x.shape[3]
    args = [dfm.data_ptr(), x.data_ptr(), B, Hin, Win, Hout, Wout, C, Cin, k, stride, dwf.data_ptr(), dwm.data_ptr()]
    if torch.are_deterministic_algorithms_enabled():
        ws = ops.det_workspace(lib.read_conv_wgrad_det_workspace_bytes(B, Hout, Wout, C, Cin, k, stride), dfm.device, "conv wgrad")
        L.check(lib.read_conv_wgrad_det(*args, ws.data_ptr(), st))
    else:
        L.check(lib.read_conv_wgrad(*args, st))


def _out_grad(gout, C):
    """The output gradient ``gout`` (NCHW) as NHWC bf16 with the C channels the conv runs at: a conv run padded to C gets 0 as
    the gradient of its padded channels."""
    gp = gout.float()
    if gp.shape[1] < C:
        gp = torch.cat([gp, gp.new_zeros((gp.shape[0], C - gp.shape[1]) + tuple(gp.shape[2:]))], 1)
    return ops.nchw_to_nhwc(gp.contiguous(), True)


def _param_grads(lib, g, fm, c, dfm, srcs, need, cout):
    """[dwf, dbias_f, dwm, dbias_m, dgamma, dbeta] of the FoldedConv ``c`` from its output gradient ``g`` and recomputed [f | m]:
    the gate backward into ``dfm``, then the weight gradient over each NHWC source in ``srcs`` (skipped when no weight needs one,
    as for a frozen net).  ``need`` are the 6 parameters' needs_input_grad flags: a gradient nobody asks for is None, the others
    are sliced to the conv's ``cout`` real channels."""
    red = gate_backward(lib, g, fm, c, dfm)
    dwf = dwm = None
    if need[0] or need[2]:
        B, Hout, Wout, _ = dfm.shape
        dws = [[torch.zeros((c.C, s.shape[3], c.k, c.k), dtype=torch.float32, device=dfm.device) for _ in range(2)] for s in srcs]
        for s, (wf_s, wm_s) in zip(srcs, dws):
            conv_wgrad(lib, dfm, s, B, Hout, Wout, c.C, c.k, c.stride, wf_s, wm_s, L.stream_ptr())
        dwf, dwm = dws[0] if len(srcs) == 1 else (torch.cat(w, 1) for w in zip(*dws))
    grads = [dwf, red[0], dwm, red[1], red[2], red[3]]
    return [gr[:cout] if n else None for gr, n in zip(grads, need)]


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
    _launch_raw(lib, dfm, cin // 2, conv.w_dgrad, out, residual)
    return out


def padded_channels(c):
    """The channel count a conv with C = c runs at: 16, 32, 64 or a multiple of 64 (the counts the gate backward, the weight
    gradient and the RAW 1x1 plans take)."""
    return 16 if c <= 16 else 32 if c <= 32 else 64 * ((c + 63) // 64)


def recompute_fm(lib, srcs, c):
    """[f | m] (RAW column order) of the FoldedConv ``c`` over the NHWC sources, launched with the conv's own epilogue
    parameters (RAW output reads none of them).  A RAW 1x1 plan takes at most 64 output channels (one N tile), so a wider 1x1
    conv is recomputed per 64-channel block with that block's filters: block b of the RAW order is [f | m] of channels
    64b .. 64b + 63."""
    d = _desc(srcs, c.C, c.k, c.stride)
    B, H, W = d.B, d.Hout, d.Wout
    if c.k != 1 or c.C <= 64:
        fm = torch.empty((B, H, W, 2 * c.C), dtype=torch.bfloat16, device=srcs[0].device)
        _launch(lib, srcs, c.C, c.w_tc, c.par, c.elu, L.OUT_RAW_NHWC, fm, k=c.k, stride=c.stride)
        return fm
    blocks_ = []
    for w in _fm64_filters(lib, c.pk, c.C, srcs):
        out = torch.empty((B, H, W, 128), dtype=torch.bfloat16, device=srcs[0].device)
        _launch(lib, srcs, 64, w, c.par, c.elu, L.OUT_RAW_NHWC, out, k=1)
        blocks_.append(out)
    return torch.cat(blocks_, -1)


def dgrad_1x1(dfm, c, c0, cs):
    """Input gradient [B,H,W,cs] (bf16) of input channels c0 .. c0 + cs - 1 of the 1x1 FoldedConv ``c``: RAW 1x1 plans over
    [df | dm] with transposed filters, one per 128 channels (the plans' widest N tile); 16 channels run padded to 32."""
    lib = L.load()
    B, H, W, _ = dfm.shape
    parts = []
    for _, cn, w in _dgrad1x1_filters(lib, c.pk, c.C, c0, cs):
        n_out = max(cn, 32)
        out = torch.empty((B, H, W, n_out), dtype=torch.bfloat16, device=dfm.device)
        _launch_raw(lib, dfm, n_out // 2, w, out, k=1)
        parts.append(out if cn == n_out else out[..., :cn])
    return parts[0] if len(parts) == 1 else torch.cat(parts, -1)


def input_grad(dfm, c, src, c0, residual=None):
    """Input gradient (NHWC bf16, the shape of ``src``) of the NHWC source ``src`` of the FoldedConv ``c``, input channels
    c0 .. c0 + Cs - 1 of its concat, from [df | dm] in RAW column order: the stride-2 kernel, a 1x1 conv's RAW plans (dgrad_1x1),
    or a 3x3 stride-1 conv's dgrad, plus ``residual``."""
    if c.stride == 2:
        B, Hout, Wout, _ = dfm.shape
        dx = torch.empty_like(src)
        L.check(L.load().read_conv_dgrad_s2(dfm.data_ptr(), dgrad_s2_filters(c).data_ptr(), B, Hout, Wout, c.C,
                                            src.shape[3], c.k, dx.data_ptr(), L.stream_ptr()))
        return dx
    if c.k == 1:
        return dgrad_1x1(dfm, c, c0, src.shape[3])
    return dgrad(dfm, c, residual)


def conv_backward(lib, c, srcs, g, need, cout, need_src, residual=None, nchw=False):
    """Backward of the FoldedConv ``c`` over the NHWC sources ``srcs`` from its output gradient ``g`` (NHWC bf16): [f | m]
    recomputed, the 6 parameters' gradients (_param_grads with their flags ``need`` and real channel count ``cout``), then the
    input gradient of each source whose ``need_src`` flag is set (input_grad, ``residual`` added in a 3x3 conv's rounding), NCHW
    f32 with ``nchw``, else NHWC bf16; None for the others.  Returns (parameter gradients, input gradients)."""
    fm = recompute_fm(lib, srcs, c)
    dfm = torch.empty_like(fm)
    grads = _param_grads(lib, g, fm, c, dfm, srcs, need, cout)
    del fm                                                                 # the input gradient reads [df | dm] only
    dxs, c0 = [], 0
    for s, n in zip(srcs, need_src):
        dx = input_grad(dfm, c, s, c0, residual) if n else None
        dxs.append(ops.nhwc_to_nchw(dx.contiguous()) if nchw and n else dx)
        c0 += s.shape[3]
    return grads, dxs


def _check_cuda(x):
    if not x.is_cuda:
        raise RuntimeError("read_b200: train_precision='bf16' runs the gated 3x3 convs on the H100 kernels and needs CUDA tensors")
    L.require_device(x.device.index)


class ConvChainFn(torch.autograd.Function):
    """The gated convs ``mods`` in turn over NCHW f32 tensors.  ``tensors`` = the ``n_src`` sources, a residual slot (None, or a
    tensor the output's shape that a one-conv call adds) and per conv its 6 parameters (stack_params).  Conv 0 reads the sources
    (a 1x1 conv several as a virtual concat), conv i > 0 the output of conv i - 1.  More than one conv is a chain of ResBlocks:
    the second conv of each pair adds the pair's input.  Each conv runs at padded_channels of its C.  ``per_item``: a train-mode
    norm normalises each batch item with its own statistics."""

    @staticmethod
    def forward(ctx, mods, n_src, per_item, *tensors):
        xs, residual, params = tensors[:n_src], tensors[n_src], tensors[n_src + 1:]
        _check_cuda(xs[0])
        lib = L.load()
        nhwc = lambda t: ops.nchw_to_nhwc(t.detach().float().contiguous(), True)
        srcs = [nhwc(x) for x in xs]
        res = None if residual is None else nhwc(residual)
        items = xs[0].shape[0] if per_item else None
        # every conv's filters packed before the first launch
        convs = [FoldedConv(m, *params[6 * i: 6 * i + 6], cout=padded_channels(params[6 * i].shape[0]),
                            srcs=srcs if i == 0 else None, items=items) for i, m in enumerate(mods)]
        ins = [srcs]                                                       # the input of each conv, then the output
        for i, c in enumerate(convs):
            d = _desc(ins[i], c.C, c.k, c.stride)
            y = torch.empty((d.B, d.Hout, d.Wout, c.C), dtype=torch.bfloat16, device=srcs[0].device)
            conv_forward(lib, ins[i], c, y, residual=ins[i - 1][0] if len(convs) > 1 and i % 2 else res)
            ins.append([y])
        ctx.convs, ctx.conv, ctx.n_src = convs, convs[-1], n_src     # ctx.conv: the conv whose output the call returns
        # the parameters are saved too: the folded / packed copies in ctx.convs alias or derive from them, and saving them makes
        # autograd raise if one is modified in place between forward and backward
        ctx.save_for_backward(*(t for ts in ins[:-1] for t in ts), *params)
        y, cout = ops.nhwc_to_nchw(ins[-1][0]), params[-6].shape[0]
        return y if cout == convs[-1].C else y[:, :cout].contiguous()

    @staticmethod
    def backward(ctx, gout):
        lib, convs, n_src, need = L.load(), ctx.convs, ctx.n_src, ctx.needs_input_grad
        n_in = n_src + len(convs) - 1
        saved = ctx.saved_tensors
        ins, params = [saved[:n_src]] + [saved[i:i + 1] for i in range(n_src, n_in)], saved[n_in:]
        g = g_block = _out_grad(gout, ctx.conv.C)                           # the gradient of the output, NHWC bf16
        grads, chain = [None] * len(params), len(convs) > 1
        for i in reversed(range(len(convs))):
            if chain and i % 2 == 1:
                g_block = g                                                # the gradient of this ResBlock's output
            p = 4 + n_src + 6 * i                                          # needs_input_grad of the conv's 6 parameters
            # the first conv of a ResBlock adds the gradient that reaches its input through the skip
            grads[6 * i: 6 * i + 6], dxs = conv_backward(lib, convs[i], ins[i], g, need[p: p + 6], params[6 * i].shape[0],
                                                         need[3: 3 + n_src] if i == 0 else [True],
                                                         g_block if chain and i % 2 == 0 else None, nchw=i == 0)
            g = dxs[0]
        return (None, None, None, *dxs, gout if need[3 + n_src] else None, *grads)


def _stack_names(net, prefix):
    return [f"{prefix}.layers.{i}.main.{j}" for i in range(net.num_res) for j in (0, 1)]


def stack_convs(net, prefix):
    """The 8 GatedConvs of the stack ``prefix`` (e.g. 'Encoder.0') in forward order."""
    return [net.get_submodule(n) for n in _stack_names(net, prefix)]


def res_stack(net, prefix, x, batch_stats=False, per_item=False):
    """bf16 forward of one EBlock / DBlock of ``net`` on the wgmma kernels, differentiable (stack_forward)."""
    return stack_forward(stack_convs(net, prefix), x, batch_stats=batch_stats, names=_stack_names(net, prefix),
                         per_item=per_item)


def stack_params(mods):
    """ConvChainFn's parameter list for the GatedConvs ``mods``: per conv (conv_f.weight, conv_f.bias, conv_m.weight,
    conv_m.bias, norm.weight, norm.bias)."""
    params = []
    for m in mods:
        b = m.block
        params += [b['conv_f'].weight, b['conv_f'].bias, b['conv_m'].weight, b['conv_m'].bias, b['norm'].weight, b['norm'].bias]
    return params


def _label(mod, name):
    return name or f"GatedConv(k={mod.k}, stride={mod.stride})"


def check_norms(mods, batch_stats, pixels, names=None, per_item=False):
    """Without ``batch_stats`` every norm must be in eval mode (RuntimeError).  With it, a train-mode norm must be one the batch
    statistics kernels implement (momentum set, running statistics tracked, affine) and the conv must have at least 2 output
    pixels (``pixels`` = B * H_out * W_out, or H_out * W_out per item with ``per_item``; torch raises for 1 too); otherwise a
    ValueError names the layer."""
    for i, m in enumerate(mods):
        n = m.block['norm']
        if not n.training:
            continue
        if not batch_stats:
            raise RuntimeError("read_b200: train_precision='bf16' folds BatchNorm with its running statistics; put the net in "
                               "eval() mode (the reference trains with eval-mode BatchNorm)")
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
    return ConvChainFn.apply(list(mods), 1, per_item, x, None, *stack_params(mods))


def gated_conv(mod, x, residual=None, batch_stats=False, name=None, per_item=False):
    """bf16 forward of the gated 3x3 stride-1 conv ``mod`` (a GatedConv) on the wgmma kernels, plus ``residual`` (NCHW, the
    output's shape) when given, differentiable.  A conv with C < 16 (the RGB output conv) runs padded to C = 16 and takes no
    residual.  ``batch_stats``: a train-mode norm normalises with batch statistics (else it raises), each batch item with its own
    with ``per_item``; ``name`` labels the layer in errors."""
    if mod.k != 3 or mod.stride != 1:
        raise ValueError(f"read_b200: gated_conv runs 3x3 stride-1 convs only (got k={mod.k}, stride={mod.stride})")
    check_norms([mod], batch_stats, (1 if per_item else x.shape[0]) * x.shape[2] * x.shape[3], [name], per_item)
    cout = mod.block['conv_f'].weight.shape[0]
    if residual is not None and padded_channels(cout) != cout:
        raise ValueError("read_b200: a residual needs C >= 16")
    return ConvChainFn.apply([mod], 1, per_item, x, residual, *stack_params([mod]))


GEOMETRIES = ((1, 1), (3, 2), (4, 2))        # (k, stride) of the convs gated_conv_srcs runs


def gated_conv_srcs(mod, xs, name=None, batch_stats=False, per_item=False):
    """bf16 forward of the gated 1x1 or stride-2 conv ``mod`` (a GatedConv) over the NCHW tensors ``xs`` on the wgmma kernels,
    differentiable.  A 1x1 conv reads several sources as one concat (each a multiple of 32 channels); a stride-2 conv takes one
    source of even height and width.  A conv whose C is not 16, 32, 64 or a multiple of 64 runs padded (padded_channels).
    ``name`` labels the layer in errors.  ``batch_stats``: a train-mode norm normalises with batch statistics (else it raises),
    each batch item with its own with ``per_item``."""
    label = _label(mod, name)
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
    return ConvChainFn.apply([mod], len(xs), per_item, *xs, None, *stack_params([mod]))
