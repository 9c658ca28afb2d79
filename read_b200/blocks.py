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

BatchNorm is eval-mode (running statistics, as the reference trains: eval_in_train), folded into scale / shift like the inference
engine.  Filters are re-packed from the live fp32 parameters on every call.
"""
import ctypes

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


class FoldedConv:
    """One GatedConv's live parameters for this step: folded eval-mode BatchNorm and the bf16 filters of the forward conv (also
    used for the RAW recompute) and of the input gradient.  ``cout`` > the conv's C pads it with zero filters, biases and BatchNorm
    scale / shift (the RGB output conv, C = 3, runs as C = 16; SCM*.main.3, C = 56 / 120 / 248, as 64 / 128 / 256): the padded
    channels compute 0 and get 0 gradients.  A 1x1 or stride-2 conv (k in {1, 3, 4}, stride in {1, 2}) packs its forward filters
    for the launch over ``srcs`` (the NHWC sources, whose channel counts set a concat's K chunks); its input-gradient filters are
    packed in backward (dgrad_s2_filters, dgrad_1x1)."""

    def __init__(self, mod, wf, bf, wm, bm, gamma, beta, cout=None, srcs=None):
        lib, st = L.load(), L.stream_ptr()
        norm = mod.block['norm']
        cin = wf.shape[1]
        C = cout or wf.shape[0]
        pad = lambda t: _pad_rows(t.detach().float(), C).contiguous()
        self.C, self.elu = C, bool(mod.elu)
        self.wf, self.wm, self.bf, self.bm = pad(wf), pad(wm), pad(bf), pad(bm)
        inv = torch.rsqrt(norm.running_var.detach().float() + norm.eps)
        scale = gamma.detach().float() * inv
        self.mean, self.inv = pad(norm.running_mean), pad(inv)
        self.scale, self.shift = pad(scale), pad(beta.detach().float() - norm.running_mean.detach().float() * scale)
        self.k, self.stride = mod.k, mod.stride
        self.w_tc = torch.empty(lib.read_tc_weight_elems(C, cin, mod.k), dtype=torch.bfloat16, device=wf.device)
        self.w_dgrad = None                  # an 8-channel input's gradient kernel reads wf / wm itself
        if (mod.k, mod.stride) != (3, 1):
            L.check(lib.read_pack_weights_tc_for(ctypes.byref(_desc(srcs, C, mod.k, mod.stride)), self.wf.data_ptr(),
                                                 self.wm.data_ptr(), self.w_tc.data_ptr(), st))
            return
        L.check(lib.read_pack_weights_tc(self.wf.data_ptr(), self.wm.data_ptr(), C, cin, 3, self.w_tc.data_ptr(), st))
        if cin != 8:
            self.w_dgrad = torch.empty(lib.read_tc_weight_elems(cin // 2, 2 * C, 3), dtype=torch.bfloat16, device=wf.device)
            L.check(lib.read_pack_weights_tc_dgrad(self.wf.data_ptr(), self.wm.data_ptr(), C, cin, self.w_dgrad.data_ptr(), st))

    @property
    def par(self):
        return (self.bf, self.bm, self.scale, self.shift)


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
        _check_cuda(x)
        lib = L.load()
        convs = [FoldedConv(m, *params[6 * i: 6 * i + 6]) for i, m in enumerate(mods)]   # packed before the first conv launch
        t = ops.nchw_to_nhwc(x.detach().float().contiguous(), True)
        C = t.shape[3]
        saved = []
        for r in range(0, len(convs), 2):
            h = torch.empty_like(t)
            _launch(lib, t, C, convs[r].w_tc, convs[r].par, convs[r].elu, L.OUT_NHWC, h)
            y = torch.empty_like(t)
            _launch(lib, h, C, convs[r + 1].w_tc, convs[r + 1].par, convs[r + 1].elu, L.OUT_NHWC, y, residual=t)
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
            red = torch.zeros((4, C), dtype=torch.float32, device=dev)   # dbias_f, dbias_m, dgamma, dbeta
            L.check(lib.read_gate_backward(g.data_ptr(), fm.data_ptr(), B * H * W, C, int(c.elu), c.bf.data_ptr(), c.bm.data_ptr(),
                                           c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), dfm.data_ptr(),
                                           red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st))
            dwf = dwm = None
            if ctx.needs_input_grad[2 + 6 * i] or ctx.needs_input_grad[4 + 6 * i]:    # not for a frozen net
                dwf, dwm = torch.zeros_like(c.wf), torch.zeros_like(c.wm)
                L.check(lib.read_conv3x3_wgrad(dfm.data_ptr(), x_in.data_ptr(), B, H, W, C, C, dwf.data_ptr(), dwm.data_ptr(), st))
            grads[6 * i: 6 * i + 6] = [dwf, red[0], dwm, red[1], red[2], red[3]]
            if i > 0 or ctx.needs_input_grad[0]:
                # the first conv of a ResBlock adds the gradient that reaches its input through the skip
                g = dgrad(dfm, c, residual=g_block if i % 2 == 0 else None)
        dx = ops.nhwc_to_nchw(g) if ctx.needs_input_grad[0] else None
        grads = [gr if ctx.needs_input_grad[2 + k] else None for k, gr in enumerate(grads)]
        return (dx, None, *grads)


def stack_convs(net, prefix):
    """The 8 GatedConvs of the stack ``prefix`` (e.g. 'Encoder.0') in forward order."""
    return [net.get_submodule(f"{prefix}.layers.{i}.main.{j}") for i in range(net.num_res) for j in (0, 1)]


def res_stack(net, prefix, x):
    """bf16 forward of one EBlock / DBlock of ``net`` on the wgmma kernels, differentiable through ResStackFn."""
    return stack_forward(stack_convs(net, prefix), x)


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


def stack_forward(mods, x):
    """The ResBlocks t -> t + mods[2r+1](mods[2r](t)) applied to x in turn, bf16 on the wgmma kernels."""
    _check_eval(mods)
    return ResStackFn.apply(x, list(mods), *stack_params(mods))


class GatedConvFn(torch.autograd.Function):
    """x (NCHW f32) -> mod(x) [+ residual] for one gated 3x3 stride-1 conv ``mod``; ``params`` = (conv_f.weight, conv_f.bias,
    conv_m.weight, conv_m.bias, norm.weight, norm.bias).  A conv with C < 16 (the RGB output conv) runs padded to C = 16."""

    @staticmethod
    def forward(ctx, x, residual, mod, *params):
        _check_cuda(x)
        lib = L.load()
        cout = params[0].shape[0]
        conv = FoldedConv(mod, *params, cout=max(cout, 16))
        if residual is not None and conv.C != cout:
            raise ValueError("read_b200: a residual needs C >= 16")
        t = ops.nchw_to_nhwc(x.detach().float().contiguous(), True)
        B, H, W, _ = t.shape
        r = None if residual is None else ops.nchw_to_nhwc(residual.detach().float().contiguous(), True)
        y = torch.empty((B, H, W, conv.C), dtype=torch.bfloat16, device=t.device)
        _launch(lib, t, conv.C, conv.w_tc, conv.par, conv.elu, L.OUT_NHWC, y, residual=r)
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
        red = torch.zeros((4, C), dtype=torch.float32, device=dev)       # dbias_f, dbias_m, dgamma, dbeta
        L.check(lib.read_gate_backward(g.data_ptr(), fm.data_ptr(), B * H * W, C, int(c.elu), c.bf.data_ptr(), c.bm.data_ptr(),
                                       c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), dfm.data_ptr(),
                                       red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st))
        dwf = dwm = None
        if need[3] or need[5]:                                            # not for a frozen net
            dwf, dwm = torch.zeros_like(c.wf), torch.zeros_like(c.wm)
            L.check(lib.read_conv3x3_wgrad(dfm.data_ptr(), x_in.data_ptr(), B, H, W, C, x_in.shape[3], dwf.data_ptr(),
                                           dwm.data_ptr(), st))
        dx = ops.nhwc_to_nchw(dgrad(dfm, c)) if need[0] else None
        grads = [dwf, red[0], dwm, red[1], red[2], red[3]]
        grads = [gr[:cout] if gr is not None and need[3 + k] else None for k, gr in enumerate(grads)]
        return (dx, gout if need[1] else None, None, *grads)


def gated_conv(mod, x, residual=None):
    """bf16 forward of the gated 3x3 stride-1 conv ``mod`` (a GatedConv) on the wgmma kernels, plus ``residual`` (NCHW, the
    output's shape) when given, differentiable through GatedConvFn."""
    if mod.k != 3 or mod.stride != 1:
        raise ValueError(f"read_b200: gated_conv runs 3x3 stride-1 convs only (got k={mod.k}, stride={mod.stride})")
    _check_eval([mod])
    return GatedConvFn.apply(x, residual, mod, *stack_params([mod]))


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
    w = torch.empty(lib.read_tc_weight_elems(64, d.Cin, 1), dtype=torch.bfloat16, device=srcs[0].device)
    d64 = _desc(srcs, 64, 1, 1)
    for b in range(c.C // 64):
        L.check(lib.read_pack_weights_tc_for(ctypes.byref(d64), c.wf[64 * b: 64 * b + 64].data_ptr(),
                                             c.wm[64 * b: 64 * b + 64].data_ptr(), w.data_ptr(), L.stream_ptr()))
        out = torch.empty((B, H, W, 128), dtype=torch.bfloat16, device=srcs[0].device)
        _launch(lib, srcs, 64, w, (zeros,) * 4, False, L.OUT_RAW_NHWC, out, k=1)
        blocks_.append(out)
    return torch.cat(blocks_, -1)


def dgrad_s2_filters(c):
    """The flipped-by-phase filters [k*k][Cin][2C] (bf16) of the stride-2 input-gradient kernel for the FoldedConv ``c``."""
    lib = L.load()
    cin = c.wf.shape[1]
    w = torch.empty((c.k * c.k, cin, 2 * c.C), dtype=torch.bfloat16, device=c.wf.device)
    L.check(lib.read_pack_weights_dgrad_s2(c.wf.data_ptr(), c.wm.data_ptr(), c.C, cin, c.k, w.data_ptr(), L.stream_ptr()))
    return w


def dgrad_1x1(dfm, c, c0, cs):
    """Input gradient [B,H,W,cs] (bf16) of input channels c0 .. c0 + cs - 1 of the 1x1 FoldedConv ``c``: RAW 1x1 plans over
    [df | dm] with transposed filters, one per 128 channels (the plans' widest N tile); 16 channels run padded to 32."""
    lib, st = L.load(), L.stream_ptr()
    B, H, W, _ = dfm.shape
    cin = c.wf.shape[1]
    parts = []
    for a in range(c0, c0 + cs, 128):
        cn = min(128, c0 + cs - a)
        n_out = max(cn, 32)
        w = torch.empty(lib.read_tc_weight_elems(n_out // 2, 2 * c.C, 1), dtype=torch.bfloat16, device=dfm.device)
        L.check(lib.read_pack_weights_tc_dgrad1x1(c.wf.data_ptr(), c.wm.data_ptr(), c.C, cin, a, cn, w.data_ptr(), st))
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
        xs, params = args[:n_src], args[n_src:]
        _check_cuda(xs[0])
        lib = L.load()
        cout = params[0].shape[0]
        ts = [ops.nchw_to_nhwc(x.detach().float().contiguous(), True) for x in xs]
        conv = FoldedConv(mod, *params, cout=padded_channels(cout), srcs=ts)
        d = _desc(ts, conv.C, mod.k, mod.stride)
        y = torch.empty((d.B, d.Hout, d.Wout, conv.C), dtype=torch.bfloat16, device=ts[0].device)
        _launch(lib, ts, conv.C, conv.w_tc, conv.par, conv.elu, L.OUT_NHWC, y, k=mod.k, stride=mod.stride)
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
        B, Hin, Win, _ = ts[0].shape
        gp = gout.float()
        if cout < C:
            gp = torch.cat([gp, gp.new_zeros((B, C - cout) + tuple(gp.shape[2:]))], 1)  # the padded channels' gradient is 0
        g = ops.nchw_to_nhwc(gp.contiguous(), True)
        Hout, Wout = g.shape[1], g.shape[2]
        fm = recompute_fm(lib, ts, c)
        dfm = torch.empty_like(fm)
        red = torch.zeros((4, C), dtype=torch.float32, device=dev)        # dbias_f, dbias_m, dgamma, dbeta
        L.check(lib.read_gate_backward(g.data_ptr(), fm.data_ptr(), B * Hout * Wout, C, int(c.elu), c.bf.data_ptr(),
                                       c.bm.data_ptr(), c.scale.data_ptr(), c.mean.data_ptr(), c.inv.data_ptr(), dfm.data_ptr(),
                                       red[0].data_ptr(), red[1].data_ptr(), red[2].data_ptr(), red[3].data_ptr(), st))
        del fm
        dwf = dwm = None
        if need[n_src] or need[n_src + 2]:                                 # not for a frozen net
            kk = (c.k, c.k)
            dws = [(torch.zeros((C, t.shape[3]) + kk, device=dev), torch.zeros((C, t.shape[3]) + kk, device=dev)) for t in ts]
            for t, (wf_s, wm_s) in zip(ts, dws):
                L.check(lib.read_conv_wgrad(dfm.data_ptr(), t.data_ptr(), B, Hin, Win, Hout, Wout, C, t.shape[3], c.k, c.stride,
                                            wf_s.data_ptr(), wm_s.data_ptr(), st))
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


def gated_conv_srcs(mod, xs, name=None):
    """bf16 forward of the gated 1x1 or stride-2 conv ``mod`` (a GatedConv) over the NCHW tensors ``xs`` on the wgmma kernels,
    differentiable through MultiSourceConvFn.  A 1x1 conv reads several sources as one concat (each a multiple of 32 channels);
    a stride-2 conv takes one source of even height and width.  ``name`` labels the layer in errors."""
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
    _check_eval([mod])
    return MultiSourceConvFn.apply(mod, len(xs), *xs, *stack_params([mod]))
