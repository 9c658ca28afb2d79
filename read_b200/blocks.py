"""bf16 training of the gated 3x3 stride-1 convs (READ/models/unet.py:22-53) on the wgmma kernels.

``UNet.train_precision = 'bf16'`` sends 78 of the net's 99 convs here; the other 21 (the 1x1 and stride-2 convs), the
interpolations, concats and FAM products / sums stay on torch operators in the same autograd graph.
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


def _launch(lib, src, cout, w_tc, par, elu, out_mode, out, residual=None):
    """One 3x3 stride-1 launch of the TMA wgmma kernel over the NHWC bf16 tensor ``src``; par = (bias_f, bias_m, scale, shift)."""
    B, H, W, cin = src.shape
    d = L.ReadConvDesc()
    d.act_dtype, d.n_src = L.ACT_BF16, 1
    d.src[0].ptr = src.data_ptr()
    d.src[0].C, d.src[0].H, d.src[0].W = cin, H, W
    d.src[0].mode, d.src[0].factor = L.SRC_IDENTITY, 1
    d.B, d.Hin, d.Win, d.Cin = B, H, W, cin
    d.Hout, d.Wout, d.Cout = H, W, cout
    d.k, d.stride, d.pad, d.elu = 3, 1, 1, int(elu)
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
    scale / shift (the RGB output conv, C = 3, runs as C = 16): the padded channels compute 0 and get 0 gradients."""

    def __init__(self, mod, wf, bf, wm, bm, gamma, beta, cout=None):
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
        self.w_tc = torch.empty(lib.read_tc_weight_elems(C, cin, 3), dtype=torch.bfloat16, device=wf.device)
        L.check(lib.read_pack_weights_tc(self.wf.data_ptr(), self.wm.data_ptr(), C, cin, 3, self.w_tc.data_ptr(), st))
        self.w_dgrad = None                  # an 8-channel input's gradient kernel reads wf / wm itself
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
