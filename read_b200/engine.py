"""Refinement-net engine: lowers UNet.forward (READ/models/unet.py:202-285) to a static list of fused
gated-conv launches over NHWC activations, optionally replayed as one CUDA graph.

Every BasicConv (unet.py:22-53) is ONE kernel: conv_f + conv_m + bias + ELU + sigmoid gate + eval-BN affine,
with the graph glue folded in: torch.cat -> virtual concat, F.interpolate / nn.Upsample -> resampling operand
loader, ResBlock / FAM skip -> residual add in the epilogue, FAM product -> second epilogue output.
"""
import ctypes

import os

import torch

from . import _lib as L

_MODE = {"id": L.SRC_IDENTITY, "down": L.SRC_NEAREST_DOWN, "up": L.SRC_NEAREST_UP, "bil4": L.SRC_BILINEAR_UP4}


class _Layer:
    __slots__ = ("name", "plan", "impl", "keep", "flops", "k", "stride", "kind", "cin", "cout", "side")


class UNetEngine:
    """Static-shape executor.  ``precision``: 'bf16' (wgmma tensor-core kernels where supported) or 'fp32'
    (CUDA-core parity mode).  ``conv_impl``: 'auto' (tensor cores everywhere they apply) | 'tma_only' (TMA-fed wgmma kernel
    for the stride-1 layers, CUDA cores for the rest) | 'generic' (CUDA-core kernel everywhere)."""

    def __init__(self, state_dict, B, H, W, device, precision="bf16", conv_impl="auto", use_graph=True,
                 base=32, num_res=4):
        L.require_device(torch.device(device).index)
        if H % 16 or W % 16:
            # READ/gl/nn.py:107-109 asserts the same: the 4x4/s2 + x4-bilinear decoder needs it
            raise RuntimeError(f"set width {16 * (W // 16)} / height {16 * (H // 16)}: sizes must be multiples of 16")
        assert precision in ("bf16", "fp32") and conv_impl in ("auto", "generic", "tma_only")
        self.lib = L.load()
        self.B, self.H, self.W = B, H, W
        self.device = torch.device(device)
        self.bf16 = precision == "bf16"
        self.adt = torch.bfloat16 if self.bf16 else torch.float32
        self.act_code = L.ACT_BF16 if self.bf16 else L.ACT_F32
        self.conv_impl = conv_impl
        self.base, self.num_res = base, num_res
        self.sd = {k: v.detach().to(self.device, torch.float32).contiguous() for k, v in state_dict.items()
                   if v.dtype.is_floating_point}
        self.layers = []         # the 99 gated convs
        self.ops = []            # launch order: convs + auxiliary kernels (bilinear upsamples in bf16 mode)
        self._keep = []          # tensors the plans point into
        self.use_graph = use_graph
        self.alternate_order = os.environ.get("READ_B200_ALT_ORDER", "1") != "0"
        # Side chain (SURVEY.md §8f "small-layer tail"; OFF by default, READ_B200_SIDE_CHAIN=1): the SCM blocks of the two coarsest
        # pyramid levels depend only on the net's inputs and are first consumed deep in the encoder, and each of their launches is a few
        # tiles per SM - mostly pipeline fill and drain.  With the option they run on a second stream on SIDE_CTAS SMs while the main
        # chain (the half-resolution SCM block, the first conv) runs on the rest; one event joins them before the first consumer; both
        # chains are captured into the same CUDA graph.  Off because the cross-stream graph edges cost the programmatic-dependent-
        # launch overlap of ~10 launches and the main chain loses more on its smaller grids than the side chain hides (the whole-net
        # graph replay was slower with the option on; not re-measured on H100).  Output is identical either way.
        self.side_chain = os.environ.get("READ_B200_SIDE_CHAIN", "0") == "1" and type(self) is UNetEngine
        self._side_stream = None
        self.graph = None
        with torch.cuda.device(self.device):
            self._build()

    # ------------------------------------------------------------------ weights
    def _params(self, prefix, cin, cout, k):
        sd = self.sd
        wf, wm = sd[prefix + ".block.conv_f.weight"], sd[prefix + ".block.conv_m.weight"]
        assert tuple(wf.shape) == (cout, cin, k, k), (prefix, tuple(wf.shape), (cout, cin, k, k))
        bf, bm = sd[prefix + ".block.conv_f.bias"], sd[prefix + ".block.conv_m.bias"]
        n = prefix + ".block.norm."
        scale = (sd[n + "weight"] / torch.sqrt(sd[n + "running_var"] + 1e-5)).contiguous()   # eval BN, eps 1e-5
        shift = (sd[n + "bias"] - sd[n + "running_mean"] * scale).contiguous()
        return wf, wm, bf, bm, scale, shift

    # ------------------------------------------------------------------ one fused gated conv
    def _conv(self, prefix, srcs, cout, k, stride, elu, residual=None, out2_mul=None, final=False,
              raw=False, addin=None, cin_slice=None, name=None):
        """srcs: list of (tensor [B,h,w,c], mode, factor).  Returns out (and out2 if out2_mul).
        ``raw``: store the pre-activation accumulators [f | m] (2*cout channels) instead of the gated output;
        ``addin``: RAW tensor of the next-coarser resolution added (nearest x2) before the activation;
        ``cin_slice`` = (c0, c1): this launch covers input channels [c0, c1) of the layer's weights (one term of a 1x1 conv
        over a multi-resolution concat, see ``_aff``)."""
        lib = self.lib
        self._before_conv(srcs, k, stride, residual, out2_mul, addin)
        d = L.ReadConvDesc()
        d.act_dtype = self.act_code
        d.n_src = len(srcs)
        cin = 0
        hin = win = None
        for i, (t, mode, f) in enumerate(srcs):
            _, h, w, c = t.shape
            d.src[i].ptr = t.data_ptr()
            d.src[i].C, d.src[i].H, d.src[i].W = c, h, w
            d.src[i].mode, d.src[i].factor = _MODE[mode], f
            eh, ew = {"id": (h, w), "down": (h // f, w // f), "up": (h * f, w * f), "bil4": (h * 4, w * 4)}[mode]
            if hin is None:
                hin, win = eh, ew
            assert (eh, ew) == (hin, win), (prefix, eh, ew, hin, win)
            cin += c
        pad = int((k - 1) / 2)                                   # unet.py:29
        hout = (hin + 2 * pad - k) // stride + 1
        wout = (win + 2 * pad - k) // stride + 1
        if cin_slice is None:
            wf, wm, bf, bm, scale, shift = self._params(prefix, cin, cout, k)
        else:
            c0, c1 = cin_slice
            assert c1 - c0 == cin, (prefix, cin_slice, cin)
            sdw = self.sd[prefix + ".block.conv_f.weight"]
            wf, wm, bf, bm, scale, shift = self._params(prefix, sdw.shape[1], cout, k)
            wf, wm = wf[:, c0:c1].contiguous(), wm[:, c0:c1].contiguous()
        d.B, d.Hin, d.Win, d.Cin = self.B, hin, win, cin
        d.Hout, d.Wout, d.Cout = hout, wout, cout
        d.k, d.stride, d.pad, d.elu = k, stride, pad, int(elu)
        d.bias_f, d.bias_m, d.bn_scale, d.bn_shift = bf.data_ptr(), bm.data_ptr(), scale.data_ptr(), shift.data_ptr()
        if final:
            out = torch.empty((self.B, cout, hout, wout), dtype=torch.float32, device=self.device)
            d.out_mode = L.OUT_NCHW_F32
        elif raw:
            out = torch.empty((self.B, hout, wout, 2 * cout), dtype=self.adt, device=self.device)
            d.out_mode = L.OUT_RAW_NHWC
        else:
            out = torch.empty((self.B, hout, wout, cout), dtype=self.adt, device=self.device)
            d.out_mode = L.OUT_NHWC
        d.out = out.data_ptr()
        out2 = None
        if residual is not None:
            assert tuple(residual.shape) == (self.B, hout, wout, cout)
            d.residual = residual.data_ptr()
        if out2_mul is not None:
            assert tuple(out2_mul.shape) == (self.B, hout, wout, cout)
            out2 = torch.empty_like(out)
            d.out2, d.out2_mul = out2.data_ptr(), out2_mul.data_ptr()
        if addin is not None:
            assert tuple(addin.shape) == (self.B, (hout + 1) // 2, (wout + 1) // 2, 2 * cout), (prefix, tuple(addin.shape))
            d.addin, d.addin_H, d.addin_W = addin.data_ptr(), addin.shape[1], addin.shape[2]
        keep = [wf, wm, bf, bm, scale, shift, out, out2, residual, out2_mul, addin] + [s[0] for s in srcs]

        kind = "generic"
        if raw or addin is not None:
            d.impl = L.CONV_TCGEN05          # validation: these only exist on the TMA-fed kernel
            assert self.bf16 and lib.read_conv_tc_supported(ctypes.byref(d)), prefix
            kind = "tma"
        elif self.bf16 and self.conv_impl != "generic":
            if lib.read_conv_tc_supported(ctypes.byref(d)):
                kind = "tma"
            elif self.conv_impl == "auto" and lib.read_conv_tcg_supported(ctypes.byref(d)):
                kind = "gather"
        stream = L.stream_ptr()
        if kind == "tma":
            wtc = torch.empty(lib.read_tc_weight_elems(cout, cin, k), dtype=torch.bfloat16, device=self.device)
            L.check(lib.read_pack_weights_tc_for(ctypes.byref(d), wf.data_ptr(), wm.data_ptr(), wtc.data_ptr(), stream))
            d.w_tc, d.impl = wtc.data_ptr(), L.CONV_TCGEN05
            keep.append(wtc)
        elif kind == "gather":
            wtc = torch.empty(lib.read_tcg_weight_elems(cout, cin, k), dtype=torch.bfloat16, device=self.device)
            L.check(lib.read_pack_weights_tcg(wf.data_ptr(), wm.data_ptr(), cout, cin, k, wtc.data_ptr(), stream))
            d.w_tc, d.impl = wtc.data_ptr(), L.CONV_TCGEN05_GATHER
            keep.append(wtc)
        else:
            npad = lib.read_generic_npad(cout)
            kpad = ((k * k * cin + 15) // 16) * 16
            wg = torch.empty(kpad * npad, dtype=torch.float32, device=self.device)
            L.check(lib.read_pack_weights_generic(wf.data_ptr(), wm.data_ptr(), cout, cin, k, wg.data_ptr(), stream))
            d.w_generic, d.impl = wg.data_ptr(), L.CONV_GENERIC
            keep.append(wg)
        plan = L.c_vp()
        L.check(lib.read_conv_plan_create(ctypes.byref(d), ctypes.byref(plan)))
        if self.alternate_order and (len(self.layers) & 1):
            # consecutive launches walk the image in opposite directions: a layer starts on the tiles its producer wrote last,
            # which are the ones still in L2 (every activation tensor of the two finest levels is larger than half the L2)
            L.check(lib.read_conv_plan_set_tile_order(plan, 1))
        ly = _Layer()
        ly.name, ly.plan, ly.impl, ly.keep = (name or prefix), plan, lib.read_conv_plan_impl(plan), keep
        ly.flops = 2 * 2 * self.B * hout * wout * cout * cin * k * k
        ly.k, ly.stride, ly.kind = k, stride, "conv"
        ly.cin, ly.cout = cin, cout
        ly.side = False
        self.layers.append(ly)
        self.ops.append(ly)
        self._after_conv(srcs, k, stride, out, out2, residual, out2_mul, addin, final)
        return (out, out2) if out2_mul is not None else out

    # hooks of the strip-parallel engine (StripEngine): halo validity tracking around every conv; no-ops here
    def _before_conv(self, srcs, k, stride, residual, out2_mul, addin):
        pass

    def _after_conv(self, srcs, k, stride, out, out2, residual, out2_mul, addin, final):
        pass

    def _merge_src(self, t):
        """Decoder skip merge input: nn.Upsample(x4, bilinear) of ``t`` (unet.py:260,268,276).  In bf16 mode the upsample is a
        separate bandwidth-bound kernel so that the 1x1 merge conv gathers plain sources with cp.async; in fp32 parity mode
        it is fused into the conv's operand loader."""
        if not self.bf16 or self.conv_impl == "generic":
            return (t, "bil4", 4)
        B, h, w, c = t.shape
        out = torch.empty((B, 4 * h, 4 * w, c), dtype=self.adt, device=self.device)
        op = _Layer()
        op.name, op.plan, op.impl, op.flops, op.k, op.stride, op.kind = f"upsample4({h}x{w}x{c})", None, -1, 0, 0, 0, "upsample"
        op.keep = [t, out, (t.data_ptr(), B, h, w, c, out.data_ptr())]
        self.ops.append(op)
        return (out, "id", 1)

    # ------------------------------------------------------------------ blocks (unet.py:11-117)
    def _res(self, prefix, x, c):
        t = self._conv(prefix + ".main.0", [(x, "id", 1)], c, 3, 1, True)
        return self._conv(prefix + ".main.1", [(t, "id", 1)], c, 3, 1, False, residual=x)

    def _block(self, prefix, x, c):
        for i in range(self.num_res):
            x = self._res(f"{prefix}.layers.{i}", x, c)
        return x

    def _scm(self, prefix, x, c):
        t = self._conv(prefix + ".main.0", [(x, "id", 1)], c // 4, 3, 1, True)
        t = self._conv(prefix + ".main.1", [(t, "id", 1)], c // 2, 1, 1, True)
        t = self._conv(prefix + ".main.2", [(t, "id", 1)], c // 2, 3, 1, True)
        t = self._conv(prefix + ".main.3", [(t, "id", 1)], c - 8, 1, 1, True)
        return self._conv(prefix + ".conv", [(x, "id", 1), (t, "id", 1)], c, 1, 1, False)   # cat[x, main(x)]

    def _down_fam(self, fe, fam, x, z_scm, c):
        """feat_extract[fe] (3x3 s2, ELU) followed by FAM: z + merge(z * z_scm)  (unet.py:225-234)."""
        z, zz = self._conv(f"feat_extract.{fe}", [(x, "id", 1)], c, 3, 2, True, out2_mul=z_scm)
        return self._conv(f"{fam}.merge", [(zz, "id", 1)], c, 3, 1, False, residual=z)

    def _aff(self, idx, srcs, c):
        """AFF head (unet.py:79-89): BC1x1_elu(cat of the four scales) then BC3x3.  On the tensor-core path the 1x1 conv over
        the concat is split by linearity: a 1x1 conv commutes with nearest upsampling, so every source COARSER than the
        output is convolved at its own resolution into a RAW [f|m] tensor that is added (nearest x2, coarse to fine) to the
        next finer term; the sources at or above the output resolution are TMA sources (identity / traversal-stride) of
        the final launch.  The reference order cat[res1, res2, res3, z] fixes the weight column ranges."""
        prefix = f"AFFs.{idx}.conv.0"
        # the split pays for the full-resolution head (8x fewer MACs there); at half resolution the saving does not cover the extra launches
        chain_ok = self.bf16 and self.conv_impl == "auto" and c == self.base
        if chain_ok:
            coarse = [(i, t, f) for i, (t, mode, f) in enumerate(srcs) if mode == "up"]
            fine = [(i, sv) for i, sv in enumerate(srcs) if sv[1] != "up"]
            offs = [0]
            for t, _, _ in srcs:
                offs.append(offs[-1] + t.shape[3])
            chain_ok = len(coarse) >= 1 and all(cf == 2 ** (k + 1) for k, (_, _, cf) in enumerate(coarse)) \
                and all(t.shape[3] % 32 == 0 for t, _, _ in srcs)
        if not chain_ok:
            a = self._conv(prefix, srcs, c, 1, 1, True)
            return self._conv(f"AFFs.{idx}.conv.1", [(a, "id", 1)], c, 3, 1, False)
        partial = None
        for i, t, f in reversed(coarse):                     # coarsest first
            partial = self._conv(prefix, [(t, "id", 1)], c, 1, 1, False, raw=True, addin=partial,
                                 cin_slice=(offs[i], offs[i + 1]), name=f"{prefix}[raw 1/{f} term]")
        i0, i1 = fine[0][0], fine[-1][0]
        a = self._conv(prefix, [sv for _, sv in fine], c, 1, 1, True, addin=partial, cin_slice=(offs[i0], offs[i1 + 1]))
        return self._conv(f"AFFs.{idx}.conv.1", [(a, "id", 1)], c, 3, 1, False)

    def _build(self):
        self.inputs = self._make_inputs()
        self.output = self._build_graph(self.inputs)
        if getattr(self, "_side_range", None) is not None:
            self.set_side_chain(True)           # also caps the guard launches that follow the side range
        self.flops = sum(l.flops for l in self.layers)
        torch.cuda.current_stream().synchronize()   # weight packing done before any capture

    def _make_inputs(self):
        return [torch.zeros((self.B, self.H >> l, self.W >> l, 8), dtype=self.adt, device=self.device) for l in range(4)]

    def _build_graph(self, inputs):
        """UNet.forward (READ/models/unet.py:202-285) as a sequence of fused gated-conv launches; returns the output tensor."""
        c = self.base
        x, x2, x4, x8 = inputs
        z2 = self._scm("SCM2", x2, 2 * c)
        n0 = len(self.ops)
        z4 = self._scm("SCM1", x4, 4 * c)
        z8 = self._scm("SCM0", x8, 8 * c)
        self._mark_side(n0, len(self.ops))
        x_ = self._conv("feat_extract.0", [(x, "id", 1)], c, 3, 1, True)
        res1 = self._block("Encoder.0", x_, c)
        z = self._down_fam(1, "FAM2", res1, z2, 2 * c)
        res2 = self._block("Encoder.1", z, 2 * c)
        z = self._down_fam(2, "FAM1", res2, z4, 4 * c)
        res3 = self._block("Encoder.2", z, 4 * c)
        z = self._down_fam(6, "FAM0", res3, z8, 8 * c)
        z = self._block("Encoder.3", z, 8 * c)
        # AFFs consume the pre-AFF res1..3 and the Encoder[3] output (unet.py:239-254)
        r1 = self._aff(0, [(res1, "id", 1), (res2, "up", 2), (res3, "up", 4), (z, "up", 8)], c)
        r2 = self._aff(1, [(res1, "down", 2), (res2, "id", 1), (res3, "up", 2), (z, "up", 4)], 2 * c)
        r3 = self._aff(2, [(res1, "down", 4), (res2, "down", 2), (res3, "id", 1), (z, "up", 2)], 4 * c)
        z = self._block("Decoder.0", z, 8 * c)
        t = self._conv("feat_extract.7", [(z, "id", 1)], 4 * c, 4, 2, True)
        z = self._conv("Convs.0", [self._merge_src(t), (r3, "id", 1)], 4 * c, 1, 1, True)
        z = self._block("Decoder.1", z, 4 * c)
        t = self._conv("feat_extract.3", [(z, "id", 1)], 2 * c, 4, 2, True)
        z = self._conv("Convs.1", [self._merge_src(t), (r2, "id", 1)], 2 * c, 1, 1, True)
        z = self._block("Decoder.2", z, 2 * c)
        t = self._conv("feat_extract.4", [(z, "id", 1)], c, 4, 2, True)
        z = self._conv("Convs.2", [self._merge_src(t), (r1, "id", 1)], c, 1, 1, True)
        z = self._block("Decoder.3", z, c)
        return self._conv("feat_extract.5", [(z, "id", 1)], 3, 3, 1, False, final=True)

    SIDE_CTAS = 24          # SMs of the side chain; the main-chain launches that overlap it use the rest

    def _mark_side(self, i0, i1):
        """ops[i0:i1] form the side chain; the main-chain ops before them (the half-resolution SCM block) and the first conv after
        them share the device with it and get the complementary grid."""
        if not (getattr(self, "side_chain", False) and self.bf16 and i1 > i0 and all(o.plan is not None for o in self.ops[i0:i1])):
            return
        n_sm = torch.cuda.get_device_properties(self.device).multi_processor_count
        if n_sm <= 2 * self.SIDE_CTAS:
            return
        for o in self.ops[i0:i1]:
            o.side = True
            L.check(self.lib.read_conv_plan_set_max_ctas(o.plan, self.SIDE_CTAS))
        for o in self.ops[:i0]:
            if o.plan is not None:
                L.check(self.lib.read_conv_plan_set_max_ctas(o.plan, n_sm - self.SIDE_CTAS))
        self._side_range = (i0, i1)
        self._side_guard = 1      # main-chain launches after the side range that keep the reduced grid (the side chain may still run)

    # ------------------------------------------------------------------ execution
    def _launch_all(self):
        stream = L.stream_ptr()
        rng = getattr(self, "_side_range", None)
        if rng is None:
            for op in self.ops:
                self.launch_op(op, stream)
            return
        i0, i1 = rng
        main = torch.cuda.current_stream()
        if self._side_stream is None:
            self._side_stream = torch.cuda.Stream(device=self.device)
        side = self._side_stream
        fork = torch.cuda.Event()
        fork.record(main)                      # the inputs were written on the main stream
        side.wait_event(fork)
        sptr = side.cuda_stream
        for op in self.ops[i0:i1]:             # enqueue the side chain first: its CTAs take their SMs before the main chain's
            self.launch_op(op, sptr)
        join = torch.cuda.Event()
        join.record(side)
        for op in self.ops[:i0]:
            self.launch_op(op, stream)
        joined = False
        for op in self.ops[i1:]:
            if not joined and self._reads_side_output(op):
                main.wait_event(join)
                joined = True
            self.launch_op(op, stream)
        if not joined:
            main.wait_event(join)

    def set_side_chain(self, on):
        """Switch the two-stream schedule off (every launch on the current stream with a full grid: what per-layer timing wants)
        or back on.  Drops a captured graph."""
        rng = getattr(self, "_side_range_saved", None) or getattr(self, "_side_range", None)
        if rng is None:
            return
        i0, i1 = rng
        n_sm = torch.cuda.get_device_properties(self.device).multi_processor_count
        for j, o in enumerate(self.ops[:i1 + self._side_guard]):
            if o.plan is not None:
                cap = 0 if not on else (self.SIDE_CTAS if i0 <= j < i1 else n_sm - self.SIDE_CTAS)
                L.check(self.lib.read_conv_plan_set_max_ctas(o.plan, cap))
        self._side_range_saved = rng
        self._side_range = rng if on else None
        self.graph = None

    def _reads_side_output(self, op):
        """True if ``op`` consumes a tensor produced by the side chain (its ``keep`` list holds every tensor it touches)."""
        i0, i1 = self._side_range
        outs = getattr(self, "_side_outs", None)
        if outs is None:
            outs = self._side_outs = {id(t) for o in self.ops[i0:i1] for t in o.keep[6:8] if torch.is_tensor(t)}
        return any(torch.is_tensor(t) and id(t) in outs for t in op.keep)

    def launch_op(self, op, stream=None):
        stream = L.stream_ptr() if stream is None else stream
        if op.plan is not None:
            L.check(self.lib.read_conv_plan_launch(op.plan, stream))
        elif op.kind == "upsample":
            src, B, h, w, c, dst = op.keep[2]
            L.check(self.lib.read_upsample_bilinear4(src, self.act_code, B, h, w, c, dst, stream))
        else:
            self._launch_aux(op, stream)

    def _launch_aux(self, op, stream):
        raise RuntimeError(f"unknown engine op {op.kind}")

    def run(self):
        """Run the net on whatever is in ``self.inputs``; result in ``self.output`` ([B,3,H,W] f32)."""
        if not self.use_graph:
            self._launch_all()
            return self.output
        if self.graph is None:
            self._launch_all()                               # warm-up outside capture
            torch.cuda.current_stream().synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._launch_all()
            self.graph = g
        self.graph.replay()
        return self.output

    def n_launches(self):
        return len(self.ops)

    def impl_histogram(self):
        names = {L.CONV_GENERIC: "generic", L.CONV_TCGEN05: "wgmma_tma", L.CONV_TCGEN05_GATHER: "wgmma_gather"}
        h = {"wgmma_tma": 0, "wgmma_gather": 0, "generic": 0}
        for ly in self.layers:
            h[names[ly.impl]] += 1
        return h

    def set_inputs_nchw(self, feats):
        """feats: 4 tensors [B,8,h_l,w_l] f32 cuda -> engine input buffers (NHWC act dtype)."""
        lib, stream = self.lib, L.stream_ptr()
        for l in range(4):
            f = feats[l]
            if not (f.is_cuda and f.dtype == torch.float32 and f.is_contiguous()):
                f = f.to(self.device, torch.float32).contiguous()
            assert tuple(f.shape) == (self.B, 8, self.H >> l, self.W >> l), (tuple(f.shape), l)
            L.check(lib.read_nchw_f32_to_nhwc(f.data_ptr(), self.B, 8, self.H >> l, self.W >> l, self.act_code,
                                              self.inputs[l].data_ptr(), stream))

    def __del__(self):
        try:
            for ly in self.layers:
                if ly.plan is not None:
                    self.lib.read_conv_plan_destroy(ly.plan)
        except Exception:
            pass


class StripEngine(UNetEngine):
    """Strip-parallel refinement net (SURVEY.md §8f rank 1): rank ``rank`` of ``world`` GPUs refines rows
    [rank * H / world, (rank + 1) * H / world) of ONE frame; see ``read_b200.strips`` for the halo bookkeeping and
    ``csrc/halo.cu`` for the exchange kernel (peer-mapped mailboxes over NVLink, no NCCL between the layers).

    ``self.inputs`` are the local crops (with halos) of the feature pyramid - fill them with ``set_inputs_from_full``;
    ``self.output_interior`` is this rank's [1,3,S,W] slice of the frame.  All ranks must call ``run()`` together."""

    def __init__(self, state_dict, H, W, device, rank, world, group=None, precision="bf16", use_graph=True):
        from . import strips
        assert precision == "bf16", "the strip engine runs the production (tensor-core) path"
        self.rank, self.world, self.group = rank, world, group
        self.H_full = H
        _, H_local, self.h_top, self.h_bot = strips.strip_rows(H, world, rank, 0)
        self.S = H // world
        self._strips = strips
        self._meta = {}           # id(tensor) -> [level, valid halo rows]
        self._exch = []           # [(tensor, level)] in op order
        super().__init__(state_dict, 1, H_local, W, device, precision=precision, conv_impl="auto", use_graph=use_graph)
        self._setup_mailbox()

    # ------------------------------------------------------------------ halo bookkeeping (build time)
    def _level_of(self, rows):
        l = 0
        while (self.H >> l) != rows:
            l += 1
            assert l <= 4, (rows, self.H)
        return l

    def _v(self, t):
        m = self._meta.get(id(t))
        if m is None:             # an engine input: a crop of true data, halo fully valid
            m = self._meta[id(t)] = [self._level_of(t.shape[1]), self._strips.halo_rows(self._level_of(t.shape[1]))]
        return m

    def _exchange(self, t):
        m = self._v(t)
        op = _Layer()
        op.name, op.plan, op.impl, op.flops, op.k, op.stride, op.kind = f"halo(l{m[0]}, {t.shape[3]}ch)", None, -1, 0, 0, 0, "halo"
        op.keep = [t, len(self._exch)]
        self._exch.append((t, m[0]))
        self.ops.append(op)
        m[1] = self._strips.halo_rows(m[0])

    def _before_conv(self, srcs, k, stride, residual, out2_mul, addin):
        if self.world == 1:
            return
        st = self._strips
        need = st.conv_need(k)
        for (t, mode, f) in srcs:
            m = self._v(t)
            l_in = m[0] if mode == "id" else (m[0] + {2: 1, 4: 2, 8: 3}[f] if mode == "down" else
                                              m[0] - ({2: 1, 4: 2, 8: 3}[f] if mode == "up" else 2))
            if st.src_validity(m[1], mode, f, st.halo_rows(l_in)) < need:
                self._exchange(t)
                assert st.src_validity(m[1], mode, f, st.halo_rows(l_in)) >= need

    def _after_conv(self, srcs, k, stride, out, out2, residual, out2_mul, addin, final):
        if self.world == 1:
            return
        st = self._strips
        v_in, l_in = None, None
        for (t, mode, f) in srcs:
            m = self._v(t)
            l_in = m[0] if mode == "id" else (m[0] + {2: 1, 4: 2, 8: 3}[f] if mode == "down" else
                                              m[0] - ({2: 1, 4: 2, 8: 3}[f] if mode == "up" else 2))
            ve = st.src_validity(m[1], mode, f, st.halo_rows(l_in))
            v_in = ve if v_in is None else min(v_in, ve)
        l_out = l_in + (1 if stride == 2 else 0)
        v = min(st.conv_out_validity(v_in, k, stride), st.halo_rows(l_out))
        if residual is not None:
            v = min(v, self._v(residual)[1])
        if addin is not None:                       # RAW tensor of the next-coarser level, nearest x2
            v = min(v, 2 * self._v(addin)[1])
        self._meta[id(out)] = [l_out, v]
        if out2 is not None:
            self._meta[id(out2)] = [l_out, min(v, self._v(out2_mul)[1])]

    def _merge_src(self, t):
        # bilinear x4 reads one source row beyond the strip for its first / last interior rows
        if self.world > 1 and self._v(t)[1] < 1:
            self._exchange(t)
        src = super()._merge_src(t)
        if self.world > 1 and src[1] == "id":       # the separate bilinear-x4 kernel wrote a new tensor
            m = self._v(t)
            self._meta[id(src[0])] = [m[0] - 2, self._strips.src_validity(m[1], "bil4", 4, self._strips.halo_rows(m[0] - 2))]
        return src

    def _build(self):
        if self.world > 1:
            op = _Layer()
            op.name, op.plan, op.impl, op.flops, op.k, op.stride, op.kind, op.keep = "epoch", None, -1, 0, 0, 0, "epoch", []
            self.ops.append(op)
        super()._build()
        self.output_interior = self.output[:, :, self.h_top:self.h_top + self.S]

    # ------------------------------------------------------------------ mailboxes (after the op list is known)
    def _setup_mailbox(self):
        import torch.distributed as dist
        self._mail = None
        if self.world == 1:
            return
        assert len(self._exch) >= 2, "the mailbox protocol needs at least two exchanges per frame (csrc/halo.cu)"
        lib = self.lib
        n = len(self._exch)
        esize = 2
        # layout (identical on every rank): [flags: n x 2 u32][counters: n u32][epoch u32] padded to 1 KB, then per exchange two slots
        head = ((n * 2 + n + 1) * 4 + 1023) // 1024 * 1024
        offs, o = [], head
        for (t, lvl) in self._exch:
            nbytes = self._strips.halo_rows(lvl) * t.shape[2] * t.shape[3] * esize
            assert nbytes % 16 == 0
            offs.append((o, o + ((nbytes + 255) // 256 * 256), nbytes))
            o += 2 * ((nbytes + 255) // 256 * 256)
        ptr = L.c_vp()
        handle = ctypes.create_string_buffer(64)
        with torch.cuda.device(self.device):
            L.check(lib.read_ipc_alloc(o, ctypes.byref(ptr), handle))
        self._mail = ptr.value
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle.raw), group=self.group)
        self._peers = {}
        for nb in (self.rank - 1, self.rank + 1):
            if 0 <= nb < self.world:
                pp = L.c_vp()
                with torch.cuda.device(self.device):
                    L.check(lib.read_ipc_open(handles[nb], ctypes.byref(pp)))
                self._peers[nb] = pp.value
        up, dn = self._peers.get(self.rank - 1), self._peers.get(self.rank + 1)
        self._epoch_ptr = self._mail + (n * 3) * 4
        self._descs = []
        for e, (t, lvl) in enumerate(self._exch):
            h = self._strips.halo_rows(lvl)
            row = t.shape[2] * t.shape[3] * esize
            Hl = t.shape[1]
            ht = h if self.rank > 0 else 0
            hb = h if self.rank < self.world - 1 else 0
            slot_up, slot_dn, nbytes = offs[e]           # slot written by the upper / the lower neighbour
            d = L.ReadHaloDesc()
            base = t.data_ptr()
            if up is not None:
                d.src_up = base + ht * row                               # my first interior rows -> the upper rank's "from below" slot
                d.peer_up_slot = up + slot_dn
                d.peer_up_flag = up + (e * 2 + 1) * 4
                d.slot_from_up = self._mail + slot_up
                d.flag_from_up = self._mail + (e * 2 + 0) * 4
                d.dst_top = base
            if dn is not None:
                d.src_dn = base + (Hl - hb - h) * row                    # my last interior rows -> the lower rank's "from above" slot
                d.peer_dn_slot = dn + slot_up
                d.peer_dn_flag = dn + (e * 2 + 0) * 4
                d.slot_from_dn = self._mail + slot_dn
                d.flag_from_dn = self._mail + (e * 2 + 1) * 4
                d.dst_bot = base + (Hl - hb) * row
            d.bytes = nbytes
            d.epoch = self._epoch_ptr
            d.cta_counter = self._mail + (n * 2 + e) * 4
            self._descs.append(d)
        dist.barrier(group=self.group)                # every mailbox is mapped before anyone pushes

    def _launch_aux(self, op, stream):
        if op.kind == "epoch":
            L.check(self.lib.read_epoch_bump(self._epoch_ptr, stream))
        elif op.kind == "halo":
            L.check(self.lib.read_halo_exchange(ctypes.byref(self._descs[op.keep[1]]), stream))
        else:
            raise RuntimeError(f"unknown engine op {op.kind}")

    def n_exchanges(self):
        return len(self._exch)

    def set_inputs_from_full(self, full_feats):
        """full_feats[l]: [1, H >> l, W >> l, 8] in the engine's activation dtype (the whole frame's feature pyramid) -> copy
        this rank's crop (strip + halos) of every level into the engine inputs."""
        for l in range(4):
            a, n, _, _ = self._strips.strip_rows(self.H_full, self.world, self.rank, l)
            self.inputs[l].copy_(full_feats[l][:, a:a + n])

    def __del__(self):
        try:
            for p in getattr(self, "_peers", {}).values():
                self.lib.read_ipc_close(p)
            if getattr(self, "_mail", None):
                self.lib.read_ipc_free(self._mail)
        except Exception:
            pass
        super().__del__()
