"""Exact checks of the forward gated-conv kernels at every tile, K-chunk, source and image edge (tests/fwd_exact_util.py states
the method), and of read_upsample_bilinear4.

* TMA-fed wgmma kernel (csrc/conv_tc.cu): every geometry it accepts; RAW outputs every bf16 element the round-to-nearest of the
  exact sum; gated outputs exact on the gate-pinned channels and bounded on the others; out2 exactly bf16(stored y * mul); each
  case also with one, two and three persistent CTAs and with the reversed tile order, which must give the same bits;
* gather wgmma kernel (csrc/conv_tc_gather.cu) and CUDA-core kernel (csrc/conv_generic.cu, bf16 and fp32 activations) likewise;
* a two-plan chain whose second plan reads the first's output, with programmatic dependent launch on and off;
* every layer class the engine plans at C3, for each conv_impl, appears among the exact cases.
Every output lies inside a guard band (bwd_exact_util.Guarded): a write past the image, the padded channels or the batch fails.
"""
import ctypes
import zlib

import pytest
import torch

import bwd_exact_util as U
import fwd_exact_util as X
from gpu_util import dev
from read_b200 import _lib as L

pytestmark = pytest.mark.gpu
WORST = {}
IMPL = {"tma": L.CONV_TCGEN05, "gather": L.CONV_TCGEN05_GATHER, "generic": L.CONV_GENERIC}
MODES = {"id": L.SRC_IDENTITY, "down": L.SRC_NEAREST_DOWN, "up": L.SRC_NEAREST_UP, "bil4": L.SRC_BILINEAR_UP4}


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _worst(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    print("\nworst so far: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


class Launch:
    """A case's device operands, packed weights and guard-banded outputs; ``run`` plans and launches it once."""

    def __init__(self, c, o):
        lib, d = L.load(), dev()
        self.c, self.lib = c, lib
        adt = torch.bfloat16 if c.act == "bf16" else torch.float32
        self.keep = []
        dsc = L.ReadConvDesc()
        dsc.act_dtype = L.ACT_BF16 if c.act == "bf16" else L.ACT_F32
        dsc.n_src = len(c.srcs)
        for i, (t, (C, m, f)) in enumerate(zip(o["srcs"], c.srcs)):
            td = t.to(d, adt).contiguous()
            self.keep.append(td)
            dsc.src[i].ptr, dsc.src[i].C, dsc.src[i].H, dsc.src[i].W = td.data_ptr(), C, t.shape[1], t.shape[2]
            dsc.src[i].mode, dsc.src[i].factor = MODES[m], f
        dsc.B, dsc.Hin, dsc.Win, dsc.Cin = c.B, c.H, c.W, c.cin
        dsc.Hout, dsc.Wout, dsc.Cout = c.hout, c.wout, c.cout
        dsc.k, dsc.stride, dsc.pad, dsc.elu = c.k, c.stride, c.pad, c.elu
        dv = [o[n].to(d).contiguous() for n in ("wf", "wm", "bf", "bm", "scale", "shift")]
        self.keep += dv
        dsc.bias_f, dsc.bias_m, dsc.bn_scale, dsc.bn_shift = (t.data_ptr() for t in dv[2:])
        dsc.out_mode = {"nhwc": L.OUT_NHWC, "raw": L.OUT_RAW_NHWC, "nchw": L.OUT_NCHW_F32}[c.out]
        dsc.impl = IMPL[c.impl]
        st = L.stream_ptr()
        if c.impl == "tma":
            w = torch.empty(lib.read_tc_weight_elems(c.cout, c.cin, c.k), dtype=torch.bfloat16, device=d)
            L.check(lib.read_pack_weights_tc_for(ctypes.byref(dsc), dv[0].data_ptr(), dv[1].data_ptr(), w.data_ptr(), st))
            dsc.w_tc = w.data_ptr()
        elif c.impl == "gather":
            w = torch.empty(lib.read_tcg_weight_elems(c.cout, c.cin, c.k), dtype=torch.bfloat16, device=d)
            L.check(lib.read_pack_weights_tcg(dv[0].data_ptr(), dv[1].data_ptr(), c.cout, c.cin, c.k, w.data_ptr(), st))
            dsc.w_tc = w.data_ptr()
        else:
            w = torch.empty(lib.read_generic_npad(c.cout) * ((c.k * c.k * c.cin + 15) // 16 * 16), dtype=torch.float32, device=d)
            L.check(lib.read_pack_weights_generic(dv[0].data_ptr(), dv[1].data_ptr(), c.cout, c.cin, c.k, w.data_ptr(), st))
            dsc.w_generic = w.data_ptr()
        self.keep.append(w)
        odt = torch.float32 if c.out == "nchw" else adt
        n = c.B * c.hout * c.wout * c.out_channels
        self.out = U.Guarded(n, odt, d)
        dsc.out = self.out.out.data_ptr()
        nhwc_ops = {}
        for name in ("res", "out2_mul", "addin", "mul"):
            if o.get(name) is not None:
                nhwc_ops[name] = o[name].to(d, adt).contiguous()
                self.keep.append(nhwc_ops[name])
        if c.residual:
            dsc.residual = nhwc_ops["res"].data_ptr()
        self.out2 = None
        if c.out2:
            self.out2 = U.Guarded(n, odt, d)
            dsc.out2, dsc.out2_mul = self.out2.out.data_ptr(), nhwc_ops["out2_mul"].data_ptr()
        if c.addin:
            dsc.addin, dsc.addin_H, dsc.addin_W = nhwc_ops["addin"].data_ptr(), o["addin"].shape[1], o["addin"].shape[2]
        if c.mul:
            dsc.mul = nhwc_ops["mul"].data_ptr()
        self.dsc = dsc

    def shape(self):
        c = self.c
        return (c.B, c.cout, c.hout, c.wout) if c.out == "nchw" else (c.B, c.hout, c.wout, c.out_channels)

    def run(self, max_ctas=0, reverse=False):
        """Launch once into freshly sentinel-filled outputs; returns (out, out2) on the host."""
        lib = self.lib
        for g in (self.out, self.out2):
            if g is not None:
                g.buf.view(g.view_dtype).fill_(g.sentinel)
                g.out.zero_()
        plan = L.c_vp()
        L.check(lib.read_conv_plan_create(ctypes.byref(self.dsc), ctypes.byref(plan)))
        try:
            assert lib.read_conv_plan_impl(plan) == IMPL[self.c.impl]
            L.check(lib.read_conv_plan_set_max_ctas(plan, max_ctas))
            L.check(lib.read_conv_plan_set_tile_order(plan, int(reverse)))
            L.check(lib.read_conv_plan_launch(plan, L.stream_ptr()))
            torch.cuda.synchronize()
        finally:
            lib.read_conv_plan_destroy(plan)
        what = f"{self.c.id} max_ctas={max_ctas} reverse={reverse}"
        self.out.check(what + " out")
        got = self.out.out.view(self.shape()).cpu()
        got2 = None
        if self.out2 is not None:
            self.out2.check(what + " out2")
            got2 = self.out2.out.view(self.shape()).cpu()
        return got, got2


# ------------------------------------------------------------------ the gate's saturation, per kernel
@pytest.fixture(scope="module")
def gate_pinned():
    """Per kernel: does sigmoid(64) come out exactly 1.0?  A final-layer plan (fp32 output, so nothing hides a rounding) with
    wf = wm = 0, bias_f = 1, bias_m = 64, scale = 1, shift = 0: every output is the gate itself."""
    sat = {}
    for impl in ("tma", "gather", "generic"):
        c = X.Case("gate self-check", impl, ((32, "id", 1),), 3, 3, 1, 1, 16, 8, out="nchw")
        o = X.operands(c, _gen("self-check", impl))
        o.update(wf=torch.zeros_like(o["wf"]), wm=torch.zeros_like(o["wm"]), bf=torch.ones(3), bm=torch.full((3,), 64.0),
                 scale=torch.ones(3), shift=torch.zeros(3))
        got, _ = Launch(c, o).run()
        vals = sorted({float(v) for v in got.unique()})
        sat[impl] = vals == [1.0]
        print(f"\n{impl}: sigmoid(64) -> {vals} ({'exactly 1: pinned channels checked for equality' if sat[impl] else 'not saturated: pinned channels bounded'})")
    return sat


# ------------------------------------------------------------------ the checks
def _nonrep_ok(want, what):
    frac = U.bf16_nonrepresentable_fraction(want)
    assert frac >= 0.1, f"{what}: only {frac:.2f} of the exact sums need rounding; the round-to-nearest check would be weak"


def _check(c, o, r, got, got2, sat, what):
    names = ["b", "c", "y", "x"] if c.out == "nchw" else ["b", "y", "x", "c"]
    if c.out == "raw":
        _nonrep_ok(r["raw"], what)
        U.assert_bf16_rn(got, r["raw"], what + " RAW", names)
        return
    got = got.double()
    exact = r["exact"] if sat else torch.zeros_like(r["exact"])
    if bool(exact.any()):
        U.assert_exact(got[exact], r["y_pin"][exact], what + " gate-pinned channels", ["element"])
    tau = X.TAU_ACC if c.impl == "generic" else X.TAU_FAST
    b = X.bound(c, o, r, tau)
    ordinary = ~exact
    fam = f"{c.impl}-{c.act}{'-nchw' if c.out == 'nchw' else ''}"
    worst = U.assert_bound(got[ordinary], r["y64"][ordinary], b[ordinary], 1.0, what + " ordinary channels", names=["element"])
    _worst(f"{fam} err/bound", worst)
    _worst(f"{fam} tau share", X.tau_share(got, r["y64"], c, o, r, tau))
    if c.out2:
        # out2 is bf16(stored y * mul) on every channel, and exact wherever y is
        mul = o["out2_mul"].double()
        U.assert_exact(got2, X._round(got * mul, r["dt"]), what + " out2 = stored y * mul", names)
        if bool(exact.any()):
            U.assert_exact(got2.double()[exact], r["o2_pin"][exact], what + " out2 of the pinned channels", ["element"])


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _run_case(c, gate_pinned):
    X.precondition(c)
    o = X.make(c, _gen(c))
    r = X.ref(c, o)
    ln = Launch(c, o)
    got, got2 = ln.run()
    _check(c, o, r, got, got2, gate_pinned[c.impl], c.id)
    if c.impl == "generic":
        return
    # persistence: one CTA walks every tile (every ring and barrier phase wraps), two and three CTAs, the reversed order
    variants = [(m, False) for m in X.MAX_CTAS] + ([(0, True), (2, True)] if c.impl == "tma" else [])
    for mc, rev in variants:
        g, g2 = ln.run(mc, rev)
        assert torch.equal(_bits(g), _bits(got)), f"{c.id}: max_ctas={mc} reverse={rev} differs from the full-grid launch"
        if g2 is not None:
            assert torch.equal(_bits(g2), _bits(got2)), f"{c.id}: out2 with max_ctas={mc} reverse={rev}"


@pytest.mark.parametrize("case", X.TMA_CASES, ids=lambda c: c.id)
def test_tma_forward_is_exact(case, gate_pinned):
    _run_case(case, gate_pinned)


@pytest.mark.parametrize("case", X.GATHER_CASES, ids=lambda c: c.id)
def test_gather_forward_is_exact(case, gate_pinned):
    _run_case(case, gate_pinned)


@pytest.mark.parametrize("case", X.GENERIC_CASES, ids=lambda c: c.id)
def test_generic_forward_is_exact(case, gate_pinned):
    _run_case(case, gate_pinned)


# ------------------------------------------------------------------ programmatic dependent launch between two plans
@pytest.mark.parametrize("pdl", [1, 0])
def test_pdl_chain_second_plan_reads_the_first_output(pdl):
    """RAW 3x3 32 -> 2x16 (plan 1), then RAW 3x3 over plan 1's output (plan 2), launched back to back on one stream: plan 2's
    output is exact against the float64 composition, so it read plan 1's finished output."""
    lib = L.load()
    B, H, W = 3, 64, 96
    g = _gen("pdl", pdl)
    c1 = X.Case("pdl 1", "tma", ((32, "id", 1),), 16, 3, 1, B, H, W, out="raw")
    x = U.int_tensor((B, H, W, 32), 4, g)
    w1 = [U.int_tensor((16, 32, 3, 3), 4, g) for _ in range(2)]
    w2 = [U.int_tensor((16, 32, 3, 3), 8, g) for _ in range(2)]
    zeros = torch.zeros(16)
    o1 = dict(srcs=[x], wf=w1[0], wm=w1[1], bf=zeros, bm=zeros, scale=zeros, shift=zeros)
    want1 = U.to_raw(torch.cat([torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), w.double(), padding=1)
                                for w in w1], 1).permute(0, 2, 3, 1))
    assert float(want1.abs().max()) * 9 * 32 * 8 < X.EXACT_LIMIT
    rn1 = want1.float().bfloat16()
    want2 = U.to_raw(torch.cat([torch.nn.functional.conv2d(rn1.double().permute(0, 3, 1, 2), w.double(), padding=1)
                                for w in w2], 1).permute(0, 2, 3, 1))
    l1 = Launch(c1, o1)
    o2 = dict(srcs=[torch.zeros(B, H, W, 32)], wf=w2[0], wm=w2[1], bf=zeros, bm=zeros, scale=zeros, shift=zeros)
    l2 = Launch(X.Case("pdl 2", "tma", ((32, "id", 1),), 16, 3, 1, B, H, W, out="raw"), o2)
    l2.dsc.src[0].ptr = l1.out.out.data_ptr()                     # plan 2 reads plan 1's output
    old = 1
    L.check(lib.read_set_option(b"tc_pdl", pdl))
    try:
        for gb in (l1.out, l2.out):
            gb.buf.view(gb.view_dtype).fill_(gb.sentinel)
            gb.out.zero_()
        plans = [L.c_vp(), L.c_vp()]
        for ln, p in zip((l1, l2), plans):
            L.check(lib.read_conv_plan_create(ctypes.byref(ln.dsc), ctypes.byref(p)))
        st = L.stream_ptr()
        for p in plans:
            L.check(lib.read_conv_plan_launch(p, st))
        torch.cuda.synchronize()
        for p in plans:
            lib.read_conv_plan_destroy(p)
    finally:
        L.check(lib.read_set_option(b"tc_pdl", old))
    l1.out.check("pdl plan 1")
    l2.out.check("pdl plan 2")
    U.assert_bf16_rn(l1.out.out.view(B, H, W, 32), want1, f"pdl={pdl} plan 1", ["b", "y", "x", "c"])
    U.assert_bf16_rn(l2.out.out.view(B, H, W, 32), want2, f"pdl={pdl} plan 2", ["b", "y", "x", "c"])


# ------------------------------------------------------------------ bilinear x4 upsample
@pytest.mark.parametrize("act", ["bf16", "f32"])
@pytest.mark.parametrize("C", X.BIL_CS)
def test_upsample_bilinear4_is_exact(C, act):
    """Integers |x| <= 3 blended with the dyadic x4 weights: every output an exact multiple of 1/64 below 3, equal to F.interpolate."""
    lib = L.load()
    dt = torch.bfloat16 if act == "bf16" else torch.float32
    for h in X.BIL_HW:
        for w in X.BIL_HW:
            x = U.int_tensor((2, h, w, C), X.A_BIL, _gen("bil", h, w, C, act))
            want = X.bilinear4(x.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
            out = U.Guarded(2 * 16 * h * w * C, dt, dev())
            xd = x.to(dev(), dt).contiguous()
            L.check(lib.read_upsample_bilinear4(xd.data_ptr(), L.ACT_BF16 if act == "bf16" else L.ACT_F32, 2, h, w, C,
                                                out.out.data_ptr(), L.stream_ptr()))
            torch.cuda.synchronize()
            what = f"upsample_bilinear4 {act} {h}x{w}x{C}"
            out.check(what)
            U.assert_exact(out.out.view(2, 4 * h, 4 * w, C), want, what, ["b", "y", "x", "c"])


# ------------------------------------------------------------------ coverage census of the engine's plans
@pytest.mark.parametrize("precision,conv_impl", sorted(X.ENGINE_CENSUS))
def test_every_engine_layer_class_is_an_exact_case(precision, conv_impl, synth_sd):
    """UNetEngine at C3 (1920x1088): the class of every planned conv (kernel, k, stride, Cin, Cout, sources, epilogue flags) is
    among the exact cases, and the hard-coded census of test_fwd_exact_host.py is current."""
    from read_b200.engine import UNetEngine
    seen = set()
    names = {L.CONV_TCGEN05: "tma", L.CONV_TCGEN05_GATHER: "gather", L.CONV_GENERIC: "generic"}

    class Census(UNetEngine):
        def _conv(self, prefix, srcs, cout, k, stride, elu, residual=None, out2_mul=None, final=False, raw=False, addin=None,
                  cin_slice=None, name=None):
            r = super()._conv(prefix, srcs, cout, k, stride, elu, residual, out2_mul, final, raw, addin, cin_slice, name)
            ly = self.layers[-1]
            seen.add(X.census_class(names[ly.impl], "bf16" if self.bf16 else "f32", k, stride,
                                    [(t.shape[3], m, f) for t, m, f in srcs], cout, residual is not None, out2_mul is not None,
                                    addin is not None, False, "nchw" if final else ("raw" if raw else "nhwc")))
            return r

    eng = Census(synth_sd, 1, 1088, 1920, dev(), precision=precision, conv_impl=conv_impl, use_graph=False)
    del eng
    torch.cuda.empty_cache()
    covered = {X.case_class(c) for c in X.EXACT_CASES}
    assert seen <= covered, f"{precision}/{conv_impl}: layer classes without an exact case: {sorted(seen - covered)}"
    assert seen == X.ENGINE_CENSUS[(precision, conv_impl)], \
        (f"{precision}/{conv_impl}: census changed: new {sorted(seen - X.ENGINE_CENSUS[(precision, conv_impl)])}, "
         f"gone {sorted(X.ENGINE_CENSUS[(precision, conv_impl)] - seen)}")
