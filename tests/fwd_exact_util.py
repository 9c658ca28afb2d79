"""Exact and per-element checks of the forward gated-conv kernels (csrc/conv_tc.cu, csrc/conv_tc_gather.cu, csrc/conv_generic.cu)
and of read_upsample_bilinear4: case lists, operand generators, float64 references and the exactness precondition, shared by
test_fwd_exact_host.py (no GPU) and test_gpu_fwd_exact.py.  The generic helpers (int_tensor, Guarded, assert_exact, fm_columns,
the sentinels) are bwd_exact_util's.

Operands: activations are integers in [-A, A] (exact in bf16 for A <= 256), weights integers in [-AW, AW] times 2^-s, and every
other operand a small dyadic.  Every partial sum of every accumulator is then an integer multiple of the accumulator unit
(2^-s, or 2^-(s+6) when a bilinear x4 source is blended in) below 2^24 units, so the tensor-core and the CUDA-core accumulation
both produce the one exact value whatever their order (``precondition`` proves the bound per case).

What the kernels produce from those sums:
  RAW [f | m]          bf16 round-to-nearest of (sum + add-in [+ residual]), compared for equality in the RAW column order;
  gate pinned open     channels with wm = 0 and bias_m = 64: sigmoid(64) is 1.0 in fp32 (tanh.approx / expf saturate; each
                       kernel's self-check shows it), so with elu = 0, or elu = 1 where f + b_f > 0, the output is
                       bf16(fl32(fl32(f * scale + shift) + residual)) (fp32 outputs: without the bf16 rounding), which ``ref``
                       emulates bit for bit: the checks there are equalities;
  out2                 bf16(stored y * mul) with both factors bf16: the product is exact in fp32, so out2 is exact wherever y is;
  other channels       |got - want64| <= REL |want64| + TAU |A| |scale| + EPS32 (|A scale| + |shift| + |residual|):
                       REL is the output format's half ulp, TAU covers the gate's approximate sigmoid / ELU, EPS32 the fp32
                       roundings of the epilogue's fma and residual add (A = the activation ELU(f) or f, float64).
"""
import dataclasses
import math

import torch
import torch.nn.functional as F

import bwd_exact_util as U

# ---------------------------------------------------------------- kernel constants
TC_TH, TC_TW = 16, 8                # TMA kernel tile: 16 rows x 8 pixels
G_TH, G_TW = 8, 16                  # gather kernel tile: 8 rows x 16 pixels
TC_RESIDENT_MAX = 144 * 1024        # TMA kernel: packed weights up to this size stay resident in shared memory
EXACT_LIMIT = U.EXACT_LIMIT

# ---------------------------------------------------------------- operand amplitudes
A = 32                              # |activation| (integers)
AW = 32                             # |weight| in units of 2^-s
A_BIL = 3                           # |activation| of a source that is bilinear-upsampled x4: blends are multiples of 1/64 below 3
BIL_BITS = 6                        # 2D bilinear x4 weights are multiples of 1/64
A_MUL = 4                           # |input-side multiplier| (integers)
A_ADD = 256                         # |add-in| and |RAW residual| in accumulator units
A_BIAS = 256                        # |bias_f| (and |bias_m| of the ordinary channels) in accumulator units
PIN_BIAS_M = 64.0                   # bias_m of the gate-pinned channels: sigmoid(64) == 1.0 in fp32

# The bound constants.  TAU_FAST: the wgmma kernels' tanh.approx / ex2.approx gate.  PTX documents about 2^-11 relative error
# for tanh.approx; measured on an H100 80GB HBM3 over test_gpu_fwd_exact.py's cases, the worst share of the TAU term an ordinary
# element uses beyond its rounding and fp32 terms is 0.00164 at 2^-9 (on the fp32 final-layer outputs, where no bf16 rounding
# hides it), i.e. 0.105 at 2^-15: 9.5x headroom.  TAU_ACC: the CUDA-core kernel's expf / expm1f / division, whose error the
# EPS32 term already covered on every measured element (share 0).
TAU_FAST = 2.0 ** -15
TAU_ACC = 2.0 ** -20
EPS32 = 2.0 ** -22
REL = {"bf16": 2.0 ** -8, "f32": 2.0 ** -23}


# ---------------------------------------------------------------- cases
@dataclasses.dataclass(frozen=True)
class Case:
    """One forward conv launch.  srcs: ((C, mode, factor), ...) with mode in id / down / up / bil4; H, W: the conv input size
    (the virtual concat's); out: 'nhwc' (gated), 'raw' ([f | m] accumulators) or 'nchw' (final layer, fp32)."""
    name: str
    impl: str                       # 'tma' | 'gather' | 'generic'
    srcs: tuple
    cout: int
    k: int
    stride: int
    B: int
    H: int
    W: int
    out: str = "nhwc"
    residual: bool = False
    out2: bool = False
    addin: bool = False
    mul: bool = False
    elu: int = 0
    act: str = "bf16"

    @property
    def cin(self):
        return sum(c for c, _, _ in self.srcs)

    @property
    def pad(self):
        return (self.k - 1) // 2 if self.stride == 1 else 1

    @property
    def hout(self):
        return (self.H + 2 * self.pad - self.k) // self.stride + 1

    @property
    def wout(self):
        return (self.W + 2 * self.pad - self.k) // self.stride + 1

    @property
    def bil(self):
        return any(m == "bil4" for _, m, _ in self.srcs)

    def src_hw(self, mode, f):
        return {"id": (self.H, self.W), "down": (self.H * f, self.W * f), "up": (self.H // f, self.W // f),
                "bil4": (self.H // 4, self.W // 4)}[mode]

    @property
    def out_channels(self):
        return 2 * self.cout if self.out == "raw" else self.cout

    @property
    def id(self):
        return (f"{self.impl}-{self.act}-{self.name}-B{self.B}-{self.H}x{self.W}" + ("-elu" if self.elu else ""))


def census_class(impl, act, k, stride, srcs, cout, residual, out2, addin, mul, out):
    """The class of a planned layer: kernel (the CUDA-core one by its activation type), geometry, sources and epilogue flags."""
    kern = impl if impl != "generic" else f"generic-{act}"
    return (kern, k, stride, sum(c for c, _, _ in srcs), cout, tuple((c, m, f) for c, m, f in srcs), bool(residual),
            bool(out2), bool(addin), bool(mul), out)


def case_class(c):
    return census_class(c.impl, c.act, c.k, c.stride, c.srcs, c.cout, c.residual, c.out2, c.addin, c.mul, c.out)


def _id(C):
    return ((C, "id", 1),)


# The TMA-fed wgmma kernel: every geometry it accepts (tc_supported), at ragged tiles on both edges and B = 1 / 3.
TMA_CASES = [
    # 3x3 stride 1, one source: 16-channel K steps (Cin 8 read with a 16-channel box), 32- and 64-channel K chunks, resident
    # weights (C64 at exactly 144 KB) and streamed ones, one and two n-tiles, two CTAs per SM (N <= 64) and one
    Case("3x3 8->16", "tma", _id(8), 16, 3, 1, 3, 17, 9, elu=1),
    Case("3x3 8->32", "tma", _id(8), 32, 3, 1, 1, 33, 17, elu=1),
    Case("3x3 8->64", "tma", _id(8), 64, 3, 1, 3, 15, 7, elu=1),
    Case("3x3 32->32", "tma", _id(32), 32, 3, 1, 3, 16, 8, elu=1),
    Case("3x3 32->32 +res", "tma", _id(32), 32, 3, 1, 1, 17, 9, residual=True),
    Case("3x3 64->64 (weights 144 KB)", "tma", _id(64), 64, 3, 1, 3, 1, 17, elu=1),
    Case("3x3 64->64 +res", "tma", _id(64), 64, 3, 1, 1, 33, 7, residual=True),
    Case("3x3 128->128 streamed", "tma", _id(128), 128, 3, 1, 1, 17, 17, elu=1),
    Case("3x3 128->128 +res", "tma", _id(128), 128, 3, 1, 3, 15, 9, residual=True),
    Case("3x3 256->256 two n-tiles", "tma", _id(256), 256, 3, 1, 1, 16, 9, elu=1),
    Case("3x3 256->256 +res", "tma", _id(256), 256, 3, 1, 3, 17, 1, residual=True),
    # 1x1, one source
    Case("1x1 16->32", "tma", _id(16), 32, 1, 1, 3, 17, 9, elu=1),
    Case("1x1 32->64", "tma", _id(32), 64, 1, 1, 1, 33, 8, elu=1),
    Case("1x1 64->128 two n-tiles", "tma", _id(64), 128, 1, 1, 3, 15, 17, elu=1),
    # stride 2 (four phase tiles per stage), with the FAM product as out2; Hin = 2 Hout, ragged Hout / Wout
    Case("3x3s2 32->64 +out2", "tma", _id(32), 64, 3, 2, 3, 18, 14, out2=True, elu=1),
    Case("3x3s2 64->128 +out2", "tma", _id(64), 128, 3, 2, 1, 34, 18, out2=True, elu=1),
    Case("3x3s2 128->256 +out2", "tma", _id(128), 256, 3, 2, 3, 2, 34, out2=True, elu=1),
    Case("4x4s2 256->128", "tma", _id(256), 128, 4, 2, 1, 30, 16, elu=1),
    Case("4x4s2 128->64", "tma", _id(128), 64, 4, 2, 3, 34, 2, elu=1),
    Case("4x4s2 64->32", "tma", _id(64), 32, 4, 2, 1, 66, 18, elu=1),
    # 1x1 virtual concats of identity sources (decoder merges)
    Case("1x1 cat128+128->128", "tma", ((128, "id", 1), (128, "id", 1)), 128, 1, 1, 3, 17, 9, elu=1),
    Case("1x1 cat64+64->64", "tma", ((64, "id", 1), (64, "id", 1)), 64, 1, 1, 1, 15, 17, elu=1),
    Case("1x1 cat32+32->32", "tma", ((32, "id", 1), (32, "id", 1)), 32, 1, 1, 3, 16, 7, elu=1),
    # the AFF head split by linearity: RAW terms with the coarser term as add-in, the last one gated
    Case("RAW 1x1 256->32", "tma", _id(256), 32, 1, 1, 3, 17, 9, out="raw"),
    Case("RAW 1x1 128->32 +addin", "tma", _id(128), 32, 1, 1, 1, 33, 17, out="raw", addin=True),
    Case("RAW 1x1 64->32 +addin", "tma", _id(64), 32, 1, 1, 3, 15, 8, out="raw", addin=True),
    Case("1x1 32->32 +addin", "tma", _id(32), 32, 1, 1, 3, 17, 9, addin=True, elu=1),
    # RAW 1x1 at Cout 16 / 32 / 64 over concats of identity and nearest-down x2 / x4 / x8 sources, with and without the add-in
    Case("RAW 1x1 cat down8+id->16", "tma", ((32, "down", 8), (64, "id", 1)), 16, 1, 1, 3, 9, 7, out="raw"),
    Case("RAW 1x1 128->16 +addin", "tma", _id(128), 16, 1, 1, 1, 17, 9, out="raw", addin=True),
    Case("RAW 1x1 cat down4+down2+id->32 +addin", "tma", ((32, "down", 4), (64, "down", 2), (128, "id", 1)), 32, 1, 1, 1, 17, 9,
         out="raw", addin=True),
    Case("RAW 1x1 cat down2+id+id->64 +addin", "tma", ((64, "down", 2), (32, "id", 1), (256, "id", 1)), 64, 1, 1, 3, 15, 8,
         out="raw", addin=True),
    Case("RAW 1x1 cat down2+id->64", "tma", ((64, "down", 2), (64, "id", 1)), 64, 1, 1, 1, 16, 1, out="raw"),
    Case("1x1 cat down2+id->64 +addin", "tma", ((32, "down", 2), (64, "id", 1)), 64, 1, 1, 3, 17, 9, addin=True, elu=1),
    Case("1x1 cat down4+down2+id->32 +addin", "tma", ((32, "down", 4), (64, "down", 2), (128, "id", 1)), 32, 1, 1, 1, 33, 7,
         addin=True),
    # RAW 3x3 stride 1 over one source, with and without the [B, H, W, 2C] residual; RAW stride 2
    Case("RAW 3x3 64->32 +res", "tma", _id(64), 32, 3, 1, 3, 17, 9, out="raw", residual=True),
    Case("RAW 3x3 32->64", "tma", _id(32), 64, 3, 1, 1, 15, 17, out="raw"),
    Case("RAW 3x3 128->128 +res", "tma", _id(128), 128, 3, 1, 1, 16, 9, out="raw", residual=True),
    Case("RAW 3x3s2 64->128", "tma", _id(64), 128, 3, 2, 1, 18, 34, out="raw"),
    Case("RAW 4x4s2 128->64", "tma", _id(128), 64, 4, 2, 3, 34, 14, out="raw"),
    # the final layer: Cout 3 padded to 8, fp32 NCHW from the registers
    Case("final 3x3 32->3", "tma", _id(32), 3, 3, 1, 3, 17, 9, out="nchw"),
    Case("final 3x3 32->3 W1", "tma", _id(32), 3, 3, 1, 1, 16, 1, out="nchw"),
]

AFF1_SRCS = ((32, "down", 2), (64, "id", 1), (128, "up", 2), (256, "up", 4))
AFF2_SRCS = ((32, "down", 4), (64, "down", 2), (128, "id", 1), (256, "up", 2))
AFF0_SRCS = ((32, "id", 1), (64, "up", 2), (128, "up", 4), (256, "up", 8))

# The gather kernel: resampled sources (nearest up x2 / x4 / x8, nearest down, bilinear x4), padded Cout, stride 2 on odd
# shapes, residual and out2, NCHW; ragged 8 x 16 tiles.
GATHER_CASES = [
    Case("1x1 32->56", "gather", _id(32), 56, 1, 1, 3, 17, 9, elu=1),
    Case("1x1 64->120 two n-tiles", "gather", _id(64), 120, 1, 1, 1, 9, 33, elu=1),
    Case("1x1 128->248 (padded to 256)", "gather", _id(128), 248, 1, 1, 3, 15, 17, elu=1),
    Case("1x1 cat8+56->64", "gather", ((8, "id", 1), (56, "id", 1)), 64, 1, 1, 1, 17, 9),
    Case("1x1 cat8+120->128", "gather", ((8, "id", 1), (120, "id", 1)), 128, 1, 1, 3, 8, 17),
    Case("1x1 cat8+248->256", "gather", ((8, "id", 1), (248, "id", 1)), 256, 1, 1, 1, 9, 16),
    Case("AFF1 cat down2+id+up2+up4->64", "gather", AFF1_SRCS, 64, 1, 1, 3, 12, 20, elu=1),
    Case("AFF2 cat down4+down2+id+up2->128", "gather", AFF2_SRCS, 128, 1, 1, 1, 18, 34, elu=1),
    Case("AFF0 cat id+up2+up4+up8->32", "gather", AFF0_SRCS, 32, 1, 1, 3, 16, 24, elu=1),
    Case("1x1 cat bil4+id->128", "gather", ((128, "bil4", 4), (128, "id", 1)), 128, 1, 1, 1, 12, 20, elu=1),
    Case("1x1 cat bil4+id->32", "gather", ((32, "bil4", 4), (32, "id", 1)), 32, 1, 1, 3, 4, 36, elu=1),
    Case("3x3s2 odd 32->64 +out2", "gather", _id(32), 64, 3, 2, 3, 17, 9, out2=True, elu=1),
    Case("4x4s2 odd 64->32 +res", "gather", _id(64), 32, 4, 2, 1, 15, 33, residual=True),
    Case("3x3s2 odd 128->256", "gather", _id(128), 256, 3, 2, 1, 9, 31, elu=1),
    Case("3x3 64->64 +res +out2", "gather", _id(64), 64, 3, 1, 3, 17, 9, residual=True, out2=True),
    Case("3x3 8->32", "gather", _id(8), 32, 3, 1, 1, 9, 17, elu=1),
    Case("final 3x3 32->3", "gather", _id(32), 3, 3, 1, 3, 17, 9, out="nchw"),
]

# The CUDA-core kernel: every layer kind of the net (the engine runs all of them on it with conv_impl='generic' and in fp32, and
# the ones the TMA kernel does not take with 'tma_only'), plus the input-side FAM multiplier, in both activation types.
_GENERIC_KINDS = [
    (_id(8), 16, 3, 1, {}), (_id(8), 32, 3, 1, {}), (_id(8), 64, 3, 1, {}),
    (_id(32), 32, 3, 1, {}), (_id(32), 32, 3, 1, {"residual": True}), (_id(64), 64, 3, 1, {}),
    (_id(64), 64, 3, 1, {"residual": True}), (_id(128), 128, 3, 1, {}), (_id(128), 128, 3, 1, {"residual": True}),
    (_id(256), 256, 3, 1, {}), (_id(256), 256, 3, 1, {"residual": True}),
    (_id(16), 32, 1, 1, {}), (_id(32), 64, 1, 1, {}), (_id(64), 128, 1, 1, {}),
    (_id(32), 56, 1, 1, {}), (_id(64), 120, 1, 1, {}), (_id(128), 248, 1, 1, {}),
    (((8, "id", 1), (56, "id", 1)), 64, 1, 1, {}), (((8, "id", 1), (120, "id", 1)), 128, 1, 1, {}),
    (((8, "id", 1), (248, "id", 1)), 256, 1, 1, {}),
    (_id(32), 64, 3, 2, {"out2": True}), (_id(64), 128, 3, 2, {"out2": True}), (_id(128), 256, 3, 2, {"out2": True}),
    (_id(256), 128, 4, 2, {}), (_id(128), 64, 4, 2, {}), (_id(64), 32, 4, 2, {}),
    (AFF0_SRCS, 32, 1, 1, {}), (AFF1_SRCS, 64, 1, 1, {}), (AFF2_SRCS, 128, 1, 1, {}),
    (((128, "bil4", 4), (128, "id", 1)), 128, 1, 1, {}), (((64, "bil4", 4), (64, "id", 1)), 64, 1, 1, {}),
    (((32, "bil4", 4), (32, "id", 1)), 32, 1, 1, {}),
    (_id(32), 3, 3, 1, {"out": "nchw"}),
    (_id(32), 32, 3, 1, {"mul": True, "residual": True}),
]
# (B, H, W) rotated through the kinds; multiples of 8 where an x8 source needs them.  The CUDA-core tile is 8 x 8.
_GENERIC_SHAPES = [(3, 17, 9), (1, 9, 17), (3, 15, 7), (1, 1, 9), (3, 16, 8), (1, 33, 1)]


def _generic_cases():
    cases = []
    for act in ("bf16", "f32"):
        for i, (srcs, cout, k, stride, kw) in enumerate(_GENERIC_KINDS):
            B, H, W = _GENERIC_SHAPES[(i + (act == "f32")) % len(_GENERIC_SHAPES)]
            fmax = max([f if m in ("up", "down") else (4 if m == "bil4" else 1) for _, m, f in srcs])
            if any(m in ("up", "bil4") for _, m, _ in srcs):
                H, W = fmax * (H // fmax + 1), fmax * (W // fmax + 2)
            if stride == 2:
                H, W = 2 * H, 2 * W
            name = "{}->{} {}x{}s{}".format("+".join(f"{m}{c}" + (f"x{f}" if f > 1 else "") for c, m, f in srcs), cout, k, k, stride)
            name += "".join(f" +{n}" for n in ("residual", "out2", "mul") if kw.get(n))
            cases.append(Case(name, "generic", srcs, cout, k, stride, B, H, W, out=kw.get("out", "nhwc"),
                              residual=kw.get("residual", False), out2=kw.get("out2", False), mul=kw.get("mul", False),
                              elu=int(i % 2 == 0 and kw.get("out") != "nchw"), act=act))
    return cases


GENERIC_CASES = _generic_cases()
EXACT_CASES = TMA_CASES + GATHER_CASES + GENERIC_CASES

# read_conv_plan_set_max_ctas values every TMA / gather case also runs with (0 = one CTA per SM): one CTA walking every tile
# wraps every A, B and epilogue ring and every barrier phase
MAX_CTAS = (1, 2, 3)

# read_upsample_bilinear4 shapes
BIL_HW = (1, 2, 3, 5)
BIL_CS = (8, 16, 64, 256)


# ---------------------------------------------------------------- the engine's layer classes (conv_impl x precision at C3)
def _tma(k, s, srcs, cout, out="nhwc", res=False, out2=False, addin=False):
    return census_class("tma", "bf16", k, s, srcs, cout, res, out2, addin, False, out)


def _cls(kern, act, k, s, srcs, cout, out="nhwc", res=False, out2=False):
    return census_class(kern, act, k, s, srcs, cout, res, out2, False, False, out)


_TMA_COMMON = {
    _tma(3, 1, _id(8), 16), _tma(3, 1, _id(8), 32), _tma(3, 1, _id(8), 64),
    _tma(1, 1, _id(16), 32), _tma(1, 1, _id(32), 64), _tma(1, 1, _id(64), 128),
    _tma(3, 1, _id(32), 32), _tma(3, 1, _id(32), 32, res=True), _tma(3, 1, _id(64), 64), _tma(3, 1, _id(64), 64, res=True),
    _tma(3, 1, _id(128), 128), _tma(3, 1, _id(128), 128, res=True), _tma(3, 1, _id(256), 256),
    _tma(3, 1, _id(256), 256, res=True),
    _tma(3, 2, _id(32), 64, out2=True), _tma(3, 2, _id(64), 128, out2=True), _tma(3, 2, _id(128), 256, out2=True),
    _tma(4, 2, _id(256), 128), _tma(4, 2, _id(128), 64), _tma(4, 2, _id(64), 32),
    _tma(1, 1, ((128, "id", 1), (128, "id", 1)), 128), _tma(1, 1, ((64, "id", 1), (64, "id", 1)), 64),
    _tma(1, 1, ((32, "id", 1), (32, "id", 1)), 32),
    _tma(3, 1, _id(32), 3, out="nchw"),
}
_NOT_TMA = [(1, 1, _id(32), 56), (1, 1, _id(64), 120), (1, 1, _id(128), 248), (1, 1, ((8, "id", 1), (56, "id", 1)), 64),
            (1, 1, ((8, "id", 1), (120, "id", 1)), 128), (1, 1, ((8, "id", 1), (248, "id", 1)), 256),
            (1, 1, AFF1_SRCS, 64), (1, 1, AFF2_SRCS, 128)]
_ALL_GENERIC = [(3, 1, _id(8), 16, {}), (3, 1, _id(8), 32, {}), (3, 1, _id(8), 64, {}), (1, 1, _id(16), 32, {}),
                (1, 1, _id(32), 64, {}), (1, 1, _id(64), 128, {}), (3, 1, _id(32), 32, {}), (3, 1, _id(32), 32, {"res": True}),
                (3, 1, _id(64), 64, {}), (3, 1, _id(64), 64, {"res": True}), (3, 1, _id(128), 128, {}),
                (3, 1, _id(128), 128, {"res": True}), (3, 1, _id(256), 256, {}), (3, 1, _id(256), 256, {"res": True}),
                (3, 2, _id(32), 64, {"out2": True}), (3, 2, _id(64), 128, {"out2": True}), (3, 2, _id(128), 256, {"out2": True}),
                (4, 2, _id(256), 128, {}), (4, 2, _id(128), 64, {}), (4, 2, _id(64), 32, {}),
                (1, 1, ((128, "bil4", 4), (128, "id", 1)), 128, {}), (1, 1, ((64, "bil4", 4), (64, "id", 1)), 64, {}),
                (1, 1, ((32, "bil4", 4), (32, "id", 1)), 32, {}), (3, 1, _id(32), 3, {"out": "nchw"}),
                (1, 1, AFF0_SRCS, 32, {})] + [(k, s, srcs, cout, {}) for k, s, srcs, cout in _NOT_TMA]

ENGINE_CENSUS = {
    ("bf16", "auto"): _TMA_COMMON | {_cls("gather", "bf16", *c) for c in _NOT_TMA} | {
        _tma(1, 1, _id(256), 32, out="raw"), _tma(1, 1, _id(128), 32, out="raw", addin=True),
        _tma(1, 1, _id(64), 32, out="raw", addin=True), _tma(1, 1, _id(32), 32, addin=True)},
    ("bf16", "tma_only"): _TMA_COMMON | {_cls("generic", "bf16", *c) for c in _NOT_TMA} |
                          {_cls("generic", "bf16", 1, 1, AFF0_SRCS, 32)},
    ("bf16", "generic"): {_cls("generic", "bf16", k, s, srcs, cout, **kw) for k, s, srcs, cout, kw in _ALL_GENERIC},
    ("fp32", "generic"): {_cls("generic", "f32", k, s, srcs, cout, **kw) for k, s, srcs, cout, kw in _ALL_GENERIC},
}


# ---------------------------------------------------------------- TMA kernel geometry (conv_tc.cu: tc_geom, tc_plan_create)
def tma_geom(c):
    """(cin_blk, kchunks, n_tile, n_tiles, packed weight bytes, resident, CTAs per SM) of a TMA case."""
    gran = 32 if len(c.srcs) > 1 and any(C % 64 for C, _, _ in c.srcs) else 64
    if c.cin % 64 == 0 and c.stride == 1 and gran == 64:
        cin_blk = 64
    elif c.cin % 32 == 0:
        cin_blk = 32
    else:
        assert c.cin in (8, 16) and c.stride == 1, c.id
        cin_blk = 16
    cout_pad = 8 if c.cout <= 8 else c.cout
    n_tile = min(2 * cout_pad, 128)
    n_tiles = 2 * cout_pad // n_tile
    kchunks = -(-c.cin // cin_blk)
    halo_rows, halo_w = (TC_TH + 1, TC_TW + 1) if c.stride == 2 else (TC_TH + c.k - 1, TC_TW + c.k - 1)
    tile = -(-halo_rows * halo_w * cin_blk * 2 // 1024) * 1024
    a_bytes = 4 * tile if c.stride == 2 else tile
    total_b = c.k * c.k * kchunks * n_tile * cin_blk * 2
    e_bytes = 0 if c.out == "nchw" else (128 * (2 if c.out == "raw" else 1) * n_tile + (128 * n_tile if c.out2 else 0) +
                                         (64 * n_tile if c.addin else 0))
    fixed = 1024 + 8 * 70 + 16 * cout_pad + 64
    budget_2, budget_1 = 114 * 1024 - 1024 - fixed, 227 * 1024 - fixed
    fits = n_tiles == 1 and total_b <= TC_RESIDENT_MAX
    ctas = 2 if n_tile <= 64 and fits and total_b + 2 * e_bytes + 3 * a_bytes <= budget_2 else 1
    resident = fits and total_b + 2 * e_bytes + 2 * a_bytes <= (budget_2 if ctas == 2 else budget_1)
    return cin_blk, kchunks, n_tile, n_tiles, total_b, resident, ctas


def tma_classes(c):
    cin_blk, kchunks, n_tile, n_tiles, total_b, resident, ctas = tma_geom(c)
    cls = {f"K chunk {cin_blk}", f"{n_tiles} n-tiles", "resident weights" if resident else "streamed weights",
           f"{ctas} CTAs per SM", f"W%8=={c.wout % TC_TW}", f"H%16=={c.hout % TC_TH}", f"B=={c.B}"}
    if total_b == TC_RESIDENT_MAX and resident:
        cls.add("resident weights of exactly 144 KB")
    if kchunks > 1:
        cls.add("several K chunks")
    return cls


# ---------------------------------------------------------------- the exactness precondition
def acc_unit_bits(c):
    """log2 of 1 / (the activation grid): 0 for integer activations, BIL_BITS when a bilinear x4 source is blended in."""
    return BIL_BITS if c.bil else 0


def src_amp(c, mode):
    return A_BIL if mode == "bil4" else A


def max_partial_units(c):
    """The largest magnitude any partial sum of an accumulator (plus add-in / RAW residual, plus bias_f) can reach, in units of
    the accumulator grid 2^-(s + acc_unit_bits)."""
    g = 2 ** acc_unit_bits(c)
    mul = A_MUL if c.mul else 1
    acc = sum(C * c.k * c.k * src_amp(c, m) * g * mul * AW for C, m, _ in c.srcs)
    extra = (A_ADD if c.addin else 0) + (A_ADD if (c.residual and c.out == "raw") else 0)
    return acc + extra + (0 if c.out == "raw" else A_BIAS)


def precondition(c):
    """Refuse a case whose partial sums could leave fp32's exact integers; returns the bound."""
    m = max_partial_units(c)
    assert m < EXACT_LIMIT, f"{c.id}: partial sums reach {m} units >= 2^24"
    return m


# ---------------------------------------------------------------- resampling references (float64, NCHW)
def nearest(x, mode, f):
    """F.interpolate(mode='nearest') by an integer power-of-two factor, written as indexing (test_fwd_exact_host checks both agree)."""
    if mode == "id":
        return x
    if mode == "down":
        return x[:, :, ::f, ::f]
    return x.repeat_interleave(f, 2).repeat_interleave(f, 3)


def bilinear4(x):
    return F.interpolate(x.double(), scale_factor=4, mode="bilinear", align_corners=False)


def resample(x, mode, f):
    return bilinear4(x) if mode == "bil4" else nearest(x, mode, f)


# ---------------------------------------------------------------- operands
def dyadic(shape, num_amp, bits, gen, zero_frac=0.0, nonzero=False):
    """Integers in [-num_amp, num_amp] times 2^-bits (``nonzero``: without 0)."""
    v = U.int_tensor(shape, num_amp, gen, zero_frac)
    if nonzero:
        v = torch.where(v == 0, torch.ones_like(v), v)
    return v * 2.0 ** -bits


def operands(c, gen):
    """CPU float32 tensors of a case: sources NHWC, weights [Cout, Cin, k, k] (integers; the scale 2^-s is chosen by ``make``),
    per-channel vectors, epilogue operands NHWC."""
    o = {"srcs": []}
    for C, mode, f in c.srcs:
        h, w = c.src_hw(mode, f)
        o["srcs"].append(U.int_tensor((c.B, h, w, C), src_amp(c, mode), gen))
    o["wf"] = U.int_tensor((c.cout, c.cin, c.k, c.k), AW, gen)
    o["wm"] = U.int_tensor((c.cout, c.cin, c.k, c.k), AW, gen)
    o["mul"] = U.int_tensor((c.B, c.H, c.W, c.cin), A_MUL, gen, zero_frac=0.1) if c.mul else None
    return o


def pinned_channels(cout):
    """The gate-pinned half: the even output channels (every epilogue channel pair holds one pinned and one ordinary channel)."""
    return torch.arange(cout) % 2 == 0


def make(c, gen, pin=True):
    """Operands with the weight scale 2^-s chosen so the gate sees values of order 1, the float64 accumulators (in value units),
    and the epilogue parameters.  ``pin``: give the even channels wm = 0, bias_m = 64 (the gate pinned open)."""
    o = operands(c, gen)
    x = torch.cat([resample(t.double().permute(0, 3, 1, 2), m, f) for t, (_, m, f) in zip(o["srcs"], c.srcs)], 1)
    if c.mul:
        x = x * o["mul"].double().permute(0, 3, 1, 2)
    pinned = pinned_channels(c.cout) if (pin and c.out != "raw") else torch.zeros(c.cout, dtype=torch.bool)
    o["wm"][pinned] = 0
    conv = lambda w: F.conv2d(x, w.double(), stride=c.stride, padding=c.pad).permute(0, 2, 3, 1)   # NHWC, integer weights
    accf, accm = conv(o["wf"]), conv(o["wm"])
    spread = float(torch.cat([accf.flatten(), accm.flatten()]).std()) if accf.numel() > 1 else 1.0
    s = max(0, round(math.log2(max(spread, 1.0) / 2)))           # |f|, |m| of order 2 in value units
    g = acc_unit_bits(c)
    o["s"], o["unit"] = s, 2.0 ** -(s + g)
    sc = 2.0 ** -s
    o["wf"], o["wm"] = o["wf"] * sc, o["wm"] * sc
    o["accf"], o["accm"] = accf * sc, accm * sc
    Ho, Wo, C = c.hout, c.wout, c.cout
    o["pinned"] = pinned
    bf = dyadic((C,), A_BIAS, s + g, gen)
    bm = torch.where(pinned, torch.full((C,), PIN_BIAS_M), dyadic((C,), A_BIAS, s + g, gen))
    scale = dyadic((C,), 8, 2, gen, nonzero=True)
    shift = dyadic((C,), 16, 3, gen)
    o["bf"], o["bm"], o["scale"], o["shift"] = bf, bm, scale, shift
    if c.residual:
        o["res"] = (dyadic((c.B, Ho, Wo, 2 * C), A_ADD, s + g, gen) if c.out == "raw"
                    else dyadic((c.B, Ho, Wo, C), 64, 2, gen))
    if c.out2:
        o["out2_mul"] = dyadic((c.B, Ho, Wo, C), 64, 3, gen)
    if c.addin:
        ad = dyadic((c.B, (Ho + 1) // 2, (Wo + 1) // 2, 2 * C), A_ADD, s + g, gen)
        ad[..., C:][..., pinned] = 0                               # the pinned gates stay at bias_m = 64
        o["addin"] = ad
    return o


# ---------------------------------------------------------------- float64 references
def _round(v, dt):
    """float64 -> the output dtype by round-to-nearest-even (float64 -> float32 first: the kernels' values are fp32)."""
    v = v.float()
    return v.bfloat16() if dt == "bf16" else v


def ref(c, o):
    """The exact / float64 results of a case.  RAW: 'raw' (the exact sum, RAW column order) and 'raw_rn' (its bf16 rounding).
    Gated: 'y64' (float64), 'y_pin' (the bit-exact emulation for the gate-pinned channels), 'A', 'res', 'exact' (where y_pin
    applies: pinned channels, and with ELU only where f + b_f > 0); with out2 'o2_pin' / 'o2_64'.  NHWC, NCHW outputs permuted."""
    f, m = o["accf"], o["accm"]
    if c.addin:
        up = o["addin"].double().repeat_interleave(2, 1).repeat_interleave(2, 2)[:, :c.hout, :c.wout]
        f, m = f + up[..., :c.cout], m + up[..., c.cout:]
    r = {}
    if c.out == "raw":
        raw = U.to_raw(torch.cat([f, m], -1))
        if c.residual:
            raw = raw + o["res"].double()
        r["raw"], r["raw_rn"] = raw, _round(raw, "bf16")
        return r
    F_ = f + o["bf"].double()
    M_ = m + o["bm"].double()
    A_ = torch.where(F_ > 0, F_, torch.expm1(F_)) if c.elu else F_
    sc, sh = o["scale"].double(), o["shift"].double()
    res = o["res"].double() if c.residual else torch.zeros_like(F_)
    y64 = A_ * torch.sigmoid(M_) * sc + sh + res
    y1 = (F_ * sc + sh).float().double()                          # fmaf(f * 1.0, scale, shift)
    y2 = (y1 + res).float().double()                              # + residual in fp32
    dt = "f32" if c.out == "nchw" or c.act == "f32" else "bf16"
    r["y64"], r["y_pin"], r["A"], r["res"], r["dt"] = y64, _round(y2, dt).double(), A_, res, dt
    exact = o["pinned"].expand_as(F_)
    if c.elu:
        exact = exact & (F_ > 0)
    r["exact"] = exact
    if c.out2:
        mul = o["out2_mul"].double()
        r["o2_pin"] = _round(r["y_pin"] * mul, dt).double()
        r["o2_64"] = y64 * mul
    if c.out == "nchw":
        for k in ("y64", "y_pin", "A", "res", "exact"):
            r[k] = r[k].permute(0, 3, 1, 2)
    return r


def bound(c, o, r, tau):
    """Per-element bound of the ordinary channels (module docstring), in the layout of r['y64']."""
    sc, sh = o["scale"].double(), o["shift"].double()
    if c.out == "nchw":
        sc, sh = sc[:, None, None], sh[:, None, None]
    As = (r["A"] * sc).abs()
    return REL[r["dt"]] * r["y64"].abs() + tau * As + EPS32 * (As + sh.abs() + r["res"].abs())


def tau_share(got, want64, c, o, r, tau):
    """The worst share of the TAU term an ordinary element uses beyond its rounding and fp32 terms: what TAU's headroom is
    measured on."""
    g, w = got.detach().double().cpu(), want64.double()
    sc, sh = o["scale"].double(), o["shift"].double()
    if c.out == "nchw":
        sc, sh = sc[:, None, None], sh[:, None, None]
    As = (r["A"] * sc).abs()
    over = ((g - w).abs() - REL[r["dt"]] * w.abs() - EPS32 * (As + sh.abs() + r["res"].abs())).clamp(min=0)
    t = tau * As
    share = torch.where(t > 0, over / torch.where(t > 0, t, torch.ones_like(t)), over * math.inf)
    mask = ~r["exact"]
    return float(share[mask].nan_to_num(0.0).max()) if bool(mask.any()) else 0.0
