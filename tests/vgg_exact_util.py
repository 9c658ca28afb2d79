"""Exact checks of the VGG perceptual loss (read_b200/vgg_loss.py, csrc/vgg.cu): the census of what VGGLoss launches, the case
lists of its conv plans, operand generators, float64 conv references and float32 replays of the glue kernels, shared by
test_vgg_exact_host.py (no GPU) and test_gpu_vgg_exact.py.

Convs.  Every VGG conv is a RAW 3x3 plan of the TMA wgmma kernel: forward over read_pack_weights_tc filters of the gated pair
split_filters makes, input gradient over read_pack_weights_tc_dgrad filters (conv1_1's: read_conv3x3_dgrad_cin8).  With integer
operands every partial sum is an exact fp32 integer (fwd_exact_util / bwd_exact_util state the method), so every bf16 output is
checked for equality with the round-to-nearest of the exact sum.

Glue.  Each kernel of csrc/vgg.cu is replayed operation by operation in torch float32 on the host (IEEE round-to-nearest, like
the device's __f*_rn and plain fp32 operations), then rounded to bf16 with .bfloat16() (RNE).  Two operations are fused on the
device, as the compiled SASS shows, and the replays reproduce the fused rounding:
  vgg_post_partial   raw * ratio + bias is one FFMA: the replay forms the exact value in float64 (a bf16 times an fp32 has at
                     most 32 significant bits), proves per element with TwoSum that adding the bias was exact too, and rounds
                     once to fp32;
  the loss term      *term += s * scale is one DFMA: the replay rounds prefill + s * scale once, from exact rationals.
The term's sum s is replayed in the kernel's fixed order: each thread's fp32 sum over its grid-stride units, the CTA's double
tree, the CTAs' partials in CTA order.  On integer-valued operands every one of those partial sums is exact, so s is the exact
sum of |y_out - y_tgt|.
"""
import fractions
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

import bwd_exact_util as U
import fwd_exact_util as X
from read_b200 import vgg_loss as V

# ---------------------------------------------------------------- kernel constants (csrc/vgg.cu)
VG_THREADS = 256
VG_MAX_CTAS = 1024


def vg_blocks(units):
    return int(min(max(-(-units // VG_THREADS), 1), VG_MAX_CTAS))


# ---------------------------------------------------------------- 1. the census of what VGGLoss launches
# (conv module index, cin, cout, loss term, pool follows) of each conv of the two layer sets' walks
WALKS = {
    "LAYERS": ((0, 3, 64, True, False), (2, 64, 64, True, True), (5, 64, 128, True, False), (7, 128, 128, True, True),
               (10, 128, 256, True, False), (12, 256, 256, True, False), (14, 256, 256, True, False), (16, 256, 256, True, True),
               (19, 256, 512, True, False), (21, 512, 512, True, False), (23, 512, 512, True, False), (25, 512, 512, True, True),
               (28, 512, 512, True, False)),
    "LAYERS_OPTIMIZED": ((0, 3, 64, False, False), (2, 64, 64, True, True), (5, 64, 128, False, False),
                         (7, 128, 128, True, True), (10, 128, 256, False, False), (12, 256, 256, False, False),
                         (14, 256, 256, False, False), (16, 256, 256, True, True), (19, 256, 512, False, False),
                         (21, 512, 512, False, False), (23, 512, 512, False, False), (25, 512, 512, True, True),
                         (28, 512, 512, False, False), (30, 512, 512, False, False), (32, 512, 512, False, False),
                         (34, 512, 512, True, False)),
}
# forward RAW 3x3 plans: (Cin padded to 8, Cout = cout / 2, the gated pair's filters each)
FWD_CLASSES = {(8, 32), (64, 32), (64, 64), (128, 64), (128, 128), (256, 128), (256, 256), (512, 256)}
# input-gradient RAW 3x3 plans over _dgrad-packed filters: (Cin = the conv's cout, Cout = its cin / 2)
DGRAD_CLASSES = {(64, 32), (128, 32), (128, 64), (256, 64), (256, 128), (512, 128), (512, 256)}
# read_conv3x3_dgrad_cin8 (conv1_1): C = the pair's filters each
CIN8_CS = {32}
# split_filters: width of the channel blocks dealt alternately to wf and wm, per cout
SPLIT_BLOCKS = {64: 32, 128: 64, 256: 64, 512: 64}


def walk(layers):
    return tuple((s.conv, s.cin, s.cout, s.loss, s.pool) for s in V.layer_walk(layers))


def split_block(c):
    """The width of the channel blocks split_filters deals to wf (and alternately wm), read off its output."""
    wf, _ = V.split_filters(torch.arange(c, dtype=torch.float64).reshape(c, 1, 1, 1))
    f = wf.flatten().long().tolist()
    n = 1
    while n < len(f) and f[n] == f[n - 1] + 1:
        n += 1
    return n


def derived_census():
    """The census computed from vgg_loss itself: walks, forward / input-gradient classes, cin8 C, split blocks."""
    steps = V.layer_walk(V.LAYERS) + V.layer_walk(V.LAYERS_OPTIMIZED)
    return dict(walks={"LAYERS": walk(V.LAYERS), "LAYERS_OPTIMIZED": walk(V.LAYERS_OPTIMIZED)},
                fwd={(max(s.cin, 8), s.cout // 2) for s in steps},
                dgrad={(s.cout, s.cin // 2) for s in steps if s.cin != 3},
                cin8={s.cout // 2 for s in steps if s.cin == 3},
                split={s.cout: split_block(s.cout) for s in steps})


def launch_census():
    """What one VGGLoss forward + backward passes to blocks._launch, as (packing, Cin, Cout, k, stride, out, residual)."""
    return ({("tc", cin, cout, 3, 1, "raw", False) for cin, cout in FWD_CLASSES} |
            {("tc_dgrad", cin, cout, 3, 1, "raw", False) for cin, cout in DGRAD_CLASSES})


# ---------------------------------------------------------------- 2. forward RAW plans (fwd_exact_util cases)
def _fwd(name, cin, cout, B, H, W):
    return X.Case(f"VGG {name} RAW 3x3 {cin}->{cout}", "tma", ((cin, "id", 1),), cout, 3, 1, B, H, W, out="raw")


# one per class at ragged tiles (H = 1 and W = 1 among them, the deep layers at the sizes a 70 x 46 image gives them), then each
# class at the size a 256^2 training crop gives its layer, 2n = 2 images
VGG_FWD_CASES = [
    _fwd("conv1_1", 8, 32, 2, 33, 1),
    _fwd("conv1_2", 64, 32, 4, 17, 9),
    _fwd("conv2_1", 64, 64, 2, 15, 17),
    _fwd("conv2_2", 128, 64, 2, 1, 23),
    _fwd("conv3_1", 128, 128, 4, 9, 15),
    _fwd("conv3_x", 256, 128, 2, 17, 7),
    _fwd("conv4_1", 256, 256, 2, 8, 5),
    _fwd("conv4_x", 512, 256, 2, 9, 17),
    _fwd("conv5_x", 512, 256, 2, 4, 2),
    _fwd("conv1_1", 8, 32, 2, 256, 256),
    _fwd("conv1_2", 64, 32, 2, 256, 256),
    _fwd("conv2_1", 64, 64, 2, 128, 128),
    _fwd("conv2_2", 128, 64, 2, 128, 128),
    _fwd("conv3_1", 128, 128, 2, 64, 64),
    _fwd("conv3_x", 256, 128, 2, 64, 64),
    _fwd("conv4_1", 256, 256, 2, 32, 32),
    _fwd("conv4_x", 512, 256, 2, 32, 32),
    _fwd("conv5_x", 512, 256, 2, 16, 16),
]

# ---------------------------------------------------------------- 3. input-gradient RAW plans: (cin, C, B, H, W), bwd notation
# (the plan reads [df | dm] of 2C channels and writes cin); every class at the edges DGRAD_HW reaches (1, 8, 9, 16, 17), then at
# each layer's training-crop size
_DGRAD_LAYERS = [("conv1_2", 64, 32, 256), ("conv2_1", 64, 64, 128), ("conv2_2", 128, 64, 128), ("conv3_1", 128, 128, 64),
                 ("conv3_x", 256, 128, 64), ("conv4_1", 256, 256, 32), ("conv4_x", 512, 256, 32), ("conv5_x", 512, 256, 16)]
_DGRAD_EDGES = [(2, 1, 17), (2, 17, 1), (2, 9, 16), (3, 16, 9), (2, 8, 8), (2, 17, 17), (3, 1, 1), (1, 16, 8)]


def _dgrad_cases():
    cases, seen = [], set()
    for _, cin, C, hw in _DGRAD_LAYERS:
        if (cin, C) not in seen:
            seen.add((cin, C))
            cases += [(cin, C, B, H, W) for B, H, W in _DGRAD_EDGES]
        cases.append((cin, C, 2, hw, hw))
    return cases


VGG_DGRAD_CASES = _dgrad_cases()
DGRAD_AMP = U.DGRAD_AMP


def dgrad_class(case):
    cin, C = case[:2]
    return (2 * C, cin // 2)


def dgrad_max_partial(case):
    cin, C = case[:2]
    return U.max_partial(9 * 2 * C, DGRAD_AMP, DGRAD_AMP)


# ---------------------------------------------------------------- 4. the VGG path: integer features in torchvision's layout
PATH_AMP = 32                       # |activation|, |dy| (integers) and |weight| (integers times 2^-PATH_S)
PATH_S = 5
PATH_SHAPE = (2, 11, 13)            # 2n, h, w of every conv's launch


def int_features(gen, amp=PATH_AMP, s=PATH_S):
    """VGG19's features as torchvision builds them (Conv2d, ReLU(inplace=True), MaxPool2d(2, 2)) with integer weights times 2^-s
    and integer biases."""
    mods = []
    for k in V.vgg19_modules():
        if k == "relu":
            mods.append(nn.ReLU(inplace=True))
        elif k == "pool":
            mods.append(nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            conv = nn.Conv2d(k[1], k[2], kernel_size=3, padding=1)
            with torch.no_grad():
                conv.weight.copy_(U.int_tensor(tuple(conv.weight.shape), amp, gen) * 2.0 ** -s)
                conv.bias.copy_(U.int_tensor(tuple(conv.bias.shape), amp, gen))
            mods.append(conv)
    return nn.Sequential(*mods)


def path_max_partial(cin):
    return U.max_partial(9 * cin, PATH_AMP, PATH_AMP)


def conv_ref(x, w):
    """float64 NHWC: the plain conv (padding 1) of x [B, H, W, cin] by w [cout, cin, 3, 3]."""
    return F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), padding=1).permute(0, 2, 3, 1)


def conv_input_grad_ref(dy, w):
    """float64 NHWC: the input gradient of that conv, conv_transpose2d(dy, w) (padding 1)."""
    return F.conv_transpose2d(dy.double().permute(0, 3, 1, 2), w.double(), padding=1).permute(0, 2, 3, 1)


# ---------------------------------------------------------------- 5. operands and float32 replays of the glue kernels
def nz(t):
    """t with -0 turned into +0 (int_tensor zeroes negative values into -0, which no VGG tensor holds)."""
    return t + 0.0


def glue_raw(n, H, W, C, gen, amp=2000, tie=0.2):
    """RAW [2n, H, W, C] bf16: integers up to ``amp`` (bf16 keeps them integers), the target equal to the output on about ``tie``
    of the elements (codes 2 on a loss layer)."""
    r = U.int_tensor((2 * n, H, W, C), amp, gen, zero_frac=0.1).bfloat16().float()
    same = torch.rand((n, H, W, C), generator=gen) < tie
    r[n:][same] = r[:n][same]
    return nz(r).bfloat16()


def glue_bias(C, gen, amp=300):
    return nz(U.int_tensor((C,), amp, gen, zero_frac=0.1))


def glue_mask(n, H, W, gen, kind):
    """Byte mask [n, H, W]: 'holes' (random holes, an empty corner block on the image border, a full bottom band), 'valid', 'invalid'."""
    if kind == "valid":
        return torch.ones((n, H, W), dtype=torch.uint8)
    if kind == "invalid":
        return torch.zeros((n, H, W), dtype=torch.uint8)
    m = (torch.rand((n, H, W), generator=gen) < 0.7).to(torch.uint8)
    m[0, :4, :5] = 0
    m[-1, :, -3:] = 0
    m[-1, -2:, :] = 1
    return m


def window_count(mask):
    """[n, H, W] int: valid pixels in each 3x3 window of the byte mask, zero padding (vg_window)."""
    c = F.conv2d(mask.double()[:, None], torch.ones((1, 1, 3, 3), dtype=torch.float64), padding=1)[:, 0]
    return c.round().long()


def vg_ratio(cnt):
    """fp32 [n, H, W]: c ? fl(fl(1 / c) * 9) : 0 (vg_ratio: __frcp_rn then __fmul_rn)."""
    c = cnt.float()
    r = (torch.ones_like(c) / torch.where(c > 0, c, torch.ones_like(c))) * torch.tensor(9.0)
    return torch.where(cnt > 0, r, torch.zeros_like(r))


def _relu(v):
    """fmaxf(v, 0) of fp32 v that holds no -0 and no NaN."""
    return torch.where(v > 0, v, torch.zeros_like(v))


def fma32(a, b, c):
    """fp32 fmaf(a, b, c) per element for a bf16-valued a and fp32 b, c: a * b is exact in float64 (at most 32 significant bits);
    TwoSum proves the float64 addition exact on every element, so one rounding to fp32 is the fused result."""
    p = a.double() * b.double()
    cc = c.double()
    s = p + cc
    bb = s - p
    err = (p - (s - bb)) + (cc - bb)
    assert bool((err == 0).all()), "fma32: the float64 sum is not exact; the fused rounding cannot be replayed"
    return s.float()


def post_values(raw, bias, n, mask=None, fused=True):
    """y [2n, H, W, C] fp32 of vgg_post (ReLU(raw + bias)) or, with the byte mask, of vgg_post_partial
    (upd ? ReLU(raw * ratio + bias) : 0, raw * ratio + bias fused unless ``fused`` is False)."""
    r = raw.float()
    if mask is None:
        return _relu(r + bias)
    cnt = window_count(mask)
    ratio = torch.cat([vg_ratio(cnt)] * 2)[..., None].expand_as(r)
    v = fma32(r, ratio, bias.expand_as(r)) if fused else r * ratio + bias
    upd = torch.cat([cnt] * 2)[..., None].expand_as(r) > 0
    return torch.where(upd, _relu(v), torch.zeros_like(v))


def post_codes(y, n, loss):
    """int8 [n, H, W, C]: 0 where the output's ReLU is closed, else 2 + sign(y_out - y_tgt) on a loss layer and 2 off it."""
    yi, yt = y[:n], y[n:]
    d = yi - yt
    s = ((d > 0).to(torch.int8) - (d < 0).to(torch.int8)) if loss else torch.zeros_like(d, dtype=torch.int8)
    return torch.where(yi > 0, 2 + s, torch.zeros_like(s)).to(torch.int8)


def pool_replay(y):
    """[B, H // 2, W // 2, C] fp32: the kernel's 2x2 average, ((y00 + y01) + y10) + y11 then * 0.25; odd rows / columns dropped."""
    B, H, W, C = y.shape
    Ho, Wo = H // 2, W // 2
    v = y[:, :2 * Ho, :2 * Wo].reshape(B, Ho, 2, Wo, 2, C)
    return (((v[:, :, 0, :, 0] + v[:, :, 0, :, 1]) + v[:, :, 1, :, 0]) + v[:, :, 1, :, 1]) * torch.tensor(0.25)


def post_out(y, pool):
    """The next conv's input (bf16) written by vgg_post: y, or its pool."""
    return (pool_replay(y) if pool else y).bfloat16()


def term_sum(y, n, pool):
    """s of the loss term, in the kernel's order (module docstring), as a float (double)."""
    P = 2 if pool else 1
    _, H, W, C = y.shape
    G, Hb, Wb = C // 8, -(-H // P), -(-W // P)
    absd = (y[:n] - y[n:]).abs()
    pad = torch.zeros((n, Hb * P, Wb * P, C), dtype=torch.float32)
    pad[:, :H, :W] = absd
    vals = pad.reshape(n, Hb, P, Wb, P, G, 8).permute(0, 1, 3, 5, 2, 4, 6).reshape(-1, P * P * 8)
    units = vals.shape[0]
    grid = vg_blocks(units)
    T = grid * VG_THREADS
    K = -(-units // T)
    v = torch.zeros((K * T, P * P * 8), dtype=torch.float32)
    v[:units] = vals
    v = v.reshape(K, T, P * P * 8)
    acc = torch.zeros(T, dtype=torch.float32)
    for k in range(K):
        for e in range(P * P * 8):
            acc = acc + v[k, :, e]
    red = acc.double().reshape(grid, VG_THREADS)
    s = VG_THREADS // 2
    while s:
        red[:, :s] += red[:, s:2 * s]
        s //= 2
    total = 0.0
    for p in red[:, 0].tolist():
        total += p
    return total


def term_exact_sum(y, n):
    """The exact sum of |y_out - y_tgt| (float64; exact for the integer-valued operands)."""
    return float((y[:n].double() - y[n:].double()).abs().sum())


def fused_term(prefill, s, scale):
    """*term after ``*term += s * scale`` compiled to one DFMA: prefill + s * scale rounded once."""
    return float(fractions.Fraction(prefill) + fractions.Fraction(s) * fractions.Fraction(scale))


def dgrad_in_replay(up, code, H, W, pool, g, coef, mask=None):
    """dY [n, H, W, C] bf16 of vgg_dgrad_in (or, with the byte mask, vgg_dgrad_in_partial): l1 = fl32(g * coef),
    dY = code ? u + (code - 2) * l1 : 0 (times ratio), u = up, or a quarter of the pooled up on the rows / columns it covers."""
    n, C = code.shape[0], code.shape[-1]
    l1 = torch.tensor(g, dtype=torch.float32) * torch.tensor(coef, dtype=torch.float32)
    u = torch.zeros((n, H, W, C), dtype=torch.float32)
    if up is not None:
        if pool:
            Hu, Wu = H // 2, W // 2
            u[:, :2 * Hu, :2 * Wu] = up.float().repeat_interleave(2, 1).repeat_interleave(2, 2) * torch.tensor(0.25)
        else:
            u = up.float()
    c = code.to(torch.int32)
    d = torch.where(c != 0, u + (c - 2).float() * l1, torch.zeros_like(u))
    if mask is not None:
        d = d * vg_ratio(window_count(mask))[..., None]
    return d.bfloat16()


def normalize_replay(x, t, mean, std, mask=None):
    """[2n, H, W, 8] bf16 of vgg_normalize[_masked]: (x - mean) / std (times M), channels 3..7 zero."""
    v = (torch.cat([x, t]) - mean) / std
    if mask is not None:
        m = mask[:, None].float()
        v = v * torch.cat([m, m])
    out = torch.zeros((v.shape[0], v.shape[2], v.shape[3], 8), dtype=torch.float32)
    out[..., :3] = v.permute(0, 2, 3, 1)
    return out.bfloat16()


def image_grad_replay(dx, std, mask=None):
    """[n, 3, H, W] fp32 of vgg_image_grad[_masked]: dx (times M) / std."""
    v = dx[..., :3].float().permute(0, 3, 1, 2)
    if mask is not None:
        v = v * mask[:, None].float()
    return v / std


# ---------------------------------------------------------------- checkers
_BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def assert_same_bits(got, want, what, names=None):
    """Every element of ``got`` has the bits of ``want`` (same dtype): -0 against +0 and any rounding difference fail."""
    g, w = got.detach().cpu(), want.detach().cpu()
    assert g.dtype == w.dtype and g.shape == w.shape, (what, g.dtype, w.dtype, tuple(g.shape), tuple(w.shape))
    gb, wb = g.contiguous().view(_BITS[g.element_size()]), w.contiguous().view(_BITS[w.element_size()])
    bad = gb != wb
    if bool(bad.any()):
        names = names or [f"d{i}" for i in range(g.dim())]
        first = bad.nonzero()[:6].tolist()
        detail = "; ".join(f"[{', '.join(f'{n}={i}' for n, i in zip(names, ix))}] got {g[tuple(ix)].item()!r} want "
                           f"{w[tuple(ix)].item()!r}" for ix in first)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ in their bits: {detail}")


def assert_term(got, want, what):
    assert got == want or (math.isnan(got) and math.isnan(want)), f"{what}: term {got!r}, want {want!r} ({got - want:+.3g})"
