"""Exact and per-element checks of the training backward kernels (csrc/conv_bwd.cu, the RAW plans of csrc/conv_tc.cu under
blocks.dgrad / blocks.dgrad_1x1, csrc/gather.cu, csrc/train.cu, csrc/scatter_det.cu): operand generators, float64 references,
checkers, guard bands and the edge-class shape lists, shared by test_bwd_exact_host.py (no GPU) and test_gpu_bwd_exact.py.

Integer-valued operands make every product and every partial sum exact in fp32 while its magnitude stays below 2^24, so split-K,
atomics, tensor-core accumulation and the deterministic combines all have to produce the one exact integer, whatever their order:
the checks compare every element, and one dropped, duplicated or misrouted pixel changes at least one of them.  A bf16 output
holds the round-to-nearest-even of that exact value; the operands are large enough that most exact sums are not representable in
bf16, so a truncating or double-rounding epilogue fails too.

What integers cannot reach (the gate's sigmoid / ELU, train-mode BatchNorm's correction terms) is held to per-element bounds:
  bf16 element   |got - want64| <= 2^-8 |want64| + TAU * T
  fp32 sum       |got - want64| <= TAU_S * sum of T over its pixels
T is the sum of the absolute values of the terms that form the element: for the gate, dg_terms * max(1, |A|) with
dg_terms = |scale * dy| + |k1| * (|g| + |mean|) + |k0|.  g and mean enter separately because the kernel rounds g before it
subtracts mean, so the error of g - mean scales with |g| + |mean|, not with their difference.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

# ---------------------------------------------------------------- kernel constants (csrc/conv_bwd.cu, csrc/conv_tc.cu)
SMS = 132                           # H100 SXM
WG_PX, WG_M, WG_N = 32, 64, 32      # weight gradient: pixel segment, column block, input-channel block
DG8_PX, DG8_THREADS = 64, 128       # 8-channel input gradient: pixel segment
DS_PX = 64                          # stride-2 input gradient: input pixels per segment
TC_TH, TC_TW = 16, 8                # TMA conv tile: 16 rows x 8 pixels
GB_THREADS = 256                    # gate / BatchNorm passes: ppb = 256 / (C / 8) pixels per step
EXACT_LIMIT = 2 ** 24               # fp32 holds every integer below this

# The bound constants.  Measured on an H100 80GB HBM3 (700 W) over test_gpu_bwd_exact.py's cases: the worst share of TAU a [df | dm]
# element uses beyond its bf16 rounding is 0.0149 at TAU = 2^-18, i.e. 0.119 at 2^-21 (8x headroom); the worst err / bound of the
# fp32 sums is 0.00414 at TAU_S = 2^-14, i.e. 0.066 at 2^-18 (15x headroom).  REL_BF16 is bf16's half ulp, not a tolerance.
TAU = 2.0 ** -21
TAU_S = 2.0 ** -18
REL_BF16 = 2.0 ** -8

# sentinel bit patterns of the guard bands by element size (bf16 / fp32: NaNs no kernel writes; u8 flags: neither 0 nor 1)
SENTINELS = {1: (torch.uint8, 0xA5), 2: (torch.int16, 0x7FA1), 4: (torch.int32, 0x7FA1A1A1)}
GUARD = 8192                        # guard elements on each side of an output (a multiple of 64: 128-byte aligned interiors)


# ---------------------------------------------------------------- operand generators
def int_tensor(shape, amp, gen, zero_frac=0.4):
    """float32 integers uniform in [-amp, amp] with about ``zero_frac`` extra zeros; exact in bf16 for amp <= 256."""
    v = torch.randint(-amp, amp + 1, shape, generator=gen).float()
    return v * (torch.rand(shape, generator=gen) >= zero_frac)


def bf16_nonrepresentable_fraction(want):
    """Share of the exact values ``want`` (float64, integers) that bf16 cannot hold: what the round-to-nearest check tests."""
    w = want.double()
    return float((w.float().bfloat16().double() != w).double().mean())


def gate_fm_values(P, C, gen):
    """The raw [f | m] (concat order, before bias) of P pixels: randn mixed with the hard regions of the gate.  m: 0, +-10, +-30,
    +-100 (a saturated sigmoid, 1 - s cancelling); f: +-0, tiny (the expm1f branch), f << 0 (A + 1 cancelling)."""
    f = torch.randn((P, C), generator=gen) * 2
    m = torch.randn((P, C), generator=gen) * 2
    pick = lambda vals: torch.tensor(vals)[torch.randint(0, len(vals), (P, C), generator=gen)]
    r = torch.rand((P, C), generator=gen)
    m = torch.where(r < 0.35, pick([0.0, 10.0, -10.0, 30.0, -30.0, 100.0, -100.0]), m)
    r = torch.rand((P, C), generator=gen)
    f = torch.where(r < 0.15, pick([0.0, -0.0, 1e-3, -1e-3, 3e-6, -3e-6, 1e-30, -1e-30]), f)
    f = torch.where((r >= 0.15) & (r < 0.3), pick([-20.0, -60.0, -90.0, -7.0]), f)
    return torch.cat([f, m], 1)


# ---------------------------------------------------------------- float64 references
def fm_columns(C):
    """blocks.fm_columns without the package import: the concat channel held by each RAW [f | m] column."""
    half = min(C, 64)
    j = torch.arange(2 * C)
    blk, r = j // (2 * half), j % (2 * half)
    return torch.where(r < half, blk * half + r, C + blk * half + r - half)


def to_raw(cat):
    """[..., 2C] concat order -> RAW column order."""
    return cat[..., fm_columns(cat.shape[-1] // 2)]


def wgrad_ref(dcat, x, k, stride):
    """[2C, Cin, k, k] float64: the weight gradient of [conv_f; conv_m] from dcat [B,Ho,Wo,2C] and x [B,Hi,Wi,Cin] (NHWC)."""
    return torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (dcat.shape[-1], x.shape[-1], k, k),
                                       dcat.double().permute(0, 3, 1, 2), stride=stride, padding=(k - 1) // 2)


def dgrad_ref(dcat, wcat, Hi, Wi, stride):
    """[B,Hi,Wi,Cin] float64: the input gradient of [conv_f; conv_m] (wcat [2C, Cin, k, k]) from dcat [B,Ho,Wo,2C]."""
    B, k = dcat.shape[0], wcat.shape[-1]
    return torch.nn.grad.conv2d_input((B, wcat.shape[1], Hi, Wi), wcat.double(), dcat.double().permute(0, 3, 1, 2),
                                      stride=stride, padding=(k - 1) // 2).permute(0, 2, 3, 1)


def gather_ref(go, ids, N, prefill):
    """prefill [N, D] + the scatter of grad_out [B,D,h,w] onto the clamped ids [B,h,w], float64 (np.add.at)."""
    out = np.array(prefill, np.float64)
    key = np.clip(np.asarray(ids).reshape(-1).astype(np.int64), 0, N - 1)
    D = go.shape[1]
    np.add.at(out, key, np.asarray(go, np.float64).transpose(0, 2, 3, 1).reshape(-1, D))
    return out


def gate_ref(o, C, elu, kind, items, P):
    """float64 gate / BatchNorm backward of the operands ``o`` (dy [items*P, C], fm RAW [items*P, 2C] bf16; bf, bm [C]; scale, mean,
    inv, s0 = sum_dy, s1 = sum_dy_xhat [items, C]).  kind: 'eval' (read_gate_backward), 'batch' (read_gate_backward_batch_stats,
    statistics over items*P pixels, items = 1) or 'items' (per item).  Returns dfm in RAW order, the sums, and their bounds' T."""
    fm = o["fm"].double()
    cat = torch.empty_like(fm)
    cat[:, fm_columns(C)] = fm
    f, m = cat[:, :C] + o["bf"].double(), cat[:, C:] + o["bm"].double()
    s = torch.sigmoid(m)
    A = F.elu(f) if elu else f
    Ad = torch.where(f > 0, torch.ones_like(f), A + 1) if elu else torch.ones_like(f)
    dy = o["dy"].double()
    r = torch.arange(dy.shape[0]) // P
    sc, mu, iv = (o[n].double()[r] for n in ("scale", "mean", "inv"))
    g = A * s
    if kind == "eval":
        k1 = k0 = torch.zeros_like(dy)
    else:
        # the kernel's k1 / k0 use the pixel count of the statistics: P per item, or items * P for one call-wide set
        n = P if kind == "items" else dy.shape[0]
        k1 = -sc * iv * o["s1"].double()[r] / n
        k0 = -sc * o["s0"].double()[r] / n
    dg = dy * sc + k1 * (g - mu) + k0
    dg_terms = (dy * sc).abs() + k1.abs() * (g.abs() + mu.abs()) + k0.abs()
    df, dm = dg * s * Ad, dg * A * s * (1 - s)
    T = dg_terms * torch.clamp(A.abs(), min=1.0)
    xh = dy * (g - mu) * iv
    xh_T = dy.abs() * (g.abs() + mu.abs()) * iv
    per = lambda t: t.reshape(items, P, C).sum(1)
    return dict(dfm=to_raw(torch.cat([df, dm], 1)), T_dfm=to_raw(torch.cat([T, T], 1)),
                sum_df=df.sum(0), sum_dm=dm.sum(0), T_sum=T.sum(0),
                sum_dy=per(dy), sum_xh=per(xh), T_xh=per(xh_T), dgamma=xh.sum(0), T_dgamma=xh_T.sum(0), dbeta=dy.sum(0))


# ---------------------------------------------------------------- checkers
def _where(mask, names, limit=6):
    idx = mask.nonzero()[:limit].tolist()
    return [", ".join(f"{n}={i}" for n, i in zip(names, ix)) for ix in idx]


def assert_exact(got, want, what, names=None):
    """Every element of ``got`` equals the exact ``want`` (float64); on failure the message names the first differing elements."""
    g, w = got.detach().double().cpu(), want.detach().double().cpu()
    assert g.shape == w.shape, (what, tuple(g.shape), tuple(w.shape))
    bad = ~(g == w)
    if bool(bad.any()):
        names = names or [f"d{i}" for i in range(g.dim())]
        first = bad.nonzero()[:6].tolist()
        detail = "; ".join(f"[{', '.join(f'{n}={i}' for n, i in zip(names, ix))}] got {g[tuple(ix)].item()!r} want "
                           f"{w[tuple(ix)].item()!r}" for ix in first)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ from the exact result: {detail}")


def assert_bf16_rn(got, want64, what, names=None):
    """A bf16 output holds the round-to-nearest-even of the exact integer ``want64`` (|want64| < 2^24, so float64 -> float32 is
    exact and the only rounding is float32 -> bf16)."""
    assert float(want64.abs().max()) < EXACT_LIMIT, what
    assert_exact(got.float(), want64.float().bfloat16().float(), what, names)


def bound_ratios(got, want64, T, tau, rel=0.0):
    """|got - want64| / (rel * |want64| + tau * T) per element (0 where both are 0)."""
    g, w, t = got.detach().double().cpu(), want64.detach().double().cpu(), T.detach().double().cpu()
    err = (g - w).abs()
    bound = rel * w.abs() + tau * t
    ratio = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)), torch.where(err > 0, math.inf, 0.0))
    return torch.nan_to_num(ratio, nan=math.inf)


def tau_share(got, want64, T, tau, rel):
    """The worst (|got - want64| - rel |want64|) / (tau T): how much of the tau term a bf16 output uses beyond its own rounding
    (which the rel term covers), the figure the headroom of TAU is measured on."""
    g, w, t = got.detach().double().cpu(), want64.detach().double().cpu(), T.detach().double().cpu()
    over = ((g - w).abs() - rel * w.abs()).clamp(min=0)
    return float(torch.where(t > 0, over / torch.where(t > 0, tau * t, torch.ones_like(t)), over * math.inf).nan_to_num(0.0).max())


def assert_bound(got, want64, T, tau, what, rel=0.0, names=None):
    """Every element within the bound; returns the worst err / bound (printed by the tests)."""
    r = bound_ratios(got, want64, T, tau, rel)
    worst = float(r.max()) if r.numel() else 0.0
    if not worst <= 1.0:
        names = names or [f"d{i}" for i in range(r.dim())]
        ix = np.unravel_index(int(torch.argmax(torch.nan_to_num(r, posinf=1e300))), tuple(r.shape))
        raise AssertionError(f"{what}: {int((r > 1).sum())} elements beyond the bound, worst err/bound {worst:.3g} at "
                             f"[{', '.join(f'{n}={int(i)}' for n, i in zip(names, ix))}]: got {got.reshape(r.shape)[ix].item()!r} "
                             f"want {want64.reshape(r.shape)[ix].item()!r} T {T.reshape(r.shape)[ix].item()!r}")
    return worst


class Guarded:
    """An output of ``n`` elements in the middle of a larger buffer whose GUARD elements on each side hold a sentinel bit pattern;
    ``out`` is the interior (optionally pre-filled), ``check`` asserts both guards are bit-unchanged."""

    def __init__(self, n, dtype, device, prefill=None, guard=GUARD):
        self.n, self.guard = n, guard
        self.buf = torch.empty(n + 2 * guard, dtype=dtype, device=device)
        self.view_dtype, self.sentinel = SENTINELS[self.buf.element_size()]
        self.buf.view(self.view_dtype).fill_(self.sentinel)
        self.out = self.buf[guard:guard + n]
        self.out.copy_(prefill.reshape(-1) if prefill is not None else torch.zeros(n, dtype=dtype))

    def check(self, what):
        ib = self.buf.view(self.view_dtype)
        for name, part, off in (("before", ib[:self.guard], -self.guard), ("after", ib[self.guard + self.n:], self.n)):
            bad = (part != self.sentinel).nonzero()
            if bad.numel():
                raise AssertionError(f"{what}: {bad.numel()} elements written {name} the output, e.g. at flat offsets "
                                     f"{[int(i) + off for i in bad[:6, 0].tolist()]} (the output has {self.n} elements)")


# ---------------------------------------------------------------- launch geometry and edge classes
def cdiv(a, b):
    return -(-a // b)


def wgrad_grid(B, H, W, C, Cin, k, sms=SMS):
    """(chunks, splits, uncapped splits, column blocks, z blocks) of the weight-gradient launch (conv_bwd.cu: wgrad_grid)."""
    chunks = B * H * cdiv(W, WG_PX)
    mb, nz = cdiv(2 * C, WG_M), cdiv(Cin, WG_N) * (2 if k == 4 else 1)
    s_free = cdiv(2 * sms, mb * nz)
    return chunks, min(s_free, chunks), s_free, mb, nz


def wgrad_classes(case, sms=SMS):
    """The edge classes one weight-gradient case (cin, C, k, stride, B, Ho, Wo) reaches."""
    cin, C, k, stride, B, H, W = case
    chunks, s, s_free, mb, nz = wgrad_grid(B, H, W, C, cin, k, sms)
    per_cta = cdiv(chunks, s)
    cls = {f"W%32=={W % WG_PX}", f"H=={H}", f"B=={B}"}
    if W < WG_PX:
        cls.add("W<32")
    if chunks <= s_free:
        cls.add("chunks<=splits")
    if chunks > 2 * s and per_cta % 2 == 1:
        cls.add("chunks>2*splits,odd per CTA")
    if chunks > 2 * s and per_cta % 2 == 0:
        cls.add("chunks>2*splits,even per CTA")
    if (2 * C) % WG_M:
        cls.add("partial column block")
    if cin % WG_N:
        cls.add("partial channel block")
    if k == 4:
        cls.add("4x4 row groups")
    return cls


WGRAD_REQUIRED = {"W%32==1", "W%32==31", "W%32==0", "W<32", "H==1", "H==2", "H==7", "B==1", "B==4", "B==8", "chunks<=splits",
                  "chunks>2*splits,odd per CTA"}


def tma_classes(H, W):
    cls = {f"W%8=={W % TC_TW}", f"H%16=={H % TC_TH}"}
    if W < TC_TW:
        cls.add("W<8")
    if H < TC_TH:
        cls.add("H<16")
    return cls


def dg8_classes(B, H, W, C):
    K2 = 2 * C
    smem = (9 * 8 + 3 * (DG8_PX + 2)) * (2 * K2 + 16)
    grid = min(min(200 * 1024 // smem, 8) * SMS, B * H * cdiv(W, DG8_PX))
    cls = {f"W%64=={W % DG8_PX}"}
    if W < DG8_PX:
        cls.add("W<64")
    if B * H * cdiv(W, DG8_PX) > grid:
        cls.add("CTA walks several segments")
    return cls


def ds_classes(Wi, C):
    cls = {f"Wi%64=={Wi % DS_PX}"}
    if Wi < DS_PX:
        cls.add("Wi<64")
    cls.add("one K chunk" if 2 * C == 32 else "several K chunks")
    return cls


def ppb(C):
    return GB_THREADS // (C // 8)


# ---------------------------------------------------------------- the shape lists
# (Cin, C) of every gated conv the net trains, C padded as the training path runs it (blocks.padded_channels, the RGB conv at 16)
TRAINED = {
    (3, 1): [(8, 16), (8, 32), (8, 64), (32, 16), (64, 16), (128, 16), (32, 32), (64, 64), (128, 128), (256, 256)],
    (1, 1): [(16, 32), (32, 64), (64, 32), (64, 64), (64, 128), (128, 64), (128, 128), (128, 256), (256, 128), (256, 256),
             (32, 128), (256, 32)],
    (3, 2): [(32, 64), (64, 128), (128, 256)],
    (4, 2): [(64, 32), (128, 64), (256, 128)],
}
# (k, stride, Cin, C) run padded -> the conv's real C (the RGB outputs: 3; SCM*.main.3: 56 / 120 / 248): the gate backward gives
# the padded channels' [df | dm] columns 0, so the tests zero them and the padded gradient rows must come out exactly 0
PADDED = {(3, 1, 32, 16): 3, (3, 1, 64, 16): 3, (3, 1, 128, 16): 3, (1, 1, 32, 64): 56, (1, 1, 64, 128): 120,
          (1, 1, 128, 256): 248}


def zero_padded_columns(dcat, n_real):
    """dcat [..., 2C] (concat order) with the channels n_real..C-1 of both halves zeroed."""
    C = dcat.shape[-1] // 2
    d = dcat.clone()
    d[..., n_real:C] = 0
    d[..., C + n_real:] = 0
    return d


def _wgrad_cases():
    cases = []
    edge_w, edge_h = (1, 31, 32, 33, 65), (1, 2, 7)
    for (k, stride), pairs in TRAINED.items():
        for i, (cin, C) in enumerate(pairs):
            # each pair at one tail shape, rotating through the edges
            cases.append((cin, C, k, stride, 1 + 3 * (i % 2), edge_h[i % 3], edge_w[i % 5]))
        cin, C = pairs[0]
        for W in edge_w:
            for H in edge_h:
                cases.append((cin, C, k, stride, 2, H, W))
    # training shapes: C5 is 8 crops of 256^2; the full-resolution convs, and the deeper ones at their resolution
    cases += [(8, 32, 3, 1, 8, 256, 256), (32, 16, 3, 1, 8, 256, 256), (32, 32, 3, 1, 8, 256, 256), (16, 32, 1, 1, 8, 256, 256),
              (64, 64, 3, 1, 8, 128, 128), (128, 128, 3, 1, 4, 64, 64), (256, 256, 3, 1, 8, 32, 32), (32, 64, 3, 2, 8, 128, 128),
              (64, 32, 4, 2, 8, 128, 128), (256, 128, 4, 2, 8, 32, 32), (128, 256, 3, 2, 8, 32, 32), (8, 16, 3, 1, 1, 7, 33), (64, 16, 3, 1, 4, 7, 31)]
    return cases


WGRAD_CASES = _wgrad_cases()
WGRAD_AMP = 2                       # |[df | dm]|, |x| <= 2
WGRAD_PREFILL = 1000                # |dW pre-fill| <= 1000, integers

DGRAD_HW = (1, 8, 9, 16, 17)
DGRAD3_CASES = ([(cin, C, 2, 17, 9) for cin, C in TRAINED[(3, 1)] if cin != 8] +
                [(64, 64, 2, H, W) for H in DGRAD_HW for W in DGRAD_HW] +
                [(256, 256, 3, 9, 17), (32, 32, 8, 64, 64)])
# 1x1: (source channel counts of the concat, C); each source's slice of the input gradient separately
DGRAD1_CASES = [((16,), 32, 2, 9, 17), ((32,), 64, 2, 17, 9), ((64,), 128, 3, 8, 16), ((128,), 64, 2, 1, 9),
                ((256,), 256, 2, 9, 8), ((32, 64, 128, 256), 128, 2, 9, 17), ((32, 64, 128, 256), 32, 2, 16, 1)]
DGRAD_AMP = 16                      # |[df | dm]|, |w| <= 16: most sums exceed 256
DGRAD_RES_AMP = 256

DG8_CASES = [(C, 2, H, W) for C in (16, 32, 64) for H, W in ((3, 1), (2, 63), (1, 64), (2, 65), (3, 129))] + \
            [(32, 8, 256, 256), (64, 4, 64, 64)]
DS_CASES = [(k, cin, C, 2, Hi, Wi) for (k, _s), pairs in (((3, 2), TRAINED[(3, 2)]), ((4, 2), TRAINED[(4, 2)]))
            for cin, C in pairs for Hi, Wi in ((2, 2), (4, 62), (6, 64), (2, 66), (4, 130))] + \
           [(4, 32, 16, 2, 6, 66), (3, 32, 64, 8, 256, 256)]

GATE_CS = (16, 32, 64, 128, 192, 256)


def gate_item_pixels(C):
    return (2, ppb(C) - 1, ppb(C), ppb(C) + 1)


# (C, items, pixels per item) of the exact per-item sums at training sizes: 64 items x 64^2 px, one item of 8 x 256^2 px
GATE_BIG = [(64, 64, 64 * 64), (256, 64, 64 * 64), (16, 1, 8 * 256 * 256)]


def max_partial(terms, amp_a, amp_b, extra=0):
    """The largest magnitude any partial sum of ``terms`` products of |a| <= amp_a, |b| <= amp_b can reach, plus |extra|."""
    return terms * amp_a * amp_b + extra


def wgrad_terms(case):
    cin, C, k, stride, B, H, W = case
    return B * H * W            # one product per output pixel and weight element
