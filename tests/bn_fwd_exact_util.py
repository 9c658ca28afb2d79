"""Per-element checks of train-mode BatchNorm's forward (csrc/bn_train.cu: bn_stats_kernel<PER_ITEM>, bn_apply_kernel<PER_ITEM>,
entry points read_bn_batch_stats[_items] and read_bn_apply[_items]): operands, exact statistics, error bounds, host replays, the
edge-class case lists and the planted defects the bounds must catch; shared by test_bn_fwd_exact_host.py (no GPU) and
test_gpu_bn_fwd_exact.py.

Statistics.  Every input is a bf16 integer: per channel a centre of up to +-192 and a spread of at most +-A, |g| <= 256.  The sums
S1 = sum g and S2 = sum g^2 are exact int64s, so mu = S1 / P and v = (P S2 - S1^2) / P^2 are exact up to one float64 rounding.
The kernel's arithmetic (bn_stats_body): each thread t holds n_t pixels of a channel (p0, p0 + gridDim * ppb, ...), K_t = its first
value, and sums x - K_t and (x - K_t)^2 in fp32.  Those are integers; with n_t (2A)^2 < 2^24 (asserted for every case, along with
|a1| < 2^24) both sums are exact, so the thread's only roundings are
    rn = fl(1 / n),  d = fl(a1 * rn),  M2 = fl(fma(-a1, d, a2))
and with u = 2^-24:  |d - a1 / n| <= ed = |a1 / n| (2u + u^2),  |M2 - M2_t| <= |a1| ed (1 + u) + u M2_t  (M2_t = a2 - a1^2 / n; the
fmaxf(., 0) only moves M2 toward it).  The CTA and last-CTA combines are float64 in a fixed order: their rounding is covered by
F64 times the magnitudes below, 2^13 times float64's unit roundoff, far more than the at most 512 + 256 additions in a chain.
    mean:   E_mu = sum_t n_t ed_t / P + F64 (max|g| + 1)
    P var:  E_Pv = sum_t [err M2_t + 2 n_t |m_t - mu| ed_t + 2 n_t ed_t^2] + F64 sum_t n_t (|m_t| + |mu|)^2
(m_t = K_t + a1 / n_t, the thread's exact mean: an error in m_t moves the pooled sum of squared deviations by 2 n_t (m_t - mu)
to first order; the partial means' own float64 rounding cancels to first order).  inv_std, scale and shift carry these through
their float64 expressions, and every fp32 output adds its own rounding, u (|value| + E).  test_bn_fwd_exact_host.py asserts that,
on every case, each planted defect (a dropped, a doubled, a neighbouring item's pixel, P - 1 for P) changes some output by at
least 4 times its bound: the bounds are tight enough to see one pixel.

Running statistics.  Per item the kernel applies, in item order, r = fmaf(x, m, __fmul_rn(1 - m, r)) to its own mean and the
unbiased variance it leaves in the workspace (bn_items_running_update).  The call-wide update is written
(1 - m) * r + m * (float)x; cuobjdump -sass of bn_stats_kernel<false> (sm_90a, nvcc 12.9, -O3) shows FADD R0 = 1 - m, FMUL
R10 = R0 * r, FFMA r' = x * m + R10 for both statistics: the same fmaf(x, m, fl((1 - m) r)).  Its unbiased variance is float64
inside the kernel, so the call-wide replay takes the three fp32 values nearest fl(var * P / (P - 1)) and accepts the result of
any of them.

Apply.  y = bf16_rn(fl(fl(fl(g * scale) + shift) + residual)), the kernel's comment: torch's fp32 evaluation, no contraction.
Half of the channels are built so that a contracted fma(g, scale, shift) changes the bf16 result of most of their elements with
g at the channel's centre: scale = 1 + e (e about 2^-21: g * scale is inexact), shift = -centre + a few units of the product's
last place, so fl(g * scale) + shift is a small value of few bits (exact in bf16) while the fused form keeps the product's
rounding error, which is larger than that value's bf16 half ulp.
"""
from fractions import Fraction

import numpy as np
import torch

# ---------------------------------------------------------------- kernel constants (csrc/bn_train.cu)
BN_THREADS = 256
BN_MAX_CTAS = 512
BN_PART = 3
BA_THREADS = 256
BN_CS = (16, 32, 64, 128, 192, 256)
EXACT_LIMIT = 2 ** 24

U = 2.0 ** -24                      # fp32 unit roundoff (round to nearest)
F64 = 2.0 ** -40                    # float64 combines: 2^13 x float64's unit roundoff
DEFECT_MARGIN = 4.0                 # each planted defect must move some output by this many bounds
MOMENTA = (0.1, 0.0, 1.0)
EPS = 1e-5


def cdiv(a, b):
    return -(-a // b)


def ppb(C):
    return BN_THREADS // (C // 8)


def stats_cap(sms):
    """CTAs per item of the statistics pass at most (bn_stats_grid): 2 per SM, at most 512."""
    return min(2 * sms, BN_MAX_CTAS)


def stats_grid(P, C, sms):
    return min(cdiv(P, ppb(C)), stats_cap(sms))


def apply_grid(items, P, C, sms):
    """CTAs per item of the apply pass (bn_apply_grid): the call's CTAs capped at 16 per SM, at least 1."""
    return min(cdiv(P * (C // 8), BA_THREADS), max(16 * sms // items, 1))


def ws_layout(per_item, items, C):
    """(uvar offset, partials offset, bytes) of the statistics workspace (bn_ws_layout)."""
    rnd = lambda b: cdiv(b, 256) * 256
    counters = 1 + items if per_item else 1
    uvar = rnd(counters * 4)
    part = uvar + (rnd(items * C * 4) if per_item else 0)
    return uvar, part, part + items * BN_MAX_CTAS * BN_PART * C * 8


# ---------------------------------------------------------------- cases
class Case:
    """One statistics + apply case: ``items`` items of ``P`` pixels (per_item) or one call over P pixels, C channels of which
    ``n_real`` are real, spread A, momentum."""

    def __init__(self, per_item, items, P, C, n_real=None, A=100, momentum=0.1, seed=0):
        self.per_item, self.items, self.P, self.C = per_item, items, P, C
        self.n_real = C if n_real is None else n_real
        self.A, self.momentum, self.seed = A, momentum, seed

    @property
    def id(self):
        return (f"{'items' if self.per_item else 'call'}-B{self.items}-P{self.P}-C{self.C}-n{self.n_real}-A{self.A}"
                f"-m{self.momentum}")

    def __repr__(self):
        return self.id


def stats_cases(sms):
    """The statistics cases for a device of ``sms`` SMs: every C at P = 2, 3, ppb - 1, ppb, ppb + 1 and at ceil(P / ppb) =
    cap - 1, cap, cap + 1; P with unequal pixel counts per thread; the training shapes; items 1, 2, 3, 8, 64 and 16 * sms + 1."""
    cap = stats_cap(sms)
    cases, k = [], 0
    mom = lambda: MOMENTA[k % 3]
    for C in BN_CS:
        b = ppb(C)
        n_real = {16: 3, 64: 56, 256: 248}.get(C, C)
        for P in (2, 3, b - 1, b, b + 1):
            cases.append(Case(False, 1, P, C, n_real if P == b + 1 else C, momentum=mom(), seed=k)); k += 1
            cases.append(Case(True, 3 if P == 3 else 2, P, C, n_real if P == b else C, momentum=mom(), seed=k)); k += 1
        for blocks in (cap - 1, cap, cap + 1):
            P = blocks * b - (b // 2 if blocks == cap + 1 else 0)
            cases.append(Case(blocks != cap, 2 if blocks != cap else 1, P, C, momentum=mom(), seed=k)); k += 1
        # more pixels than one pass of the grid: threads hold 3 or 4 pixels
        cases.append(Case(False, 1, 3 * cap * b + cap * b // 3 + 5, C, n_real, momentum=mom(), seed=k)); k += 1
    # training shapes: 8 crops of 256^2 per item and call-wide, 64 items of 32^2
    cases += [Case(True, 8, 256 * 256, 32, momentum=0.1, seed=101), Case(False, 1, 8 * 256 * 256, 16, A=150, momentum=0.1, seed=102),
              Case(True, 64, 32 * 32, 256, 248, momentum=0.1, seed=103)]
    cases += [Case(True, it, 37 * 11, 64, 56, momentum=MOMENTA[i % 3], seed=110 + i) for i, it in enumerate((1, 2, 3, 8, 64))]
    cases.append(Case(True, 16 * sms + 1, 3, 16, 3, momentum=0.1, seed=120))
    return cases


def stats_classes(case, sms):
    """The partition edges one case reaches."""
    C, P, b, cap = case.C, case.P, ppb(case.C), stats_cap(sms)
    grid = stats_grid(P, C, sms)
    stride = grid * b
    cls = {f"C={C}", f"items={case.items}" if case.per_item else "call-wide", f"momentum={case.momentum}"}
    if P in (2, 3):
        cls.add(f"P={P}")
    for name, v in (("ppb-1", b - 1), ("ppb", b), ("ppb+1", b + 1)):
        if P == v:
            cls.add(f"P={name}")
    nb = cdiv(P, b)
    for name, v in (("cap-1", cap - 1), ("cap", cap), ("cap+1", cap + 1)):
        if nb == v:
            cls.add(f"blocks={name}")
    if P < b:
        cls.add("threads without pixels")
    if P > stride and P % stride:
        cls.add("unequal pixels per thread")
    if C == 192:
        cls.add("idle threads (ppb*G < 256)")
    cls.add("combine lanes>1" if C <= BN_THREADS // 2 else "combine 1 lane")
    if case.n_real < C:
        cls.add("padded channels")
    if case.per_item and case.items > 16 * sms:
        cls.add("apply cap<1")
    if case.per_item and case.P == 256 * 256 and case.items == 8:
        cls.add("training 8x256^2 per item")
    if not case.per_item and case.P == 8 * 256 * 256:
        cls.add("training 8x256^2 call-wide")
    if case.per_item and case.items == 64 and case.P == 32 * 32:
        cls.add("training 64x32^2")
    return cls


def required_classes(sms):
    req = {f"C={C}" for C in BN_CS} | {f"P={n}" for n in (2, 3, "ppb-1", "ppb", "ppb+1")}
    req |= {f"blocks={n}" for n in ("cap-1", "cap", "cap+1")} | {f"items={i}" for i in (1, 2, 3, 8, 64)}
    req |= {"call-wide", "threads without pixels", "unequal pixels per thread", "idle threads (ppb*G < 256)", "combine lanes>1",
            "combine 1 lane", "padded channels", "apply cap<1", "training 8x256^2 per item", "training 8x256^2 call-wide",
            "training 64x32^2", f"items={16 * sms + 1}"} | {f"momentum={m}" for m in MOMENTA}
    return req


# ---------------------------------------------------------------- statistics operands and exact values
def stats_operands(case):
    """[items, P, C] int16 integers (bf16-exact), gamma / beta [n_real] fp32, running mean / var [n_real] fp32.  Per item and
    channel a centre in [-192, 192] and a spread in [0, A] (|g| <= 256); channel 0 constant, channel 1 (when real) a mean of
    +-192 far above its spread of 1, about a sixth of the others constant too; padded channels zero."""
    rng = np.random.default_rng(1000 + case.seed)
    items, P, C, nr = case.items, case.P, case.C, case.n_real
    centre = rng.integers(-192, 193, (items, 1, C))
    spread = np.minimum(rng.integers(0, case.A + 1, (items, 1, C)), 256 - np.abs(centre))
    spread[rng.random((items, 1, C)) < 1 / 6] = 0
    spread[:, :, 0] = 0
    if nr > 1:
        centre[:, :, 1] = np.where(np.arange(items) % 2 == 0, 192, -192)[:, None]
        spread[:, :, 1] = 1
    x = rng.integers(centre - spread, centre + spread + 1, (items, P, C), dtype=np.int64).astype(np.int16)
    x[:, :, nr:] = 0
    gamma = (rng.random(nr) * 1.5 + 0.25).astype(np.float32) * np.where(rng.random(nr) < 0.2, -1, 1).astype(np.float32)
    beta = rng.standard_normal(nr).astype(np.float32)
    rm = rng.standard_normal(nr).astype(np.float32)
    rv = (rng.random(nr) * 2 + 0.5).astype(np.float32)
    return x, gamma, beta, rm, rv


def exact_stats(x):
    """Per item and channel (float64 [items, C]) mean, biased and unbiased variance from int64 sums."""
    P = x.shape[1]
    S1 = x.sum(1, dtype=np.int64)
    S2 = (x.astype(np.int64) ** 2).sum(1)
    num = P * S2 - S1 * S1                                       # P^2 v, exact in int64 for P <= 2^20, |g| <= 256
    return S1 / P, num / float(P * P), num / float(P * (P - 1))


def thread_sums(x, grid, b):
    """The kernel's per-thread state for each item: K [items, T, C], n [T], a1, a2 [items, T, C] int64 for the T threads that
    hold pixels (thread slot s = pixel index mod gridDim * ppb holds pixels s, s + stride, ...)."""
    items, P, C = x.shape
    S = grid * b
    T, nmax = min(P, S), cdiv(P, S)
    pad = np.zeros((items, nmax * S, C), np.int32)
    pad[:, :P] = x
    xr = pad.reshape(items, nmax, S, C)
    mask = (np.arange(nmax * S) < P).reshape(nmax, S)
    K = xr[:, 0].copy()
    d = (xr - K[:, None]) * mask[None, :, :, None]
    n = mask.sum(0)
    return K[:, :T], n[:T], d.sum(1, dtype=np.int64)[:, :T], (d.astype(np.int64) ** 2).sum(1)[:, :T]


def sums_precondition(case, x, sms):
    """Both fp32 thread sums are exact integers: |a1|, a2 < 2^24 (returns the largest a2 and |a1|)."""
    b = ppb(case.C)
    _, _, a1, a2 = thread_sums(x, stats_grid(case.P, case.C, sms), b)
    return int(a2.max()), int(np.abs(a1).max())


def stats_bounds(x, sms, gamma, beta, n_real, eps=EPS):
    """want (float64) and bound of every statistic output [items, C]: mean, var, uvar, inv_std, scale, shift."""
    items, P, C = x.shape
    b = ppb(C)
    mu, v, uv = exact_stats(x)
    K, n, a1, a2 = thread_sums(x, stats_grid(P, C, sms), b)
    nn = n[None, :, None].astype(np.float64)
    ed = np.abs(a1 / nn) * (2 * U + U * U)
    m2t = a2 - a1.astype(np.float64) ** 2 / nn
    em2 = np.abs(a1) * ed * (1 + U) + U * np.abs(m2t)
    mt = K + a1 / nn
    E_mu = (nn * ed).sum(1) / P + F64 * (np.abs(x).max(1) + 1)
    E_Pv = (em2 + 2 * nn * np.abs(mt - mu[:, None]) * ed + 2 * nn * ed * ed).sum(1) + \
        F64 * (nn * (np.abs(mt) + np.abs(mu[:, None])) ** 2).sum(1)
    E_v = E_Pv / P + 2.0 ** -50 * v
    E_uv = E_v * P / (P - 1)
    eps64 = float(np.float32(eps))
    inv = 1.0 / np.sqrt(v + eps64)
    E_is = 0.5 * (np.maximum(v - E_v, 0) + eps64) ** -1.5 * E_v + 2.0 ** -50 * inv
    real = np.arange(C) < n_real
    gm = np.zeros(C); gm[:n_real] = gamma
    bt = np.zeros(C); bt[:n_real] = beta
    sc = gm * inv
    E_sc = np.abs(gm) * E_is
    sh = np.where(real, bt - mu * sc, 0.0)
    E_sh = np.where(real, E_mu * (np.abs(sc) + E_sc) + (np.abs(mu) + E_mu) * E_sc + 2.0 ** -50 * np.abs(sh), 0.0)
    out = lambda w, e: (w, e + U * (np.abs(w) + e))
    return {"mean": out(mu, E_mu), "var": out(v, E_v), "uvar": out(uv, E_uv), "inv_std": out(inv, E_is),
            "scale": out(sc, E_sc), "shift": out(sh, E_sh)}


def check_stats(got, bounds, what, keys=None):
    """Every element of each output within its bound; returns {output: worst err / bound}."""
    worst = {}
    for k in keys or got:
        g = np.asarray(got[k], np.float64)
        w, e = bounds[k]
        err = np.abs(g - w)
        r = np.where(e > 0, err / np.where(e > 0, e, 1), np.where(err > 0, np.inf, 0))
        r = np.nan_to_num(r, nan=np.inf)
        if not r.max(initial=0) <= 1.0:
            ix = np.unravel_index(int(np.argmax(r)), r.shape)
            raise AssertionError(f"{what} {k}: {int((r > 1).sum())} of {r.size} elements beyond the bound, worst err/bound "
                                 f"{r.max():.3g} at [item={ix[0]}, c={ix[1]}]: got {g[ix]!r} want {w[ix]!r} bound {e[ix]!r}")
        worst[k] = float(r.max(initial=0))
    return worst


# ---------------------------------------------------------------- planted defects (the bounds' tightness)
def _stats_of(xs, divisor=None):
    """exact (mean, var) per channel of the integer rows xs [P, C], the sums divided by ``divisor`` (default P)."""
    P = xs.shape[0] if divisor is None else divisor
    S1 = xs.sum(0, dtype=np.int64).astype(object)
    S2 = (xs.astype(np.int64) ** 2).sum(0).astype(object)
    mu = [Fraction(int(s), P) for s in S1]
    v = [Fraction(int(s2), P) - m * m for s2, m in zip(S2, mu)]
    return np.array([float(m) for m in mu]), np.array([float(t) for t in v])


def defects(x):
    """{name: [items, P', C] integer rows or (rows, divisor)} of the planted defects of item 0's statistics: its last pixel dropped,
    its last pixel counted twice, its last pixel read from item 1 (when there is one), and P - 1 for P."""
    x0 = x[0]
    out = {"drop": x0[:-1], "double": np.concatenate([x0, x0[-1:]]), "p-1": (x0, x0.shape[0] - 1)}
    if x.shape[0] > 1:
        y = x0.copy()
        y[-1] = x[1, -1]
        out["neighbour"] = y
    return out


def defect_ratios(x, bounds, gamma, n_real, eps=EPS):
    """{defect: the largest change / bound over item 0's mean, var, inv_std and scale}."""
    C = x.shape[2]
    eps64 = float(np.float32(eps))
    gm = np.zeros(C); gm[:n_real] = gamma
    res = {}
    for name, d in defects(x).items():
        rows, div = d if isinstance(d, tuple) else (d, None)
        mu, v = _stats_of(rows, div)
        inv = 1.0 / np.sqrt(np.maximum(v, 0) + eps64)
        best = 0.0
        for k, val in (("mean", mu), ("var", v), ("inv_std", inv), ("scale", gm * inv)):
            w, e = bounds[k]
            ch = np.abs(val - w[0])
            r = np.where(e[0] > 0, ch / np.where(e[0] > 0, e[0], 1), np.where(ch > 0, np.inf, 0))
            best = max(best, float(r.max()))
        res[name] = best
    return res


# ---------------------------------------------------------------- running statistics
def f32(v):
    return np.asarray(v, np.float32)


def fma32(a, b, c):
    """fp32 fmaf(a, b, c) per element: a * b of two fp32 values is exact in float64, and TwoSum splits p + c exactly into
    s = fl64(p + c) and err.  Where err == 0 the one rounding of s to fp32 is the fused result.  Elsewhere |err| is below half an
    ulp of s, so rounding s to fp32 rounds p + c the same way unless s is itself the midpoint of two fp32 values: then the sign of
    err decides (an fp32 midpoint has 25 significant bits, so no other double lies between s and p + c)."""
    a, b, c = np.broadcast_arrays(f32(a), f32(b), f32(c))
    p = a.astype(np.float64) * b.astype(np.float64)
    cc = c.astype(np.float64)
    s = p + cc
    bb = s - p
    err = (p - (s - bb)) + (cc - bb)
    out = s.astype(np.float32)
    fix = err != 0
    if fix.any():
        f, sf, ef = out[fix], s[fix], err[fix]
        up, dn = np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))
        f64 = f.astype(np.float64)
        tie_up = sf == (f64 + up.astype(np.float64)) / 2          # s halfway between f and the fp32 above it
        tie_dn = sf == (f64 + dn.astype(np.float64)) / 2
        f = np.where(tie_up, np.where(ef > 0, up, f), f)
        f = np.where(tie_dn, np.where(ef < 0, dn, f), f)
        out[fix] = f
    return out


def round32(q):
    """The fp32 nearest (ties to even) to the rational q."""
    f = np.float32(float(q))
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    cands = [c for c in cands if np.isfinite(c)]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c).view(np.int32)) & 1))
    return np.float32(best)


def running_items_replay(rm, rv, mean, uvar, momentum):
    """bn_items_running_update: r = fmaf(x_i, m, fl((1 - m) r)) for items i = 0, 1, ... in order (mean / uvar [items, n_real])."""
    m = np.float32(momentum)
    om = np.float32(np.float32(1) - m)
    rm, rv = f32(rm).copy(), f32(rv).copy()
    for i in range(mean.shape[0]):
        rm = fma32(mean[i], m, om * rm)
        rv = fma32(uvar[i], m, om * rv)
    return rm, rv


def running_call_candidates(rv, var, P, momentum):
    """The call-wide running_var for the three fp32 values nearest fl(var * P / (P - 1)) (the kernel's unbiased variance is
    float64): [3, n_real], ascending in the unbiased value."""
    m = np.float32(momentum)
    om = np.float32(np.float32(1) - m)
    u = f32(np.asarray(var, np.float64) * P / (P - 1))
    cands = [np.nextafter(u, np.float32(-np.inf)), u, np.nextafter(u, np.float32(np.inf))]
    return np.stack([fma32(c, m, om * f32(rv)) for c in cands])


def running_bound(rm0, rv0, mean_b, uvar_b, momentum):
    """float64 (want, bound) of the running statistics after the items' updates in order, from the exact statistics (want, bound
    of the fp32 mean / uvar per item [items, n_real])."""
    m = float(np.float32(momentum))
    om = float(np.float32(1 - np.float32(momentum)))
    res = []
    for r0, (w, e) in ((rm0, mean_b), (rv0, uvar_b)):
        r, er = np.asarray(r0, np.float64), np.zeros(len(r0))
        for i in range(w.shape[0]):
            a, bb = om * r, m * w[i]
            r = a + bb
            er = om * er + m * e[i] + 2 * U * (np.abs(a) + np.abs(r) + m * e[i] + om * er)
        res.append((r, er))
    return res


# ---------------------------------------------------------------- apply
def apply_operands(items, P, C, residual, seed):
    """g [items, P, C] int16, scale / shift [items, C] fp32, residual [items, P, C] int16 or None.  Even channels: the
    cancellation channels (module docstring), 60 % of their pixels at the channel's centre with a zero residual; odd channels:
    any integer |g| <= 256, random scale and shift, residual |r| <= 256."""
    rng = np.random.default_rng(5000 + seed)
    even = (np.arange(C) % 2 == 0)
    centre = rng.integers(65, 193, (items, 1, C)) * rng.choice([-1, 1], (items, 1, C))
    g_c = centre + rng.integers(-8, 9, (items, P, C))
    g_c = np.where(rng.random((items, P, C)) < 0.6, centre, g_c)
    g_o = rng.integers(-256, 257, (items, P, C))
    g = np.where(even, g_c, g_o).astype(np.int16)
    s_c = f32(1.0 + (1.0 + rng.random((items, C))) * 2.0 ** -21)
    h_c = f32(-centre[:, 0, :] + rng.integers(-3, 4, (items, C)) * 2.0 ** -17)
    s_o = f32(rng.standard_normal((items, C)) * 2.0 ** rng.integers(-6, 3, (items, C)))
    h_o = f32(rng.standard_normal((items, C)) * 8)
    scale = np.where(even, s_c, s_o).astype(np.float32)
    shift = np.where(even, h_c, h_o).astype(np.float32)
    r = None
    if residual:
        r = rng.integers(-256, 257, (items, P, C))
        r = np.where(even & (g == centre), 0, r).astype(np.int16)
    return g, scale, shift, r


def bf16_bits(v32):
    """round-to-nearest-even bf16 bit patterns (int16) of fp32 values (no NaNs)."""
    u = np.asarray(v32, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16).view(np.int16)


def apply_replay(g, scale, shift, r, fused=False):
    """bf16 bits [items, P, C] of fl(fl(fl(g * scale) + shift) + r) (fused: fl(fma(g, scale, shift) + r), the contracted form)."""
    gf = g.astype(np.float32)
    sc, sh = scale[:, None, :], shift[:, None, :]
    v = fma32(gf, sc, sh) if fused else (gf * sc) + sh
    if r is not None:
        v = v + r.astype(np.float32)
    return bf16_bits(v)


def fused_difference_share(g, scale, shift, r):
    """Share of the elements whose bf16 result the contracted FMA would change."""
    return float((apply_replay(g, scale, shift, r) != apply_replay(g, scale, shift, r, fused=True)).mean())


def apply_cases(sms):
    """(items, P, C) of the apply checks: every C at ppb-edge pixel counts, strided grids, the training shapes and an item count
    above 16 * sms (apply grid 1 per item)."""
    cases = []
    for C in BN_CS:
        b = ppb(C)
        cases += [(1, 2, C), (2, b + 1, C), (3, 37, C)]
    cases += [(1, 16 * sms * BA_THREADS // 2 + 77, 16), (8, 256 * 256, 32), (64, 32 * 32, 256), (16 * sms + 1, 3, 16)]
    return cases


def apply_classes(case, sms):
    items, P, C = case
    cls = {f"C={C}", "per item" if items > 1 else "one item"}
    if P * (C // 8) > apply_grid(items, P, C, sms) * BA_THREADS:
        cls.add("grid-stride")
    if 16 * sms // items < 1:
        cls.add("cap<1")
    return cls
