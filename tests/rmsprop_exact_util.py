"""Per-element checks of the sparse descriptor optimizer (csrc/train.cu: sparse_rmsprop_kernel<REG>, square_avg_materialize_kernel,
compact_touched_kernel, scatter_pairs_kernel): operands, host replays and the case lists, shared by test_rmsprop_exact_host.py (no
GPU) and test_gpu_rmsprop_exact.py.

A point the step processes (touched, or every point in the REG instance) with dt = step - last_step:
    g  = touched ? grad : 0;  REG: g = fl(g + fl(k * p));  weight decay: g = fmaf(wd, p, g)
    q' = fmaf(decay, q, fl(fl((1 - alpha) * g) * g)),  decay = alpha if dt == 1 else powf(alpha, dt)
    p' = p - fl(fl(lr * g) / fl(sqrtf(q') + eps))
build.py compiles without fast-math, so the division and sqrtf are IEEE round-to-nearest and numpy's float32 ops replay them; an
fmaf is replayed by bn_fwd_exact_util.fma32 (an exact float64 product and a TwoSum split of the sum, rounded once to fp32).  At dt == 1 every output is replayed bit for bit.  powf is not correctly rounded: the CUDA C++ Programming Guide's table
of single-precision functions gives powf(x, y) a maximum error of 4 ulp over its full range, so for dt > 1 square_avg must lie
between the replays with decay at the fp32 values 5 ulp below and above the float64 alpha^dt (4 ulp plus the half ulp of rounding
alpha^dt to fp32), and the parameter must be the bit-exact replay on the kernel's own square_avg.
"""
import numpy as np

from bn_fwd_exact_util import f32, fma32

DS = (8, 1, 3, 16)
ALPHAS = (0.99, 0.9, 0.0)
GAPS = (1, 2, 7, 1000, 100_000)
POWF_ULP = 4
STEP = 200_000                      # > the largest gap: last_step stays >= 0


def big_n(sms):
    """The points one pass of the grid covers (grid_for: 16 CTAs of 256 threads per SM)."""
    return 16 * sms * 256


def cases(sms):
    """(D, N, variant, alpha) of the step checks: variant 'plain' (read_sparse_rmsprop_step), 'wd' (with weight decay), 'reg'
    (read_sparse_rmsprop_step_reg) and 'reg0' (the REG instance with a zero coefficient and weight decay, SparseRMSprop's
    weight-decay step)."""
    B = big_n(sms)
    out, k = [], 0
    variants = ("plain", "wd", "reg", "reg0")
    for D in DS:
        for N in (1, 255, 257, B - 1, B + 1):
            out.append((D, N, variants[k % 4], ALPHAS[k % 3])); k += 1
    for v in variants:
        for a in ALPHAS:
            out.append((8 if v != "wd" else 3, 257, v, a))
    out.append((1, 2 ** 24 + 1, "plain", 0.99))
    return out


def case_classes(case, sms):
    D, N, v, a = case
    cls = {f"D={D}", f"variant={v}", f"alpha={a}", "vector path" if D == 8 else "generic loop"}
    if N > big_n(sms):
        cls.add("grid-stride tail")
    if N in (1, 255, 257):
        cls.add(f"N={N}")
    if N == 2 ** 24 + 1:
        cls.add("N=2^24+1")
    return cls


def operands(D, N, seed, all_touched=False):
    """param_cn [D, N], grad_nd [N, D], square_avg [N, D] (fp32), touched [N] u8, last_step [N] int32 for step STEP: gaps from
    GAPS, about a third of the points touched, a tenth of the square_avg rows 0 with gradients ~1e-9 (eps dominates the
    denominator), some exact zeros; the untouched rows hold non-zero values the step must neither read nor clear."""
    rng = np.random.default_rng(seed)
    p = f32(rng.uniform(-1, 1, (D, N)))
    g = f32(rng.standard_normal((N, D)) * 0.3)
    g[rng.random((N, D)) < 0.05] = 0
    q = f32(rng.random((N, D)) * 0.05)
    tiny = rng.random(N) < 0.1
    q[tiny] = 0
    g[tiny] = f32(rng.standard_normal((int(tiny.sum()), D)) * 1e-9)
    touched = (rng.random(N) < 0.35).astype(np.uint8) if not all_touched else np.ones(N, np.uint8)
    last = (STEP - np.asarray(GAPS)[rng.integers(0, len(GAPS), N)]).astype(np.int32)
    return p, g, q, touched, last


def decay_range(alpha, dt):
    """fp32 (lo, hi) that contain powf(alpha, dt): 5 ulp either side of the float64 alpha^dt's fp32 rounding, not below 0."""
    true = np.float64(np.float32(alpha)) ** np.asarray(dt, np.float64)
    lo = hi = true.astype(np.float32)
    for _ in range(POWF_ULP + 1):
        lo = np.nextafter(lo, np.float32(0))
        hi = np.nextafter(hi, np.float32(np.inf))
    return np.maximum(lo, np.float32(0)), hi


def step_replay(p, g, q, touched, last, lr, alpha, eps, wd, k=None, step=STEP, q_kernel=None):
    """The step's outputs on the host: dict of param [D, N], shadow [N, D], grad, square_avg (lo and hi for dt > 1, and mid: the
    replay with decay = fp32(alpha^dt)), last_step, touched, and the mask of processed points.  k: the REG instance's coefficient (None: read_sparse_rmsprop_step).  With
    q_kernel [N, D] the parameter is replayed on the kernel's own square_avg (exact wherever that lies in [lo, hi])."""
    D, N = p.shape
    proc = np.ones(N, bool) if k is not None else touched.astype(bool)
    t = touched.astype(bool)
    pp = p.T[proc]
    gg = np.where(t[proc, None], g[proc], np.float32(0))
    if k is not None:
        gg = gg + np.float32(k) * pp
    if wd != 0:
        gg = fma32(np.float32(wd), pp, gg)
    a = np.float32(alpha)
    t2 = (np.float32(np.float32(1) - a) * gg) * gg
    dt = step - last[proc].astype(np.int64)
    lo, hi = decay_range(alpha, dt)
    one = dt == 1
    lo, hi = np.where(one, a, lo)[:, None], np.where(one, a, hi)[:, None]
    q_lo, q_hi = fma32(lo, q[proc], t2), fma32(hi, q[proc], t2)
    mid = np.where(one, a, (np.float64(a) ** dt.astype(np.float64)).astype(np.float32))[:, None]
    q_mid = fma32(mid, q[proc], t2)
    qq = q_kernel[proc] if q_kernel is not None else q_lo
    newp = pp - (np.float32(lr) * gg) / (np.sqrt(qq) + np.float32(eps))
    P, Q_lo, Q_hi, Q_mid, G = p.copy(), q.copy(), q.copy(), q.copy(), g.copy()
    P[:, proc] = newp.T
    Q_lo[proc], Q_hi[proc], Q_mid[proc] = q_lo, q_hi, q_mid
    G[t] = 0                                   # every touched row is processed and cleared; the others keep their values
    L = last.copy()
    L[proc] = step
    return {"param": P, "shadow": np.ascontiguousarray(P.T), "grad": G, "sq_lo": Q_lo, "sq_hi": Q_hi, "sq_mid": Q_mid, "last": L,
            "touched": np.zeros_like(touched), "proc": proc}


def dense_replay(q, last, step, alpha):
    """read_square_avg_dense: [D, N] (lo, hi) of decay * square_avg, decay = 1 for dt <= 0 (exact) else powf(alpha, dt)."""
    dt = step - last.astype(np.int64)
    lo, hi = decay_range(alpha, np.maximum(dt, 1))
    keep = dt <= 0
    lo, hi = np.where(keep, np.float32(1), lo)[:, None], np.where(keep, np.float32(1), hi)[:, None]
    return (lo * q).T.copy(), (hi * q).T.copy()
