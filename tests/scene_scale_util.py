"""Host restatements for the culled segmented rasterizer (ops.raster_project_segments_culled): the kernel's per-point float32
frustum test, its float64 chunk-cull rule and the unit table it compacts.  Shared by the host and GPU test files."""
import numpy as np

TWO_M21, TWO_M140, TWO_126 = 2.0 ** -21, 2.0 ** -140, 2.0 ** 126


def f32_fma(a, b, c):
    """fmaf(a, b, c) on float32 arrays: a*b + c rounded once to float32.  a*b is exact in float64; s + e == a*b + c exactly
    (TwoSum), and rounding s to float32 is correct except at a float32 midpoint, where e decides."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    with np.errstate(all="ignore"):
        p = a.astype(np.float64) * b.astype(np.float64)
        c64 = c.astype(np.float64)
        s = p + c64
        bb = s - p
        e = (p - (s - bb)) + (c64 - bb)
        r = s.astype(np.float32)
        d = s - r.astype(np.float64)
        toward = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        half = (toward.astype(np.float64) - r.astype(np.float64)) * 0.5
        mid = (d != 0) & (d == half) & np.isfinite(s)
        fix = mid & (np.sign(e) == np.sign(d))
        r = np.where(fix, toward, r)
        r = np.where((s == 0) & (e != 0), e.astype(np.float32), r)
        r = np.where(np.isfinite(s), r, (p + c64).astype(np.float32))
    return r.astype(np.float32)


def clip_coords(m, pts):
    """The kernel's clip_point dot products: m [4,4] float32 rows, pts [n,3] float32 -> c [n,4] float32."""
    m = np.asarray(m, np.float32)
    x, y, z = (np.asarray(pts, np.float32)[:, j] for j in range(3))
    out = []
    with np.errstate(all="ignore"):
        for i in range(4):
            t = x * m[i, 0]
            t = f32_fma(y, np.full_like(y, m[i, 1]), t)
            t = f32_fma(z, np.full_like(z, m[i, 2]), t)
            out.append((t + m[i, 3]).astype(np.float32))
    return np.stack(out, 1)


def point_in(m, pts):
    """clip_point's ``in``: |c_i| <= |c_3| for i = 0, 1, 2 in float32 (NaN fails)."""
    c = clip_coords(m, pts)
    aw = np.abs(c[:, 3])
    with np.errstate(invalid="ignore"):
        return (np.abs(c[:, 0]) <= aw) & (np.abs(c[:, 1]) <= aw) & (np.abs(c[:, 2]) <= aw)


def box_culled(m, lo, hi):
    """The cull rule of raster.cu's box_culled, same float64 operations in the same order.  m [4,4] float32; lo, hi [n,3] finite
    float32 -> [n] bool: True when the box is provably outside the clip volume of this view."""
    m = np.asarray(m, np.float32).astype(np.float64)
    lo = np.asarray(lo, np.float32).astype(np.float64).reshape(-1, 3)
    hi = np.asarray(hi, np.float32).astype(np.float64).reshape(-1, 3)
    n = lo.shape[0]
    if not np.all(np.isfinite(m)):
        return np.zeros(n, bool)
    A = np.maximum(np.abs(lo), np.abs(hi))
    S = []
    for r in range(4):
        s = np.full(n, abs(m[r, 3]))
        for j in range(3):
            s = s + abs(m[r, j]) * A[:, j]
        S.append(s)
    corners = [[(hi if (k >> j) & 1 else lo)[:, j] for j in range(3)] for k in range(8)]
    out = np.zeros(n, bool)
    for i in range(3):
        tot = S[i] + S[3]
        ok = tot < TWO_126
        delta = tot * TWO_M21 + TWO_M140
        above = np.ones(n, bool)
        below = np.ones(n, bool)
        for x, y, z in corners:
            ci = ((m[i, 0] * x + m[i, 1] * y) + m[i, 2] * z) + m[i, 3]
            c3 = ((m[3, 0] * x + m[3, 1] * y) + m[3, 2] * z) + m[3, 3]
            a, b = ci - c3, ci + c3
            above &= (a > delta) & (b > delta)
            below &= (a < -delta) & (b < -delta)
        out |= ok & (above | below)
    return out


def unit_dropped(seg_m_s, lo, hi):
    """Whether the kernel drops the units of these boxes under one segment's matrices seg_m_s [B,4,4]: an empty box always, a
    non-finite box never, otherwise when every view culls it."""
    lo = np.asarray(lo, np.float32).reshape(-1, 3)
    hi = np.asarray(hi, np.float32).reshape(-1, 3)
    empty = ~(lo[:, 0] <= hi[:, 0])
    finite = np.all(np.isfinite(lo) & np.isfinite(hi), 1)
    drop = np.ones(lo.shape[0], bool)
    for b in range(seg_m_s.shape[0]):
        drop &= box_culled(seg_m_s[b], np.where(finite[:, None], lo, 0), np.where(finite[:, None], hi, 0))
    return empty | (finite & drop)


def kept_units(store, seg_m, visible=None):
    """[(physical chunk, matrix slot)] of the units the culled rasterizer draws, in its order (segment, then chunk)."""
    boxes = store.boxes.cpu().numpy()
    vis = list(store.visible)[:store.nseg] if visible is None else list(visible)
    out = []
    for s in range(store.nseg):
        f, c = store.first_chunk[s], store.chunks[s]
        if not vis[s] or c == 0:
            continue
        drop = unit_dropped(np.asarray(seg_m[s]), boxes[f:f + c, :3], boxes[f:f + c, 3:])
        out += [(f + j, s) for j in range(c) if not drop[j]]
    return out
