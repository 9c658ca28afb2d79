"""Host restatement of the cylindrical panorama rasterizer (read_b200.panorama, DESIGN.md §4.4), in numpy float32 / float64 with
the kernels' operations in their order: the per-point projection, the level-0 keys by a 64-bit min, levels 1-3 by the 2x2 min,
and the radial chunk-cull rule.  Shared by the host and GPU test files."""
import numpy as np

from scene_scale_util import clip_coords, TWO_M140

F32 = np.float32
EMPTY = np.uint64(0x7FFFFFFFFFFFFFFF)             # ZBUF_EMPTY
PI_F, HALF_PI_F = F32(np.pi), F32(np.pi / 2)
# pano_atan2's polynomial in s^2, highest power first (raster.cu)
ATAN_COEF = [F32(float.fromhex(h)) for h in ("0x1.be9836p-8", "-0x1.135a34p-5", "0x1.462d4p-4", "-0x1.0f077cp-3",
                                                "0x1.95aab2p-3", "-0x1.552b84p-2", "0x1.ffff7ep-1")]


def atan2_f32(x, f):
    """raster.cu's pano_atan2 on float32 arrays."""
    x, f = np.asarray(x, F32), np.asarray(f, F32)
    with np.errstate(all="ignore"):
        ax, af = np.abs(x), np.abs(f)
        lo, hi = np.minimum(ax, af), np.maximum(ax, af)
        s = np.where(hi > 0, lo / np.where(hi > 0, hi, F32(1)), F32(0)).astype(F32)
        s2 = (s * s).astype(F32)
        p = np.full_like(s, ATAN_COEF[0])
        for c in ATAN_COEF[1:]:
            p = ((p * s2).astype(F32) + c).astype(F32)
        t = (p * s).astype(F32)
        t = np.where(ax > af, (HALF_PI_F - t).astype(F32), t)
        t = np.where(f < 0, (PI_F - t).astype(F32), t)
        return np.where(np.signbit(x), -t, t).astype(F32)


def project(m, pts, ids, pano):
    """One view: m [4,4] float32 world -> camera, pts [n,3] float32, ids [n] -> (vis, key uint64, idx0, two, idx1) as pano_project
    computes them, for pano (a read_b200.panorama.Panorama)."""
    c = pano.constants()
    W, M, H, full = pano.width, pano.margin, pano.height, pano.full
    wp = W + 2 * M
    cc = clip_coords(m, pts)
    x, y, f = cc[:, 0], cc[:, 1], (-cc[:, 2]).astype(F32)
    with np.errstate(all="ignore"):
        r = np.sqrt(((x * x).astype(F32) + (f * f).astype(F32)).astype(F32)).astype(F32)
        v = ((c["t_hi"] - (y / r).astype(F32)).astype(F32) * c["k_h"]).astype(F32)
        u = ((atan2_f32(x, f) + c["theta_half"]).astype(F32) * c["k_w"]).astype(F32)
        vis = (r >= c["znear"]) & (r <= c["zfar"]) & (v >= 0) & (v < F32(H)) & (u >= 0)
        if not full:
            vis &= u < F32(W)
        col = np.where(vis, u, 0).astype(np.int64)
        row = np.where(vis, v, 0).astype(np.int64)
    if full:
        col = np.where(col == W, 0, col)
    vis &= col < W
    two = vis & full & ((col < M) | (col >= W - M))
    key = (r.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.asarray(ids, np.uint64)
    idx0 = row * wp + col + M
    idx1 = idx0 + np.where(col < M, W, -W)
    return vis, key, idx0, two, idx1


def level0(pts, ids, view_m, pano):
    """[B, H, W + 2M] uint64 level-0 keys for the views view_m [B,4,4] (EMPTY where no point lands)."""
    view_m = np.asarray(view_m, F32).reshape(-1, 4, 4)
    wp = pano.plane_width
    out = np.full((view_m.shape[0], pano.height * wp), EMPTY, np.uint64)
    for b, m in enumerate(view_m):
        vis, key, i0, two, i1 = project(m, pts, ids, pano)
        np.minimum.at(out[b], i0[vis], key[vis])
        np.minimum.at(out[b], i1[two], key[two])
    return out.reshape(-1, pano.height, wp)


def derive(z, L=4):
    """Levels 0 .. L-1 from level 0 [B, H, W]: each the 2x2 min of the one before."""
    out = [z]
    for _ in range(1, L):
        a = out[-1]
        out.append(np.minimum(np.minimum(a[:, 0::2, 0::2], a[:, 0::2, 1::2]), np.minimum(a[:, 1::2, 0::2], a[:, 1::2, 1::2])))
    return out


def pyramid(pts, ids, view_m, pano, L=4):
    return derive(level0(pts, ids, view_m, pano), L)


def box_beyond(m, lo, hi, zfar):
    """raster.cu's box_beyond, same float64 operations in the same order.  m [4,4] float32, lo / hi [n,3] finite float32, zfar the
    float32 zfar -> [n] bool: True when every point of the box provably has a float32 radial distance above zfar."""
    m = np.asarray(m, F32).astype(np.float64)
    lo = np.asarray(lo, F32).astype(np.float64).reshape(-1, 3)
    hi = np.asarray(hi, F32).astype(np.float64).reshape(-1, 3)
    n = lo.shape[0]
    if not np.all(np.isfinite(m[:3])):
        return np.zeros(n, bool)
    zfar = float(F32(zfar))
    c = (lo + hi) * 0.5
    d = (hi - lo) * 0.5
    e2 = np.zeros(n)
    for j in range(3):
        e2 = e2 + d[:, j] * d[:, j]
    A = np.maximum(np.abs(lo), np.abs(hi))
    S, nn = np.zeros(n), 0.0
    for r in (0, 2):
        S = S + abs(m[r, 3])
        for j in range(3):
            S = S + abs(m[r, j]) * A[:, j]
            nn = nn + m[r, j] * m[r, j]
    xc = ((m[0, 0] * c[:, 0] + m[0, 1] * c[:, 1]) + m[0, 2] * c[:, 2]) + m[0, 3]
    zc = ((m[2, 0] * c[:, 0] + m[2, 1] * c[:, 1]) + m[2, 2] * c[:, 2]) + m[2, 3]
    reach = np.sqrt(e2) * np.sqrt(nn)
    delta = (S + zfar) * 2.0 ** -20 + TWO_M140
    return (S < 2.0 ** 126) & (np.sqrt(xc * xc + zc * zc) - reach > zfar + delta)


def kept_units(store, seg_m, pano, visible=None):
    """[(physical chunk, matrix slot)] of the units the culled panorama rasterizer draws, in its order (segment, then chunk)."""
    boxes = store.boxes.cpu().numpy()
    vis = list(store.visible)[:store.nseg] if visible is None else list(visible)
    out = []
    for s in range(store.nseg):
        f, cnt = store.first_chunk[s], store.chunks[s]
        if not vis[s] or cnt == 0:
            continue
        lo, hi = boxes[f:f + cnt, :3], boxes[f:f + cnt, 3:]
        empty = ~(lo[:, 0] <= hi[:, 0])
        finite = np.all(np.isfinite(lo) & np.isfinite(hi), 1)
        drop = np.ones(cnt, bool)
        for m in np.asarray(seg_m[s]):
            drop &= box_beyond(m, np.where(finite[:, None], lo, 0), np.where(finite[:, None], hi, 0), pano.constants()["zfar"])
        drop = empty | (finite & drop)
        out += [(f + j, s) for j in range(cnt) if not drop[j]]
    return out


def segmented_pyramid(store, seg_m, pano, L=4):
    """The pyramid of a SegmentedPoints store: every visible segment's points under its own matrices (world -> camera)."""
    pts4 = store.pts4.cpu().numpy()
    xyz, ids = pts4[:, :3], pts4[:, 3].view(np.uint32)
    B = np.asarray(seg_m).shape[1]
    wp = pano.plane_width
    z = np.full((B, pano.height * wp), EMPTY, np.uint64)
    for s in range(store.nseg):
        if not store.visible[s]:
            continue
        r0, r1 = store.first_chunk[s] * 1024, (store.first_chunk[s] + store.chunks[s]) * 1024
        zs = level0(xyz[r0:r1], ids[r0:r1], np.asarray(seg_m[s]), pano).reshape(B, -1)
        z = np.minimum(z, zs)
    return derive(z.reshape(B, pano.height, wp), L)


# ------------------------------------------------------------------------------------------------------------------------------
# Edge point sets.  Every set is drawn with EDGE_VIEW, whose float32 dot products return the point's coordinates exactly (row 0
# carries -0 so that x = -0 survives for points behind the camera with y > 0); tests/test_panorama_host.py proves each planted
# outcome with the kernel's arithmetic, tests/test_gpu_panorama.py draws the sets.
EDGE_VIEW = np.array([[1, -0.0, -0.0, -0.0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1]], F32)


def _ordered(v):
    """float32 -> int64 that orders like the float (+0 above -0)."""
    b = np.asarray(v, F32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7FFFFFFF) - 1, b)


def _from_ordered(k):
    k = np.int64(k)
    b = k if k >= 0 else -(k + 1) | -0x80000000
    return np.array([b], np.int64).astype(np.int32).view(F32)[0]


def _crossing(fn, a, b):
    """fn: float32 -> bool, False at a and True at b, monotone between them along the float32 order (a < b or a > b).  Returns the
    adjacent pair (last False, first True)."""
    ka, kb = _ordered(F32(a)), _ordered(F32(b))
    assert not fn(F32(a)) and fn(F32(b))
    while abs(kb - ka) > 1:
        km = (ka + kb) // 2
        if fn(_from_ordered(km)):
            kb = km
        else:
            ka = km
    return _from_ordered(ka), _from_ordered(kb)


def one(p, pano):
    """(vis, col, row, two) of one point under EDGE_VIEW."""
    vis, key, i0, two, i1 = project(EDGE_VIEW, np.asarray(p, F32).reshape(1, 3), [0], pano)
    wp = pano.plane_width
    return bool(vis[0]), int(i0[0] % wp) - pano.margin, int(i0[0] // wp), bool(two[0])


def _column_pair(k, pano, y=0.0, d=10.0):
    """Two points with adjacent float32 coordinates whose columns are k - 1 and k (k in 1 .. W - 1), at distance about d."""
    c = pano.constants()
    theta = (k / float(c["k_w"])) - float(c["theta_half"])

    def col(p):                          # int(u) before the seam wraps it
        x, y, z = (np.asarray([v], F32) for v in p)
        f = (-z).astype(F32)
        return int(((atan2_f32(x, f) + c["theta_half"]).astype(F32) * c["k_w"]).astype(F32)[0])
    if abs(theta) <= np.pi / 4:          # ahead: x grows with theta
        lo, hi = _crossing(lambda x: col((x, y, -d)) >= k, -2 * d, 2 * d)
        return (lo, y, -d), (hi, y, -d)
    if abs(theta) <= 3 * np.pi / 4:      # to the side: theta falls as f (= -z) grows
        s = d if theta > 0 else -d
        lo, hi = _crossing(lambda z: col((s, y, z)) >= k, -2 * d, 2 * d) if theta > 0 else \
            _crossing(lambda z: col((s, y, z)) >= k, 2 * d, -2 * d)
        return (s, y, lo), (s, y, hi)
    # behind (f < 0): theta falls as x grows, on either side of x = 0
    if theta > 0:
        lo, hi = _crossing(lambda x: col((x, y, d)) >= k, 2 * d, F32(0.0))
    else:
        lo, hi = _crossing(lambda x: col((x, y, d)) >= k, F32(-0.0), -2 * d)
    return (lo, y, d), (hi, y, d)


def edge_set(pano):
    """(pts [n,3] float32, labels [n], expect [n] of (vis, col, row) or None) for one panorama: the azimuths 0, +-pi/2, +-pi;
    adjacent points either side of column boundaries, including those of columns M - 1, M, W - M - 1, W - M and the seam; rows at
    v = 0 and just below H; radial distances at znear, zfar and one ulp beyond, and 0; depth ties."""
    W, H, M = pano.width, pano.height, pano.margin
    c = pano.constants()
    pts, labels, expect = [], [], []

    def add(p, label, want=None):
        pts.append(np.asarray(p, F32))
        labels.append(label)
        expect.append(want)

    d = F32(10.0)
    # E1 azimuths: theta = 0, +-pi/2 (f = 0), +-pi (x = +-0 behind the camera, y > 0 keeps the sign through EDGE_VIEW)
    for p in [(0.0, 0.0, -d), (d, 0.0, 0.0), (-d, 0.0, 0.0), (0.0, 0.5, d), (-0.0, 0.5, d)]:
        add(p, "E1")
    # E2 column boundaries
    ks = {1, 2, 37, W // 4, W // 2, W // 2 + 1, 3 * W // 4, W - 2, W - 1}
    if M:
        ks |= {M - 1, M, M + 1, W - M - 1, W - M, W - M + 1}
    for k in sorted(k for k in ks if 1 <= k <= W - 1):
        lo, hi = _column_pair(k, pano)
        add(lo, "E2", (True, k - 1, None))
        add(hi, "E2", (True, k, None))
    # E3 rows: v = 0 exactly (y / r = t_hi with r = 1), above the top row, and the last float32 v below H
    add((0.0, c["t_hi"], -1.0), "E3", (True, None, 0))
    add((0.0, np.nextafter(c["t_hi"], F32(np.inf)), -1.0), "E3", (False, None, None))
    y_lo, y_hi = _crossing(lambda y: one((0.0, y, -1.0), pano)[0], F32(-1e6), c["t_hi"])   # first visible y from below
    add((0.0, y_lo, -1.0), "E3", (False, None, None))
    add((0.0, y_hi, -1.0), "E3", (True, None, H - 1))
    # E4 radial distances: r = sqrt(rn(f * f)) == |f| exactly
    zn, zf = c["znear"], c["zfar"]
    for f, vis in [(zn, True), (np.nextafter(zn, F32(0)), False), (zf, True), (np.nextafter(zf, F32(0)), True),
                   (np.nextafter(zf, F32(np.inf)), False)]:
        add((0.0, 0.0, -f), "E4", (vis, None, None))
    add((0.0, 0.0, 0.0), "E4", (False, None, None))
    # E6 depth ties: equal r (it depends on x and f only) in one pixel, and in a seam pixel and its copy
    for k in ([W // 2] + ([M // 2, W - M // 2] if M else [])):
        lo, hi = _column_pair(k, pano)
        for dy in (0.0, 1e-6):
            add((hi[0], hi[1] + dy, hi[2]), "E6", (True, k, None))
    return np.stack(pts).astype(F32), labels, expect


def edge_store_rows(pts, ids, nan_rows=64):
    """The rows of a hand-laid store: the points with NaN padding rows spread among them, and every seam point next to an
    ordinary one, so that ring blocks mix one- and two-splat lanes.  -> (xyz [m,3] f32, ids [m] uint32); NaN rows carry id 0."""
    n = pts.shape[0]
    rows, rid = [], []
    for i in range(n):
        rows.append(pts[i])
        rid.append(ids[i])
        if i % 3 == 0 and nan_rows > 0:
            rows.append(np.full(3, np.nan, F32))
            rid.append(0)
            nan_rows -= 1
    for _ in range(nan_rows):
        rows.append(np.full(3, np.nan, F32))
        rid.append(0)
    return np.stack(rows).astype(F32), np.asarray(rid, np.uint32)
