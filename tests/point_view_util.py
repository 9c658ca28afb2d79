"""Host restatements of the point-cloud views (read_b200.point_views, read_point_view in include/read_b200.h): the per-mode colour
in numpy float32, operation by operation in the kernel's order, the same colours in float64 straight from the GLSL formulas
(READ/gl/programs.py:104-160), and the exact PCA of the ``--pca`` colours through numpy's SVD.  Shared by the host and GPU tests."""
import numpy as np

from scene_scale_util import clip_coords

F = np.float32
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def normalize32(v):
    """v [..., 3] float32 -> v_i / sqrt((v0*v0 + v1*v1) + v2*v2), each operation rounded to float32."""
    v = np.asarray(v, F)
    with np.errstate(all="ignore"):
        s = np.sqrt((v[..., 0] * v[..., 0] + v[..., 1] * v[..., 1]) + v[..., 2] * v[..., 2])
        return (v / s[..., None]).astype(F)


def _half(v):
    return (np.asarray(v, F) * F(0.5) + F(0.5)).astype(F)


def _dot32(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def view_frame(view_matrix):
    """(m_view, cam) of a view matrix: np.linalg.inv of its float32 copy (as total_matrix forms it) and its translation."""
    view = np.asarray(view_matrix, F)
    return np.linalg.inv(view).astype(F), view[:3, 3].copy()


def shade32(mode, submode, ids, colors=None, normals=None, xyz=None, total_m=None, view_matrix=None, lo=None, hi=None):
    """RGB [P, 3] float32 of the points ``ids`` ([P] int64, ids < N) under ``mode`` / ``submode``, as read_point_view computes
    them.  colors / normals: [N, 3]; xyz [N, 3]; total_m [4, 4] float32."""
    ids = np.asarray(ids, np.int64)
    P = ids.shape[0]
    z = np.zeros(P, F)
    with np.errstate(all="ignore"):
        if mode in ("color", "pca"):
            return np.asarray(colors, F)[ids, :3].copy()
        if mode == "uv":
            return np.stack([ids.astype(F) if submode == 0 else z, z, z], 1)
        if mode == "label":
            return np.stack([(np.asarray(normals, F)[ids, 0] / F(255)).astype(F), z, z], 1)
        p = None if xyz is None else np.asarray(xyz, F)[ids]
        if mode == "depth":
            c2 = clip_coords(np.asarray(total_m, F), p)[:, 2]
            return np.stack([c2, c2, c2], 1)
        if mode == "xyz":
            lo, hi = np.asarray(lo, F), np.asarray(hi, F)
            return ((p - lo) / ((hi - lo) + F(1e-9))).astype(F)
        assert mode == "normals", mode
        n = np.asarray(normals, F)[ids, :3]
        m_view, cam = view_frame(view_matrix)
        if submode == 0:
            return _half(n)
        if submode == 1:
            d = normalize32(cam - p)
            k = (F(2) * _dot32(n, d)).astype(F)
            return _half(normalize32(d - k[:, None] * n))
        if submode == 2:
            w = (cam + n).astype(F)
            rows = [(_dot32(np.broadcast_to(m_view[i, :3], w.shape), w) + m_view[i, 3]).astype(F) for i in range(3)]
            return _half(normalize32(np.stack(rows, 1)))
        if submode == 3:
            return _half(normalize32(cam - p))
        return n.copy()


def shade64(mode, submode, ids, colors=None, normals=None, xyz=None, total_m=None, view_matrix=None, lo=None, hi=None):
    """The same colours in float64 from the GLSL formulas (reflect, normalize, mat4 * vec4), for ulp comparisons."""
    ids = np.asarray(ids, np.int64)
    D = np.float64
    norm = lambda v: v / np.linalg.norm(v, axis=-1, keepdims=True)
    view = np.asarray(view_matrix, F).astype(D) if view_matrix is not None else None
    if mode == "normals":
        n = np.asarray(normals, F)[ids, :3].astype(D)
        cam = view[:3, 3]
        if submode == 0:
            return n * 0.5 + 0.5
        if submode == 1:
            d = norm(cam - np.asarray(xyz, F)[ids].astype(D))
            return norm(d - 2.0 * np.sum(n * d, 1, keepdims=True) * n) * 0.5 + 0.5
        if submode == 2:
            m_view = np.linalg.inv(np.asarray(view_matrix, F)).astype(F).astype(D)
            w = np.concatenate([cam + n, np.ones((n.shape[0], 1))], 1)
            return norm((w @ m_view.T)[:, :3]) * 0.5 + 0.5
        if submode == 3:
            return norm(cam - np.asarray(xyz, F)[ids].astype(D)) * 0.5 + 0.5
        return n
    if mode == "xyz":
        p = np.asarray(xyz, F)[ids].astype(D)
        lo, hi = np.asarray(lo, F).astype(D), np.asarray(hi, F).astype(D)
        return (p - lo) / (hi - lo + 1e-9)
    if mode == "depth":
        p = np.asarray(xyz, F)[ids].astype(D)
        c2 = p @ np.asarray(total_m, F)[2, :3].astype(D) + D(np.asarray(total_m, F)[2, 3])
        return np.stack([c2] * 3, 1)
    return shade32(mode, submode, ids, colors, normals).astype(D)


def view_rgba(keys, flip_vertical=False, clear=(0., 0., 0., 1.), **kw):
    """The whole view: keys [H, W] uint64 (the level-0 z-buffer, EMPTY where no point) -> [H, W, 4] float32, with rows flipped
    as read_point_view flips them."""
    keys = np.asarray(keys, np.uint64)
    H, W = keys.shape
    empty = keys == EMPTY
    ids = (keys & np.uint64(0xFFFFFFFF)).astype(np.int64)
    out = np.empty((H, W, 4), F)
    out[...] = np.asarray(clear, F)
    rgb = shade32(ids=ids[~empty], **kw)
    out[~empty, :3] = rgb
    out[~empty, 3] = 1.0
    return out[::-1].copy() if flip_vertical else out


def keys_from_maps(index, depth):
    """(index [H, W] f32/int, depth [H, W] f32) maps of the oracle (depth 0 = empty) -> the z-buffer keys the views shade."""
    empty = np.asarray(depth) == 0
    k = (np.asarray(depth, F).view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.asarray(index).astype(np.int64).astype(np.uint64)
    return np.where(empty, EMPTY, k)


def pca_exact(tex_dn):
    """The exact PCA colours of [D, N] descriptors through numpy's SVD: the mean-free data's right singular vectors, each flipped
    so its entry of largest magnitude is positive (svd_flip(u_based_decision=False)), the projections normalised with
    np.percentile 10 / 90 over all 3N values and clipped to [0, 1].  float64 [N, 3]."""
    x = np.asarray(tex_dn, np.float64).T
    xc = x - x.mean(0)
    _, _, vt = np.linalg.svd(xc, full_matrices=False)
    v = vt[:3]
    v = v * np.sign(v[np.arange(3), np.abs(v).argmax(1)])[:, None]
    p = xc @ v.T
    p10, p90 = np.percentile(p, 10), np.percentile(p, 90)
    return np.clip((p - p10) / (p90 - p10), 0, 1)


def separated_descriptors(n, seed):
    """[1, 8, n] float32 descriptors with well separated covariance eigenvalues (a random rotation of scaled axes)."""
    rng = np.random.default_rng(seed)
    scale = np.array([3.0, 2.0, 1.3, 0.6, 0.3, 0.2, 0.1, 0.05])
    q, _ = np.linalg.qr(rng.standard_normal((8, 8)))
    x = (rng.standard_normal((n, 8)) * scale) @ q.T + rng.standard_normal(8)
    return x.T[None].astype(np.float32)
