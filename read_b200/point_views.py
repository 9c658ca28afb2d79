"""Point-cloud views: the reference viewer's non-neural render path (viewer.py:263-285, NNScene's GLSL program in
READ/gl/programs.py:60-300) on our rasterizer.  ``FrameRenderer.render_points`` / ``SceneRenderer.render_points`` draw one level-0
z-buffer of the frame (the exact winning point per pixel, 1-pixel or as point sprites) and ONE kernel (read_point_view) colours
every pixel from its winning point's attributes; the mode semantics and their arithmetic are stated in include/read_b200.h.

Tables are point-major ``[N, 4]`` f32 in original-id (or global-id) order: 16-byte rows, one sector per drawn pixel.  The PCA
colours (``--pca``, viewer.py:202-209) are computed here once per texture version, in float64 torch operations on the device."""
import ctypes
import math

import numpy as np
import torch

from . import _lib as L
from . import ops

MODES = ("color", "pca", "normals", "depth", "uv", "xyz", "label")
ID_MODES = ("color", "pca", "uv", "label")        # what a composed scene draws: the pixel's id alone identifies the point
_TABLE = {"color": "colors", "pca": "pca", "normals": "normals", "label": "normals"}


def check_view_args(mode, submode, point_size, clear_color):
    """ValueError, naming the argument, for an unknown mode, a submode outside 0..4, a point_size outside 1..64 or a clear colour
    that is not 4 finite values.  Returns the clear colour as a tuple of 4 floats."""
    if mode not in MODES:
        raise ValueError(f"read_b200: mode must be one of {MODES}, got {mode!r}")
    if isinstance(submode, bool) or not isinstance(submode, (int, np.integer)) or not 0 <= int(submode) <= 4:
        raise ValueError(f"read_b200: submode must be an integer in 0..4, got {submode!r}")
    try:
        ps = float(point_size)
    except (TypeError, ValueError):
        raise ValueError(f"read_b200: point_size must be a number in 1..{L.MAX_POINT_SIZE}, got {point_size!r}") from None
    if not 1.0 <= ps <= L.MAX_POINT_SIZE:
        raise ValueError(f"read_b200: point_size must be a number in 1..{L.MAX_POINT_SIZE}, got {point_size!r}")
    try:
        c = np.asarray(clear_color, dtype=np.float64)
    except (TypeError, ValueError):
        raise ValueError(f"read_b200: clear_color must be 4 finite values, got {clear_color!r}") from None
    if c.shape != (4,) or not np.all(np.isfinite(c)):
        raise ValueError(f"read_b200: clear_color must be 4 finite values, got {clear_color!r}")
    return tuple(float(v) for v in c)


def attribute_table(values, n, name, device):
    """``values`` ([n, 3] float array or tensor) -> [n, 4] f32 on ``device`` (fourth column 0).  ValueError for another shape or a
    non-finite value."""
    t = (values.detach() if torch.is_tensor(values) else torch.as_tensor(np.asarray(values))).to("cpu", torch.float32)
    if t.dim() != 2 or t.shape[0] != n or t.shape[1] != 3:
        raise ValueError(f"read_b200: {name} must be [{n}, 3], got {tuple(t.shape)}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"read_b200: {name} must be finite (no NaN or inf)")
    out = torch.zeros((n, 4), dtype=torch.float32)
    out[:, :3] = t
    return out.to(device)


def percentile(sorted_values, q):
    """``np.percentile(a, q)`` (method 'linear') of the values ``sorted_values`` (ascending, 1-D float64 tensor), as numpy
    computes it: virtual index (n - 1) * (q / 100) and its lerp, taken from the upper neighbour when the weight is >= 0.5."""
    n = sorted_values.numel()
    vi = (n - 1) * (q / 100.0)
    if vi >= n - 1:
        return sorted_values[n - 1]
    lo = math.floor(vi)
    g = vi - lo
    a, b = sorted_values[lo], sorted_values[lo + 1]
    d = b - a
    return b - d * (1 - g) if g >= 0.5 else a + d * g


def pca_colors(texture_):
    """The ``--pca`` colours of the descriptors ``texture_`` ([1, D, N] or [D, N]): the projections of the mean-free [N, D]
    descriptors onto the 3 eigenvectors of their covariance with the largest eigenvalues (each with its entry of largest
    magnitude positive, sklearn's svd_flip(u_based_decision=False)), then clip((x - p10) / (p90 - p10), 0, 1) with p10 / p90
    the linear percentiles of all 3N values (viewer.py:207-208).  float64 on the texture's device, rounded once; -> [N, 4] f32.
    The reference fits IncrementalPCA(3, batch_size=64), an approximation of this exact PCA."""
    t = texture_.detach()
    x = t.reshape(t.shape[-2], t.shape[-1]).t().to(torch.float64)
    if x.shape[0] < 1 or x.shape[1] < 3:
        raise ValueError(f"read_b200: the PCA view needs >= 1 point and >= 3 descriptor channels, got {tuple(x.shape)}")
    xc = x - x.mean(0)
    w, v = torch.linalg.eigh(xc.t() @ xc)
    v = v[:, torch.argsort(w, descending=True)[:3]]
    top = v.abs().argmax(0)
    v = v * torch.sign(v[top, torch.arange(3, device=v.device)])
    p = xc @ v
    flat = torch.sort(p.reshape(-1)).values
    p10, p90 = percentile(flat, 10), percentile(flat, 90)
    out = torch.zeros((p.shape[0], 4), dtype=torch.float32, device=p.device)
    out[:, :3] = ((p - p10) / (p90 - p10)).clamp(0, 1).to(torch.float32)
    return out


class ViewState:
    """What a renderer keeps for its point views: the 1-level pyramid they draw into and the PCA colours of the last texture
    version seen (the neural path's pyramid and fused-resolve state are separate)."""

    def __init__(self, W, H, device):
        self.W, self.H, self.device = W, H, device
        self.pyr = None
        self._pca_key, self._pca = None, None

    def pyramid(self):
        if self.pyr is None:
            self.pyr = ops.Pyramid(1, self.W, self.H, 1, self.device)
        self.pyr.clear()
        return self.pyr

    def pca(self, texture_):
        key = (texture_.data_ptr(), tuple(texture_.shape), texture_._version)
        if key != self._pca_key:
            self._pca, self._pca_key = pca_colors(texture_), key
        return self._pca


def table_for(mode, colors, normals, pca):
    """The [N, 4] table ``mode`` reads (``pca``: a callable giving the PCA colours), or None for modes that read none; ValueError
    when no scene provided it."""
    which = _TABLE.get(mode)
    if which is None:
        return None
    t = pca() if which == "pca" else (colors if which == "colors" else normals)
    if t is None:
        raise ValueError(f"read_b200: mode {mode!r} needs {which}; pass {which}= to the renderer (or add_scene)")
    return t


def view_desc(mode, submode, table, xyz, total_m, view_matrix, lo, hi, clear, flip_vertical):
    """The C ABI's read_point_view_desc of one view."""
    d = L.ReadPointViewDesc()
    d.mode = L.VIEW_MODES["color" if mode == "pca" else mode]
    d.submode = int(submode)
    if mode in ("color", "pca"):
        d.colors, d.n = table.data_ptr(), table.shape[0]
    elif mode in ("normals", "label"):
        d.normals, d.n = table.data_ptr(), table.shape[0]
    if xyz is not None:
        d.xyz = xyz.data_ptr()
        d.n = xyz.shape[0] if table is None else d.n
    if total_m is not None:
        view = np.asarray(view_matrix, dtype=np.float32)
        d.total_m[:] = [float(v) for v in np.asarray(total_m, np.float32).reshape(16)]
        d.m_view[:] = [float(v) for v in np.linalg.inv(view).astype(np.float32).reshape(16)]
        d.cam[:] = [float(v) for v in view[:3, 3]]
        d.lo[:], d.hi[:] = [float(v) for v in lo], [float(v) for v in hi]
    d.clear[:] = list(clear)
    d.flip_vertical = int(bool(flip_vertical))
    return d


def launch(pyr, d, out):
    """read_point_view of level 0 of the 1-view pyramid ``pyr`` with descriptor ``d`` into ``out`` ([H, W, 4] f32)."""
    L.check(L.load().read_point_view(pyr.buf.data_ptr(), pyr.H, pyr.W, ctypes.byref(d), out.data_ptr(), L.stream_ptr()))


def shade(pyr, mode, submode, table, xyz, total_m, view_matrix, lo, hi, clear, flip_vertical):
    """Colour level 0 of the 1-view pyramid ``pyr`` -> a fresh [H, W, 4] f32 tensor (read_point_view)."""
    out = torch.empty((pyr.H, pyr.W, 4), dtype=torch.float32, device=pyr.buf.device)
    launch(pyr, view_desc(mode, submode, table, xyz, total_m, view_matrix, lo, hi, clear, flip_vertical), out)
    return out
