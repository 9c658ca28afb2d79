"""Cylindrical panoramas (DESIGN.md §4.4): a second projection of the rasterizer, up to 360 degrees in one image.

Columns are uniform in azimuth and rows linear in tan(elevation), so every column is a pinhole column (vertical lines stay
straight) and the horizontal pixel density is the same all around.  ``Panorama`` holds the geometry and turns it into the float32
constants the kernels take (include/read_b200.h, read_panorama_desc); ``raster_panorama_sorted`` and
``raster_panorama_segments_culled`` draw level 0 of a (W + 2M) x H pyramid from a ``ops.SortedPoints`` or ``ops.SegmentedPoints``
store.  At 360 degrees the plane carries M wrapped columns on each side, so the net sees the scene across the seam;
``NetAndTexture.render(..., panorama=p)`` crops them off its output."""
import ctypes
import math

import numpy as np

from . import _lib as L
from . import ops

DEFAULT_MARGIN = 128          # wrapped columns on each side of a 360-degree panorama (capped at half the width)


def _mult16(v, name, positive=True):
    if isinstance(v, bool) or int(v) != v or v % 16 or (positive and v <= 0) or v < 0:
        raise ValueError(f"read_b200: the panorama's {name} must be a {'positive ' if positive else ''}multiple of 16, got {v}")
    return int(v)


class Panorama:
    """A cylindrical camera: ``width`` x ``height`` pixels covering ``hfov_deg`` (at most 360) degrees of azimuth, centred on the
    camera's forward axis (-z), and elevations ``elevation_deg = (lo, hi)`` (-89 < lo < hi < 89) from the bottom row to the top
    one, with radial distances from ``znear`` to ``zfar``.  ``margin``: the wrapped columns drawn on each side of a 360-degree
    panorama (a multiple of 16, at most width / 2; default ``DEFAULT_MARGIN`` capped at width / 2); 0 below 360 degrees.
    ``width``, ``height`` and the margin are multiples of 16, the net's granularity.  ValueError for anything else."""

    def __init__(self, width, height, hfov_deg=360.0, elevation_deg=(-30.0, 30.0), znear=0.1, zfar=1000.0, margin=None):
        self.width = _mult16(width, "width")
        self.height = _mult16(height, "height")
        if self.width > L.PANORAMA_MAX_WIDTH:
            raise ValueError(f"read_b200: the panorama is at most {L.PANORAMA_MAX_WIDTH} pixels wide, got {width}")
        self.hfov_deg = float(hfov_deg)
        if not 0.0 < self.hfov_deg <= 360.0:
            raise ValueError(f"read_b200: the panorama's horizontal field of view must lie in (0, 360] degrees, got {hfov_deg}")
        self.full = self.hfov_deg == 360.0
        lo, hi = (float(e) for e in elevation_deg)
        if not -89.0 < lo < hi < 89.0:
            raise ValueError(f"read_b200: the elevations must satisfy -89 < lo < hi < 89 degrees, got {elevation_deg}")
        self.elevation_deg = (lo, hi)
        self.znear, self.zfar = float(znear), float(zfar)
        if not (math.isfinite(self.znear) and math.isfinite(self.zfar) and 0.0 < self.znear < self.zfar):
            raise ValueError(f"read_b200: the panorama needs finite 0 < znear < zfar, got {znear}, {zfar}")
        if margin is None:
            margin = min(DEFAULT_MARGIN, self.width // 2 // 16 * 16) if self.full else 0
        self.margin = _mult16(margin, "margin", positive=False)
        if 2 * self.margin > self.width:
            raise ValueError(f"read_b200: the margin {margin} is more than half the width {width}")
        if self.margin and not self.full:
            raise ValueError("read_b200: a panorama below 360 degrees has no margin (nothing wraps around)")

    @property
    def plane_width(self):
        """Width of the rendered level 0 and of the net's input: width + 2 margin."""
        return self.width + 2 * self.margin

    def scaled(self, ss):
        """The same panorama at ``ss`` times the resolution (supersampling): width, height and margin times ss."""
        ss = int(ss)
        if ss == 1:
            return self
        return Panorama(self.width * ss, self.height * ss, self.hfov_deg, self.elevation_deg, self.znear, self.zfar,
                        self.margin * ss)

    def constants(self):
        """The float32 constants of the projection, each computed in float64 and rounded once: theta_half = hfov / 2 (float32 pi
        at 360 degrees), k_w = width / hfov, t_hi = tan(hi), k_h = height / (tan(hi) - tan(lo)), znear, zfar."""
        hfov = math.radians(self.hfov_deg) if not self.full else 2.0 * math.pi
        lo, hi = (math.radians(e) for e in self.elevation_deg)
        f32 = np.float32
        return {"theta_half": f32(hfov / 2.0), "k_w": f32(self.width / hfov), "t_hi": f32(math.tan(hi)),
                "k_h": f32(self.height / (math.tan(hi) - math.tan(lo))), "znear": f32(self.znear), "zfar": f32(self.zfar)}

    def desc(self):
        """The kernels' ``read_panorama_desc``."""
        c = self.constants()
        return L.ReadPanoramaDesc(float(c["theta_half"]), float(c["k_w"]), float(c["t_hi"]), float(c["k_h"]), float(c["znear"]),
                                  float(c["zfar"]), self.width, self.margin, int(self.full))

    @staticmethod
    def world_to_camera(view_matrix):
        """The matrix the panorama kernels take: inv(view_matrix) in float32, for a camera-to-world ``view_matrix`` [4,4] or
        [B,4,4] in the GL convention (x right, y up, looking down -z), as ``FrameRenderer.total_matrix`` inverts it."""
        return np.linalg.inv(np.asarray(view_matrix, dtype=np.float32)).astype(np.float32)

    def __repr__(self):
        return (f"Panorama({self.width}x{self.height}, hfov {self.hfov_deg} deg, elevation {self.elevation_deg}, "
                f"z [{self.znear}, {self.zfar}], margin {self.margin})")


def _check(pyr, pano):
    if not isinstance(pano, Panorama):
        raise TypeError("read_b200: panorama must be a read_b200.panorama.Panorama")
    if (pyr.W, pyr.H) != (pano.plane_width, pano.height):
        raise RuntimeError(f"read_b200: a {pano!r} draws a {pano.plane_width}x{pano.height} pyramid, got {pyr.W}x{pyr.H}")
    if pyr.direct_mask != 1:
        raise RuntimeError("the panorama rasterizer needs nested pyramid levels")


def raster_panorama_sorted(pyr, store, view_m, pano):
    """Level 0 of a cleared (width + 2 margin) x height pyramid from a SortedPoints store, one pass over the store per 8 views
    (finish with ops.raster_derive / ops.pyramid_resolve_gather).  view_m: [B,4,4] world -> camera matrices
    (``Panorama.world_to_camera``), f32 contiguous on the device."""
    L.require_device()
    ops._f32c(view_m, "view_m")
    ops._f32c(store.pts4, "sorted store")
    if view_m.dim() != 3 or view_m.shape[0] != pyr.B:
        raise RuntimeError("batch_size check")
    _check(pyr, pano)
    lib, sp, d = L.load(), L.stream_ptr(), pano.desc()
    plane = pyr.W * pyr.H * 8                                    # bytes of one view's level-0 plane
    for v0 in range(0, pyr.B, 8):
        nb = min(8, pyr.B - v0)
        L.check(lib.read_raster_panorama_sorted(store.pts4.data_ptr(), store.n, view_m[v0:v0 + nb].data_ptr(), nb, pyr.W, pyr.H,
                                                pyr.L, ctypes.byref(d), pyr.buf.data_ptr() + v0 * plane, sp))


def raster_panorama_segments_culled(pyr, store, seg_m, pano, visible=None):
    """Level 0 of a cleared (width + 2 margin) x height pyramid from a SegmentedPoints store, drawing only the visible (segment,
    chunk) units whose box may come within zfar of some view's camera (culled and compacted on the device, no host
    synchronisation; ``ops.last_surviving_units`` reads the count).  seg_m: [nseg, B, 4, 4] world -> camera matrices per segment
    (``SceneComposer.segment_matrices(Panorama.world_to_camera(view))``), B <= 8; visible as in
    ops.raster_project_segments_culled."""
    ops._check_segmented(pyr, store, seg_m)
    _check(pyr, pano)
    visible, ws = ops._culled_inputs(store, seg_m, visible)
    d = pano.desc()
    L.check(L.load().read_raster_panorama_segments_culled(store.pts4.data_ptr(), store.n, store.seg_table.data_ptr(), store.nseg,
                                                          store.nunits, store.boxes.data_ptr(), visible.data_ptr(),
                                                          seg_m.data_ptr(), ws.data_ptr(), ws.numel(), pyr.B, pyr.W, pyr.H, pyr.L,
                                                          ctypes.byref(d), pyr.buf.data_ptr(), L.stream_ptr()))
