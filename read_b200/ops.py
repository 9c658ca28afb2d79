"""Thin torch-tensor wrappers over the C ABI (device memory + current stream only; no math here)."""
import ctypes

import torch

from . import _lib as L


def level_sizes(W, H, n_levels):
    """(w_l, h_l) = (int(W*0.5**l), int(H*0.5**l)) — src/READ/gl/myrender.py:33-34."""
    return [(int(W * (0.5 ** i)), int(H * (0.5 ** i))) for i in range(n_levels)]


class Pyramid:
    """Packed (depth|id) z-buffer pyramid for B views, L levels (see include/read_b200.h)."""

    def __init__(self, B, W, H, n_levels, device):
        lib = L.load()
        self.B, self.W, self.H, self.L = B, W, H, n_levels
        self.sizes = level_sizes(W, H, n_levels)
        self.entries = lib.read_pyramid_entries(B, W, H, n_levels)
        if self.entries < 0:
            raise RuntimeError("read_b200: bad pyramid geometry")
        self.offsets = [lib.read_pyramid_level_offset(B, W, H, l) for l in range(n_levels)]
        self.buf = torch.empty(max(self.entries, 1), dtype=torch.int64, device=device)
        self.direct_mask = lib.read_raster_direct_mask(W, H, n_levels)

    def level(self, l):
        w, h = self.sizes[l]
        return self.buf[self.offsets[l]: self.offsets[l] + self.B * w * h]

    def clear(self):
        L.check(L.load().read_zbuf_clear(self.buf.data_ptr(), self.entries, L.stream_ptr()))

    def direct_levels(self):
        return [l for l in range(self.L) if (self.direct_mask >> l) & 1]


def _f32c(t, name):
    if t.dtype != torch.float32:
        raise RuntimeError(f"{name} must be a float tensor")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    return t


def raster_project(pyr, xyz, total_m, id_base=0, derive=True):
    """Project xyz [n,3] (cuda f32) through total_m [B,4,4] (cuda f32) into an already-cleared pyramid."""
    L.require_device()
    _f32c(xyz, "in_points")
    _f32c(total_m, "total_m")
    if total_m.dim() != 3 or total_m.shape[0] != pyr.B:
        raise RuntimeError("batch_size check")
    fn = L.load().read_raster_project if derive else L.load().read_raster_project_direct
    L.check(fn(xyz.data_ptr(), xyz.shape[0], id_base, total_m.data_ptr(), pyr.B, pyr.W, pyr.H, pyr.L,
               pyr.buf.data_ptr(), L.stream_ptr()))


class SortedPoints:
    """Spatially sorted, device-resident point store for the single-view frame path (the counterpart of
    ``MyRender.update_ds`` uploading ``scene_data['pointcloud']['xyz']``, src/READ/gl/myrender.py:17-21; SURVEY.md §8f rank 3).

    ``pts4`` is ``[N,4]`` f32 = (x, y, z, bit pattern of the ORIGINAL point id); rows are ordered by the Morton code of the
    point's 3-D grid cell (``cell`` metres, ties in original order), so consecutive rows are neighbours in space.  The
    original ids travel with the points: index maps, checkpoints and ``PointTexture`` keep the reference's numbering.
    Built once per scene with torch ops on the device (scene load, not the per-frame path)."""

    def __init__(self, xyz, cell=0.25):
        # the sort itself is plain torch (runs wherever xyz lives); only the rasterizer needs the device
        if xyz.dtype != torch.float32:
            raise RuntimeError("in_points must be a float tensor")
        if not xyz.is_contiguous():
            raise RuntimeError("in_points must be contiguous")
        if xyz.dim() != 2 or xyz.shape[1] != 3:
            raise RuntimeError("in_points must be [N,3]")
        n = xyz.shape[0]
        if n >= 1 << 32:
            raise RuntimeError("point ids must fit 32 bits")
        self.n, self.cell = n, float(cell)
        if n == 0:
            self.pts4 = torch.empty((0, 4), dtype=torch.float32, device=xyz.device)
            self.perm = torch.empty((0,), dtype=torch.int64, device=xyz.device)
            return
        lo = xyz.min(0).values
        q = torch.floor((xyz - lo) / self.cell).to(torch.int64).clamp_(0, (1 << 21) - 1)

        def part1by2(v):                      # spread the low 21 bits: bit i -> bit 3i
            v = v & 0x1FFFFF
            v = (v | (v << 32)) & 0x1F00000000FFFF
            v = (v | (v << 16)) & 0x1F0000FF0000FF
            v = (v | (v << 8)) & 0x100F00F00F00F00F
            v = (v | (v << 4)) & 0x10C30C30C30C30C3
            v = (v | (v << 2)) & 0x1249249249249249
            return v

        code = part1by2(q[:, 0]) | (part1by2(q[:, 1]) << 1) | (part1by2(q[:, 2]) << 2)
        self.perm = torch.argsort(code, stable=True)
        ids = self.perm.to(torch.int32)       # ids < 2^32: keep the low 32 bits (two's complement for ids >= 2^31)
        pts4 = torch.empty((n, 4), dtype=torch.float32, device=xyz.device)
        pts4[:, :3] = xyz[self.perm]
        pts4[:, 3] = ids.view(torch.float32)
        self.pts4 = pts4


    def shard(self, start, count):
        """Rows [start, start+count) of the sorted store as a store of their own: a contiguous range of the Morton order
        is a compact spatial tile of the scene (the multi-GPU partition, SURVEY.md §8e)."""
        sub = object.__new__(SortedPoints)
        sub.n, sub.cell = int(count), self.cell
        sub.pts4 = self.pts4[start:start + count]
        sub.perm = self.perm[start:start + count]
        return sub


def raster_project_sorted(pyr, store, total_m):
    """Level 0 of a cleared pyramid from a SortedPoints store, all views in one pass over the store (finish with raster_derive /
    pyramid_resolve_gather).  total_m: [B,4,4] contiguous."""
    L.require_device()
    _f32c(total_m, "total_m")
    _f32c(store.pts4, "sorted store")
    if total_m.dim() != 3 or total_m.shape[0] != pyr.B:
        raise RuntimeError("batch_size check")
    if pyr.direct_mask != 1:
        raise RuntimeError("the sorted-store rasterizer needs nested pyramid levels")
    lib, sp = L.load(), L.stream_ptr()
    plane = pyr.W * pyr.H * 8                                    # bytes of one view's level-0 plane
    for v0 in range(0, pyr.B, 8):                               # one pass over the store per 8 views
        nb = min(8, pyr.B - v0)
        L.check(lib.read_raster_project_sorted_views(store.pts4.data_ptr(), store.n, total_m[v0:v0 + nb].data_ptr(), nb, pyr.W,
                                                     pyr.H, pyr.L, pyr.buf.data_ptr() + v0 * plane, sp))


def raster_derive(pyr):
    L.check(L.load().read_raster_derive_levels(pyr.B, pyr.W, pyr.H, pyr.L, pyr.buf.data_ptr(), L.stream_ptr()))


def zbuf_resolve(pyr, l, want_index=True, want_depth=True):
    w, h = pyr.sizes[l]
    z = pyr.level(l)
    idx = torch.empty((pyr.B, h, w), dtype=torch.float32, device=z.device) if want_index else None
    dep = torch.empty((pyr.B, h, w), dtype=torch.float32, device=z.device) if want_depth else None
    L.check(L.load().read_zbuf_resolve(z.data_ptr(), pyr.B * w * h, L.ptr(idx), L.ptr(dep), L.stream_ptr()))
    return idx, dep


def pcpr_forward_device(xyz, total_m, w, h):
    """One level, B views, everything on device. Returns (index [B,h,w], depth [B,h,w]) cuda f32."""
    L.require_device()
    _f32c(xyz, "in_points")
    _f32c(total_m, "total_m")
    if total_m.dim() != 3:
        raise RuntimeError("batch_size check")
    B = total_m.shape[0]
    ws = torch.empty(max(B * w * h, 1), dtype=torch.int64, device=xyz.device)
    idx = torch.empty((B, h, w), dtype=torch.float32, device=xyz.device)
    dep = torch.empty((B, h, w), dtype=torch.float32, device=xyz.device)
    L.check(L.load().read_pcpr_forward(xyz.data_ptr(), xyz.shape[0], total_m.data_ptr(), B, w, h, ws.data_ptr(),
                                       idx.data_ptr(), dep.data_ptr(), L.stream_ptr()))
    return idx, dep


def texture_to_point_major(tex_cn):
    """[1,D,N] (or [D,N]) f32 cuda -> [N,D] f32 cuda."""
    L.require_device()
    t = tex_cn.reshape(tex_cn.shape[-2], tex_cn.shape[-1])
    _f32c(t, "texture")
    D, N = t.shape
    out = torch.empty((N, D), dtype=torch.float32, device=t.device)
    L.check(L.load().read_texture_to_point_major(t.data_ptr(), D, N, out.data_ptr(), L.stream_ptr()))
    return out


def texture_to_channel_major(tex_nd):
    _f32c(tex_nd, "texture")
    N, D = tex_nd.shape
    out = torch.empty((1, D, N), dtype=torch.float32, device=tex_nd.device)
    L.check(L.load().read_texture_to_channel_major(tex_nd.data_ptr(), D, N, out.data_ptr(), L.stream_ptr()))
    return out


_LAYOUT_DTYPE = {L.FEAT_NCHW_F32: torch.float32, L.FEAT_NHWC_F32: torch.float32, L.FEAT_NHWC_BF16: torch.bfloat16}


def _feat_out(B, D, h, w, layout, device, out):
    shape = (B, D, h, w) if layout == L.FEAT_NCHW_F32 else (B, h, w, D)
    if out is None:
        out = torch.empty(shape, dtype=_LAYOUT_DTYPE[layout], device=device)
    return out


def gather_from_index(tex_nd, ids, layout=L.FEAT_NCHW_F32, activation="none", out=None):
    """ids [B,h,w] f32 cuda (contiguous) -> features."""
    _f32c(ids, "ids")
    B, h, w = ids.shape
    N, D = tex_nd.shape
    out = _feat_out(B, D, h, w, layout, ids.device, out)
    L.check(L.load().read_gather_from_index(tex_nd.data_ptr(), D, N, ids.data_ptr(), B, h, w, layout,
                                            L.TEXACT[activation], out.data_ptr(), L.stream_ptr()))
    return out


def gather_from_zbuf(tex_nd, pyr, l, layout=L.FEAT_NHWC_BF16, activation="none", out=None):
    w, h = pyr.sizes[l]
    N, D = tex_nd.shape
    z = pyr.level(l)
    out = _feat_out(pyr.B, D, h, w, layout, z.device, out)
    L.check(L.load().read_gather_from_zbuf(tex_nd.data_ptr(), D, N, z.data_ptr(), pyr.B, h, w, layout,
                                           L.TEXACT[activation], out.data_ptr(), L.stream_ptr()))
    return out


def pyramid_resolve_gather(tex_nd, pyr, outs, layout=L.FEAT_NHWC_BF16, view0=0, nviews=None, reset_level0=False):
    """Fused per-frame path: derive levels 1..3, gather all 4 feature maps into ``outs`` (list of 4 NHWC tensors holding
    ``nviews`` views), optionally leave level 0 cleared.  Needs a 4-level nested pyramid and 8-d descriptors; call after
    ``raster_project(..., derive=False)``."""
    N, D = tex_nd.shape
    nviews = pyr.B if nviews is None else nviews
    if not fused_resolve_supported(pyr, D):
        raise RuntimeError("read_b200: fused pyramid resolve needs L == 4 nested levels, W,H % 8 == 0 and D == 8")
    arr = (L.c_vp * 4)(*[o.data_ptr() for o in outs])
    L.check(L.load().read_pyramid_resolve_gather(tex_nd.data_ptr(), D, N, pyr.buf.data_ptr(), pyr.B, view0, nviews, pyr.W,
                                                 pyr.H, pyr.L, layout, arr, int(bool(reset_level0)), L.stream_ptr()))


def fused_resolve_supported(pyr, D=8):
    return pyr.L == 4 and D == 8 and pyr.direct_mask == 1 and pyr.W % 8 == 0 and pyr.H % 8 == 0


def gather_backward(grad_out, ids, N):
    """grad_out [B,D,h,w] f32, ids [B,h,w] f32 -> grad [N,D] f32 (scatter-add).  Under torch.use_deterministic_algorithms(True) the
    additions run in the fixed order of read_gather_backward_det, so the result is the same bits on every call."""
    grad_out = grad_out.contiguous()
    _f32c(grad_out, "grad_out")
    B, D, h, w = grad_out.shape
    g = torch.zeros((N, D), dtype=torch.float32, device=grad_out.device)
    lib = L.load()
    if torch.are_deterministic_algorithms_enabled():
        ws = det_workspace(lib.read_gather_backward_det_workspace_bytes(B, D, h, w, N), grad_out.device, "gather backward")
        L.check(lib.read_gather_backward_det(grad_out.data_ptr(), ids.data_ptr(), B, D, h, w, N, g.data_ptr(), ws.data_ptr(),
                                             L.stream_ptr()))
        return g
    L.check(lib.read_gather_backward(grad_out.data_ptr(), ids.data_ptr(), B, D, h, w, N, g.data_ptr(), L.stream_ptr()))
    return g


def det_workspace(nbytes, device, what):
    """Workspace of a deterministic entry point (nbytes from its *_workspace_bytes query; -1: the shape is not supported)."""
    if nbytes < 0:
        raise RuntimeError(f"read_b200: {what}: shape not supported by the deterministic kernels")
    return torch.empty(max(nbytes, 16), dtype=torch.uint8, device=device)


def nchw_to_nhwc(x, act_bf16):
    _f32c(x, "input")
    B, C, H, W = x.shape
    out = torch.empty((B, H, W, C), dtype=torch.bfloat16 if act_bf16 else torch.float32, device=x.device)
    L.check(L.load().read_nchw_f32_to_nhwc(x.data_ptr(), B, C, H, W, L.ACT_BF16 if act_bf16 else L.ACT_F32,
                                           out.data_ptr(), L.stream_ptr()))
    return out


def nhwc_to_nchw(x):
    B, H, W, C = x.shape
    out = torch.empty((B, C, H, W), dtype=torch.float32, device=x.device)
    L.check(L.load().read_nhwc_to_nchw_f32(x.data_ptr(), L.ACT_BF16 if x.dtype == torch.bfloat16 else L.ACT_F32,
                                           B, C, H, W, out.data_ptr(), L.stream_ptr()))
    return out


def launch_count():
    return int(L.load().read_launch_count())
