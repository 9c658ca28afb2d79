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


FLOAT_EXACT_POINTS = (1 << 24) + 1      # float32 holds every integer 0 .. 2^24: the ids of a cloud of up to 2^24 + 1 points


def index_map_dtype(n_points):
    """dtype of the index maps of a cloud of ``n_points`` points: float32, the reference's ``pcpr`` format, while float32 holds every
    id 0 .. n_points - 1 exactly (n_points <= 2^24 + 1); int32 above, with the same values (the point id, 0 for an empty pixel).
    Clouds of 2^31 points or more raise ValueError: their ids do not fit an int32 map."""
    n = int(n_points)
    if n >= 1 << 31:
        raise ValueError(f"read_b200: a cloud of {n} points is too large; point ids must stay below 2^31")
    return torch.int32 if n > FLOAT_EXACT_POINTS else torch.float32


def _ids(t, name="ids"):
    """Check an index map for the gather kernels: float32 or int32, contiguous, on the device.  Returns the suffix of the matching
    entry points ('' for float32, '_i32' for int32)."""
    if t.dtype not in (torch.float32, torch.int32):
        raise RuntimeError(f"{name} must be a float32 or int32 index map, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor")
    return "_i32" if t.dtype == torch.int32 else ""


def index_map(ids, device):
    """An index map as the gather kernels take it: int32 maps stay int32, any other dtype becomes float32 (the reference's format),
    contiguous on ``device``."""
    return ids.to(device, torch.int32 if ids.dtype == torch.int32 else torch.float32).contiguous()


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


def zbuf_resolve(pyr, l, want_index=True, want_depth=True, index_dtype=torch.float32):
    """Level ``l`` as (index [B,h,w], depth [B,h,w] f32) maps; ``index_dtype`` float32 or int32 (``index_map_dtype``)."""
    if index_dtype not in (torch.float32, torch.int32):
        raise RuntimeError(f"read_b200: index maps are float32 or int32, not {index_dtype}")
    w, h = pyr.sizes[l]
    z = pyr.level(l)
    idx = torch.empty((pyr.B, h, w), dtype=index_dtype, device=z.device) if want_index else None
    dep = torch.empty((pyr.B, h, w), dtype=torch.float32, device=z.device) if want_depth else None
    fn = L.load().read_zbuf_resolve_i32 if index_dtype == torch.int32 else L.load().read_zbuf_resolve
    L.check(fn(z.data_ptr(), pyr.B * w * h, L.ptr(idx), L.ptr(dep), L.stream_ptr()))
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
    """ids [B,h,w] f32 or int32 cuda (contiguous) -> features."""
    sfx = _ids(ids)
    B, h, w = ids.shape
    N, D = tex_nd.shape
    out = _feat_out(B, D, h, w, layout, ids.device, out)
    L.check(getattr(L.load(), "read_gather_from_index" + sfx)(tex_nd.data_ptr(), D, N, ids.data_ptr(), B, h, w, layout,
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


def _gather_backward(grad_out, ids, N, grad=None, touched=None, slots=None):
    """The descriptor-gradient scatter behind gather_backward, gather_backward_sparse and gather_backward_items: grad_out [B,D,h,w]
    f32 is added into ``grad`` ([N,D] f32; None: a fresh zeroed one, returned) and, when ``touched`` is given (the sparse form),
    touched[id] is set.  With ``slots``, item b's pixels go to slot slots[b] and N, grad and touched are per-slot lists (D = 8).
    Under torch.use_deterministic_algorithms(True) the additions run in the fixed order of the *_det entry points."""
    sfx = _ids(ids)
    _f32c(grad_out, "grad_out")
    B, D, h, w = grad_out.shape
    if slots is None:
        n_keys = N
        if grad is None:
            grad = torch.zeros((N, D), dtype=torch.float32, device=grad_out.device)
        args = [B, D, h, w, N, grad.data_ptr()] + ([] if touched is None else [touched.data_ptr()])
    else:
        if D != 8 or tuple(ids.shape) != (B, h, w) or B != len(slots):
            raise RuntimeError("read_b200: multi-texture gather backward: shape mismatch")
        n_keys, table = sum(int(n) for n in N), tex_table(slots, N, grad=grad, touched=touched)
        args = [ctypes.byref(table), h, w]
    name = "read_gather_backward" + ("" if touched is None else "_sparse") + ("" if slots is None else "_items")
    lib, ws = L.load(), None
    if torch.are_deterministic_algorithms_enabled():
        ws = det_workspace(lib.read_gather_backward_det_workspace_bytes(B, D, h, w, n_keys), grad_out.device, name)
        name, args = name + "_det", args + [ws.data_ptr()]
    L.check(getattr(lib, name + sfx)(grad_out.data_ptr(), ids.data_ptr(), *args, L.stream_ptr()))
    return grad


def gather_backward(grad_out, ids, N):
    """grad_out [B,D,h,w] f32, ids [B,h,w] f32 or int32 -> grad [N,D] f32 (scatter-add).  Under
    torch.use_deterministic_algorithms(True) the additions run in the fixed order of read_gather_backward_det, so the result is the
    same bits on every call."""
    return _gather_backward(grad_out.contiguous(), ids, N)


def gather_backward_sparse(grad_out, ids, N, grad_nd, touched):
    """Sparse form of gather_backward: scatter-add into the persistent [N,D] accumulator ``grad_nd`` and set ``touched`` [N] u8
    (read_gather_backward_sparse; under torch.use_deterministic_algorithms(True), read_gather_backward_sparse_det).
    grad_out [B,D,h,w] f32 contiguous, ids [B,h,w] f32 or int32."""
    _gather_backward(grad_out, ids, N, grad_nd, touched)


def tex_table(slots, N, tex=None, grad=None, touched=None):
    """The multi-texture kernels' table (read_tex_table): item b samples slot ``slots[b]``; per slot its point count ``N[s]`` and,
    as the call needs them, its [N, 8] descriptors ``tex[s]``, its [N, 8] accumulator ``grad[s]`` (None: the slot receives nothing)
    and its [N] ``touched`` flags."""
    if not 1 <= len(N) <= L.MAX_TEX_SLOTS or not 1 <= len(slots) <= L.MAX_TEX_ITEMS:
        raise RuntimeError(f"read_b200: a texture table holds 1..{L.MAX_TEX_SLOTS} textures and 1..{L.MAX_TEX_ITEMS} items")
    t = L.ReadTexTable()
    t.n_slots, t.n_items = len(N), len(slots)
    for s, n in enumerate(N):
        t.N[s] = int(n)
        for field, seq in (("tex_nd", tex), ("grad_nd", grad), ("touched", touched)):
            if seq is not None and seq[s] is not None:
                getattr(t, field)[s] = seq[s].data_ptr()
    for b, s in enumerate(slots):
        t.slot[b] = int(s)
    return t


def gather_from_index_items(tex_nds, slots, ids, layout=L.FEAT_NCHW_F32, activation="none", out=None):
    """gather_from_index for a batch whose item b samples ``tex_nds[slots[b]]`` ([N_s, 8] f32 point-major): one launch.
    ids [B,h,w] f32 or int32 cuda (contiguous), B = len(slots)."""
    sfx = _ids(ids)
    B, h, w = ids.shape
    if B != len(slots):
        raise RuntimeError("read_b200: one slot per item")
    for nd in tex_nds:
        _f32c(nd, "texture")
        if nd.dim() != 2 or nd.shape[1] != 8:
            raise RuntimeError("read_b200: the multi-texture gather takes [N, 8] descriptors")
    out = _feat_out(B, 8, h, w, layout, ids.device, out)
    t = tex_table(slots, [nd.shape[0] for nd in tex_nds], tex=tex_nds)
    L.check(getattr(L.load(), "read_gather_from_index_items" + sfx)(ctypes.byref(t), ids.data_ptr(), h, w, layout,
                                                                  L.TEXACT[activation], out.data_ptr(), L.stream_ptr()))
    return out


def gather_backward_items(grad_out, ids, slots, N, grads, touched=None):
    """Backward of gather_from_index_items: item b's pixels scatter-add into ``grads[slots[b]]`` ([N_s, 8] f32 accumulators; None: the
    slot receives nothing) and, when ``touched`` is given (the sparse form), set ``touched[slots[b]]``.  grad_out [B,8,h,w] f32.  Under
    torch.use_deterministic_algorithms(True) the additions run in the fixed order of read_gather_backward_items_det."""
    _gather_backward(grad_out.contiguous(), ids, N, grads, touched, slots)


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
