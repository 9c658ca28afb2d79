"""Thin torch-tensor wrappers over the C ABI (device memory + current stream only; no math here)."""
import ctypes

import torch

from . import _lib as L
from . import sprites


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
    Built once per scene with torch ops on the device (scene load, not the per-frame path).

    ``point_sizes``: optional [N] per-point sprite sizes (``scene_data['point_sizes']``, see read_b200.sprites), permuted with the
    points into ``psize`` (float32 on the store's device, padded with zeros to whole SEGMENT_CHUNK chunks); None otherwise."""

    def __init__(self, xyz, cell=0.25, point_sizes=None):
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
        sizes = None if point_sizes is None else sprites.check_point_sizes(point_sizes, n).to(xyz.device)
        self.psize = None
        if n == 0:
            self.pts4 = torch.empty((0, 4), dtype=torch.float32, device=xyz.device)
            self.perm = torch.empty((0,), dtype=torch.int64, device=xyz.device)
            if sizes is not None:
                self.psize = _padded_sizes(sizes)
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
        if sizes is not None:
            self.psize = _padded_sizes(sizes[self.perm])


    def shard(self, start, count):
        """Rows [start, start+count) of the sorted store as a store of their own: a contiguous range of the Morton order
        is a compact spatial tile of the scene (the multi-GPU partition, SURVEY.md §8e)."""
        if self.psize is not None:
            raise ValueError("read_b200: a store with point sizes is not sharded (point sprites are single-GPU)")
        sub = object.__new__(SortedPoints)
        sub.n, sub.cell, sub.psize = int(count), self.cell, None
        sub.pts4 = self.pts4[start:start + count]
        sub.perm = self.perm[start:start + count]
        return sub


def _padded_sizes(sizes):
    """[n] f32 -> [ceil(n / SEGMENT_CHUNK) * SEGMENT_CHUNK] f32, zero-padded: the rasterizer streams whole chunks of sizes."""
    n = sizes.shape[0]
    out = torch.zeros(max(-(-n // SEGMENT_CHUNK), 1) * SEGMENT_CHUNK, dtype=torch.float32, device=sizes.device)
    out[:n] = sizes
    return out


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


SEGMENT_CHUNK = 1024                     # rows per chunk of the segmented rasterizer; every segment is padded to whole chunks
MAX_SEGMENTS = L.MAX_SEGMENTS_CULLED     # per store; the table-in-parameters entry (raster_project_segments) takes 128


class SegmentedPoints:
    """Composed, device-resident point store for scene editing and stitching (read_b200.scene_edit).

    Built from ``parts``: a list of ``(xyz [n,3] f32, ids [n] int64)`` or ``(xyz, ids, point_sizes [n])``, each a group of points with their GLOBAL ids (the row of
    their descriptors in the composed descriptor table).  Each part becomes one block of ``pts4`` rows: its points sorted on
    their own as a ``SortedPoints`` store, with the global id in the id word, then padded to whole ``SEGMENT_CHUNK`` chunks with
    rows (NaN, NaN, NaN, id 0) that the rasterizer culls, so that a chunk never spans two segments.  ``segments`` lists, per
    segment, the part whose rows it draws (default: one segment per part); several segments over one part are instances.

    Per segment: ``first_chunk`` / ``chunks`` (its row range in chunks), ``visible`` (host flag, set with ``set_visible``) and
    ``ids`` (its part's global ids).  ``n`` is the row count including padding, ``n_ids`` the number of global ids (the index
    maps' dtype follows ``index_map_dtype(n_ids)``).

    For the culled rasterizer (``raster_project_segments_culled``), built once per layout on the store's device:
    ``boxes`` [n / SEGMENT_CHUNK, 6] f32, the axis-aligned box (min x, y, z, max x, y, z) of the rows of each chunk that hold a
    point (padding rows left out; a chunk of padding only gets the empty box +inf / -inf, which always culls); ``seg_table``
    [nseg, 3] int32, (first chunk, chunk count, matrix slot = the segment's index) per segment; ``nunits`` the number of
    (segment, chunk) units, the sum of the chunk counts.

    ``psize``: when some part has point sizes, [n] f32 per row (permuted with the rows; 0 for padding rows and for the points of
    parts without sizes, which keep the keys' sizes); None otherwise."""

    def __init__(self, parts, segments=None, n_ids=None, cell=0.25):
        segments = list(range(len(parts))) if segments is None else [int(s) for s in segments]
        if len(segments) > MAX_SEGMENTS:
            raise ValueError(f"read_b200: {len(segments)} segments; at most {MAX_SEGMENTS} per store")
        if any(not 0 <= s < len(parts) for s in segments):
            raise ValueError("read_b200: a segment refers to a part that does not exist")
        blocks, boxes, part_rows, row = [], [], [], 0
        self.part_ids = []
        sized = any(len(p) > 2 and p[2] is not None for p in parts)
        size_blocks = []
        for part in parts:
            xyz, ids = part[0], part[1]
            ids = torch.as_tensor(ids, dtype=torch.int64, device=xyz.device).reshape(-1)
            if ids.shape[0] != xyz.shape[0]:
                raise ValueError("read_b200: one global id per point")
            if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= 1 << 31):
                raise ValueError("read_b200: global point ids must lie in [0, 2^31)")
            sp = SortedPoints(xyz.contiguous(), cell)
            rows = -(-sp.n // SEGMENT_CHUNK) * SEGMENT_CHUNK
            blk = torch.empty((rows, 4), dtype=torch.float32, device=xyz.device)
            blk[sp.n:, :3] = float("nan")
            blk[sp.n:, 3] = 0.0                                            # id word 0 (0xFFFFFFFF would stall the ring)
            if sp.n:
                blk[:sp.n, :3] = sp.pts4[:, :3]
                blk[:sp.n, 3] = ids[sp.perm].to(torch.int32).view(torch.float32)
            if sized:
                sz = torch.zeros(rows, dtype=torch.float32, device=xyz.device)
                if len(part) > 2 and part[2] is not None and sp.n:
                    sz[:sp.n] = sprites.check_point_sizes(part[2], sp.n).to(xyz.device)[sp.perm]
                elif len(part) > 2 and part[2] is not None:
                    sprites.check_point_sizes(part[2], 0)
                size_blocks.append(sz)
            blocks.append(blk)
            boxes.append(_chunk_boxes(blk))
            part_rows.append((row, rows))
            self.part_ids.append(ids)
            row += rows
        dev = parts[0][0].device if parts else torch.device("cpu")
        self.pts4 = torch.cat(blocks) if blocks else torch.empty((0, 4), dtype=torch.float32, device=dev)
        self.n = self.pts4.shape[0]
        self.psize = torch.cat(size_blocks) if sized else None
        self.n_ids = int(n_ids) if n_ids is not None else sum(int(i.numel()) for i in self.part_ids)
        self.segment_part = segments
        self.nseg = len(segments)
        self.first_chunk = (ctypes.c_int64 * max(self.nseg, 1))(*[part_rows[p][0] // SEGMENT_CHUNK for p in segments])
        self.chunks = (ctypes.c_int64 * max(self.nseg, 1))(*[part_rows[p][1] // SEGMENT_CHUNK for p in segments])
        self.visible = (ctypes.c_uint8 * max(self.nseg, 1))(*([1] * self.nseg))
        self.boxes = torch.cat(boxes) if boxes else torch.empty((0, 6), dtype=torch.float32, device=dev)
        self.seg_table = torch.tensor([[self.first_chunk[s], self.chunks[s], s] for s in range(self.nseg)],
                                      dtype=torch.int32).reshape(-1, 3).to(dev)
        self.nunits = sum(self.chunks[s] for s in range(self.nseg))
        self._cull_ws = None                     # workspace of the culled rasterizer; its first word: the last surviving count

    def ids(self, seg):
        """Global ids of the points segment ``seg`` draws (in their part's order)."""
        return self.part_ids[self.segment_part[seg]]

    def set_visible(self, seg, visible):
        self.visible[seg] = 1 if visible else 0

    def visible_flags(self):
        """The host visibility flags as a [nseg] uint8 tensor sharing their memory (writes show in ``visible``)."""
        return torch.frombuffer(self.visible, dtype=torch.uint8)[:self.nseg]


def _chunk_boxes(blk):
    """[rows / SEGMENT_CHUNK, 6] (min xyz, max xyz) over the rows of each chunk without NaN (padding); +inf / -inf if none."""
    v = blk.view(-1, SEGMENT_CHUNK, 4)[:, :, :3]
    pad = torch.isnan(v).any(2, keepdim=True)
    return torch.cat([torch.where(pad, float("inf"), v).amin(1), torch.where(pad, float("-inf"), v).amax(1)], 1)


def _check_segmented(pyr, store, seg_m, nested=True):
    """The checks the segmented rasterizer wrappers make: seg_m [nseg, B, 4, 4] f32 contiguous on the device, the store's rows
    f32 contiguous on the device, nested pyramid levels (not for point sprites)."""
    L.require_device()
    _f32c(seg_m, "seg_m")
    _f32c(store.pts4, "segmented store")
    if seg_m.dim() != 4 or tuple(seg_m.shape[:2]) != (store.nseg, pyr.B) or tuple(seg_m.shape[2:]) != (4, 4):
        raise RuntimeError(f"read_b200: seg_m must be [{store.nseg}, {pyr.B}, 4, 4], got {tuple(seg_m.shape)}")
    if nested and pyr.direct_mask != 1:
        raise RuntimeError("the segmented rasterizer needs nested pyramid levels")


def raster_project_segments(pyr, store, seg_m):
    """Level 0 of a cleared pyramid from a SegmentedPoints store in one pass over its visible segments (finish with raster_derive
    / pyramid_resolve_gather).  seg_m: [nseg, B, 4, 4] f32 contiguous on the device, segment s drawn with seg_m[s], B <= 8."""
    _check_segmented(pyr, store, seg_m)
    L.check(L.load().read_raster_project_segments(store.pts4.data_ptr(), store.n, store.first_chunk, store.chunks, store.visible,
                                                  store.nseg, seg_m.data_ptr(), pyr.B, pyr.W, pyr.H, pyr.L, pyr.buf.data_ptr(),
                                                  L.stream_ptr()))


def _culled_inputs(store, seg_m, visible):
    """(visible flags on the device, the store's workspace) for the culled rasterizers."""
    if visible is None:
        visible = store.visible_flags().to(seg_m.device)
    if visible.dtype != torch.uint8 or tuple(visible.shape) != (store.nseg,) or not visible.is_contiguous() or not visible.is_cuda:
        raise RuntimeError(f"read_b200: visible must be a contiguous [{store.nseg}] uint8 CUDA tensor")
    need = L.load().read_raster_cull_workspace_bytes(store.nunits)
    if store._cull_ws is None or store._cull_ws.numel() < need or store._cull_ws.device != seg_m.device:
        store._cull_ws = torch.empty(need, dtype=torch.uint8, device=seg_m.device)
    return visible, store._cull_ws


def raster_project_segments_culled(pyr, store, seg_m, visible=None):
    """Level 0 of a cleared pyramid from a SegmentedPoints store of up to MAX_SEGMENTS segments, drawing only the (segment,
    chunk) units that are visible and whose chunk box may intersect the clip volume of some view (culled and compacted on the
    device, no host synchronisation; finish with raster_derive / pyramid_resolve_gather).  The pyramid is bit-identical to
    raster_project_segments'.  seg_m: [nseg, B, 4, 4] f32 contiguous on the device, B <= 8; visible: [nseg] uint8 on the device,
    or None to upload the store's host flags here."""
    _check_segmented(pyr, store, seg_m)
    visible, ws = _culled_inputs(store, seg_m, visible)
    lib = L.load()
    L.check(lib.read_raster_project_segments_culled(store.pts4.data_ptr(), store.n, store.seg_table.data_ptr(), store.nseg,
                                                    store.nunits, store.boxes.data_ptr(), visible.data_ptr(), seg_m.data_ptr(),
                                                    ws.data_ptr(), ws.numel(), pyr.B, pyr.W, pyr.H, pyr.L, pyr.buf.data_ptr(),
                                                    L.stream_ptr()))


def raster_project_sprites(pyr, store, total_m, levels, kernel="culled", visible=None):
    """Every level of a cleared pyramid from a SortedPoints or SegmentedPoints store, drawn as point sprites (read_b200.sprites):
    ``levels`` [(N, relative)] per level; the store's ``psize`` (if any) gives the per-point sizes.  One pass over the store per
    8 views (sorted store) or for all B <= 8 views (segmented store); the levels need not nest, and no derive step follows.
    total_m: [B,4,4] (sorted store) or seg_m [nseg, B, 4, 4] (segmented store) f32 contiguous on the device.  A segmented store
    is drawn by the culled rasterizer (``kernel="culled"``, with ``visible`` as in raster_project_segments_culled) or the
    parameter-table one (``kernel="segments"``)."""
    if len(levels) != pyr.L:
        raise ValueError(f"read_b200: {len(levels)} sprite levels for a {pyr.L}-level pyramid")
    d = sprites.desc(levels, store.psize)
    lib, sp = L.load(), L.stream_ptr()
    if isinstance(store, SortedPoints):
        L.require_device()
        _f32c(total_m, "total_m")
        _f32c(store.pts4, "sorted store")
        if total_m.dim() != 3 or total_m.shape[0] != pyr.B:
            raise RuntimeError("batch_size check")
        L.check(lib.read_raster_sprites_sorted(store.pts4.data_ptr(), store.n, total_m.data_ptr(), pyr.B, pyr.W, pyr.H, pyr.L,
                                               ctypes.byref(d), pyr.buf.data_ptr(), sp))
        return
    _check_segmented(pyr, store, total_m, nested=False)
    if kernel == "segments":
        L.check(lib.read_raster_sprites_segments(store.pts4.data_ptr(), store.n, store.first_chunk, store.chunks, store.visible,
                                                 store.nseg, total_m.data_ptr(), pyr.B, pyr.W, pyr.H, pyr.L, ctypes.byref(d),
                                                 pyr.buf.data_ptr(), sp))
        return
    if kernel != "culled":
        raise ValueError(f"read_b200: unknown segmented rasterizer {kernel!r}")
    visible, ws = _culled_inputs(store, total_m, visible)
    L.check(lib.read_raster_sprites_segments_culled(store.pts4.data_ptr(), store.n, store.seg_table.data_ptr(), store.nseg,
                                                    store.nunits, store.boxes.data_ptr(), visible.data_ptr(), total_m.data_ptr(),
                                                    ws.data_ptr(), ws.numel(), pyr.B, pyr.W, pyr.H, pyr.L, ctypes.byref(d),
                                                    pyr.buf.data_ptr(), sp))


def last_surviving_units(store):
    """Synchronise the device and return how many (segment, chunk) units the last raster_project_segments_culled call on
    ``store`` drew (None before the first).  For tests and benchmarks: it stalls the pipeline."""
    if store._cull_ws is None:
        return None
    torch.cuda.synchronize(store._cull_ws.device)
    return int(store._cull_ws[:4].cpu().view(torch.int32)[0])


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
