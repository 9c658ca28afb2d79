"""-m gpu: every rasterizer path at the projection's edges, key for key against the sequential oracle.

The point sets (tests/raster_edge_util.py, proven by tests/test_raster_edges_host.py) sit on the frustum planes and one ulp either
side, at the edges of the shared-reciprocal range of w and beyond it (0, denormal, FLT_MAX, inf, NaN), at d = 0 and the first
floats above it, on pixel boundaries, in depth ties and, for sprites, at every size edge.  Each path's pyramid is compared with
``oracle_sprite.sprite_zbuf`` (1-pixel levels for the 1-pixel paths: its semantics are the rasterizer's, NaN and d == 0 never
drawn, the lowest key wins), and with ``oracle.pcpr_forward`` where no point is degenerate."""
import contextlib
import ctypes
import functools

import numpy as np
import pytest
import torch

import oracle_sprite
import raster_edge_util as E
from read_b200 import _lib as Lb
from read_b200 import ops

pytestmark = pytest.mark.gpu
DEFAULTS = {"raster_mode": 2, "raster_pipelined": 1, "raster_bulk_tma": 1, "raster_stream": 1, "raster_dedup": 0,
            "raster_nbr_filter": 0, "raster_run": 0, "raster_stages": 2, "raster_occupancy": 0}
LOW = np.uint64(0xFFFFFFFF)
ZBUF_EMPTY = np.uint64(0x7FFFFFFFFFFFFFFF)          # the rasterizer's empty key; the oracle's is ~0
SMALL = (64, 48, 3)
# at 1920 x 1088 / 1080 the per-view runs take the w classes that exercise both branches of the division
BIG_VIEWS = ["w=1", "w=2^-57", "w=pred(2^-57)", "w=pred(2^58)", "w=2^58", "w=+0", "w=2^-140", "w=FLT_MAX", "w=+inf"]


def _dev():
    return torch.device("cuda", 0)


@contextlib.contextmanager
def options(**kv):
    lib = Lb.load()
    try:
        for k, v in kv.items():
            Lb.check(lib.read_set_option(k.encode(), int(v)))
        yield
    finally:
        for k in kv:
            Lb.check(lib.read_set_option(k.encode(), DEFAULTS[k]))


def _keys(pyr):
    """Every level's keys, the empty key in the oracle's encoding."""
    torch.cuda.synchronize()
    out = []
    for l, (w, h) in enumerate(pyr.sizes):
        k = pyr.level(l).cpu().numpy().view(np.uint64).reshape(pyr.B, h, w)
        out.append(np.where(k == ZBUF_EMPTY, oracle_sprite.EMPTY, k))
    return out


def _assert_keys(got, want, labels, path, opts=None):
    """Key-for-key equality of every level; the message names the path, the options, the level, the first differing pixel and
    the edge class of the points there."""
    for l, (g, w) in enumerate(zip(got, want)):
        bad = g != w
        if bad.any():
            b, y, x = (int(v) for v in np.argwhere(bad)[0])

            def cls(k):
                return "empty" if k == oracle_sprite.EMPTY else labels[int(k & LOW)] if int(k & LOW) < len(labels) else "?"
            raise AssertionError(
                f"{path} {opts or {}}: level {l} view {b} pixel (x={x}, y={y}), {int(bad.sum())} pixels differ: got "
                f"{int(g[b, y, x]):#018x} ({cls(g[b, y, x])}), want {int(w[b, y, x]):#018x} ({cls(w[b, y, x])})")


@functools.lru_cache(maxsize=None)
def view_set(W, H):
    return E.view_set(W, H)


@functools.lru_cache(maxsize=None)
def ring_store(W, H):
    return E.ring_store(W, H)


@functools.lru_cache(maxsize=4)
def one_pixel_ref(name, W, H, L, views):
    """Oracle keys of a point set ('view' or 'point') under the matrices of `views` (indices), 1-pixel levels."""
    xyz, M = _set(name, W, H, views)
    return oracle_sprite.sprite_zbuf(xyz, M, W, H, [(1, False)] * L)


def _set(name, W, H, views):
    if name == "view":
        xyz, _, M = view_set(W, H)
        return xyz, M[list(views)]
    return ring_store(W, H)["xyz"], np.stack([E.point_matrix(E.C_VALUES[v]) for v in views])


def _labels(name, W, H):
    return view_set(W, H)[1] if name == "view" else ring_store(W, H)["labels"]


def _direct(xyz_t, M, W, H, L, id_base=0):
    pyr = ops.Pyramid(M.shape[0], W, H, L, _dev())
    pyr.clear()
    ops.raster_project(pyr, xyz_t, torch.from_numpy(np.ascontiguousarray(M)).to(_dev()), id_base=id_base)
    return pyr


def _view_indices(W, H, big_subset):
    names = [n for n, _ in E.VIEW_W]
    return [names.index(n) for n in BIG_VIEWS] if big_subset else list(range(len(names)))


def _check_direct_per_view(W, H, L, opts, path, xyz_t=None):
    """B = 1 launches, one per w class of the per-view set and one per cz of the per-point set."""
    for name, views in (("view", _view_indices(W, H, W > 64)), ("point", range(len(E.C_VALUES)))):
        xyz, M = _set(name, W, H, tuple(views))
        x = torch.from_numpy(xyz).to(_dev()) if xyz_t is None or name == "point" else xyz_t
        want = one_pixel_ref(name, W, H, L, tuple(views))
        for k in range(len(views)):
            got = _keys(_direct(x, M[k:k + 1], W, H, L))
            _assert_keys(got, [w[k:k + 1] for w in want], _labels(name, W, H), f"{path} {name} set view {k}", opts)


@pytest.mark.parametrize("W,H,L", [SMALL, (1920, 1088, 4), (1920, 1080, 4)])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_direct_single_view_kernels(mode, W, H, L):
    """raster_mode 0 (staged kernel, literal IEEE cull), 1 / 2 / 3 (lean kernel: RED only, early-z, shared-memory filter)."""
    with options(raster_mode=mode):
        _check_direct_per_view(W, H, L, {"raster_mode": mode}, "raster_project B=1")


@pytest.mark.parametrize("pipelined", [0, 1])
@pytest.mark.parametrize("bulk", [0, 1])
def test_direct_staged_pipelined_and_bulk(pipelined, bulk):
    o = {"raster_mode": 0, "raster_pipelined": pipelined, "raster_bulk_tma": bulk}
    with options(**o):
        _check_direct_per_view(*SMALL, o, "raster_project staged")


@pytest.mark.parametrize("B,W,H,L", [(3, 64, 48, 3), (17, 64, 48, 3), (3, 1920, 1088, 2)])
def test_direct_staged_multi_view(oracle_mod, B, W, H, L):
    """B > 1 runs the staged kernel; B = 17 > RP_MAXB = 16 takes two launches, the second with offset matrices."""
    views = tuple(_view_indices(W, H, W > 64)[:B]) if B < 17 else tuple(range(17))
    xyz, M = _set("view", W, H, views)
    got = _keys(_direct(torch.from_numpy(xyz).to(_dev()), M, W, H, L))
    _assert_keys(got, one_pixel_ref("view", W, H, L, views), _labels("view", W, H), f"raster_project B={B}")


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("W,H,L", [(100, 50, 3), (33, 17, 3)])
def test_direct_non_nested_levels(oracle_mod, W, H, L, B):
    """Levels that do not nest are drawn directly (the staged kernel's level loop), the others derived."""
    for name, views in (("view", tuple(range(B)) if B > 1 else (11,)), ("point", tuple(range(B)))):
        xyz, M = _set(name, W, H, views)
        got = _keys(_direct(torch.from_numpy(xyz).to(_dev()), M, W, H, L))
        _assert_keys(got, one_pixel_ref(name, W, H, L, views), _labels(name, W, H), f"raster_project {W}x{H} {name} B={B}")
        if all(oracle_mod.count_degenerate(xyz, m) == 0 for m in M):
            _check_pcpr(oracle_mod, xyz, M, got, W, H)


def _check_pcpr(oracle_mod, xyz, M, got, W, H):
    for l, (w, h) in enumerate(oracle_mod.level_sizes(W, H, len(got))):
        oi, od = oracle_mod.pcpr_forward(xyz, M, w, h)
        gi, gd = oracle_sprite.resolve(got[l])
        np.testing.assert_array_equal(gi, oi, err_msg=f"pcpr index level {l}")
        np.testing.assert_array_equal(gd.view(np.uint32), od.view(np.uint32), err_msg=f"pcpr depth level {l}")


def test_direct_pcpr_where_nothing_is_degenerate(oracle_mod):
    """The per-point set with its degenerate points (NaN, d == 0) moved outside the frustum also matches pcpr_forward, in every view
    whose cz is not -1."""
    W, H, L = SMALL
    xyz = ring_store(W, H)["xyz"].copy()
    views = [v for v, c in enumerate(E.C_VALUES) if c != -1]
    M = np.stack([E.point_matrix(E.C_VALUES[v]) for v in views])
    for m in M:
        p = E.project(m, xyz, W, H)
        xyz[np.isnan(p["q"]).any(1) | (p["d"] == 0)] = (4, 4, 1)
    assert all(oracle_mod.count_degenerate(xyz, m) == 0 for m in M)
    _check_pcpr(oracle_mod, xyz, M, _keys(_direct(torch.from_numpy(xyz).to(_dev()), M, W, H, L)), W, H)


@pytest.mark.parametrize("mode", [0, 2])
def test_direct_unaligned_points_pointer(mode):
    """xyz at a 12-byte offset: the staged kernel loads without bulk copies, the lean kernel reads it as is."""
    W, H, L = SMALL
    xyz, _, _ = view_set(W, H)
    big = torch.zeros((xyz.shape[0] + 1, 3), dtype=torch.float32, device=_dev())
    big[1:] = torch.from_numpy(xyz).to(_dev())
    sub = big[1:]
    assert sub.data_ptr() % 16 != 0 and sub.is_contiguous()
    with options(raster_mode=mode):
        _check_direct_per_view(W, H, L, {"raster_mode": mode, "xyz": "unaligned"}, "raster_project", xyz_t=sub)


def test_direct_id_base_with_int32_maps():
    """id_base > 2^24: keys carry id_base + row, and the int32 index maps resolve them."""
    W, H, L = SMALL
    xyz, labels, M = view_set(W, H)
    base = (1 << 31) - xyz.shape[0] - 7
    views = (0, 2, 9, 12)
    want = one_pixel_ref("view", W, H, L, views)
    want = [np.where(w == oracle_sprite.EMPTY, w, w + np.uint64(base)) for w in want]
    pyr = _direct(torch.from_numpy(xyz).to(_dev()), M[list(views)], W, H, L, id_base=base)
    got = _keys(pyr)
    _assert_keys(got, want, _Shifted(labels, base), "raster_project id_base")
    for l in range(L):
        idx, dep = ops.zbuf_resolve(pyr, l, index_dtype=torch.int32)
        wi, wd = oracle_sprite.resolve(want[l], np.int64)
        assert np.array_equal(idx.cpu().numpy().astype(np.int64), wi), f"int32 index map level {l}"
        assert np.array_equal(dep.cpu().numpy().view(np.uint32), wd.view(np.uint32)), f"depth map level {l}"


class _Shifted:
    """The labels of ids base, base + 1, ..."""

    def __init__(self, labels, base):
        self.labels, self.base = labels, base

    def __len__(self):
        return self.base + len(self.labels)

    def __getitem__(self, i):
        return self.labels[i - self.base] if i >= self.base else "?"


def _store(pts4, psize_rows=None):
    s = object.__new__(ops.SortedPoints)
    s.n, s.cell, s.perm = pts4.shape[0], 0.0, None
    s.pts4 = torch.from_numpy(np.ascontiguousarray(pts4)).to(_dev())
    s.psize = None if psize_rows is None else ops._padded_sizes(torch.from_numpy(psize_rows).to(_dev()))
    return s


def _sorted_draw(store, M, W, H, L):
    pyr = ops.Pyramid(M.shape[0], W, H, L, _dev())
    pyr.clear()
    ops.raster_project_sorted(pyr, store, torch.from_numpy(np.ascontiguousarray(M)).to(_dev()))
    ops.raster_derive(pyr)
    return _keys(pyr)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("run", [1, 16])
@pytest.mark.parametrize("nbr", [0, 1])
@pytest.mark.parametrize("dedup", [0, 1])
def test_legacy_sorted_kernel(dedup, nbr, run, B):
    """raster_stream 0: the LDG kernel over the hand-laid store (ties with higher ids in lower lanes, across warps and chunks)."""
    W, H, L = SMALL
    rs = ring_store(W, H)
    views = tuple(range(B)) if B == 1 else (0, 4)
    o = {"raster_stream": 0, "raster_dedup": dedup, "raster_nbr_filter": nbr, "raster_run": run}
    with options(**o):
        got = _sorted_draw(_store(rs["pts4"]), _set("point", W, H, views)[1], W, H, L)
    _assert_keys(got, one_pixel_ref("point", W, H, L, views), rs["labels"], f"legacy sorted B={B}", o)


@pytest.mark.parametrize("occupancy", [0, 4])
@pytest.mark.parametrize("stages", [2, 3])
@pytest.mark.parametrize("B", [1, 3, 8])
def test_ring_whole_store(B, stages, occupancy):
    """The streaming kernel over the hand-laid store: warps whose vote sees one visible unsafe row (lane 0, lane 31, u = 3), only a
    culled one, every row unsafe, and a partial last chunk."""
    W, H, L = SMALL
    rs = ring_store(W, H)
    views = tuple(range(B))
    o = {"raster_stages": stages, "raster_occupancy": occupancy}
    with options(**o):
        got = _sorted_draw(_store(rs["pts4"]), _set("point", W, H, views)[1], W, H, L)
    _assert_keys(got, one_pixel_ref("point", W, H, L, views), rs["labels"], f"ring whole store B={B}", o)


def test_ring_whole_store_1920():
    W, H, L = 1920, 1088, 4
    rs = ring_store(W, H)
    views = (0, 3, 6)
    got = _sorted_draw(_store(rs["pts4"]), _set("point", W, H, views)[1], W, H, L)
    _assert_keys(got, one_pixel_ref("point", W, H, L, views), rs["labels"], "ring whole store 1920x1088 B=3")


def _segmented(lay, segments, visible):
    """A SegmentedPoints over hand-laid rows: segment s draws part segments[s]; visible flags per segment."""
    s = object.__new__(ops.SegmentedPoints)
    s.pts4 = torch.from_numpy(lay["pts4"]).to(_dev())
    s.n = s.pts4.shape[0]
    s.psize = None if lay["psize"] is None else torch.from_numpy(lay["psize"]).to(_dev())
    s.segment_part = list(segments)
    s.nseg = len(segments)
    parts = lay["parts"]
    s.first_chunk = (ctypes.c_int64 * s.nseg)(*[parts[p][0] for p in segments])
    s.chunks = (ctypes.c_int64 * s.nseg)(*[parts[p][1] for p in segments])
    s.visible = (ctypes.c_uint8 * s.nseg)(*[1 if v else 0 for v in visible])
    s.boxes = ops._chunk_boxes(s.pts4)
    s.seg_table = torch.tensor([[s.first_chunk[i], s.chunks[i], i] for i in range(s.nseg)], dtype=torch.int32).to(_dev())
    s.nunits = sum(s.chunks[i] for i in range(s.nseg))
    s._cull_ws = None
    return s


def _segmented_ref(lay, segments, visible, seg_m, W, H, levels):
    """Min over the visible segments of each segment's oracle keys, its local ids moved to global ids."""
    out = None
    for s, p in enumerate(segments):
        if not visible[s]:
            continue
        _, _, xyz, base, sz = lay["parts"][p]
        keys = oracle_sprite.sprite_zbuf(xyz, seg_m[s], W, H, levels, sz)
        keys = [np.where(k == oracle_sprite.EMPTY, k, k + np.uint64(base)) for k in keys]
        out = keys if out is None else [np.minimum(a, b) for a, b in zip(out, keys)]
    return out


SEGMENTS = [0, 1, 2, 3, 0, 2]              # 4: an instance of part 0 under other matrices; 5: hidden
VISIBLE = [1, 1, 1, 1, 1, 0]


def _seg_matrices(B):
    return np.stack([np.stack([E.point_matrix(E.C_VALUES[(s * 3 + b) % len(E.C_VALUES)]) for b in range(B)])
                     for s in range(len(SEGMENTS))]).astype(np.float32)


@pytest.mark.parametrize("B", [1, 8])
@pytest.mark.parametrize("kernel", ["segments", "culled"])
def test_ring_segmented(kernel, B):
    """The parameter-table and culled-table kernels: unsafe rows, chunk boxes touching the x = w plane from inside and outside, a
    hidden segment and an instance."""
    W, H, L = SMALL
    lay = E.segmented_store(W, H)
    store = _segmented(lay, SEGMENTS, VISIBLE)
    seg_m = _seg_matrices(B)
    pyr = ops.Pyramid(B, W, H, L, _dev())
    pyr.clear()
    fn = ops.raster_project_segments if kernel == "segments" else ops.raster_project_segments_culled
    fn(pyr, store, torch.from_numpy(seg_m).to(_dev()))
    ops.raster_derive(pyr)
    want = _segmented_ref(lay, SEGMENTS, VISIBLE, seg_m, W, H, [(1, False)] * L)
    _assert_keys(_keys(pyr), want, lay["labels"], f"ring {kernel} B={B}")


# sprites: the edge set under per-view w = 1 (m23 = -0), w = 0, FLT_MAX and 2^-140
SPRITE_VIEWS = [(1.0, -0.0), (0.0, -0.0), (float(E.FLT_MAX), 0.0), (float(E.DENORM), 0.0)]
SPRITE_LEVELS = {"1px": [(1, False)] * 3, "fixed": [(2, False), (3, False), (64, False)],
                 "fractional": [(2.5, False), (63.5, False), (1, False)], "relative": [(4, True), (16, True), (1, True)]}


@functools.lru_cache(maxsize=None)
def sprite_set(W, H):
    xyz, labels, sizes = E.sprite_set(W, H)
    extra = np.array([[0, 0, 0], [-0.0, -0.0, -0.0], [0.5, 0, 0]], np.float32)          # numerators over w = 0
    return np.concatenate([xyz, extra]), labels + ["E2 numerators over w=0"] * 3, np.concatenate([sizes, np.zeros(3, np.float32)])


@pytest.mark.parametrize("sized", [False, True])
@pytest.mark.parametrize("levels", sorted(SPRITE_LEVELS))
@pytest.mark.parametrize("W,H", [(64, 32), (6, 130), (130, 6)])
@pytest.mark.parametrize("kernel", ["sorted", "segments", "culled"])
def test_sprites(kernel, W, H, levels, sized):
    """Point sprites at the size edges (relative sizes over c2 = +-0, negative and denormal; per-point sizes NaN, negative,
    denormal, inf, 64 +- 0.5; even widths at u - xx = 0.5 exactly) crossing every border, on levels 1 pixel wide or high."""
    lv = SPRITE_LEVELS[levels]
    xyz, labels, sizes = sprite_set(W, H)
    sizes = sizes if sized else None
    M = np.stack([E.view_matrix(w, m23) for w, m23 in SPRITE_VIEWS])
    B = M.shape[0]
    pyr = ops.Pyramid(B, W, H, len(lv), _dev())
    pyr.clear()
    if kernel == "sorted":
        rng = np.random.default_rng(W)
        ids = rng.permutation(xyz.shape[0])
        ops.raster_project_sprites(pyr, _store(E.pts4_of(xyz[ids], ids), None if sizes is None else sizes[ids]),
                                   torch.from_numpy(M).to(_dev()), lv)
        want = oracle_sprite.sprite_zbuf(xyz, M, W, H, lv, sizes)
    else:
        lay = E.lay_segments([(xyz, labels, sizes), (xyz[::-1].copy(), labels[::-1], None if sizes is None else sizes[::-1].copy())])
        store = _segmented(lay, [0, 1, 0], [1, 1, 0])
        seg_m = np.stack([M, M[::-1], M]).astype(np.float32)
        ops.raster_project_sprites(pyr, store, torch.from_numpy(np.ascontiguousarray(seg_m)).to(_dev()), lv, kernel=kernel)
        want = _segmented_ref(lay, [0, 1, 0], [1, 1, 0], seg_m, W, H, lv)
        labels = lay["labels"]
    _assert_keys(_keys(pyr), want, labels, f"sprites {kernel} {W}x{H} levels {lv}", {"sized": sized})
