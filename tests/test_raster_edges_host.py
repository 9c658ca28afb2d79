"""No GPU: the edge point sets of tests/raster_edge_util.py hit the edges they claim, bit for bit, in the kernel's float32
arithmetic (scene_scale_util.clip_coords restates its dot products; numpy's float32 division, addition and multiplication are
correctly rounded like the kernel's)."""
import numpy as np
import pytest
import torch

import raster_edge_util as E
import scene_scale_util as S
from read_b200 import ops

F32 = np.float32


def _biased_exp(x):
    return int((E.bits(x) >> np.uint32(23)) & np.uint32(0xFF))


def test_shared_reciprocal_range_is_exponents_70_to_184():
    """div_safe_den accepts |w| in [2^-57, 2^58): the set's w classes sit on both sides of both ends."""
    assert _biased_exp(E.SAFE_LO) == 70 and _biased_exp(E.down(E.SAFE_LO)) == 69
    assert _biased_exp(E.down(E.SAFE_HI)) == 184 and _biased_exp(E.SAFE_HI) == 185
    w = np.array([E.SAFE_LO, -E.SAFE_LO, E.down(E.SAFE_HI), -E.down(E.SAFE_HI), E.p2(57), F32(1)], F32)
    assert E.div_safe(w).all()
    w = np.array([E.down(E.SAFE_LO), E.SAFE_HI, -E.SAFE_HI, 0, -0.0, E.DENORM, E.FLT_MAX, np.inf, -np.inf, np.nan], F32)
    assert not E.div_safe(w).any()
    names = {n for n, _ in E.VIEW_W}
    assert {"w=2^-57", "w=pred(2^-57)", "w=pred(2^58)", "w=2^58", "w=+0", "w=-0", "w=2^-140", "w=FLT_MAX", "w=+inf"} <= names


@pytest.mark.parametrize("W,H", [(64, 48), (1920, 1088)])
def test_view_matrices_plant_w_and_the_frustum_planes_exactly(W, H):
    xyz, labels, M = E.view_set(W, H)
    labels = np.array(labels)
    hits = 0
    for (name, w), m in zip(E.VIEW_W, M):
        c = S.clip_coords(m, xyz)
        fin = np.isfinite(xyz).all(1)
        assert np.array_equal(np.abs(c[fin, 3]), np.full(fin.sum(), abs(w), F32))      # c_3 == w for every finite point
        exact = np.isfinite(w) and w != 0 and E.bits(abs(w)) & np.uint32(0x7FFFFF) == 0 and _biased_exp(w) > 0
        if not exact:
            continue
        pre = "raw " if name == "w=1" else f"{name}: "
        for i in range(3):
            for s in "+-":
                rows = np.char.startswith(labels, f"{pre}E1 plane c{i}={s}w")
                on = rows & np.char.endswith(labels, " on")
                inside = rows & np.char.endswith(labels, " inside")
                outside = rows & np.char.endswith(labels, " outside")
                aw = F32(abs(w))
                assert on.sum() == 1 and E.bits(np.abs(c[on, i])) == E.bits(aw)                   # |c_i| == |c_3| bit for bit
                assert np.abs(c[inside, i]) == E.down(aw) and np.abs(c[outside, i]) == E.up(aw)   # one ulp either side
                hits += 1
        p = E.project(m, xyz, W, H)
        corner = np.char.startswith(labels, f"{pre}E1 edge/corner")
        assert (p["vis"] & corner).any() and (~p["vis"] & corner).any()
    assert hits >= 6 * 8


def test_zero_and_infinite_denominators():
    W, H = 64, 48
    xyz, labels, M = E.view_set(W, H)
    labels = np.array(labels)
    names = [n for n, _ in E.VIEW_W]
    raw = np.char.startswith(labels, "raw ")
    for name in ("w=+inf", "w=-inf"):                            # a finite numerator over inf: the pixel centre at d = 0.5
        p = E.project(M[names.index(name)], xyz, W, H)
        assert (p["d"][raw] == F32(0.5)).all() and (p["u"][raw] == F32(W / 2)).all() and (p["v"][raw] == F32(H / 2)).all()
        assert p["vis"][raw].all()
    zero = labels == "E2 zero or nonzero numerator over w=0"
    for name in ("w=+0", "w=-0"):
        p = E.project(M[names.index(name)], xyz, W, H)
        c = p["c"][zero]
        assert (c[:, 3] == 0).all() and (c[:, :3] == 0).all(1).any() and (c[:, :3] != 0).any(1).any()
        assert np.isnan(p["q"][zero]).any(1).all() or not p["vis"][zero].any()
        assert E.clip_in(M[names.index(name)], xyz[zero]).any()    # (0,0,0) passes the division-free test: the fallback must cull it
    p = E.project(M[names.index("w=2^-140")], xyz, W, H)
    assert p["vis"].any() and _biased_exp(E.DENORM) == 0
    p = E.project(M[names.index("w=FLT_MAX")], xyz, W, H)
    assert p["vis"].any()


def test_depth_edges():
    """d == 0 at cz = -1 (never drawn), d = k 2^-25 for cz = -1 + k ulp, and cz = 1; the per-point views put the rounding of the
    quotient fl(fl(c w) / w) into d."""
    W, H = 64, 48
    A, labels = E.normalized_rows(W, H)
    labels = np.array(labels)
    p = E.project(E.view_matrix(F32(1)), A, W, H)
    for k in range(5):
        d = p["d"][labels == f"E3 cz=-1+{k}ulp"]
        assert E.bits(d) == E.bits(F32(k * 2.0 ** -25))
    assert not p["vis"][labels == "E3 cz=-1+0ulp"].any() and p["vis"][labels == "E3 cz=-1+1ulp"].all()
    assert p["d"][labels == "E3 cz=1"] == 1
    rs = E.ring_store(W, H)
    safe = np.array(rs["labels"]) == "safe"
    for c in E.C_VALUES[:4]:
        q = E.project(E.point_matrix(c), rs["xyz"], W, H)
        ds = q["d"][safe & q["vis"]]
        assert len(np.unique(ds)) >= 2, c                           # inexact quotients: several d per cz
        assert np.abs(E.bits(ds).astype(np.int64) - E.bits((c + F32(1)) * F32(0.5))).max() >= 1
    q = E.project(E.point_matrix(F32(-1)), rs["xyz"], W, H)
    assert not q["vis"].any() and (q["d"][E.clip_in(E.point_matrix(F32(-1)), rs["xyz"]) & ~np.isnan(q["d"])] == 0).all()


@pytest.mark.parametrize("n", [64, 48, 1920, 1088, 1080])
def test_pixel_boundaries(n):
    """For every planted target j with u == j exactly, the float below gives pixel j - 1 and the one above pixel j; cx = 1 gives
    u = n, which is dropped.  Power-of-two axes hit every target; others the ends, the middle and the multiples of their odd
    part."""
    pow2 = n & (n - 1) == 0
    for j in E.boundary_targets(n):
        x = E.boundary_first(n, j)
        assert int(E.pixel_u(n, x)) == j and x in E.boundary_coords(n)
        if j > 0:
            assert int(E.pixel_u(n, E.down(x))) == j - 1 and E.down(x) in E.boundary_coords(n)
        if E.boundary_x(n, j) is None:
            assert not pow2 and j not in (0, n // 2, n), j
    assert E.pixel_u(n, F32(1)) == n
    p = E.project(E.view_matrix(F32(1)), np.array([[1, 0, 0.5], [0, -1, 0.5]], F32), n, n)
    assert not p["vis"].any()


def test_tiny_quotients_are_denormal_or_zero():
    t = E.tiny_rows()
    for w in (F32(1), E.SAFE_LO, E.down(E.SAFE_HI)):
        p = E.project(E.view_matrix(w), t, 64, 48)
        q = np.abs(p["q"])
        assert ((q < 2.0 ** -126) | (q < 2.0 ** -60)).all()
    q = np.abs(E.project(E.view_matrix(F32(1)), t, 64, 48)["q"])
    assert ((q > 0) & (q < 2.0 ** -126)).any()                     # quotients in the denormal range, absorbed by the + 1
    assert E.project(E.view_matrix(F32(1)), t, 64, 48)["vis"].all()


@pytest.mark.parametrize("W,H", [(64, 48), (1920, 1088)])
def test_ties_and_mode3_slot_collisions(W, H):
    A, labels = E.normalized_rows(W, H)
    labels = np.array(labels)
    p = E.project(E.view_matrix(F32(1)), A, W, H)
    pairs = E.slot_collisions(W, H)
    assert len(pairs) == 3
    for (ax, ay), (bx, by) in pairs:
        ia, ib = ay * W + ax, by * W + bx
        assert ia != ib and (ia ^ (ia >> 11)) & 2047 == (ib ^ (ib >> 11)) & 2047
    slot = labels == "E6 slot"
    assert p["vis"][slot].all()
    keys = set(zip(p["xx"][slot], p["yy"][slot]))
    assert keys == {q for pr in pairs for q in pr}
    tie = labels == "E6 tie"
    key = np.stack([p["xx"][tie], p["yy"][tie], E.bits(p["d"][tie])], 1)
    assert len(np.unique(key, axis=0)) == 3 and p["vis"][tie].all()


def test_ring_store_blocks_have_their_make_up():
    """Per 128-row block (the rows one compute warp votes over) and every per-point view: safe blocks hold no unsafe row; the
    one-unsafe blocks exactly one unsafe row that passes the division-free test, at lane 0, lane 31 or u = 3; the culled block one
    unsafe row that fails it; the all-unsafe block only unsafe rows.  Ties carry descending ids along the rows."""
    rs = E.ring_store(64, 48)
    pts4 = rs["pts4"]
    n = pts4.shape[0]
    assert n % E.CHUNK != 0 and n > 3 * E.CHUNK                    # a partial last chunk
    ids = E.bits(pts4[:, 3]).astype(np.int64)
    assert np.array_equal(ids, rs["ids"]) and np.array_equal(np.sort(ids), np.arange(n)) and ids.max() < E.ID_STALL
    assert np.array_equal(pts4[:, :3], rs["xyz"][ids])
    unsafe = ~E.div_safe(pts4[:, :3][:, 2])                       # c_3 == w == z for every per-point matrix
    want_spot = {"unsafe_lane0": 0, "unsafe_lane31": 31, "unsafe_u3": 113}
    seen = set()
    for c in E.C_VALUES:
        m = E.point_matrix(c)
        cin = E.clip_in(m, pts4[:, :3])
        fin = np.isfinite(pts4[:, :3]).all(1)
        assert np.array_equal(S.clip_coords(m, pts4[fin, :3])[:, 3], pts4[fin, 2])
        for k, kind in enumerate(rs["kinds"]):
            u, ci = unsafe[k * E.BLOCK:(k + 1) * E.BLOCK], cin[k * E.BLOCK:(k + 1) * E.BLOCK]
            if kind in ("safe", "ties"):
                assert not u.any()
            elif kind in want_spot:
                assert np.array_equal(np.nonzero(u)[0], [want_spot[kind]]) and ci[want_spot[kind]]
            elif kind == "unsafe_culled":
                assert u.sum() == 1 and not ci[u].any()
            else:
                assert u.all()
            seen.add(kind)
    assert {"safe", "unsafe_lane0", "unsafe_lane31", "unsafe_u3", "unsafe_culled", "all_unsafe", "ties"} <= seen
    tie = np.nonzero(np.array(rs["labels"])[ids] == "E6 tie")[0]
    assert len(tie) >= 2 * E.BLOCK and np.all(np.diff(ids[tie]) < 0)
    assert len({r // E.CHUNK for r in tie}) >= 2 and len({(r // 32) for r in tie}) >= 8


def test_ring_store_visible_unsafe_rows_are_drawn_by_the_oracle():
    """The visible unsafe rows are ones a shared reciprocal would get wrong (FLT_MAX: a flushed reciprocal; denormals) and that the
    oracle draws, so a kernel that skipped the IEEE fallback would differ."""
    rs = E.ring_store(64, 48)
    lab = np.array(rs["labels"])
    vis_unsafe = lab == "E2 visible unsafe w"
    p = E.project(E.point_matrix(F32(0.25)), rs["xyz"], 64, 48)
    assert p["vis"][vis_unsafe].all()
    w = rs["xyz"][vis_unsafe, 2]
    assert (np.abs(w) == E.FLT_MAX).any() and (_biased_exp_arr(w) == 0).any()


def _biased_exp_arr(x):
    return ((E.bits(x) >> np.uint32(23)) & np.uint32(0xFF)).astype(int)


def test_segmented_store_padding_and_boxes():
    W, H = 64, 48
    lay = E.segmented_store(W, H)
    pts4 = lay["pts4"]
    assert pts4.shape[0] % E.CHUNK == 0
    pad = np.isnan(pts4[:, 0])
    assert np.isnan(pts4[pad, :3]).all() and (E.bits(pts4[pad, 3]) == 0).all() and pad.any()
    assert E.bits(pts4[:, 3]).max() < E.ID_STALL
    boxes = ops._chunk_boxes(torch.from_numpy(pts4)).numpy()
    m = np.stack([E.point_matrix(F32(0.25))])
    dropped = {}
    for (first, chunks, xyz, base, _), tag in zip(lay["parts"], ("mixed", "inside", "just outside", "far outside")):
        b = boxes[first:first + chunks]
        dropped[tag] = S.unit_dropped(m, b[:, :3], b[:, 3:])
        if tag == "inside":
            assert (b[:, 3] == 1).all()                          # the box's hi x lies on the x = w plane
        if tag == "just outside":
            assert (b[:, 0] == E.ONE_P).all()
    assert not dropped["inside"].any() and dropped["far outside"].all() and not dropped["mixed"].any()


def test_sprite_edges():
    W, H = 64, 32
    xyz, labels, sizes = E.sprite_set(W, H)
    labels = np.array(labels)
    c = S.clip_coords(E.view_matrix(F32(1), -0.0), xyz)
    first = lambda tag: np.nonzero(np.char.startswith(labels, f"E7 relative {tag}"))[0]
    assert (E.bits(c[first("c2=+0"), 2]) == 0).all() and (E.bits(c[first("c2=-0"), 2]) == 0x80000000).all()
    assert (c[first("c2 denormal"), 2] == E.DENORM).all() and (c[first("c2<0"), 2] < 0).all()
    with np.errstate(divide="ignore"):
        assert np.isinf(F32(4) / c[first("c2=+0"), 2]).all() and (F32(4) / c[first("c2=-0"), 2] == -np.inf).all()
    p = E.project(E.view_matrix(F32(1), -0.0), xyz, W, H)
    half = np.char.startswith(labels, "E7 half-pixel centre")
    frac_u = p["u"][half] - p["xx"][half].astype(F32)
    assert (frac_u == F32(0.5)).any() and (frac_u < F32(0.5)).any() and (frac_u > F32(0.5)).any()
    wd = lambda s: int(min(max(np.floor(F32(s) + F32(0.5)), 1), 64))
    assert [wd(s) for s in (0.5, E.down(0.5), 1.5, 2.5, 63.5, E.down(63.5), 64.5, E.DENORM)] == [1, 1, 2, 3, 64, 63, 64, 1]
    names = {n for n, _ in E.SPRITE_SIZES}
    assert {"nan", "negative", "denormal", "+inf", "63.5", "pred(63.5)", "64.5"} <= names
    border = np.char.startswith(labels, "E7 border")
    assert p["vis"][border].any() and (p["xx"][border & p["vis"]] == 0).any() and (p["yy"][border & p["vis"]] == H - 1).any()


def test_the_generator_refuses_a_stalling_id():
    with pytest.raises(AssertionError):
        E.pts4_of(np.zeros((1, 3), F32), [E.ID_STALL])
