"""Cylindrical panoramas without a GPU: Panorama's validation and float32 constants, the single-precision atan2 of the kernel,
the numpy restatement of the projection (tests/oracle_panorama.py) and the edge point sets it plants, proven bit for bit."""
import ctypes
import math

import numpy as np
import pytest

import oracle_panorama as O
from read_b200 import _lib
from read_b200.panorama import Panorama, DEFAULT_MARGIN

F32 = np.float32
PANOS = [Panorama(1024, 256, margin=64), Panorama(512, 128, hfov_deg=180), Panorama(256, 64, elevation_deg=(-10, 40), margin=32),
         Panorama(4096, 1024, margin=128), Panorama(640, 64, hfov_deg=150, elevation_deg=(-60, 5))]


@pytest.mark.parametrize("kw", [
    dict(width=100, height=64), dict(width=0, height=64), dict(width=256, height=40), dict(width=256, height=64, margin=8),
    dict(width=256, height=64, margin=144), dict(width=256, height=64, hfov_deg=0), dict(width=256, height=64, hfov_deg=361),
    dict(width=256, height=64, hfov_deg=180, margin=16), dict(width=256, height=64, elevation_deg=(-89, 10)),
    dict(width=256, height=64, elevation_deg=(10, 10)), dict(width=256, height=64, elevation_deg=(20, 10)),
    dict(width=256, height=64, znear=0), dict(width=256, height=64, znear=5, zfar=5), dict(width=256, height=64, zfar=math.inf),
    dict(width=256, height=64, znear=math.nan), dict(width=1 << 17, height=64)])
def test_panorama_rejects_bad_geometry(kw):
    with pytest.raises(ValueError):
        Panorama(**kw)


def test_panorama_default_margin_and_plane():
    assert Panorama(1024, 256).margin == DEFAULT_MARGIN == 128
    assert Panorama(128, 64).margin == 64                   # capped at half the width
    assert Panorama(96, 64).margin == 48
    assert Panorama(1024, 256, hfov_deg=180).margin == 0
    p = Panorama(1024, 256, margin=64)
    assert p.full and p.plane_width == 1152
    q = p.scaled(2)
    assert (q.width, q.height, q.margin, q.elevation_deg, q.hfov_deg) == (2048, 512, 128, p.elevation_deg, 360.0)
    assert p.scaled(1) is p


@pytest.mark.parametrize("p", PANOS, ids=repr)
def test_panorama_constants_are_float64_rounded_once(p):
    c = p.constants()
    hfov = 2 * math.pi if p.full else math.radians(p.hfov_deg)
    lo, hi = (math.radians(e) for e in p.elevation_deg)
    assert all(v.dtype == np.float32 for v in c.values())
    assert c["theta_half"] == F32(hfov / 2)
    assert c["k_w"] == F32(p.width / hfov)
    assert c["t_hi"] == F32(math.tan(hi))
    assert c["k_h"] == F32(p.height / (math.tan(hi) - math.tan(lo)))
    assert (c["znear"], c["zfar"]) == (F32(p.znear), F32(p.zfar))
    if p.full:
        assert c["theta_half"] == O.PI_F                    # the kernel's pi: theta + theta_half >= 0
    d = p.desc()
    assert (d.theta_half, d.k_w, d.t_hi, d.k_h, d.znear, d.zfar) == tuple(float(c[k]) for k in
                                                                          ("theta_half", "k_w", "t_hi", "k_h", "znear", "zfar"))
    assert (d.width, d.margin, d.full) == (p.width, p.margin, int(p.full))


def test_desc_layout_matches_the_header():
    # read_panorama_desc: six floats then three int32, no padding
    assert ctypes.sizeof(_lib.ReadPanoramaDesc) == 36
    assert _lib.ReadPanoramaDesc.width.offset == 24 and _lib.ReadPanoramaDesc.full.offset == 32
    for name in ("read_raster_panorama_sorted", "read_raster_panorama_segments_culled"):
        assert name in _lib.EXPORTS


def test_world_to_camera_is_the_float32_inverse():
    rng = np.random.default_rng(3)
    a = rng.normal(size=(3, 3))
    q, _ = np.linalg.qr(a)
    view = np.eye(4, dtype=np.float32)
    view[:3, :3] = q
    view[:3, 3] = (4.0, -1.5, 20.0)
    v = Panorama.world_to_camera(view)
    assert v.dtype == np.float32 and np.array_equal(v, np.linalg.inv(view.astype(np.float32)).astype(np.float32))
    assert Panorama.world_to_camera(np.stack([view, view])).shape == (2, 4, 4)


def test_atan2_sweep_error_monotonicity_and_range():
    th = np.linspace(-np.pi, np.pi, 4_000_001)
    for r in (1.0, 1e-3, 7e4):
        x, f = (r * np.sin(th)).astype(F32), (r * np.cos(th)).astype(F32)
        t = O.atan2_f32(x, f)
        ref = np.arctan2(x.astype(np.float64), f.astype(np.float64))
        err = np.abs(t.astype(np.float64) - ref)
        err = np.minimum(err, np.abs(err - 2 * np.pi))                  # +-pi are the same direction
        assert err.max() <= 2e-6
        order = np.argsort(ref, kind="stable")
        assert np.all(np.diff(t[order]) >= 0)                           # non-decreasing along the sweep
        assert np.all(np.abs(t) <= O.PI_F)
        assert np.all((t + O.PI_F).astype(F32) >= 0)
    # the axes and the seam exactly
    z = F32(0)
    cases = [(z, F32(1), 0.0), (F32(1), z, O.HALF_PI_F), (F32(-1), z, -O.HALF_PI_F), (z, F32(-1), O.PI_F),
             (F32(-0.0), F32(-1), -O.PI_F), (F32(1), F32(1), None)]
    for x, f, want in cases:
        got = O.atan2_f32(np.array([x]), np.array([f]))[0]
        if want is not None:
            assert got == F32(want) and np.signbit(got) == np.signbit(F32(want))
    assert O.atan2_f32(np.array([z]), np.array([z]))[0] == 0


def _brute_keys(pts, ids, m, p):
    """Level 0 by a plain loop over the points: the reference for np.minimum.at."""
    vis, key, i0, two, i1 = O.project(m, pts, ids, p)
    out = {}
    for i in range(len(pts)):
        for ok, idx in ((vis[i], i0[i]), (two[i], i1[i])):
            if ok:
                out[int(idx)] = min(out.get(int(idx), int(O.EMPTY)), int(key[i]))
    return out


@pytest.mark.parametrize("p", PANOS[:3], ids=repr)
def test_oracle_level0_and_levels(p):
    rng = np.random.default_rng(7)
    n = 4000
    pts = np.concatenate([rng.normal(0, 15, (n, 2)), rng.uniform(-2, 3, (n, 1))], 1)[:, [0, 2, 1]].astype(F32)
    ids = np.arange(n, dtype=np.uint64) * 7 % n
    m = O.EDGE_VIEW
    z = O.level0(pts, ids, m, p)
    assert z.shape == (1, p.height, p.plane_width)
    flat = z.reshape(-1)
    want = _brute_keys(pts, ids, m, p)
    got = {i: int(v) for i, v in enumerate(flat) if v != O.EMPTY}
    assert got == want and len(got) > 100
    lv = O.derive(z)
    for l in range(1, 4):
        a = lv[l - 1][0]
        assert lv[l].shape[1:] == (p.height >> l, p.plane_width >> l)
        assert lv[l][0][1, 1] == min(a[2, 2], a[2, 3], a[3, 2], a[3, 3])
    if p.full and p.margin:
        M, W = p.margin, p.width
        for l in range(4):
            s = lv[l][0]
            assert np.array_equal(s[:, :M >> l], s[:, W >> l:(W + M) >> l])          # left margin = the panorama's right end
            assert np.array_equal(s[:, (W + M) >> l:], s[:, M >> l:(2 * M) >> l])     # right margin = its left end


@pytest.mark.parametrize("p", PANOS, ids=repr)
def test_edge_sets_are_planted_bit_for_bit(p):
    pts, labels, expect = O.edge_set(p)
    assert {"E1", "E2", "E3", "E4", "E6"} <= set(labels)
    for q, label, want in zip(pts, labels, expect):
        vis, col, row, two = O.one(q, p)
        if want is None:
            continue
        assert vis == want[0], (label, q)
        if want[1] is not None:
            assert col == want[1], (label, q, col)
        if want[2] is not None:
            assert row == want[2], (label, q, row)
    E2 = [q for q, lab in zip(pts, labels) if lab == "E2"]
    for a, b in zip(E2[0::2], E2[1::2]):          # adjacent float32 coordinates: the two points straddle the boundary
        k = np.flatnonzero((a != b))
        assert len(k) == 1 and np.nextafter(a[k[0]], b[k[0]]) == b[k[0]]
    if p.full:
        # x = +0 behind the camera: u is exactly W before the seam wraps it to column 0; x = -0: u = 0
        c = p.constants()
        u = lambda x: (((O.atan2_f32(np.array([x]), np.array([F32(-10)])) + c["theta_half"]).astype(F32)) * c["k_w"]).astype(F32)
        assert int(u(F32(0.0))[0]) in (p.width, p.width - 1) and u(F32(-0.0))[0] == 0
        assert O.one((0.0, 0.5, 10.0), p)[1] == 0 and O.one((-0.0, 0.5, 10.0), p)[1] == 0
        M = p.margin
        cols = [O.one(q, p) for q, lab in zip(pts, labels) if lab == "E2"]
        assert any(t for _, _, _, t in cols) and any(v and not t for v, _, _, t in cols)
        assert {M - 1, M, p.width - M - 1, p.width - M} <= {c for _, c, _, _ in cols}


def test_edge_ties_resolve_to_the_lowest_id():
    p = PANOS[0]
    pts, labels, _ = O.edge_set(p)
    ties = pts[[i for i, lab in enumerate(labels) if lab == "E6"]]
    ids = np.arange(len(ties), 0, -1).astype(np.uint64)              # the later point of each pair has the lower id
    vis, key, i0, two, i1 = O.project(O.EDGE_VIEW, ties, ids, p)
    assert np.all(vis)
    z = O.level0(ties, ids, O.EDGE_VIEW, p).reshape(-1)
    for j in range(0, len(ties), 2):
        assert key[j] >> np.uint64(32) == key[j + 1] >> np.uint64(32) and i0[j] == i0[j + 1]
        assert z[i0[j]] == key[j + 1]
        if two[j]:
            assert z[i1[j]] == key[j + 1]


def test_edge_store_rows_mix_seam_and_padding_in_every_block():
    p = PANOS[0]
    pts, _, _ = O.edge_set(p)
    rows, ids = O.edge_store_rows(pts, np.arange(1, len(pts) + 1, dtype=np.uint32))
    nan = np.isnan(rows[:, 0])
    assert nan.sum() == 64 and np.all(ids[nan] == 0)
    _, _, _, two, _ = O.project(O.EDGE_VIEW, rows, ids, p)
    first = rows[:32]
    t = O.project(O.EDGE_VIEW, first, ids[:32], p)
    assert t[3].any() and (t[0] & ~t[3]).any() and np.isnan(first[:, 0]).any()   # one warp: two-splat, one-splat and padding
    assert two.sum() > 4


def _box_points(lo, hi, n, rng):
    return (lo + (hi - lo) * rng.random((n, 3))).astype(F32)


def test_radial_cull_is_conservative():
    """A box culled by box_beyond holds no point the kernel would draw, whatever the matrix (rigid, scaled or sheared)."""
    rng = np.random.default_rng(11)
    p = Panorama(256, 64, zfar=50.0, margin=16)
    zfar = p.constants()["zfar"]
    culled = kept = 0
    for trial in range(300):
        m = np.eye(4, dtype=F32)
        m[:3, :3] = rng.normal(size=(3, 3)) * rng.choice([0.2, 1.0, 3.0])
        m[:3, 3] = rng.normal(0, 40, 3)
        lo = rng.normal(0, 40, 3).astype(F32)
        hi = (lo + rng.uniform(0, 8, 3)).astype(F32)
        beyond = O.box_beyond(m, lo[None], hi[None], zfar)[0]
        pts = np.concatenate([_box_points(lo, hi, 200, rng), np.array([[a, b, c] for a in (lo[0], hi[0]) for b in (lo[1], hi[1])
                                                                        for c in (lo[2], hi[2])], F32)])
        cc = O.clip_coords(m, pts)
        x, f = cc[:, 0], (-cc[:, 2]).astype(F32)
        r = np.sqrt(((x * x).astype(F32) + (f * f).astype(F32)).astype(F32)).astype(F32)
        if beyond:
            culled += 1
            assert np.all(r > zfar)
        else:
            kept += 1
    assert culled > 20 and kept > 20
    # tight: a unit box whose nearest point is one metre beyond zfar is culled, one straddling zfar is not
    m = np.eye(4, dtype=F32)
    assert O.box_beyond(m, np.array([[0, 0, 51]], F32), np.array([[1, 1, 52]], F32), zfar)[0]
    assert not O.box_beyond(m, np.array([[0, 0, 49.5]], F32), np.array([[1, 1, 50.5]], F32), zfar)[0]
    bad = m.copy()
    bad[0, 0] = np.nan
    assert not O.box_beyond(bad, np.array([[0, 0, 500]], F32), np.array([[1, 1, 501]], F32), zfar)[0]
