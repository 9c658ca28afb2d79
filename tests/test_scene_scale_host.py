"""Scene editing at scale without a GPU: the float64 chunk-cull rule against the kernel's float32 per-point test, the store's
chunk boxes and unit table, the limits, ``add_instances`` and the vectorised matrix rule (read_b200.ops.SegmentedPoints,
read_b200.scene_edit.SceneComposer, read_raster_project_segments_culled)."""
import ctypes
from fractions import Fraction

import numpy as np
import pytest
import torch

from read_b200 import _lib, ops, synth
from read_b200.scene_edit import SceneComposer, segment_matrices
from scene_scale_util import box_culled, f32_fma, point_in, unit_dropped

CHUNK = ops.SEGMENT_CHUNK


def _round_f32(v):
    """Correctly rounded float32 of the exact rational v (ties to even)."""
    r = np.float32(float(v))
    cands = [r, np.nextafter(r, np.float32(np.inf)), np.nextafter(r, np.float32(-np.inf))]
    cands = [c for c in cands if np.isfinite(c)]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - v), int(np.array(c).view(np.uint32)) & 1))
    return best


def test_f32_fma_restatement_is_the_correctly_rounded_fma():
    rng = np.random.default_rng(0)
    a = rng.normal(size=3000).astype(np.float32) * np.float32(2.0) ** rng.integers(-20, 20, 3000).astype(np.float32)
    b = rng.normal(size=3000).astype(np.float32)
    c = -(a.astype(np.float64) * b).astype(np.float32)                  # heavy cancellation: the rounding of a*b decides
    c[::3] = rng.normal(size=1000).astype(np.float32)
    # exact float32 midpoints: a*b + c lands half-way between two float32 values, with and without a tiny remainder
    a[:200] = np.float32(1.0) + np.float32(2.0 ** -23) * rng.integers(1, 1000, 200).astype(np.float32)
    b[:200] = np.float32(1.0) + np.float32(2.0 ** -12)
    c[:200] = np.float32(2.0 ** 24) * np.sign(rng.normal(size=200)).astype(np.float32)
    got = f32_fma(a, b, c)
    for i in range(a.size):
        want = _round_f32(Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i])))
        assert got[i].view(np.uint32) == np.float32(want).view(np.uint32), (i, a[i], b[i], c[i])


def _samples(lo, hi, rng, k=48):
    """Corners, random interior points and points on every face of the float32 box [lo, hi]."""
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    corners = np.array([[hi[j] if (c >> j) & 1 else lo[j] for j in range(3)] for c in range(8)], np.float32)
    t = rng.uniform(0, 1, (k, 3))
    inner = (lo + t * (hi.astype(np.float64) - lo)).astype(np.float32)
    inner = np.clip(inner, lo, hi)
    faces = np.repeat(inner[:6], 1, 0).copy()
    for f in range(6):
        faces[f, f % 3] = (lo if f < 3 else hi)[f % 3]
    return np.concatenate([corners, inner, faces])


def _assert_conservative(m, lo, hi, rng):
    culled = box_culled(m, lo, hi)
    for i in np.nonzero(culled)[0]:
        pts = _samples(lo[i], hi[i], rng)
        inside = point_in(m, pts)
        assert not inside.any(), (m, lo[i], hi[i], pts[inside][:3])
    return culled


def _camera_matrix(rng, W=256, H=128):
    proj, _ = synth.camera_batch(W, H, [0])
    pose = np.eye(4)
    a = rng.uniform(-np.pi, np.pi)
    pose[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    pose[:3, 3] = rng.uniform(-50, 50, 3)
    return synth.total_matrix(proj, pose[None].astype(np.float32))[0]


def test_cull_rule_is_conservative_on_random_boxes_and_matrices():
    rng = np.random.default_rng(1)
    n_culled = n_total = 0
    for trial in range(40):
        m = _camera_matrix(rng) if trial % 2 == 0 else rng.normal(size=(4, 4)).astype(np.float32)
        c = rng.uniform(-200, 200, (300, 3))
        ext = rng.uniform(0, 1, (300, 3)) * 10.0 ** rng.uniform(-3, 2, (300, 1))
        lo, hi = (c - ext).astype(np.float32), (c + ext).astype(np.float32)
        culled = _assert_conservative(m, lo, hi, rng)
        n_culled += int(culled.sum())
        n_total += culled.size
    assert 0.2 * n_total < n_culled < n_total                       # the rule does cull, and not everything


def test_cull_rule_faces_one_ulp_inside_and_outside_every_plane():
    """Matrix with c_i = x_i and c_3 = 1: the clip volume is the cube |x_i| <= 1 exactly.  A box whose near face lies 1 ulp
    inside a plane, or on it, holds a drawn point and must not be culled; 1 ulp outside, every point is culled, and the rule
    may not cull unless all of them are."""
    rng = np.random.default_rng(2)
    m = np.eye(4, dtype=np.float32)
    one = np.float32(1.0)
    for axis in range(3):
        for sign in (1.0, -1.0):
            for face, drawn in ((np.nextafter(one, np.float32(0)), True), (one, True), (np.nextafter(one, np.float32(2)), False)):
                lo = np.full(3, -0.5, np.float32)
                hi = np.full(3, 0.5, np.float32)
                if sign > 0:
                    lo[axis], hi[axis] = face, np.float32(3.0)
                else:
                    lo[axis], hi[axis] = np.float32(-3.0), -face
                corner = np.where(np.arange(3) == axis, lo if sign > 0 else hi, np.float32(0.0))[None].astype(np.float32)
                assert bool(point_in(m, corner)[0]) == drawn
                culled = _assert_conservative(m, lo[None], hi[None], rng)[0]
                assert not (drawn and culled)
            # a box well outside the plane is culled
            lo = np.full(3, -0.5, np.float32)
            hi = np.full(3, 0.5, np.float32)
            (lo, hi)[0 if sign > 0 else 1][axis] = np.float32(1.01 * sign)
            (lo, hi)[1 if sign > 0 else 0][axis] = np.float32(3.0 * sign)
            assert box_culled(m, lo[None], hi[None])[0]


def test_cull_rule_behind_the_camera_near_w_zero_and_huge_coordinates():
    rng = np.random.default_rng(3)
    proj, view = synth.camera_batch(256, 128, [0])
    m = synth.total_matrix(proj, view)[0]
    # behind the camera (the camera looks along -z): boxes at z > 0
    c = np.stack([rng.uniform(-30, 30, 500), rng.uniform(-5, 5, 500), rng.uniform(0.5, 300, 500)], 1)
    lo, hi = (c - 0.5).astype(np.float32), (c + 0.5).astype(np.float32)
    behind = _assert_conservative(m, lo, hi, rng)
    assert behind.mean() > 0.9
    # straddling w = 0 (the camera plane): never culled by a rule that must hold for every point
    c = np.stack([rng.uniform(-1, 1, 200), rng.uniform(-1, 1, 200), rng.uniform(-1e-3, 1e-3, 200)], 1)
    lo, hi = (c - 1e-2).astype(np.float32), (c + 1e-2).astype(np.float32)
    _assert_conservative(m, lo, hi, rng)
    wz = np.array([[0.0, 0.0, -1e-30]], np.float32)
    _assert_conservative(m, wz - np.float32(1e-38), wz + np.float32(1e-38), rng)
    # huge coordinates: products near the float32 range give no claim (float32 could overflow), smaller ones stay exact
    for scale in (1e15, 1e30, 1e36, 3e38):
        c = rng.uniform(-1, 1, (200, 3)) * scale
        lo, hi = (c - 0.1 * scale).astype(np.float32), np.minimum(c + 0.1 * scale, 3.4e38).astype(np.float32)
        _assert_conservative(m, lo, hi, rng)
    big = np.array([[1e37, 1e37, 1e37]], np.float32)
    assert not box_culled(m * np.float32(1e3), big, big * np.float32(2))[0]


def test_non_finite_matrices_and_boxes_never_cull():
    far_lo, far_hi = np.array([[100.0, 100.0, 100.0]], np.float32), np.array([[101.0, 101.0, 101.0]], np.float32)
    m = np.eye(4, dtype=np.float32)
    assert box_culled(m, far_lo, far_hi)[0]
    for bad in (np.nan, np.inf, -np.inf):
        for k in (0, 5, 15):
            mb = m.copy()
            mb.reshape(-1)[k] = bad
            assert not box_culled(mb, far_lo, far_hi)[0]
    seg_m = m[None]
    assert unit_dropped(seg_m, far_lo, far_hi)[0]
    for bad in (np.inf, -np.inf):
        lo, hi = far_lo.copy(), far_hi.copy()
        hi[0, 1] = bad if bad > 0 else hi[0, 1]
        lo[0, 1] = bad if bad < 0 else lo[0, 1]
        assert not unit_dropped(seg_m, lo, hi)[0]                          # a point at infinity may pass |c| <= |w|
    empty_lo, empty_hi = np.full((1, 3), np.inf, np.float32), np.full((1, 3), -np.inf, np.float32)
    assert unit_dropped(seg_m, empty_lo, empty_hi)[0]                      # padding only: always dropped


# ---------------------------------------------------------------------------------------------------------- store and table
def _scene(n, seed):
    xyz = torch.from_numpy(synth.street_scene(n, depth=40.0, seed=seed))
    return xyz, torch.rand((1, 8, n), generator=torch.Generator().manual_seed(seed))


def test_chunk_boxes_leave_padding_out():
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(5000, 1)
    s = comp.add_scene(xyz, tex)
    for start, size in ((0, 1), (10, 1023), (2000, 1024), (3100, 1025)):
        comp.add_object(s, np.arange(start, start + size))
    st = comp.store
    assert st.boxes.shape == (st.n // CHUNK, 6) and st.boxes.dtype == torch.float32
    rows = st.pts4.view(-1, CHUNK, 4)
    for c in range(st.n // CHUNK):
        real = rows[c][~torch.isnan(rows[c][:, :3]).any(1), :3]
        assert real.shape[0] > 0                                             # ceil(n / 1024) chunks: none is padding only
        assert torch.equal(st.boxes[c, :3], real.min(0).values) and torch.equal(st.boxes[c, 3:], real.max(0).values)
    # a chunk of padding only gets the empty box; a NaN row of a real chunk is left out too
    blk = torch.full((3 * CHUNK, 4), float("nan"))
    blk[:, 3] = 0.0
    blk[:5, :3] = torch.tensor([[1.0, 2.0, 3.0], [-1.0, 0.5, 7.0], [0.0, 0.0, 0.0], [4.0, -3.0, 1.0], [2.0, 2.0, 2.0]])
    blk[2 * CHUNK, :3] = torch.tensor([5.0, 6.0, 7.0])
    blk[2 * CHUNK + 1, :3] = torch.tensor([float("nan"), 100.0, 100.0])
    boxes = ops._chunk_boxes(blk)
    assert boxes[0].tolist() == [-1.0, -3.0, 0.0, 4.0, 2.0, 7.0]
    assert boxes[1].tolist() == [float("inf")] * 3 + [float("-inf")] * 3
    assert boxes[2].tolist() == [5.0, 6.0, 7.0, 5.0, 6.0, 7.0]
    assert unit_dropped(np.eye(4, dtype=np.float32)[None], boxes[1:2, :3].numpy(), boxes[1:2, 3:].numpy())[0]


def test_unit_table_mirrors_the_segment_table():
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(6000, 2)
    s = comp.add_scene(xyz, tex)
    o = comp.add_object(s, np.arange(100, 2200))
    comp.add_object(s, [])                                                   # an empty object: a segment of no chunks
    comp.add_instances(o, np.stack([np.eye(4)] * 3))
    st = comp.store
    want = [[st.first_chunk[i], st.chunks[i], i] for i in range(st.nseg)]
    assert st.seg_table.dtype == torch.int32 and st.seg_table.tolist() == want
    assert st.nunits == sum(st.chunks[i] for i in range(st.nseg)) == 4 + 3 + 0 + 3 * 3
    assert st.visible_flags().tolist() == [1] * st.nseg
    st.set_visible(1, False)
    assert st.visible_flags().tolist()[1] == 0 and st.visible[1] == 0      # one buffer behind both views


# ---------------------------------------------------------------------------------------------------------------- limits
def test_limits_and_their_errors():
    assert ops.MAX_SEGMENTS == _lib.MAX_SEGMENTS_CULLED == 4096 and _lib.MAX_SEGMENTS == 128
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(2000, 4)
    o = comp.add_object(comp.add_scene(xyz, tex), [0, 1, 2])
    hs = comp.add_instances(o, np.stack([np.eye(4)] * (ops.MAX_SEGMENTS - 2)))
    assert len(hs) == ops.MAX_SEGMENTS - 2 and comp.store.nseg == ops.MAX_SEGMENTS
    with pytest.raises(ValueError, match="segments"):
        comp.add_instances(o, np.eye(4)[None])
    with pytest.raises(ValueError, match="finite"):
        comp.add_instances(o, np.full((1, 4, 4), np.nan))
    with pytest.raises(ValueError, match="finite"):
        comp.add_instances(o, np.eye(4))                                     # [4,4], not [K,4,4]


def test_culled_entry_point_rejects_bad_arguments_before_device_work():
    lib = _lib.load()
    ptr = 0x100000
    ws_need = lib.read_raster_cull_workspace_bytes(4)
    assert ws_need >= 16 + 2 * 8 * 4 and lib.read_raster_cull_workspace_bytes(-1) == -1

    def call(n=2 * CHUNK, nseg=2, nunits=4, B=1, W=64, H=32, L=4, pts=ptr, ws=ptr, ws_bytes=ws_need, table=ptr):
        return lib.read_raster_project_segments_culled(pts, n, table, nseg, nunits, ptr, ptr, ptr, ws, ws_bytes, B, W, H, L, ptr,
                                                       None)

    cases = ((dict(n=CHUNK + 1), b"whole"), (dict(pts=ptr + 4), b"aligned"),
             (dict(nseg=ops.MAX_SEGMENTS + 1), b"segments"), (dict(nseg=-1), b"segments"), (dict(table=None), b"null"),
             (dict(nunits=-1), b"units"), (dict(nunits=1 << 31), b"units"), (dict(nseg=0), b"units"),
             (dict(B=9), b"views"), (dict(B=0), b"views"), (dict(W=64, H=30), b"nested"), (dict(W=0), b"positive"),
             (dict(ws=None), b"workspace"), (dict(ws=ptr + 8), b"workspace"), (dict(ws_bytes=ws_need - 1), b"workspace"))
    for kw, msg in cases:
        assert call(**kw) != 0, kw
        assert msg in lib.read_last_error(), (kw, lib.read_last_error())
    # the parameter-table entry keeps its own limit of 128
    first = (ctypes.c_int64 * 1)(0)
    assert lib.read_raster_project_segments(ptr, CHUNK, first, first, (ctypes.c_uint8 * 1)(1), 129, ptr, 1, 64, 32, 4, ptr,
                                            None) != 0
    assert b"segments" in lib.read_last_error()


# ---------------------------------------------------------------------------------------------- composer: vectorised host work
def _loop_transforms(comp):
    """The per-segment rule as it was written before the arrays: P for a scene's static part, P @ M otherwise."""
    out = np.empty((len(comp._segments), 4, 4))
    for s, (h, si) in enumerate(comp._segments):
        P = comp._scenes[si]["P"]
        out[s] = P if h.kind == "scene" else P @ comp._entry(h)["M"]
    return out


def _big_composer(rng, n_inst=300):
    comp = SceneComposer(device="cpu")
    scenes = []
    for k in range(3):
        xyz, tex = _scene(3000, 10 + k)
        P = np.eye(4)
        P[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        P[:3, 3] = rng.normal(size=3) * 50
        scenes.append(comp.add_scene(xyz, tex, placement=P))
    objs = [comp.add_object(scenes[k % 3], np.arange(100 * (k // 3), 100 * (k // 3) + 50)) for k in range(12)]

    def rigid():
        M = np.eye(4)
        M[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        M[:3, 3] = rng.normal(size=3) * 10
        return M
    for o in objs:
        comp.set_transform(o, rigid())
    insts = comp.add_instances(objs[0], np.stack([rigid() for _ in range(n_inst)]))
    insts += comp.add_instances(objs[5], np.stack([rigid() for _ in range(20)]))
    return comp, scenes, objs, insts, rigid


def test_vectorised_transforms_and_matrices_equal_the_per_segment_rule_bit_for_bit():
    rng = np.random.default_rng(5)
    comp, scenes, objs, insts, rigid = _big_composer(rng)
    proj, view = synth.camera_batch(256, 128, [1, 7, 13])
    total = synth.total_matrix(proj, view)
    for edit in range(4):
        got = comp.segment_transforms()
        want = _loop_transforms(comp)
        assert got.tobytes() == want.tobytes(), edit
        assert comp.segment_matrices(total).tobytes() == segment_matrices(total, want).tobytes()
        comp.set_transform(scenes[edit % 3], rigid())                      # edits between frames: arrays follow
        comp.set_transform(objs[edit], rigid())
        comp.set_transform(insts[7 * edit], rigid())
    # visibility: vectorised flags equal the per-segment rule
    comp.set_visible(objs[0], False)
    comp.set_visible(insts[3], False)
    comp.set_visible(scenes[1], False)
    want = [int(comp._scenes[si]["visible"] and (h.kind == "scene" or comp._entry(h)["visible"])) for h, si in comp._segments]
    assert comp.store.visible_flags().tolist() == want
    assert want.count(0) == 1 + 1 + 4 + 1                                    # object 0, instance 3, scene 1 + its 4 objects


def test_add_instances_equals_repeated_add_instance():
    rng = np.random.default_rng(6)
    Ms = np.stack([np.eye(4) + np.pad(rng.normal(size=(3, 4)), ((0, 1), (0, 0))) for _ in range(17)])
    xyz, tex = _scene(3000, 7)
    comps = []
    for batched in (False, True):
        comp = SceneComposer(device="cpu")
        o = comp.add_object(comp.add_scene(xyz, tex), np.arange(500, 1700))
        hs = comp.add_instances(o, Ms) if batched else [comp.add_instance(o, M) for M in Ms]
        assert [(h.kind, h.index) for h in hs] == [("instance", i) for i in range(17)]
        comps.append(comp)
    a, b = comps[0].store, comps[1].store
    assert a.nseg == b.nseg == 19 and torch.equal(a.seg_table, b.seg_table)
    assert torch.equal(torch.nan_to_num(a.pts4, nan=9.0), torch.nan_to_num(b.pts4, nan=9.0)) and torch.equal(a.boxes, b.boxes)
    total = synth.total_matrix(*synth.camera_batch(128, 64, [2]))
    assert comps[0].segment_matrices(total).tobytes() == comps[1].segment_matrices(total).tobytes()
