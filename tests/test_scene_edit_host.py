"""Scene editing and stitching without a GPU: the segmented store's layout, the matrix rule and the argument errors
(read_b200.ops.SegmentedPoints, read_b200.scene_edit.SceneComposer)."""
import ctypes

import numpy as np
import pytest
import torch

from read_b200 import _lib, ops, synth
from read_b200.scene_edit import SceneComposer, segment_matrices
from read_b200.texture import PointTexture

CHUNK = ops.SEGMENT_CHUNK


def _scene(n, seed):
    xyz = torch.from_numpy(synth.street_scene(n, depth=40.0, seed=seed))
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(seed))
    return xyz, tex


def _composer():
    comp = SceneComposer(device="cpu")
    xyz_a, tex_a = _scene(5000, 1)
    xyz_b, tex_b = _scene(3000, 2)
    a = comp.add_scene(xyz_a, tex_a)
    place = np.eye(4)
    place[:3, 3] = [40.0, 0.0, -8.0]
    b = comp.add_scene(xyz_b, tex_b, placement=place)
    sizes = [0, 1, 1023, 1024, 1025]
    objs, start = [], 0
    for s in sizes:
        objs.append(comp.add_object(a, np.arange(start, start + s)))
        start += s
    inst = comp.add_instance(objs[3], np.diag([1.0, 1.0, 1.0, 1.0]))
    return comp, (a, b), objs, inst, (xyz_a, xyz_b), (tex_a, tex_b), sizes


def _ids_of_rows(pts4):
    return pts4[:, 3].contiguous().view(torch.int32).to(torch.int64)


def test_segment_layout_padding_and_global_ids():
    comp, (a, b), objs, inst, (xyz_a, xyz_b), _, sizes = _composer()
    st = comp.store
    assert b.base == 5000 and comp.total == 8000 and st.n_ids == 8000
    assert st.nseg == 2 + len(sizes) + 1 and st.n % CHUNK == 0
    # segment order: scene a's static part, its objects, scene b, then the instance
    carved = sum(sizes)
    want_rows = [5000 - carved] + sizes + [3000] + [sizes[3]]
    world = [xyz_a, xyz_b]
    seen_rows = set()
    for s in range(st.nseg):
        f, c = st.first_chunk[s], st.chunks[s]
        assert c == -(-want_rows[s] // CHUNK), s                                   # padded to whole chunks
        rows = st.pts4[f * CHUNK:(f + c) * CHUNK]
        n = want_rows[s]
        real, pad = rows[:n], rows[n:]
        assert torch.isnan(pad[:, :3]).all() and (_ids_of_rows(pad) == 0).all()   # NaN coordinates, id word 0 (not all ones)
        assert not torch.isnan(real[:, :3]).any()
        gid = _ids_of_rows(real)
        assert torch.equal(torch.sort(gid).values, torch.sort(st.ids(s)).values)
        scene = 1 if s == len(sizes) + 1 else 0
        base = 5000 if scene else 0
        assert torch.equal(real[:, :3], world[scene][gid - base])                 # each row carries its point's global id
        if s < st.nseg - 1:
            assert (f, c) not in seen_rows or c == 0
            seen_rows.add((f, c))
    # the instance draws the SAME rows as its object
    o3 = 1 + 3
    assert (st.first_chunk[st.nseg - 1], st.chunks[st.nseg - 1]) == (st.first_chunk[o3], st.chunks[o3])
    assert torch.equal(st.ids(st.nseg - 1), st.ids(o3))
    # every global id appears exactly once outside the instance
    all_ids = torch.cat([st.ids(s) for s in range(st.nseg - 1)])
    assert torch.equal(torch.sort(all_ids).values, torch.arange(8000))


def test_composed_texture_is_the_concatenation():
    comp, _, _, _, _, (tex_a, tex_b), _ = _composer()
    assert torch.equal(comp.texture.texture_.detach(), torch.cat([tex_a, tex_b], 2))


def _restated(total_m, P, M):
    """T[i][k] = sum_j total_m[i][j] * (P @ M)[j][k], every operation in float64 (Python floats), rounded once to float32."""
    PM = [[sum(P[i][j] * M[j][k] for j in range(4)) for k in range(4)] for i in range(4)]
    T = [[0.0] * 4 for _ in range(4)]
    for i in range(4):
        for k in range(4):
            acc = float(total_m[i][0]) * PM[0][k]
            for j in range(1, 4):
                acc = acc + float(total_m[i][j]) * PM[j][k]
            T[i][k] = acc
    return np.array(T, dtype=np.float64).astype(np.float32)


def test_matrix_rule_against_a_float64_restatement():
    comp, (a, b), objs, inst, *_ = _composer()
    rng = np.random.default_rng(0)
    M = np.eye(4)
    M[:3, :3] = np.linalg.qr(rng.normal(size=(3, 3)))[0]
    M[:3, 3] = rng.normal(size=3) * 3
    comp.set_transform(objs[2], M)
    comp.set_transform(inst, M @ M)
    proj, view = synth.camera_batch(256, 128, [3, 11])
    total = synth.total_matrix(proj, view)
    seg_m = comp.segment_matrices(total)
    assert seg_m.dtype == np.float32 and seg_m.shape == (comp.store.nseg, 2, 4, 4)
    P_b = comp._scenes[1]["P"]
    for bb in range(2):
        np.testing.assert_array_equal(seg_m[3, bb], _restated(total[bb], np.eye(4), M))              # object 2 of scene a
        np.testing.assert_array_equal(seg_m[6, bb], _restated(total[bb], P_b, np.eye(4)))            # scene b (placed)
        np.testing.assert_array_equal(seg_m[7, bb], _restated(total[bb], np.eye(4), M @ M))          # the instance


def test_identity_placement_and_transform_give_total_m_bit_for_bit():
    comp, (a, b), *_ = _composer()
    comp.set_transform(b, np.eye(4))                             # scene b back at the origin
    proj, view = synth.camera_batch(256, 128, [0, 5, 9])
    total = synth.total_matrix(proj, view)
    seg_m = comp.segment_matrices(total)
    for s in range(seg_m.shape[0]):
        assert seg_m[s].tobytes() == total.tobytes()
    one = segment_matrices(total[0], np.eye(4)[None])             # [4,4] total_m: B = 1
    assert one.shape == (1, 1, 4, 4) and one[0, 0].tobytes() == total[0].tobytes()


def test_overlapping_objects_raise():
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(2000, 3)
    s = comp.add_scene(xyz, tex)
    comp.add_object(s, np.arange(0, 100))
    with pytest.raises(ValueError, match="at most one object"):
        comp.add_object(s, np.arange(50, 150))
    with pytest.raises(ValueError):
        comp.add_object(s, [5000])                              # not a point of the scene
    with pytest.raises(ValueError):
        comp.add_object(s, [200, 200])


def test_more_segments_than_the_limit_raise():
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(2000, 4)
    s = comp.add_scene(xyz, tex)
    o = comp.add_object(s, [0])
    for _ in range(ops.MAX_SEGMENTS - 2):
        comp.add_instance(o, np.eye(4))
    assert comp.store.nseg == ops.MAX_SEGMENTS
    with pytest.raises(ValueError, match="segments"):
        comp.add_instance(o, np.eye(4))
    part = (xyz[:10], torch.arange(10))
    with pytest.raises(ValueError, match="segments"):
        ops.SegmentedPoints([part], [0] * (ops.MAX_SEGMENTS + 1))


def test_two_to_the_31_points_raise():
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(1000, 5)
    comp.add_scene(xyz, tex)
    big = torch.zeros((1, 3)).expand((1 << 31) - 1000, 3)       # a shape, never materialised
    with pytest.raises(ValueError, match="2\\^31"):
        comp.add_scene(big, torch.zeros((1, 8, 1)).expand(1, 8, big.shape[0]))
    assert ops.index_map_dtype(comp.total) == torch.float32


def test_mismatched_descriptors_or_activation_raise():
    comp = SceneComposer(device="cpu")
    xyz, tex = _scene(1000, 6)
    comp.add_scene(xyz, tex)
    with pytest.raises(ValueError, match="D = 8"):
        comp.add_scene(xyz, torch.zeros((1, 4, 1000)))
    sig = PointTexture(8, 1000, activation='sigmoid')
    with pytest.raises(ValueError, match="activation"):
        comp.add_scene(xyz, sig)
    with pytest.raises(ValueError):
        comp.add_scene(xyz, torch.zeros((1, 8, 999)))


def test_raster_entry_point_rejects_bad_tables_and_geometry():
    """read_raster_project_segments validates before it touches the device (fake, aligned pointers suffice)."""
    lib = _lib.load()
    ptr = 0x100000
    first = (ctypes.c_int64 * 2)(0, 1)
    cnt = (ctypes.c_int64 * 2)(1, 1)
    vis = (ctypes.c_uint8 * 2)(1, 1)

    def call(n=2 * CHUNK, nseg=2, B=1, W=64, H=32, L=4, pts=ptr, first=first, cnt=cnt):
        return lib.read_raster_project_segments(pts, n, first, cnt, vis, nseg, ptr, B, W, H, L, ptr, None)

    for kw, msg in ((dict(n=CHUNK + 1), b"whole"), (dict(pts=ptr + 4), b"aligned"), (dict(nseg=ops.MAX_SEGMENTS + 1), b"segments"),
                    (dict(B=9), b"views"), (dict(W=64, H=30), b"nested"),
                    (dict(cnt=(ctypes.c_int64 * 2)(1, 2)), b"outside"), (dict(first=(ctypes.c_int64 * 2)(-1, 0)), b"outside")):
        assert call(**kw) != 0, kw
        assert msg in lib.read_last_error(), (kw, lib.read_last_error())
    assert call(nseg=0) == 0                                      # nothing visible: nothing to launch


def test_set_transform_and_set_visible_copy_no_point_data():
    comp, (a, b), objs, inst, *_ = _composer()
    st = comp.store
    ptr, snapshot = st.pts4.data_ptr(), st.pts4.clone()
    M = np.eye(4)
    M[:3, 3] = [1.0, 2.0, 3.0]
    for h in (a, b, objs[1], inst):
        comp.set_transform(h, M)
    comp.set_visible(objs[2], False)
    comp.set_visible(b, False)
    assert comp.store is st and st.pts4.data_ptr() == ptr
    assert torch.equal(torch.nan_to_num(st.pts4, nan=7.0), torch.nan_to_num(snapshot, nan=7.0))
    vis = list(st.visible)[:st.nseg]
    assert vis == [1, 1, 1, 0, 1, 1, 0, 1]                       # object 2 and scene b hidden; the rest drawn
    comp.set_visible(objs[3], False)                              # hiding an object leaves its instance
    assert list(st.visible)[:st.nseg][4] == 0 and list(st.visible)[:st.nseg][-1] == 1
    comp.set_visible(a, False)                                    # hiding a scene hides its objects and instances
    assert sum(list(st.visible)[:st.nseg]) == 0
    comp.set_visible(a, True)
    comp.set_visible(b, True)
    assert list(st.visible)[:st.nseg] == [1, 1, 1, 0, 0, 1, 1, 1]
    seg_m = comp.segment_matrices(np.eye(4, dtype=np.float32))
    np.testing.assert_array_equal(seg_m[0, 0], M.astype(np.float32))                   # the scene placement
    np.testing.assert_array_equal(seg_m[2, 0], (M @ M).astype(np.float32))             # object 1: placement @ transform
