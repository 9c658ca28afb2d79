"""-m gpu: scene editing and stitching (read_b200.scene_edit, ops.raster_project_segments, viewer.SceneRenderer).

The oracle of a composed frame: every visible segment rendered by ``oracle.pcpr_forward`` with its matrix
T = total_m @ P_scene @ M (read_b200.scene_edit's matrix rule), its local ids mapped to global ids, and the segments merged by the
minimum of the packed (depth bits, global id) key - the z-buffer's own order.  Index and depth maps must match bit for bit."""
import numpy as np
import pytest
import torch

from read_b200 import ops, synth
from read_b200.compose import NetAndTexture
from read_b200.scene_edit import SceneComposer
from read_b200.texture import PointTexture
from read_b200.unet import UNet
from read_b200.viewer import FrameRenderer, SceneRenderer

pytestmark = pytest.mark.gpu
TOL_FP32 = 2e-4
TOL_BF16 = 3e-2
CHUNK = ops.SEGMENT_CHUNK
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _dev():
    return torch.device("cuda", 0)


def _segment_points(store, s):
    """(xyz [n,3] f32, global ids [n]) of segment s, read back from the store's rows, ordered by global id (so that the oracle's
    lowest-local-id tie rule is the z-buffer's lowest-global-id rule)."""
    f, c = store.first_chunk[s], store.chunks[s]
    rows = store.pts4[f * CHUNK:(f + c) * CHUNK].cpu()
    rows = rows[~torch.isnan(rows[:, 0])]
    gid = rows[:, 3].contiguous().view(torch.int32).to(torch.int64)
    order = torch.argsort(gid)
    return rows[order, :3].numpy().copy(), gid[order].numpy()


def _oracle(oracle_mod, groups, W, H, L):
    """groups: [(xyz, global ids, T [B,4,4] f32)] -> per level (index [B,h,w] f32, depth [B,h,w] f32) of their merged render."""
    out, B = [], groups[0][2].shape[0]
    for (w, h) in ops.level_sizes(W, H, L):
        best = None
        for xyz, gid, T in groups:
            if len(gid) == 0:
                continue
            idx, dep = oracle_mod.pcpr_forward(xyz, T, w, h)
            key = (dep.view(np.uint32).astype(np.uint64) << np.uint64(32)) | gid[idx.astype(np.int64)].astype(np.uint64)
            key = np.where(dep == 0, EMPTY, key)
            best = key if best is None else np.minimum(best, key)
        if best is None:
            best = np.full((B, h, w), EMPTY)
        empty = best == EMPTY
        index = np.where(empty, 0, best & np.uint64(0xFFFFFFFF)).astype(np.float32)
        depth = np.where(empty, 0, best >> np.uint64(32)).astype(np.uint32).view(np.float32)
        out.append((index, depth))
    return out


def _composed_oracle(oracle_mod, comp, seg_m, W, H, L):
    st = comp.store
    groups = [(*_segment_points(st, s), seg_m[s]) for s in range(st.nseg) if st.visible[s]]
    return _oracle(oracle_mod, groups, W, H, L)


def _render_maps(comp, seg_m, W, H, L):
    pyr = ops.Pyramid(seg_m.shape[1], W, H, L, _dev())
    pyr.clear()
    ops.raster_project_segments(pyr, comp.store, torch.from_numpy(seg_m).to(_dev()))
    ops.raster_derive(pyr)
    maps = [ops.zbuf_resolve(pyr, l) for l in range(L)]
    torch.cuda.synchronize()
    return [(i.cpu().numpy(), d.cpu().numpy()) for i, d in maps], pyr


def _assert_maps_equal(got, want, what=""):
    for l, ((gi, gd), (wi, wd)) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(gi, wi, err_msg=f"{what} index level {l}")
        np.testing.assert_array_equal(gd.view(np.uint32), wd.view(np.uint32), err_msg=f"{what} depth bits level {l}")


def _clutter_objects(n, sizes):
    """Consecutive id ranges of the given sizes inside street_scene's box clutter (the last 20 % of the ids)."""
    start, out = int(0.8 * n), []
    for s in sizes:
        out.append(np.arange(start, start + s))
        start += s
    assert start <= n
    return out


def _rigid(rng, shift=1.0):
    M = np.eye(4)
    a = rng.uniform(-0.3, 0.3)
    M[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    M[:3, 3] = rng.uniform(-shift, shift, 3)
    return M


# ----------------------------------------------------------------------------------------------------------- 1. split == unsplit
def test_split_scene_equals_the_unsplit_store(synth_sd):
    W, H, n = 256, 128, 150_000
    xyz = synth.street_scene(n, depth=50.0, seed=21)
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(4))
    comp = SceneComposer(_dev())
    s = comp.add_scene(xyz, tex)
    for ids in _clutter_objects(n, [0, 1, 1023, 1024, 1025] + [300] * 40):
        comp.add_object(s, ids)
    proj, view = synth.camera_batch(W, H, [2, 9])
    total = synth.total_matrix(proj, view)
    seg_m = comp.segment_matrices(total)
    _, pyr = _render_maps(comp, seg_m, W, H, 4)
    ref = ops.Pyramid(2, W, H, 4, _dev())
    ref.clear()
    ops.raster_project_sorted(ref, ops.SortedPoints(torch.from_numpy(xyz).to(_dev())), torch.from_numpy(total).to(_dev()))
    ops.raster_derive(ref)
    torch.cuda.synchronize()
    assert torch.equal(pyr.buf, ref.buf)
    # through infer: the composed renderer's frame is FrameRenderer's, bit for bit
    fr = FrameRenderer(xyz, synth_sd, tex, (W, H))
    sr = SceneRenderer(comp, synth_sd, (W, H))
    for t in (2, 9):
        p, v = synth.camera_batch(W, H, [t])
        a, b = fr.infer(p[0], v[0]), sr.infer(p[0], v[0])
        assert torch.equal(a['output'], b['output'])
        for x, y in zip(a['net_input'], b['net_input']):
            assert torch.equal(x, y)


# ------------------------------------------------------------------------------------- 2. transforms / visibility vs the oracle
def _edited_composition(rng, n_a=60_000, n_b=20_000):
    xyz_a = synth.street_scene(n_a, depth=30.0, seed=31)
    xyz_b = synth.street_scene(n_b, depth=30.0, seed=32)
    comp = SceneComposer(_dev())
    a = comp.add_scene(xyz_a, torch.rand((1, 8, n_a)))
    place = np.eye(4)
    place[:3, 3] = [3.0, 0.0, -12.0]
    b = comp.add_scene(xyz_b, torch.rand((1, 8, n_b)), placement=place)
    sizes = [0, 1, 1023, 1024, 1025] + [97] * 58 + [150]            # 64 objects
    objs = [comp.add_object(a, ids) for ids in _clutter_objects(n_a, sizes)]
    assert len(objs) == 64
    for i, o in enumerate(objs):
        comp.set_transform(o, _rigid(rng))
        if i % 5 == 3:
            comp.set_visible(o, False)
    comp.set_transform(objs[4], np.diag([2.0 ** 60] * 4))            # |w| ~ 2^60: the project_point fallback
    comp.add_instance(objs[4], _rigid(rng, 2.0))
    comp.add_instance(objs[2], _rigid(rng, 2.0))
    return comp, (a, b), objs


@pytest.mark.parametrize("ts", [[4], [0, 2, 4, 6, 8, 10, 12, 14]])
def test_moved_hidden_instanced_and_stitched_against_the_oracle(oracle_mod, ts):
    W, H, L = 128, 64, 4
    comp, (a, b), objs = _edited_composition(np.random.default_rng(len(ts)))
    assert comp.store.nseg == 2 + 64 + 2
    proj, view = synth.camera_batch(W, H, ts)
    seg_m = comp.segment_matrices(synth.total_matrix(proj, view))
    np.testing.assert_array_equal(seg_m[5], np.float32(2.0 ** 60) * seg_m[0])
    got, _ = _render_maps(comp, seg_m, W, H, L)
    want = _composed_oracle(oracle_mod, comp, seg_m, W, H, L)
    _assert_maps_equal(got, want)
    assert (want[0][0] != 0).sum() > 0.2 * W * H * len(ts)
    # hide the whole second scene and show an object again: the next render follows
    comp.set_visible(b, False)
    comp.set_visible(objs[3], True)
    got, _ = _render_maps(comp, seg_m, W, H, L)
    _assert_maps_equal(got, _composed_oracle(oracle_mod, comp, seg_m, W, H, L), "after edit")


# ------------------------------------------------------------------------------------------------- 3. semantics pinned exactly
def _dyadic_scene(n, seed):
    """Coordinates k/16 inside the frustum of _DYADIC_M (z in [-8, -1.5]); every product with _DYADIC_M and a dyadic shift is exact."""
    rng = np.random.default_rng(seed)
    z = -rng.integers(24, 128, n) / 16.0
    x = np.round(rng.uniform(-0.8, 0.8, n) * -z * 16) / 16
    y = np.round(rng.uniform(-0.8, 0.8, n) * -z * 16) / 16
    return np.stack([x, y, z], 1).astype(np.float32)


_DYADIC_M = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, -1, -2], [0, 0, -1, 0]], np.float32)[None]


def test_moving_equals_pretranslating_and_hiding_equals_deleting(oracle_mod):
    W, H, L, n = 64, 32, 4, 30_000
    xyz = _dyadic_scene(n, 5)
    obj = np.arange(1000, 4000)
    shift = np.array([0.25, -0.125, -0.5])
    M = np.eye(4)
    M[:3, 3] = shift
    tex = torch.rand((1, 8, n))
    moved = SceneComposer(_dev())
    s = moved.add_scene(xyz, tex)
    o = moved.add_object(s, obj, M)
    pre_xyz = xyz.copy()
    pre_xyz[obj] += shift.astype(np.float32)
    assert np.array_equal(pre_xyz[obj] - shift.astype(np.float32), xyz[obj])          # the shift is exact
    pre = SceneComposer(_dev())
    pre.add_object(pre.add_scene(pre_xyz, tex), obj)
    got, _ = _render_maps(moved, moved.segment_matrices(_DYADIC_M), W, H, L)
    want, _ = _render_maps(pre, pre.segment_matrices(_DYADIC_M), W, H, L)
    _assert_maps_equal(got, want, "moved vs pre-translated")
    assert (got[0][0] != 0).sum() > 0.3 * W * H
    # hiding == deleting the points (the others keep their ids)
    moved.set_visible(o, False)
    got, _ = _render_maps(moved, moved.segment_matrices(_DYADIC_M), W, H, L)
    keep = np.setdiff1d(np.arange(n), obj)
    want = _oracle(oracle_mod, [(xyz[keep], keep, _DYADIC_M)], W, H, L)
    _assert_maps_equal(got, want, "hidden vs deleted")


# --------------------------------------------------------------------------------------------------------------- 4. net path
def _net_and_texture(sd, tex, ss, temporal, precision):
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.precision = precision
    t = PointTexture(8, tex.shape[2])
    with torch.no_grad():
        t.texture_.copy_(tex)
    m = NetAndTexture(net, {0: t}, ss, temporal_average=temporal)
    m.load_textures(0)
    return m.cuda().eval()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_composed_net_path_equals_forward_on_oracle_maps(oracle_mod, synth_sd, precision):
    W, H, ss = 128, 64, 2
    comp, _, _ = _edited_composition(np.random.default_rng(7), n_a=50_000, n_b=15_000)
    sr = SceneRenderer(comp, synth_sd, (W, H), supersampling=ss, temporal_average=True, flip_vertical=True)
    sr.model.net.precision = precision
    ref = _net_and_texture(synth_sd, comp.texture.texture_.detach().cpu(), ss, True, "fp32")
    for t in (3, 4, 5):
        proj, view = synth.camera_batch(W, H, [t])
        seg_m = comp.segment_matrices(FrameRenderer.total_matrix(proj[0], view[0]))
        maps = _composed_oracle(oracle_mod, comp, seg_m, W * ss, H * ss, 4)
        inputs = {(f"uv_1d_p1_ds{l}" if l else "uv_1d_p1"): torch.from_numpy(maps[l][0][:, None]).cuda() for l in range(4)}
        inputs["id"] = 0
        got = sr.infer(proj[0], view[0])
        with torch.no_grad():
            want, want_in = ref(inputs, return_input=True)
        rgb = got['output'][..., :3]
        assert tuple(got['output'].shape) == (H, W, 4) and bool((got['output'][..., 3] == 1).all())
        exp = want[0].permute(1, 2, 0).flip(0)
        if precision == "fp32":
            for x, y in zip(got['net_input'], want_in):
                assert tuple(x.shape) == tuple(y.shape)
                assert float((x - y).abs().max()) < 1e-6
            assert float((rgb - exp).abs().max()) < TOL_FP32
        else:
            assert float((rgb - exp).abs().max()) < TOL_BF16


# --------------------------------------------------------------------------------------------- 5. edits show on the next frame
def test_edits_take_effect_on_the_next_frame(synth_sd):
    W, H, n = 128, 64, 40_000
    xyz = synth.street_scene(n, depth=30.0, seed=8)
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(8))
    comp = SceneComposer(_dev())
    s = comp.add_scene(xyz, tex)
    objs = [comp.add_object(s, ids) for ids in _clutter_objects(n, [2000, 2000])]
    r = SceneRenderer(comp, synth_sd, (W, H))
    proj, view = synth.camera_batch(W, H, [3])
    f1 = r.infer(proj[0], view[0])
    keep1 = f1['output'].clone()
    M = np.eye(4)
    M[:3, 3] = [1.5, 0.0, 0.5]
    comp.set_transform(objs[0], M)
    comp.set_visible(objs[1], False)
    f2 = r.infer(proj[0], view[0])
    fresh = SceneRenderer(comp, synth_sd, (W, H)).infer(proj[0], view[0])
    torch.cuda.synchronize()
    assert torch.equal(f2['output'], fresh['output'])
    assert not torch.equal(f2['output'], keep1)
    assert torch.equal(f1['output'], keep1)                                 # frames are fresh tensors
    assert f1['output'].data_ptr() != f2['output'].data_ptr()
    # a layout edit (one more scene, one more instance) between frames
    comp.add_instance(objs[0], np.eye(4))
    place = np.eye(4)
    place[:3, 3] = [0.0, 0.0, -20.0]
    comp.add_scene(synth.street_scene(10_000, depth=20.0, seed=9), torch.rand((1, 8, 10_000)), placement=place)
    f3 = r.infer(proj[0], view[0])
    fresh = SceneRenderer(comp, synth_sd, (W, H)).infer(proj[0], view[0])
    torch.cuda.synchronize()
    assert torch.equal(f3['output'], fresh['output']) and not torch.equal(f3['output'], f2['output'])
