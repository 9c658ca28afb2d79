"""-m gpu: cylindrical panoramas (read_b200.panorama, DESIGN.md §4.4) against the numpy restatement in tests/oracle_panorama.py.

Every level's (depth | id) keys must equal the oracle's key for key: the level-0 key is the min over the points' splats (two near
the seam of a 360-degree view), levels 1-3 its 2x2 mins.  The frame of ``infer_panorama`` is the refinement engine run on the
features gathered from the oracle's index maps, cropped to the panorama."""
import numpy as np
import pytest
import torch

import oracle_panorama as O
from gpu_util import psnr
from read_b200 import _lib as Lb
from read_b200 import ops, synth
from read_b200.compose import NetAndTexture
from read_b200.panorama import Panorama, raster_panorama_sorted, raster_panorama_segments_culled
from read_b200.scene_edit import SceneComposer
from read_b200.texture import PointTexture
from read_b200.unet import UNet
from read_b200.viewer import FrameRenderer, SceneRenderer

pytestmark = pytest.mark.gpu
F32 = np.float32
TOL_BF16, PSNR_MIN = 3e-2, 45.0


def _dev():
    return torch.device("cuda", 0)


def _view(yaw_deg, z, x=0.0):
    """A camera-to-world GL view matrix in the middle of the street: eye (x, 0, z), turned by yaw_deg about y."""
    a = np.deg2rad(yaw_deg)
    m = np.eye(4)
    m[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    m[:3, 3] = (x, 0.0, z)
    return m.astype(F32)


def _keys(pyr):
    torch.cuda.synchronize()
    buf = pyr.buf.cpu().numpy().view(np.uint64)
    out = []
    for l in range(pyr.L):
        w, h = pyr.sizes[l]
        out.append(buf[pyr.offsets[l]:pyr.offsets[l] + pyr.B * w * h].reshape(pyr.B, h, w))
    return out


def _assert_levels(got, want, what):
    for l, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape, (what, l)
        bad = np.flatnonzero(g.reshape(-1) != w.reshape(-1))
        assert bad.size == 0, f"{what}: level {l}: {bad.size} keys differ, first at {bad[:5]}"


def _assert_seam(levels, p, what):
    """Rendered columns [0, M) hold what [W, W + M) holds, at every level: the wrapped copies of the panorama's ends."""
    M, W = p.margin, p.width
    for l, z in enumerate(levels):
        assert np.array_equal(z[:, :, :M >> l], z[:, :, W >> l:(W + M) >> l]), (what, l)
        assert np.array_equal(z[:, :, (W + M) >> l:], z[:, :, M >> l:(2 * M) >> l]), (what, l)


def _sorted_pyramid(store, V, p, L=4):
    pyr = ops.Pyramid(V.shape[0], p.plane_width, p.height, L, _dev())
    pyr.clear()
    raster_panorama_sorted(pyr, store, torch.from_numpy(np.ascontiguousarray(V)).to(_dev()), p)
    ops.raster_derive(pyr)
    return _keys(pyr)


@pytest.fixture(scope="module")
def street():
    xyz = synth.street_scene(1_000_000, depth=120.0, seed=5)
    return xyz, ops.SortedPoints(torch.from_numpy(xyz).to(_dev()))


PANOS = {
    "360": Panorama(1024, 256, margin=64, zfar=200.0),
    "180": Panorama(1024, 256, hfov_deg=180, zfar=200.0),
    "asym": Panorama(512, 128, elevation_deg=(-55.0, 12.0), margin=64, zfar=200.0),
    "150": Panorama(640, 128, hfov_deg=150, elevation_deg=(-20.0, 35.0)),
}


@pytest.mark.parametrize("name", list(PANOS))
@pytest.mark.parametrize("B", [1, 2])
def test_street_scene_keys_equal_the_oracle(street, name, B):
    xyz, store = street
    p = PANOS[name]
    views = [_view(20.0, -60.0), _view(-135.0, -30.0, 3.0)][:B]
    V = Panorama.world_to_camera(np.stack(views))
    got = _sorted_pyramid(store, V, p)
    want = O.pyramid(xyz, np.arange(len(xyz), dtype=np.uint64), V, p)
    _assert_levels(got, want, f"{name} B={B}")
    assert (got[0] != O.EMPTY).mean() > 0.1                            # the scene is all around
    if p.full:
        _assert_seam(got, p, name)


def _hand_store(rows, ids):
    """A sorted-store object over hand-laid rows (the rasterizer reads pts4 and n only)."""
    st = object.__new__(ops.SortedPoints)
    pts4 = np.empty((len(rows), 4), F32)
    pts4[:, :3] = rows
    pts4[:, 3] = np.asarray(ids, np.uint32).view(F32)
    st.pts4 = torch.from_numpy(pts4).to(_dev())
    st.n, st.cell, st.psize, st.perm = len(rows), 0.25, None, None
    return st


EDGE_PANOS = [Panorama(1024, 256, margin=64), Panorama(512, 128, hfov_deg=180), Panorama(256, 64, elevation_deg=(-10, 40), margin=32),
              Panorama(4096, 1024, margin=128)]


@pytest.mark.parametrize("p", EDGE_PANOS, ids=repr)
def test_edge_sets_sorted_and_culled(p):
    pts, labels, _ = O.edge_set(p)
    # each point twice (ids i and n + i) and the ties with descending ids: every tie resolves by the id
    pts = np.concatenate([pts, pts[::-1]])
    ids = np.arange(1, len(pts) + 1, dtype=np.uint32)
    rows, rid = O.edge_store_rows(pts, ids)
    V = np.stack([O.EDGE_VIEW, O.EDGE_VIEW])
    want = O.pyramid(rows, rid.astype(np.uint64), V, p)
    got = _sorted_pyramid(_hand_store(rows, rid), V, p)
    _assert_levels(got, want, f"sorted {p!r}")
    if p.full:
        _assert_seam(got, p, "edges")
    # the same points through the segmented store and the culled table (padding rows: NaN, id 0)
    seg = ops.SegmentedPoints([(torch.from_numpy(pts).to(_dev()), torch.from_numpy(ids.astype(np.int64)))])
    seg_m = torch.from_numpy(np.ascontiguousarray(V[None])).to(_dev())
    pyr = ops.Pyramid(2, p.plane_width, p.height, 4, _dev())
    pyr.clear()
    raster_panorama_segments_culled(pyr, seg, seg_m, p)
    ops.raster_derive(pyr)
    _assert_levels(_keys(pyr), O.segmented_pyramid(seg, V[None], p), f"culled {p!r}")


def _model(sd, n, seed=1, ss=1, temporal=False):
    net = UNet()
    net.load_state_dict(sd, strict=True)
    tex = PointTexture(8, n)
    with torch.no_grad():
        tex.texture_.copy_(torch.rand((1, 8, n), generator=torch.Generator().manual_seed(seed)))
    model = NetAndTexture(net, {0: tex}, ss, temporal_average=temporal)
    model.load_textures(0)
    return model.to(_dev()).eval(), tex


def test_supersampling_maps_equal_the_oracle(street, synth_sd):
    xyz, store = street
    p = Panorama(256, 64, margin=32, zfar=200.0)
    model, _ = _model(synth_sd, len(xyz), ss=2)
    V = Panorama.world_to_camera(_view(40.0, -50.0)[None])
    out, maps = model.render(store, torch.from_numpy(V).to(_dev()), p.width, p.height, want_maps=True, panorama=p)
    assert tuple(out.shape) == (1, 3, p.height, p.width)
    want = O.pyramid(xyz, np.arange(len(xyz), dtype=np.uint64), V, p.scaled(2))
    for l, (idx, dep) in enumerate(maps):
        k = want[l]
        empty = k == O.EMPTY
        assert idx.shape[-1] == (2 * p.plane_width) >> l
        np.testing.assert_array_equal(idx.cpu().numpy(), np.where(empty, 0, k & np.uint64(0xFFFFFFFF)).astype(F32))
        np.testing.assert_array_equal(dep.cpu().numpy().view(np.uint32), np.where(empty, 0, k >> np.uint64(32)).astype(np.uint32))


def _clutter_objects(n, sizes):
    start, out = int(0.8 * n), []
    for s in sizes:
        out.append(np.arange(start, start + s))
        start += s
    return out


def _rigid(rng, shift=1.0, scale=1.0):
    M = np.eye(4)
    a = rng.uniform(-0.3, 0.3)
    M[:3, :3] = scale * np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    M[:3, 3] = rng.uniform(-shift, shift, 3)
    return M


def test_scene_renderer_edits_and_radial_cull(synth_sd):
    rng = np.random.default_rng(17)
    n_a, n_b = 120_000, 40_000
    xyz_a = synth.street_scene(n_a, depth=150.0, seed=41)
    xyz_b = synth.street_scene(n_b, depth=40.0, seed=42)
    comp = SceneComposer(_dev())
    a = comp.add_scene(xyz_a, torch.rand((1, 8, n_a)))
    place = np.eye(4)
    place[:3, 3] = (0.0, 0.0, -160.0)
    comp.add_scene(xyz_b, torch.rand((1, 8, n_b)), placement=place)
    objs = [comp.add_object(a, ids) for ids in _clutter_objects(n_a, [2000, 1500, 1025, 3000, 700])]
    comp.set_transform(objs[0], _rigid(rng, 2.0))
    comp.set_transform(objs[1], _rigid(rng, 1.0, scale=1.5))
    comp.set_visible(objs[2], False)
    comp.add_instance(objs[3], _rigid(rng, 20.0))
    comp.add_instance(objs[4], _rigid(rng, 5.0))
    store = comp.store
    for zfar, culls in [(1000.0, False), (45.0, True)]:
        p = Panorama(512, 128, margin=64, zfar=zfar)
        V = Panorama.world_to_camera(np.stack([_view(10.0, -60.0), _view(200.0, -20.0)]))
        seg_m = comp.segment_matrices(V)
        pyr = ops.Pyramid(2, p.plane_width, p.height, 4, _dev())
        pyr.clear()
        raster_panorama_segments_culled(pyr, store, torch.from_numpy(seg_m).to(_dev()), p)
        ops.raster_derive(pyr)
        _assert_levels(_keys(pyr), O.segmented_pyramid(store, seg_m, p), f"composed zfar {zfar}")
        drawn = ops.last_surviving_units(store)
        assert drawn == len(O.kept_units(store, seg_m, p))
        if culls:
            assert drawn < sum(store.chunks[s] for s in range(store.nseg) if store.visible[s])
        else:
            assert drawn == sum(store.chunks[s] for s in range(store.nseg) if store.visible[s])
    # through SceneRenderer.infer_panorama: the net input's level 0 is drawn from the same pyramid
    sr = SceneRenderer(comp, synth_sd, (256, 64))
    p = Panorama(256, 64, margin=32, zfar=45.0)
    res = sr.infer_panorama(_view(10.0, -60.0), p)
    assert tuple(res['output'].shape) == (64, 256, 4) and tuple(res['net_input'][0].shape) == (1, 8, 64, 320)
    assert torch.isfinite(res['output']).all()


def test_infer_panorama_equals_the_engine_on_oracle_features(street, synth_sd):
    from oracle import unet_ref
    xyz, _ = street
    n = len(xyz)
    p = Panorama(512, 128, margin=64, zfar=200.0)
    g = torch.Generator().manual_seed(9)
    tex_cpu = torch.rand((1, 8, n), generator=g)
    fr = FrameRenderer(xyz, synth_sd, tex_cpu, (256, 128), flip_vertical=True)
    view = _view(-30.0, -55.0)
    res = fr.infer_panorama(view, p)
    rgba = res['output'].cpu()
    # the oracle's index maps -> the engine's gather -> the engine, cropped
    V = Panorama.world_to_camera(view[None])
    keys = O.pyramid(xyz, np.arange(n, dtype=np.uint64), V, p)
    maps = [torch.from_numpy(np.where(k == O.EMPTY, 0, k & np.uint64(0xFFFFFFFF)).astype(F32)) for k in keys]
    eng = fr.model.net.engine(1, p.height, p.plane_width, _dev())
    tex = fr.model._texture(0)
    layout = Lb.FEAT_NHWC_BF16 if eng.bf16 else Lb.FEAT_NHWC_F32
    for l, mp in enumerate(maps):
        ops.gather_from_index(tex.point_major(), mp.to(_dev()).contiguous(), layout, tex.activation, out=eng.inputs[l])
    ref = eng.run()[0, :, :, p.margin:p.margin + p.width].permute(1, 2, 0).flip(0).cpu()
    assert torch.equal(rgba[..., :3], ref)
    assert torch.all(rgba[..., 3] == 1)
    # the fp32 torch net on the same maps
    with torch.no_grad():
        want = unet_ref.net_and_texture(synth_sd, tex_cpu, [m[None] for m in maps])
    want = want[0, :, :, p.margin:p.margin + p.width].permute(1, 2, 0).flip(0)
    err = float((rgba[..., :3] - want).abs().max())
    assert err <= TOL_BF16 and psnr(rgba[..., :3].numpy(), want.numpy()) >= PSNR_MIN, err
    for l, x in enumerate(res['net_input']):
        assert tuple(x.shape) == (1, 8, p.height >> l, p.plane_width >> l)


def test_point_sprites_on_a_panorama_raise(synth_sd):
    xyz = synth.street_scene(20_000, depth=30.0, seed=3)
    tex = torch.rand((1, 8, len(xyz)))
    p = Panorama(256, 64, margin=32)
    fr = FrameRenderer(xyz, synth_sd, tex, (128, 64), input_format="uv_1d_p2, uv_1d_p1_ds1, uv_1d_p1_ds2, uv_1d_p1_ds3")
    with pytest.raises(ValueError):
        fr.infer_panorama(_view(0.0, -10.0), p)
    fr = FrameRenderer(xyz, synth_sd, tex, (128, 64), point_sizes=np.full(len(xyz), 2.0, F32))
    with pytest.raises(ValueError):
        fr.infer_panorama(_view(0.0, -10.0), p)
    model, _ = _model(synth_sd, len(xyz))
    with pytest.raises(ValueError):                                      # a plain [N,3] cloud: panoramas need a store
        model.render(torch.from_numpy(xyz).to(_dev()), torch.eye(4, device=_dev())[None], 256, 64, panorama=p)


def test_alternating_frames_and_panoramas_keep_their_histories(synth_sd):
    xyz = synth.street_scene(60_000, depth=40.0, seed=8)
    tex = torch.rand((1, 8, len(xyz)), generator=torch.Generator().manual_seed(2))
    W, H = 128, 64
    p = Panorama(256, 64, margin=32)
    kw = dict(supersampling=2, temporal_average=True)
    both = FrameRenderer(xyz, synth_sd, tex, (W, H), **kw)
    frames = FrameRenderer(xyz, synth_sd, tex, (W, H), **kw)
    panos = FrameRenderer(xyz, synth_sd, tex, (W, H), **kw)
    for t in (2, 5, 9):
        proj, view = synth.camera_batch(W, H, [t])
        a = both.infer(proj[0], view[0])
        b = both.infer_panorama(_view(3.0 * t, -0.5 * t - 10.0), p)
        c = frames.infer(proj[0], view[0])
        d = panos.infer_panorama(_view(3.0 * t, -0.5 * t - 10.0), p)
        assert torch.equal(a['output'], c['output']) and torch.equal(b['output'], d['output'])
        for x, y in zip(b['net_input'], d['net_input']):
            assert torch.equal(x, y)
    # and the history does matter: a fresh renderer's first panorama differs from the third one of a sequence
    fresh = FrameRenderer(xyz, synth_sd, tex, (W, H), **kw).infer_panorama(_view(27.0, -14.5), p)
    assert not torch.equal(fresh['output'], d['output'])
