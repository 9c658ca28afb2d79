"""-m gpu: point-cloud views (FrameRenderer.render_points / SceneRenderer.render_points, read_point_view).

The pixel sets come from the oracle z-buffers (oracle.pcpr_forward for 1-pixel views, tests/zbuffer_sprite.c for sprites, the
composed oracle of the point-sprite tests for composed scenes; depth 0 = empty), and every view is compared bit for bit with the
numpy restatement (tests/point_view_util.py) applied to the oracle's ids; the PCA colours within 1 float32 ulp of the float64
exact PCA."""
import numpy as np
import pytest
import torch

import oracle_sprite
import point_view_util as pv
from read_b200 import synth
from read_b200.scene_edit import SceneComposer
from read_b200.viewer import FrameRenderer, SceneRenderer
from test_gpu_point_sprites import _composed_oracle

pytestmark = pytest.mark.gpu
MODES = [("color", 0)] + [("normals", s) for s in range(5)] + [("depth", 0), ("xyz", 0), ("label", 0)] + \
        [("uv", s) for s in range(5)]


def _attrs(n, seed):
    rng = np.random.default_rng(seed)
    nrm = rng.standard_normal((n, 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
    lab = rng.random(n) < 0.1
    nrm[lab, 0] = rng.integers(0, 256, int(lab.sum()))             # labels 0..255, one per point, live in the normals' x
    return rng.random((n, 3)).astype(np.float32), nrm


def _texture(n, seed):
    return torch.from_numpy(pv.separated_descriptors(n, seed))


def _same(got, want, what):
    """Bit-identical, NaN payloads aside (the device's canonical NaN is not numpy's)."""
    g, w = got.cpu().numpy() if torch.is_tensor(got) else got, want
    nan = np.isnan(w)
    assert np.array_equal(np.isnan(g), nan), what
    bad = (g.view(np.uint32) != w.view(np.uint32)) & ~nan
    assert not bad.any(), f"{what}: {int(bad.sum())} values differ"


def _keys(xyz, total, W, H, oracle_mod, levels=None, sizes=None):
    if levels is None:
        idx, dep = oracle_mod.pcpr_forward(xyz, total[None], W, H)
        return pv.keys_from_maps(idx[0], dep[0])
    return oracle_sprite.sprite_zbuf(xyz, total[None], W, H, levels, sizes)[0][0]


def _check_modes(fr, keys, P, V, xyz, colors, normals, tex, modes=MODES, **kw):
    total = FrameRenderer.total_matrix(P, V)
    ctx = dict(colors=colors, normals=normals, xyz=xyz, total_m=total, view_matrix=V, lo=xyz.min(0), hi=xyz.max(0))
    for mode, sub in modes:
        got = fr.render_points(P, V, mode, sub, **kw)['output']
        assert tuple(got.shape) == (fr.H, fr.W, 4) and got.dtype == torch.float32
        want = pv.view_rgba(keys, flip_vertical=fr.flip_vertical, clear=kw.get("clear_color", (0., 0., 0., 1.)), mode=mode,
                            submode=sub, **ctx)
        _same(got, want, f"{mode}/{sub}")
    # PCA: within 1 float32 ulp of the float64 exact PCA at every drawn pixel, the clear colour elsewhere
    got = fr.render_points(P, V, 'pca', **kw)['output'].cpu().numpy()
    if fr.flip_vertical:
        got = got[::-1]
    drawn = keys != pv.EMPTY
    want = pv.pca_exact(tex[0].numpy())[(keys[drawn] & np.uint64(0xFFFFFFFF)).astype(np.int64)]
    err = np.abs(got[drawn][:, :3].astype(np.float64) - want) / np.spacing(want.astype(np.float32))
    assert float(err.max()) <= 1.0, float(err.max())
    assert np.array_equal(got[~drawn], np.broadcast_to(np.float32(kw.get("clear_color", (0., 0., 0., 1.))), got[~drawn].shape))


@pytest.mark.parametrize("W,H,n", [(128, 64, 60_000), (1920, 1088, 400_000)])
def test_every_mode_matches_the_restatement(synth_sd, oracle_mod, W, H, n):
    xyz = synth.street_scene(n, depth=60.0, seed=5)
    colors, normals = _attrs(n, 5)
    tex = _texture(n, 5)
    fr = FrameRenderer(xyz, synth_sd, tex, (W, H), colors=colors, normals=torch.from_numpy(normals))
    proj, view = synth.camera_batch(W, H, [2])
    keys = _keys(xyz, FrameRenderer.total_matrix(proj[0], view[0]), W, H, oracle_mod)
    assert (keys != pv.EMPTY).mean() > 0.05
    _check_modes(fr, keys, proj[0], view[0], xyz, colors, normals, tex)


def test_clear_colour_flip_and_a_renderer_without_a_store(synth_sd, oracle_mod):
    W, H, n = 128, 80, 40_000
    xyz = synth.street_scene(n, depth=40.0, seed=6)
    colors, normals = _attrs(n, 6)
    tex = _texture(n, 6)
    # six levels of 80 rows do not nest: the frame path keeps no sorted store and the view rasterises the cloud itself
    fr = FrameRenderer(xyz, synth_sd, tex, (W, H), n_levels=6, flip_vertical=True, colors=colors, normals=normals)
    assert fr.store is None
    proj, view = synth.camera_batch(W, H, [4])
    keys = _keys(xyz, FrameRenderer.total_matrix(proj[0], view[0]), W, H, oracle_mod)
    _check_modes(fr, keys, proj[0], view[0], xyz, colors, normals, tex, modes=[("color", 0), ("depth", 0), ("normals", 1)],
                 clear_color=(0.25, 0.5, -1.0, 0.0))
    # sprites on a renderer without a store: it builds its sorted store once
    lv = [(3.0, False)]
    keys3 = _keys(xyz, FrameRenderer.total_matrix(proj[0], view[0]), W, H, oracle_mod, levels=lv)
    got = fr.render_points(proj[0], view[0], 'uv', point_size=3)['output']
    _same(got, pv.view_rgba(keys3, flip_vertical=True, mode='uv', submode=0), "uv p3 without store")


def test_nothing_in_front_of_the_camera_is_all_clear_colour(synth_sd, oracle_mod):
    W, H, n = 128, 64, 20_000
    xyz = synth.street_scene(n, depth=40.0, seed=7)
    xyz[:, 2] += 1000.0                                                  # behind the camera (it looks down -z)
    colors, normals = _attrs(n, 7)
    fr = FrameRenderer(xyz, synth_sd, _texture(n, 7), (W, H), colors=colors, normals=normals)
    proj, view = synth.camera_batch(W, H, [0])
    assert (_keys(xyz, FrameRenderer.total_matrix(proj[0], view[0]), W, H, oracle_mod) == pv.EMPTY).all()
    for mode in ('color', 'depth', 'pca'):
        got = fr.render_points(proj[0], view[0], mode, clear_color=(0.1, 0.2, 0.3, 0.4))['output'].cpu().numpy()
        assert np.array_equal(got, np.broadcast_to(np.float32([0.1, 0.2, 0.3, 0.4]), got.shape)), mode


def _sizes(n, seed):
    rng = np.random.default_rng(seed)
    s = rng.uniform(0.5, 9.0, n).astype(np.float32)
    s[rng.random(n) < 0.3] = 0.0                                         # keeps point_size
    s[rng.random(n) < 0.02] = 200.0                                      # above the 64-pixel limit
    return s


@pytest.mark.parametrize("point_size,relative,sized", [(3, False, False), (64, False, False), (8, True, False),
                                                        (2, False, True), (1, True, True)])
def test_point_sprites_match_the_sprite_oracle(synth_sd, point_size, relative, sized):
    W, H, n = 160, 96, 30_000
    xyz = synth.street_scene(n, depth=40.0, seed=8)
    colors, normals = _attrs(n, 8)
    tex = _texture(n, 8)
    sizes = _sizes(n, 8) if sized else None
    fr = FrameRenderer(xyz, synth_sd, tex, (W, H), colors=colors, normals=normals, point_sizes=sizes)
    proj, view = synth.camera_batch(W, H, [3])
    total = FrameRenderer.total_matrix(proj[0], view[0])
    keys = oracle_sprite.sprite_zbuf(xyz, total[None], W, H, [(float(point_size), relative)], sizes)[0][0]
    _check_modes(fr, keys, proj[0], view[0], xyz, colors, normals, tex,
                 modes=[("color", 0), ("normals", 3), ("depth", 0), ("xyz", 0), ("uv", 0)],
                 point_size=point_size, relative=relative)


def _composition(with_colors_b=False):
    na, nb = 40_000, 15_000
    xa = synth.street_scene(na, depth=40.0, seed=21)
    xb = synth.street_scene(nb, depth=25.0, seed=22)
    ca, la = _attrs(na, 21)
    cb, lb = _attrs(nb, 22)
    comp = SceneComposer(torch.device("cuda", 0))
    a = comp.add_scene(xa, _texture(na, 1), colors=ca, normals=la)
    P = np.eye(4)
    P[:3, 3] = [3.0, 0.0, -30.0]
    b = comp.add_scene(xb, _texture(nb, 2), P, normals=lb, colors=cb if with_colors_b else None)
    moved = comp.add_object(a, np.arange(5000, 9000))
    M = np.eye(4)
    M[:3, 3] = [0.5, 0.2, -1.0]
    comp.set_transform(moved, M)
    inst_obj = comp.add_object(b, np.arange(100, 2100))
    Mi = np.eye(4)
    Mi[:3, 3] = [-2.0, 0.0, 4.0]
    comp.add_instance(inst_obj, Mi)
    hidden = comp.add_object(a, np.arange(20_000, 22_000))
    comp.set_visible(hidden, False)
    colors = np.concatenate([ca, cb if with_colors_b else np.zeros_like(cb)])
    return comp, colors, np.concatenate([la, lb])


@pytest.mark.parametrize("point_size", [1, 3])
def test_scene_renderer_id_modes_match_the_composed_oracle(synth_sd, point_size):
    W, H = 128, 64
    comp, colors, normals = _composition()
    sr = SceneRenderer(comp, synth_sd, (W, H), flip_vertical=True)
    proj, view = synth.camera_batch(W, H, [2])
    seg_m = comp.segment_matrices(FrameRenderer.total_matrix(proj[0], view[0]))
    idx, dep = _composed_oracle(comp, seg_m, W, H, [(float(point_size), False)], None)[0]
    keys = pv.keys_from_maps(idx[0], dep[0])
    assert (keys != pv.EMPTY).mean() > 0.2
    for mode, sub in [("color", 0), ("label", 0), ("uv", 0), ("uv", 3)]:
        got = sr.render_points(proj[0], view[0], mode, sub, point_size=point_size)['output']
        _same(got, pv.view_rgba(keys, flip_vertical=True, mode=mode, submode=sub, colors=colors, normals=normals), mode)
    got = sr.render_points(proj[0], view[0], 'pca', point_size=point_size)['output'].cpu().numpy()[::-1]
    drawn = keys != pv.EMPTY
    want = pv.pca_exact(comp.texture.texture_.detach().cpu()[0].numpy())[(keys[drawn] & np.uint64(0xFFFFFFFF)).astype(np.int64)]
    err = np.abs(got[drawn][:, :3].astype(np.float64) - want) / np.spacing(want.astype(np.float32))
    assert float(err.max()) <= 1.0, float(err.max())
    for mode in ('normals', 'depth', 'xyz'):
        with pytest.raises(ValueError, match=mode):
            sr.render_points(proj[0], view[0], mode)


def test_composed_tables_follow_later_scenes(synth_sd):
    comp, _, _ = _composition(with_colors_b=True)
    n = comp.total
    assert tuple(comp.colors.shape) == (n, 4) and tuple(comp.normals.shape) == (n, 4)
    extra = comp.add_scene(synth.street_scene(1000, depth=10.0, seed=3), _texture(1000, 3))
    assert comp.colors.shape[0] == n + 1000 and not comp.colors[extra.base:].any()
    c = SceneComposer(torch.device("cuda", 0))
    c.add_scene(synth.street_scene(1000, depth=10.0, seed=3), _texture(1000, 3))
    sr = SceneRenderer(c, synth_sd, (64, 32))
    proj, view = synth.camera_batch(64, 32, [0])
    for mode, what in (("color", "colors"), ("label", "normals")):
        with pytest.raises(ValueError, match=what):
            sr.render_points(proj[0], view[0], mode)


@pytest.mark.parametrize("ss,temporal", [(1, False), (1, True), (2, False)])
def test_infer_is_unchanged_by_views_in_between(synth_sd, ss, temporal):
    W, H, n = 128, 64, 50_000
    xyz = synth.street_scene(n, depth=40.0, seed=9)
    colors, normals = _attrs(n, 9)
    tex = _texture(n, 9)
    kw = dict(supersampling=ss, temporal_average=temporal, return_net_input=False)
    plain = FrameRenderer(xyz, synth_sd, tex, (W, H), **kw)
    viewed = FrameRenderer(xyz, synth_sd, tex, (W, H), colors=colors, normals=normals, **kw)
    for t in range(3):
        proj, view = synth.camera_batch(W * ss, H * ss, [t])
        want = plain.infer(proj[0], view[0])['output']
        for mode, size in (("color", 1), ("pca", 3), ("depth", 1)):
            viewed.render_points(proj[0], view[0], mode, point_size=size)
        got = viewed.infer(proj[0], view[0])['output']
        assert torch.equal(got, want), t
