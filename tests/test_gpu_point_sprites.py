"""-m gpu: point sprites (read_b200.sprites, ops.raster_project_sprites, the input_format / point_sizes surfaces).

Parity target: the sprite restatement of the sequential z-buffer (tests/zbuffer_sprite.c via tests/oracle_sprite.py).  Index and
depth maps must match bit for bit, for the whole-store, segmented and culled-table kernels alike."""
import numpy as np
import pytest
import torch

import oracle_sprite
from read_b200 import ops, synth
from read_b200.compose import NetAndTexture
from read_b200.myrender import MyRender
from read_b200.scene_edit import SceneComposer
from read_b200.texture import PointTexture
from read_b200.unet import UNet
from read_b200.viewer import FrameRenderer, SceneRenderer

pytestmark = pytest.mark.gpu
CHUNK = ops.SEGMENT_CHUNK
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _dev():
    return torch.device("cuda", 0)


def _maps(pyr):
    out = [ops.zbuf_resolve(pyr, l) for l in range(pyr.L)]
    torch.cuda.synchronize()
    return [(i.cpu().numpy(), d.cpu().numpy()) for i, d in out]


def _assert_maps_equal(got, want, what=""):
    for l, ((gi, gd), (wi, wd)) in enumerate(zip(got, want)):
        assert np.array_equal(gd, wd), f"{what} depth level {l}: {int((gd != wd).sum())} pixels differ"
        assert np.array_equal(gi, wi), f"{what} index level {l}: {int((gi != wi).sum())} pixels differ"


def _sprite_pyramid(store, m, W, H, levels, kernel="culled"):
    pyr = ops.Pyramid(m.shape[1] if isinstance(store, ops.SegmentedPoints) else m.shape[0], W, H, len(levels), _dev())
    pyr.clear()
    ops.raster_project_sprites(pyr, store, m, levels, kernel=kernel)
    return pyr


def _sizes(n, seed):
    """Per-point sizes with zeros (the key's N), small, ordinary and above-the-clamp values."""
    rng = np.random.default_rng(seed)
    s = rng.uniform(0.2, 9.0, n).astype(np.float32)
    s[rng.random(n) < 0.3] = 0.0
    s[rng.random(n) < 0.02] = 200.0
    return s


LEVEL_SETS = {
    "p2347": [(2, False), (3, False), (4, False), (7, False)],
    "p64": [(64, False), (1, False), (64, False), (1, False)],
    "ps4_ps16": [(4, True), (16, True), (1, False), (1, False)],
    "mixed": [(1, False), (3, False), (1, False), (1, False)],
}


@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("levels", sorted(LEVEL_SETS))
@pytest.mark.parametrize("sized", [False, True])
@pytest.mark.parametrize("W,H,L", [(128, 64, 4), (100, 50, 3)])       # nested; 50 -> 25 -> 12 does not nest
def test_three_kernels_match_the_oracle(B, levels, sized, W, H, L):
    n = 40_000 if B < 8 else 12_000
    lv = LEVEL_SETS[levels][:L]
    xyz = synth.street_scene(n, depth=40.0, seed=B + L)
    proj, view = synth.camera_batch(W, H, list(range(0, 2 * B, 2)))
    M = synth.total_matrix(proj, view)
    sizes = _sizes(n, B) if sized else None
    want = oracle_sprite.sprite_maps(xyz, M, W, H, lv, sizes)
    x = torch.from_numpy(xyz).to(_dev())
    m = torch.from_numpy(M).to(_dev())
    got = _maps(_sprite_pyramid(ops.SortedPoints(x, point_sizes=sizes), m, W, H, lv))
    _assert_maps_equal(got, want, "whole store")
    ids = torch.arange(n, device=_dev())
    seg = ops.SegmentedPoints([(x, ids, sizes)])
    assert seg.psize is not None if sized else seg.psize is None
    seg_m = m[None].contiguous()
    for kernel in ("segments", "culled"):
        _assert_maps_equal(_maps(_sprite_pyramid(seg, seg_m, W, H, lv, kernel)), want, kernel)
    assert sum(int((i != 0).sum()) for i, _ in want) > 0.2 * B * W * H


def test_odd_width_is_a_min_filter_of_the_one_pixel_zbuffer():
    W, H, n = 256, 128, 300_000
    xyz = synth.street_scene(n, depth=60.0, seed=4)
    proj, view = synth.camera_batch(W, H, [1, 5])
    m = torch.from_numpy(synth.total_matrix(proj, view)).to(_dev())
    store = ops.SortedPoints(torch.from_numpy(xyz).to(_dev()))
    one = _sprite_pyramid(store, m, W, H, [(1, False)]).level(0).view(2, H, W)
    big = torch.iinfo(torch.int64).max                      # the empty key: every point's key is smaller
    assert int(one.max()) == big and int(one.min()) > 0
    base = one
    for w in (3, 5, 9):
        k = w // 2
        pad = torch.full((2, H + 2 * k, W + 2 * k), big, dtype=torch.int64, device=base.device)
        pad[:, k:k + H, k:k + W] = base
        filt = torch.full_like(base, big)
        for dy in range(w):
            for dx in range(w):
                filt = torch.minimum(filt, pad[:, dy:dy + H, dx:dx + W])
        got = _sprite_pyramid(store, m, W, H, [(w, False)]).level(0).view(2, H, W)
        assert torch.equal(got, filt), w


def test_one_pixel_sprites_equal_the_existing_path():
    W, H, L, n = 128, 64, 4, 100_000
    xyz = synth.street_scene(n, depth=60.0, seed=6)
    proj, view = synth.camera_batch(W, H, [0, 3, 7])
    M = synth.total_matrix(proj, view)
    x, m = torch.from_numpy(xyz).to(_dev()), torch.from_numpy(M).to(_dev())
    ref = ops.Pyramid(3, W, H, L, _dev())
    ref.clear()
    ops.raster_project(ref, x, m)
    want = _maps(ref)
    _assert_maps_equal(_maps(_sprite_pyramid(ops.SortedPoints(x), m, W, H, [(1, False)] * L)), want, "_p1")
    # _ps with per-point sizes whose relative size always rounds to 1 (s / c2 = 1.4 where c2 > 0; c2 <= 0 gives max(1, -) = 1)
    c2 = (xyz.astype(np.float64) @ M[0, 2, :3].astype(np.float64)) + M[0, 2, 3]
    sizes = np.where(c2 > 0, 1.4 * c2, 1.0).astype(np.float32)
    got = _maps(_sprite_pyramid(ops.SortedPoints(x, point_sizes=sizes), m[:1].contiguous(), W, H, [(1, True)] * L))
    _assert_maps_equal(got, [(i[:1], d[:1]) for i, d in want], "_ps sizes rounding to 1")


class _DS:
    def __init__(self, i, xyz, W, H, fmt, sizes=None):
        self.id, self.tgt_sh, self.input_format = i, (W, H), fmt
        self.scene_data = {'pointcloud': {'xyz': xyz}, 'point_sizes': sizes}


FMT = "uv_1d_p2, uv_1d_ps8_ds1, uv_1d_p1_ds2, uv_1d_p3_ds3, uv_1d_p1_ds4"


def test_myrender_point_sprites_match_the_oracle(oracle_mod):
    W, H = 160, 96
    xa = synth.street_scene(30_000, depth=40.0, seed=1)
    xb = synth.street_scene(20_000, depth=30.0, seed=2)
    sb = _sizes(20_000, 9)
    dss = [_DS(0, xa, W, H, FMT), _DS(1, xb, W, H, FMT, sb)]
    proj, view = synth.camera_batch(W, H, [0, 2, 4, 6])
    data = {'input': {'id': torch.tensor([0, 1, 1, 0])}, 'proj_matrix': torch.from_numpy(proj),
            'view_matrix': torch.from_numpy(view)}
    out, dep = MyRender(dss, point_sprites=True).render(data)
    levels = [(2, False), (8, True), (1, False), (3, False), (1, False)]
    M = (proj @ np.linalg.inv(view)).astype(np.float32)
    keys = [k.strip() for k in FMT.split(',')]
    for sel, xyz, sz in (([0, 3], xa, None), ([1, 2], xb, sb)):
        want = oracle_sprite.sprite_maps(xyz, M[sel], W, H, levels, sz)
        for l, k in enumerate(keys):
            assert np.array_equal(out[k][sel, 0].numpy(), want[l][0]), (sel, k)
            assert np.array_equal(dep[k][sel, 0].numpy(), want[l][1]), (sel, k)
    # the default ignores the sizes: today's 1-pixel maps
    out1, _ = MyRender(dss).render(data)
    for sel, xyz in (([0, 3], xa), ([1, 2], xb)):
        for l, k in enumerate(keys):
            w, h = ops.level_sizes(W, H, 5)[l]
            idx, _ = oracle_mod.pcpr_forward(xyz, M[sel], w, h)
            assert np.array_equal(out1[k][sel, 0].numpy(), idx), (sel, k)


def _texture(n, seed):
    return torch.rand((1, 8, n), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("ss,temporal", [(1, False), (2, False), (1, True)])
def test_frame_renderer_equals_forward_on_myrender_maps(synth_sd, ss, temporal):
    W, H, n = 128, 64, 60_000
    fmt = "uv_1d_p2, uv_1d_ps8_ds1, uv_1d_p1_ds2, uv_1d_p3_ds3"
    xyz = synth.street_scene(n, depth=40.0, seed=12)
    sizes = _sizes(n, 12)
    tex = _texture(n, 12)
    fr = FrameRenderer(xyz, synth_sd, tex, (W, H), supersampling=ss, temporal_average=temporal, input_format=fmt,
                       point_sizes=sizes)
    ref = _net(synth_sd, tex, ss, temporal, fr.model.net.precision)
    mr = MyRender([_DS(0, xyz, W * ss, H * ss, fmt, sizes)], device_outputs=True, point_sprites=True)
    for t in (3, 4):
        proj, view = synth.camera_batch(W * ss, H * ss, [t])
        got = fr.infer(proj[0], view[0])
        maps, _ = mr.render({'input': {'id': torch.tensor([0])}, 'proj_matrix': torch.from_numpy(proj),
                             'view_matrix': torch.from_numpy(view)})
        with torch.no_grad():
            want = ref(maps)
        exp = want[0].permute(1, 2, 0)
        err = float((got['output'][..., :3] - exp).abs().max())
        if ss == 1 and not temporal:
            assert err == 0.0, err
        else:   # forward reduces and averages with torch ops, render with its staging kernel (same as the 1-pixel tests)
            assert err < (2e-4 if fr.model.net.precision == "fp32" else 3e-2), err


def _net(sd, tex, ss, temporal, precision):
    net = UNet()
    net.load_state_dict(sd, strict=True)
    net.precision = precision
    t = PointTexture(8, tex.shape[2])
    with torch.no_grad():
        t.texture_.copy_(tex)
    m = NetAndTexture(net, {0: t}, ss, temporal_average=temporal)
    m.load_textures(0)
    return m.cuda().eval()


def _composed_oracle(comp, seg_m, W, H, levels, sizes_of):
    """The sprite oracle over every visible segment with its own matrix, local ids mapped to global ids, merged by key."""
    store = comp.store
    vis = store.visible_flags().numpy()
    best = None
    for s in range(store.nseg):
        if not vis[s]:
            continue
        f, c = store.first_chunk[s], store.chunks[s]
        rows = store.pts4[f * CHUNK:(f + c) * CHUNK].cpu()
        real = ~torch.isnan(rows[:, 0])
        rows = rows[real]
        gid = rows[:, 3].contiguous().view(torch.int32).to(torch.int64)
        order = torch.argsort(gid)
        xyz, gid = rows[order, :3].numpy().copy(), gid[order].numpy()
        if store.psize is not None:                         # the store's sizes travel with their rows
            ps = store.psize[f * CHUNK:(f + c) * CHUNK].cpu()[real][order].numpy()
            assert np.array_equal(ps, sizes_of(gid))
        else:
            ps = None
        keys = oracle_sprite.sprite_zbuf(xyz, seg_m[s], W, H, levels, ps)
        merged = []
        for k in keys:
            empty = k == EMPTY
            local = np.where(empty, 0, k & np.uint64(0xFFFFFFFF)).astype(np.int64)
            merged.append(np.where(empty, EMPTY, (k & ~np.uint64(0xFFFFFFFF)) | gid[local].astype(np.uint64)))
        keys = merged
        best = keys if best is None else [np.minimum(a, b) for a, b in zip(best, keys)]
    return [oracle_sprite.resolve(k) for k in best]


def test_scene_renderer_composition_matches_the_oracle(synth_sd):
    W, H = 128, 64
    fmt = "uv_1d_p3, uv_1d_ps8_ds1, uv_1d_p2_ds2, uv_1d_ds3"
    levels = [(3, False), (8, True), (2, False), (1, False)]
    na, nb = 40_000, 15_000
    xa = synth.street_scene(na, depth=40.0, seed=21)
    xb = synth.street_scene(nb, depth=25.0, seed=22)
    sb = _sizes(nb, 22)
    comp = SceneComposer(_dev())
    a = comp.add_scene(xa, _texture(na, 1))
    P = np.eye(4)
    P[:3, 3] = [3.0, 0.0, -30.0]                                       # far along the street: partly outside the view
    b = comp.add_scene(xb, _texture(nb, 2), P, point_sizes=sb)
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
    sizes_global = np.concatenate([np.zeros(na, np.float32), sb])
    sr = SceneRenderer(comp, synth_sd, (W, H), input_format=fmt)
    proj, view = synth.camera_batch(W, H, [2])
    seg_m = comp.segment_matrices(FrameRenderer.total_matrix(proj[0], view[0]))
    frame = sr.infer(proj[0], view[0])
    assert tuple(frame['output'].shape) == (H, W, 4)
    m = torch.from_numpy(seg_m).to(_dev())
    _, maps = sr.model.render(comp.store, m, W, H, want_maps=True, input_format=fmt)
    got = [(i.cpu().numpy(), d.cpu().numpy()) for i, d in maps]
    _assert_maps_equal(got, _composed_oracle(comp, seg_m, W, H, levels, lambda g: sizes_global[g]), "composed")
    units = ops.last_surviving_units(comp.store)
    assert 0 < units < comp.store.nunits                              # part of the cloud was culled


def test_descriptor_gradient_through_sprite_maps():
    W, H, n = 96, 64, 5_000
    xyz = synth.street_scene(n, depth=30.0, seed=31)
    proj, view = synth.camera_batch(W, H, [0, 1])
    m = torch.from_numpy(synth.total_matrix(proj, view)).to(_dev())
    store = ops.SortedPoints(torch.from_numpy(xyz).to(_dev()))
    pyr = _sprite_pyramid(store, m, W, H, [(9, False)])
    ids, _ = ops.zbuf_resolve(pyr, 0)
    counts = torch.bincount(ids.reshape(-1).long(), minlength=n)
    assert int(counts[1:].max()) >= 20                                # one id covers many pixels
    g = torch.Generator().manual_seed(3)
    go = torch.randn((2, 8, H, W), generator=g).to(_dev())
    got = ops.gather_backward(go, ids, n).cpu()
    want = torch.zeros((n, 8), dtype=torch.float64).index_add_(
        0, ids.reshape(-1).long().cpu(), go.permute(0, 2, 3, 1).reshape(-1, 8).double().cpu())
    err = (got.double() - want).abs().max() / want.abs().max()
    assert float(err) < 1e-5, float(err)
