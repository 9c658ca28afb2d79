"""Point sprites without a GPU: the input-format parser, the sprite oracle's known answers, and the host-side validation."""
import numpy as np
import pytest
import torch

import oracle
import oracle_sprite
from read_b200 import ops, sprites, synth


@pytest.mark.parametrize("key,want", [
    ("uv_1d", (1, False)), ("uv_1d_ds1", (1, False)), ("uv_1d_p3_ds1", (3, False)), ("uv_1d_ps8", (8, True)),
    ("uv_1d_ps8_ds1", (8, True)), ("uv_1d_p2_ps16", (16, True)), ("uv_1d_ps4_p7", (7, False)), ("uv_2d_p12", (12, False)),
])
def test_parser_takes_the_last_size_match(key, want):
    assert sprites.parse_point_size(key) == want


def test_sprite_levels_and_their_errors():
    assert sprites.sprite_levels("uv_1d_p2, uv_1d_ps8_ds1, uv_1d_ds2, uv_1d_p3_ds3", 4) == [(2, False), (8, True), (1, False),
                                                                                             (3, False)]
    assert sprites.sprite_levels(["uv_1d_p2", "uv_1d", "colors", "x"], 2) == [(2, False), (1, False)]   # only n_levels keys
    for fmt, name in (("colors_p2,uv_1d", "colors_p2"), ("uv_1d_p0,uv_1d", "uv_1d_p0"), ("uv_1d,uv_1d_p65", "uv_1d_p65"),
                      ("uv_1d,uv_1d_p2_ds2", "uv_1d_p2_ds2"), ("uv_1d_ds1,uv_1d", "uv_1d_ds1")):
        with pytest.raises(ValueError, match=name):
            sprites.sprite_levels(fmt, 2)
    with pytest.raises(ValueError):
        sprites.sprite_levels("uv_1d", 2)
    assert sprites.sprite_levels("uv_1d_p64", 1) == [(64, False)]
    assert sprites.one_pixel([(1, False)] * 3) and not sprites.one_pixel([(1, False)], np.ones(3))
    assert not sprites.one_pixel([(1, True)])


def test_point_size_validation():
    assert sprites.check_point_sizes(np.array([0.0, 1.5, 80.0]), 3).dtype == torch.float32
    for bad in (np.ones(4), np.array([1.0, -0.5, 2.0]), np.array([1.0, np.nan, 2.0]), np.array([1.0, np.inf, 2.0])):
        with pytest.raises(ValueError):
            sprites.check_point_sizes(bad, 3)
    xyz = torch.zeros((3, 3))
    with pytest.raises(ValueError):
        ops.SortedPoints(xyz, point_sizes=np.array([1.0, -1.0, 2.0]))
    with pytest.raises(ValueError):
        ops.SegmentedPoints([(xyz, torch.arange(3), np.ones(2))])


def test_stores_permute_and_pad_the_sizes():
    rng = np.random.default_rng(0)
    xyz = torch.from_numpy(rng.uniform(-5, 5, (3000, 3)).astype(np.float32))
    sizes = rng.uniform(0, 10, 3000).astype(np.float32)
    st = ops.SortedPoints(xyz, cell=0.5, point_sizes=sizes)
    assert st.psize.shape[0] == 3072 and bool((st.psize[3000:] == 0).all())
    ids = st.pts4[:, 3].contiguous().view(torch.int32).long()
    assert torch.equal(st.psize[:3000], torch.from_numpy(sizes)[ids])
    seg = ops.SegmentedPoints([(xyz, torch.arange(3000) + 7, sizes), (xyz[:10], torch.arange(10))])
    assert seg.psize.shape[0] == seg.n
    gid = seg.pts4[:, 3].contiguous().view(torch.int32).long()
    real = ~torch.isnan(seg.pts4[:, 0])
    first = real.clone()
    first[3072:] = False
    assert torch.equal(seg.psize[first], torch.from_numpy(sizes)[gid[first] - 7])
    assert bool((seg.psize[~first] == 0).all())                      # padding and the part without sizes
    assert ops.SegmentedPoints([(xyz, torch.arange(3000))]).psize is None
    with pytest.raises(ValueError):
        st.shard(0, 100)


# ---------------------------------------------------------------------------------------------- oracle known answers
_ID = np.eye(4, dtype=np.float32)[None]


def _one_point(u, v, W, H, z=0.5):
    """A point whose centre lands at (u, v) under the identity matrix: cx = 2u/W - 1, cy = 1 - 2v/H (exact for dyadic u, v)."""
    return np.array([[2.0 * u / W - 1.0, 1.0 - 2.0 * v / H, z]], np.float32)


@pytest.mark.parametrize("u", [10.25, 10.5, 10.75])
@pytest.mark.parametrize("wd", [1, 2, 3, 4])
def test_oracle_squares(u, wd):
    W = H = 32
    (idx, dep), = oracle_sprite.sprite_maps(_one_point(u, 20.25, W, H), _ID, W, H, [(wd, False)])
    k = wd // 2
    x0 = 10 - k if wd % 2 else 10 + (u - 10 >= 0.5) - k
    y0 = 20 - k if wd % 2 else 20 - k                               # v = 20.25: below the half pixel
    want = np.zeros((H, W), bool)
    want[y0:y0 + wd, x0:x0 + wd] = True
    assert np.array_equal(dep[0] != 0, want)
    assert np.all(dep[0][want] == np.float32(0.75)) and np.all(idx[0][want] == 0)


def test_oracle_corners_and_edges_clip():
    W, H = 16, 8
    for (u, v), n_px in (((0.25, 0.25), 9), ((15.75, 7.75), 9), ((0.25, 4.25), 15), ((8.25, 7.9), 15)):
        (_, dep), = oracle_sprite.sprite_maps(_one_point(u, v, W, H), _ID, W, H, [(5, False)])
        assert int((dep[0] != 0).sum()) == n_px, (u, v)
    # a centre outside the frame draws nothing, however large the point
    (_, dep), = oracle_sprite.sprite_maps(np.array([[1.2, 0.0, 0.5]], np.float32), _ID, W, H, [(64, False)])
    assert not dep.any()


def test_oracle_relative_size_and_per_point_sizes():
    W = H = 64
    pts = np.concatenate([_one_point(20.25, 20.25, W, H, 0.5), _one_point(40.25, 40.25, W, H, 0.25)])
    # clip z = z under the identity: 8 / 0.5 = 16 and 8 / 0.25 = 32 pixels; per-point 0 keeps N, 2 -> 4 / 8 pixels
    (_, dep), = oracle_sprite.sprite_maps(pts, _ID, W, H, [(8, True)])
    # the squares (columns and rows 12..27 and 24..55) overlap in 4 x 4 pixels, which go to the nearer point (depth 0.625)
    assert int((dep[0] == np.float32(0.625)).sum()) == 32 * 32
    assert int((dep[0] == np.float32(0.75)).sum()) == 16 * 16 - 4 * 4
    (_, dep), = oracle_sprite.sprite_maps(pts, _ID, W, H, [(8, True)], np.array([0.0, 2.0], np.float32))
    assert int((dep[0] == np.float32(0.625)).sum()) == 8 * 8
    (_, dep), = oracle_sprite.sprite_maps(pts, _ID, W, H, [(3, False)], np.array([200.0, 0.0], np.float32))
    # 200 clamps to 64: columns and rows -12..51, clipped to 0..51; the nearer 3 x 3 point keeps its pixels
    assert int((dep[0] == np.float32(0.625)).sum()) == 9
    assert int((dep[0] == np.float32(0.75)).sum()) == 52 * 52 - 9


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_oracle_width_one_equals_the_pcpr_oracle(seed):
    W, H, L = 96, 48, 3
    xyz = synth.street_scene(20_000, depth=50.0, seed=seed)
    proj, view = synth.camera_batch(W, H, [seed, seed + 3])
    M, idx, dep = oracle.render_pyramid(xyz, proj, view, W, H, L)
    for l, (i, d) in enumerate(oracle_sprite.sprite_maps(xyz, M, W, H, [(1, False)] * L)):
        assert np.array_equal(i, idx[l][:, 0]) and np.array_equal(d, dep[l][:, 0])
