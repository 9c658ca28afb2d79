"""Point-cloud views on the host: the numpy float32 restatement of every mode against hand-derived values and against the float64
GLSL formulas, the exact PCA of the ``--pca`` colours against numpy's SVD and against the reference's own ``pca_color``, and the
argument checks of render_points."""
import numpy as np
import pytest
import torch

import point_view_util as pv
from conftest import load_golden
from read_b200 import point_views

F = np.float32
EYE_AT_5 = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 5], [0, 0, 0, 1]], F)     # camera at (0, 0, 5), axes aligned


def _normals(n, submode, p=(0., 0., 1.), view=EYE_AT_5):
    n = np.asarray(n, F).reshape(-1, 3)
    xyz = np.repeat(np.asarray(p, F).reshape(1, 3), n.shape[0], 0)
    return pv.shade32("normals", submode, np.arange(n.shape[0]), normals=n, xyz=xyz, view_matrix=view)


AXES = np.eye(3, dtype=F)


def test_axis_normals_under_each_submode():
    assert np.array_equal(_normals(AXES, 0), 0.5 * AXES + 0.5)
    assert np.array_equal(_normals(AXES, 4), AXES)
    # view direction from p = (0, 0, 1) to the camera at (0, 0, 5) is +z, whatever the normal
    assert np.array_equal(_normals(AXES, 3), np.tile(F([0.5, 0.5, 1.0]), (3, 1)))
    # reflect(d, n) = d - 2 dot(n, d) n with d = +z: x and y normals leave it, the z normal turns it round
    assert np.array_equal(_normals(AXES, 1), F([[0.5, 0.5, 1.0], [0.5, 0.5, 1.0], [0.5, 0.5, 0.0]]))
    # camera frame: m_view (cam + n, 1) = n for an axis-aligned camera
    assert np.array_equal(_normals(AXES, 2), 0.5 * AXES + 0.5)
    # a camera whose z axis is the world's x axis (view = camera-to-world pose, m_view = inv(view)) sees the x normal as +z
    rot = np.array([[0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 5], [0, 0, 0, 1]], F)
    got = _normals(AXES[:1], 2, view=rot)
    assert np.allclose(got, F([[0.5, 0.5, 1.0]]), atol=1e-6), got


def test_zero_vectors_normalise_to_nan():
    assert np.all(np.isnan(_normals(AXES[:1], 3, p=(0., 0., 5.))))         # the point sits on the camera
    assert np.all(np.isnan(_normals(AXES[:1], 1, p=(0., 0., 5.))))
    # camera frame of a zero normal: m_view (cam, 1) = 0
    assert np.all(np.isnan(_normals(np.zeros((1, 3)), 2)))


def test_xyz_maps_the_bounding_box_corners_to_0_and_1():
    lo, hi = F([-1.0, -2.0, -3.0]), F([1.0, 2.0, 7.5])
    corners = np.array([[(hi if (c >> a) & 1 else lo)[a] for a in range(3)] for c in range(8)], F)
    got = pv.shade32("xyz", 0, np.arange(8), xyz=corners, lo=lo, hi=hi)
    want = np.array([[(c >> a) & 1 for a in range(3)] for c in range(8)], F)     # (hi - lo) + 1e-9 rounds to hi - lo in float32
    assert np.array_equal(got, want)


def test_uv_rounds_ids_to_float32():
    ids = np.array([0, 7, (1 << 24) + 1, (1 << 31) - 1], np.int64)
    got = pv.shade32("uv", 0, ids)
    assert got[:, 0].tolist() == [0.0, 7.0, float(1 << 24), float(1 << 31)]
    assert not got[:, 1:].any()
    for sub in range(1, 5):
        assert not pv.shade32("uv", sub, ids).any()


def test_label_is_normal_x_over_255():
    n = F([[0, 9, 9], [255, 9, 9], [17, 0, 0]])
    got = pv.shade32("label", 0, np.arange(3), normals=n)
    assert got[:, 0].tolist() == [0.0, 1.0, float(F(17) / F(255))]
    assert not got[:, 1:].any()


def _scene(n, seed):
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(-20, 20, (n, 3)).astype(F)
    nrm = rng.standard_normal((n, 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(F)
    ang = rng.uniform(0, 2 * np.pi)
    view = np.eye(4, dtype=F)
    view[:3, :3] = np.array([[np.cos(ang), 0, np.sin(ang)], [0, 1, 0], [-np.sin(ang), 0, np.cos(ang)]], F)
    view[:3, 3] = rng.uniform(-5, 5, 3)
    proj = np.array([[1.2, 0, 0, 0], [0, 1.6, 0, 0], [0, 0, -1.0002, -0.20002], [0, 0, -1, 0]], F)
    total = (proj @ np.linalg.inv(view)).astype(F)
    return dict(xyz=xyz, normals=nrm, total_m=total, view_matrix=view, lo=xyz.min(0), hi=xyz.max(0),
                colors=rng.random((n, 3)).astype(F))


CASES = [("normals", s) for s in range(5)] + [("depth", 0), ("xyz", 0), ("label", 0), ("color", 0), ("uv", 0)]


@pytest.mark.parametrize("mode,submode", CASES)
def test_restatement_is_within_a_few_ulps_of_the_glsl_formulas(mode, submode):
    kw = _scene(20_000, 3)
    ids = np.arange(20_000)
    got = pv.shade32(mode, submode, ids, **kw)
    want = pv.shade64(mode, submode, ids, **kw)
    # half(v) = v*0.5 + 0.5 of a unit vector's component: its error is a few ulps of 0.5, whatever the result's size; in the
    # camera frame, m_view (cam + n, 1) cancels the camera position, so the error grows with |cam|
    floor = 0.5 if mode == "normals" and submode < 4 else 0.0
    if mode == "normals" and submode == 2:
        floor *= 1 + float(np.abs(kw["view_matrix"][:3, 3]).max())
    ulp = np.spacing(np.maximum(np.abs(want), floor).astype(F)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want)
    if mode == "depth":   # c2 itself: 2 fma + add over terms of either sign, relative to the largest term
        scale = np.abs(kw["xyz"].astype(np.float64) * kw["total_m"][2, :3]).max(1)[:, None] + abs(float(kw["total_m"][2, 3]))
        assert float((err / np.spacing(scale.astype(F))).max()) <= 3
    else:
        assert float((err / ulp).max()) <= 4, float((err / ulp).max())


def test_pca_is_the_exact_pca_of_numpy_svd():
    tex = pv.separated_descriptors(5000, 11)
    got = point_views.pca_colors(torch.from_numpy(tex))
    assert got.dtype == torch.float32 and tuple(got.shape) == (5000, 4) and not got[:, 3].any()
    want = pv.pca_exact(tex[0])
    err = np.abs(got[:, :3].numpy().astype(np.float64) - want) / np.spacing(want.astype(F))
    assert float(err.max()) <= 1.0, float(err.max())
    # the sign rule fixes the basis, not the data's sign: negated descriptors project to -x, and the percentile normalisation
    # turns that into 1 - colour
    neg = point_views.pca_colors(torch.from_numpy(-tex))
    assert float((neg[:, :3].double() - (1 - torch.from_numpy(want))).abs().max()) < 1e-6


@pytest.mark.parametrize("n,q", [(1, 10), (2, 10), (10, 90), (11, 10), (12345, 10), (12345, 90), (3 * 7, 50)])
def test_percentile_is_numpys_linear_percentile(n, q):
    v = np.sort(np.random.default_rng(n).standard_normal(n))
    got = float(point_views.percentile(torch.from_numpy(v), q))
    assert got == float(np.percentile(v, q)), (got, np.percentile(v, q))


def test_pca_matches_the_reference_pca_color_golden():
    g = load_golden("ref_pca")
    tex = pv.separated_descriptors(int(g["n"]), int(g["seed"]))
    got = point_views.pca_colors(torch.from_numpy(tex))[:, :3].numpy()
    err = float(np.abs(got - g["colors"]).max())
    # IncrementalPCA(3, batch_size=64) approximates the exact PCA; measured 4.2e-4 on this fixture, frozen with margin
    assert err < 5e-4, err


@pytest.mark.parametrize("kw,name", [
    (dict(mode="rgb"), "mode"), (dict(mode=None), "mode"),
    (dict(submode=5), "submode"), (dict(submode=-1), "submode"), (dict(submode=1.5), "submode"),
    (dict(point_size=0), "point_size"), (dict(point_size=65), "point_size"), (dict(point_size=float("nan")), "point_size"),
    (dict(point_size="big"), "point_size"),
    (dict(clear_color=(0, 0, 0)), "clear_color"), (dict(clear_color=(0, 0, 0, float("inf"))), "clear_color"),
    (dict(clear_color="black"), "clear_color"),
])
def test_bad_view_arguments_raise_naming_the_argument(kw, name):
    args = dict(mode="color", submode=0, point_size=1, clear_color=(0., 0., 0., 1.))
    args.update(kw)
    with pytest.raises(ValueError, match=name):
        point_views.check_view_args(**args)


def test_good_view_arguments():
    assert point_views.check_view_args("pca", 4, 64, [0, 0.5, 1, 1]) == (0.0, 0.5, 1.0, 1.0)
    assert point_views.check_view_args("uv", np.int64(0), 1.5, np.zeros(4)) == (0.0,) * 4


def test_missing_tables_raise_naming_the_attribute():
    for mode, name in (("color", "colors"), ("normals", "normals"), ("label", "normals")):
        with pytest.raises(ValueError, match=name):
            point_views.table_for(mode, None, None, lambda: None)
    assert point_views.table_for("uv", None, None, None) is None
    assert point_views.table_for("depth", None, None, None) is None


def test_attribute_tables_are_checked():
    with pytest.raises(ValueError, match="colors"):
        point_views.attribute_table(np.zeros((4, 4)), 4, "colors", "cpu")
    with pytest.raises(ValueError, match="normals"):
        point_views.attribute_table(np.zeros((3, 3)), 4, "normals", "cpu")
    bad = np.zeros((4, 3))
    bad[2, 1] = np.nan
    with pytest.raises(ValueError, match="finite"):
        point_views.attribute_table(bad, 4, "colors", "cpu")
    t = point_views.attribute_table(torch.arange(12.).reshape(4, 3), 4, "colors", "cpu")
    assert t.dtype == torch.float32 and t.shape == (4, 4) and t[:, :3].tolist() == torch.arange(12.).reshape(4, 3).tolist()
    assert not t[:, 3].any()
