"""-m gpu: the UNMODIFIED reference CUDA rasterizer (pcpr.forward, compiled from the reference's own sources by
oracle/build_ref.py) against the oracle and against our kernel (SURVEY.md §8c(3)), through its outputs on the two scenes below
as recorded by tests/golden/make_ref_pcpr_golden.py.

The reference kernel is nondeterministic under pixel contention (its lock drops contended writes), so:
  * on a collision-free scene (at most one point per pixel) all three must agree exactly;
  * on a dense scene the reference may only be WORSE than the true z-buffer: ref_depth >= oracle_depth wherever
    both are non-empty, and it never invents coverage.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from gpu_util import render_gpu, scene_and_cams

pytestmark = pytest.mark.gpu


def _ref(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


def test_collision_free_scene_all_three_agree(oracle_mod):
    W, H = 64, 48
    ys, xs = np.mgrid[0:H, 0:W]
    # one point per pixel centre (identity matrix: u = W(x+1)/2), random depths, shuffled ids
    x = (xs.ravel() + 0.5) / W * 2 - 1
    y = 1 - (ys.ravel() + 0.5) / H * 2
    rng = np.random.default_rng(0)
    z = rng.uniform(-0.9, 0.9, x.size)
    xyz = np.stack([x, y, z], 1).astype(np.float32)[rng.permutation(x.size)]
    xyz = np.concatenate([np.full((1, 3), 9, np.float32), xyz])       # id 0 off-screen ("0 denotes empty")
    M = np.eye(4, dtype=np.float32)[None]
    oi, od = oracle_mod.pcpr_forward(xyz, M, W, H)
    g = _ref("ref_pcpr_collision_free")
    ri, rd = g["index"], g["depth"]
    gi, gd, _ = render_gpu(xyz, M, W, H, 1)
    assert (oi != 0).all()
    np.testing.assert_array_equal(ri, oi)
    np.testing.assert_array_equal(rd, od)
    np.testing.assert_array_equal(gi[0], oi)
    np.testing.assert_array_equal(gd[0], od)


def test_dense_scene_reference_is_never_better_than_the_zbuffer(oracle_mod):
    xyz, M = scene_and_cams(300_000, 128, 96, [0], depth=60.0)
    oi, od = oracle_mod.pcpr_forward(xyz, M, 128, 96)
    rd = _ref("ref_pcpr_dense")["depth"]
    assert ((rd == 0) >= (od == 0)).all()                  # reference covers no pixel the z-buffer leaves empty
    both = (rd != 0) & (od != 0)
    assert (rd[both] >= od[both]).all()
    print(f"reference depth equals the sequential z-buffer on {100 * float((rd == od).mean()):.2f}% of pixels")
    gi, gd, _ = render_gpu(xyz, M, 128, 96, 1)
    np.testing.assert_array_equal(gi[0], oi)               # ours is exact
