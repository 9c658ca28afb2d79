"""Clouds of more than 2^24 + 1 points, host side (no GPU): the index-map dtype rule at its edges, the 2^31-point limit where a cloud
enters, the ctypes bindings of the int32 entry points, the dtype checks of the gather wrappers, and the int32 oracle z-buffer
(tests/zbuffer_i32.c) against oracle/zbuffer.c.
tests/test_gpu_large_scene.py checks the kernels on an H100."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

import oracle_i32
from conftest import ROOT
from read_b200 import _lib, ops, synth
from read_b200.compose import NetAndTexture
from read_b200.myrender import MyRender
from read_b200.texture import PointTexture

I32_TWINS = ["read_zbuf_resolve", "read_gather_from_index", "read_gather_from_index_items", "read_gather_backward",
             "read_gather_backward_sparse", "read_gather_backward_items", "read_gather_backward_sparse_items",
             "read_gather_backward_det", "read_gather_backward_sparse_det", "read_gather_backward_items_det",
             "read_gather_backward_sparse_items_det"]


def test_index_map_dtype_at_its_edges():
    assert ops.index_map_dtype(0) == torch.float32
    assert ops.index_map_dtype(10_000_000) == torch.float32
    assert ops.index_map_dtype(2 ** 24) == torch.float32
    assert ops.index_map_dtype(2 ** 24 + 1) == torch.float32       # largest id 2^24: float32 holds it
    assert ops.index_map_dtype(2 ** 24 + 2) == torch.int32         # id 2^24 + 1 has no float32
    assert ops.index_map_dtype(2 ** 25) == torch.int32
    assert ops.index_map_dtype(2 ** 31 - 1) == torch.int32
    for n in (2 ** 31, 2 ** 31 + 1, 2 ** 32):
        with pytest.raises(ValueError, match="2\\^31"):
            ops.index_map_dtype(n)


def test_the_edge_is_where_float32_stops_holding_ids():
    ids = np.arange(2 ** 24 - 4, 2 ** 24 + 6, dtype=np.int64)
    exact = ids.astype(np.float32).astype(np.int64) == ids
    assert exact[ids <= 2 ** 24].all() and not exact[ids == 2 ** 24 + 1].any()


def _ds(xyz, ds_id=0):
    import types
    return types.SimpleNamespace(id=ds_id, tgt_sh=(64, 64), input_format="uv_1d_p1", scene_data={'pointcloud': {'xyz': xyz}})


def test_clouds_of_2_31_points_are_rejected_where_they_enter():
    huge = np.broadcast_to(np.zeros(3, np.float32), (2 ** 31, 3))          # no memory behind it
    with pytest.raises(ValueError, match="2\\^31"):
        MyRender().update_ds([_ds(np.zeros((10, 3), np.float32), 0), _ds(huge, 1)])
    model = NetAndTexture(nn.Identity(), {0: PointTexture(8, 4)})
    with pytest.raises(ValueError, match="2\\^31"):
        model.render(torch.zeros(3).expand(2 ** 31, 3), torch.eye(4)[None], 64, 64)


def test_i32_entry_points_are_bound_like_their_float_twins():
    sigs = _lib._SIGS
    assert sorted(n for n in sigs if n.endswith("_i32")) == sorted(n + "_i32" for n in I32_TWINS)
    for name in I32_TWINS:
        assert sigs[name + "_i32"] == sigs[name], name
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "read_b200.h")).read(), flags=re.S)
    for name in I32_TWINS:
        decl = re.search(r"\b" + name + r"_i32\s*\(([^;]*)\)\s*;", header).group(1)
        twin = re.search(r"\b" + name + r"\s*\(([^;]*)\)\s*;", header).group(1)
        n_args = lambda d: len([a for a in d.split(",") if a.strip()])
        assert n_args(decl) == n_args(twin), name
        # the index map is the one argument whose type changes: float -> int32_t
        assert re.sub(r"\s+", " ", twin.replace("float *ids", "int32_t *ids").replace("float *index_out", "int32_t *index_out")) \
            == re.sub(r"\s+", " ", decl), name


def test_gather_wrappers_take_float32_or_int32_maps_only():
    tex = torch.zeros((4, 8))
    for dt in (torch.int64, torch.float64, torch.int16, torch.uint8):
        ids = torch.zeros((1, 2, 2), dtype=dt)
        with pytest.raises(RuntimeError, match="float32 or int32"):
            ops.gather_from_index(tex, ids)
        with pytest.raises(RuntimeError, match="float32 or int32"):
            ops.gather_from_index_items([tex], [0], ids)
        with pytest.raises(RuntimeError, match="float32 or int32"):
            ops.gather_backward(torch.zeros((1, 8, 2, 2)), ids, 4)


def test_index_map_keeps_int32_and_converts_everything_else_to_float32():
    cpu = torch.device("cpu")
    i32 = torch.tensor([[0, 2 ** 24 + 1]], dtype=torch.int32)
    assert ops.index_map(i32, cpu).dtype == torch.int32 and torch.equal(ops.index_map(i32, cpu), i32)
    for dt in (torch.float32, torch.float64, torch.int64):
        assert ops.index_map(torch.zeros((2, 3), dtype=dt).t(), cpu).dtype == torch.float32
    assert ops.index_map(torch.zeros((2, 3), dtype=torch.int32).t(), cpu).is_contiguous()


def test_int32_oracle_equals_the_float_oracle_on_a_small_scene(oracle_mod):
    xyz = synth.street_scene(60_000, depth=60.0, seed=5)
    proj, view = synth.camera_batch(96, 64, [0, 3])
    tm = synth.total_matrix(proj, view)
    for w, h in oracle_mod.level_sizes(96, 64, 3):
        fi, fd = oracle_mod.pcpr_forward(xyz, tm, w, h)
        ii, idp = oracle_i32.pcpr_forward_i32(xyz, tm, w, h)
        assert ii.dtype == np.int32 and np.array_equal(ii, fi.astype(np.int32)) and np.array_equal(idp, fd)
        assert (ii > 0).sum() > 0.2 * ii.size


def test_int32_oracle_gives_exact_ids_where_float32_cannot(oracle_mod):
    """A cloud of 2^24 + 8 points, all behind the camera but the last six, which land on six pixels of their own."""
    n = 2 ** 24 + 8
    xyz = np.zeros((n, 3), np.float32)
    xyz[:, 2] = 5.0                                                  # behind the camera (GL: -z forward): culled
    W = H = 64
    proj, view = synth.camera_batch(W, H, [0])
    tm = synth.total_matrix(proj, view)
    last = np.arange(n - 6, n)
    xyz[last] = np.stack([np.linspace(-2, 2, 6), np.zeros(6), np.full(6, -10.0)], 1).astype(np.float32)
    fi, fd = oracle_mod.pcpr_forward(xyz, tm, W, H)
    ii, idp = oracle_i32.pcpr_forward_i32(xyz, tm, W, H)
    assert np.array_equal(idp, fd)
    assert sorted(ii[ii > 0].tolist()) == last.tolist()
    wrong = fi[ii > 0].astype(np.int64) != ii[ii > 0]
    assert wrong.sum() == 3                                          # the odd ids above 2^24 round to a neighbour in float32
