"""-m gpu: scene editing at scale (ops.raster_project_segments_culled, thousands of segments, view-frustum culling of the store's
chunks on the device).

The world: stitched street scenes along -z and a "garage" scene of compact cars whose points are all carved into objects; the
cars are placed on the street by their transforms and instanced hundreds to thousands of times.  The camera stands inside the
world, so most chunks lie behind it or outside the field of view.  The culled path must give the parameter-table path's
z-buffer bit for bit (<= 128 segments), the merged per-segment oracle's maps at 1000 and 4096 segments, and draw exactly the
units the host restatement of the cull rule keeps."""
import numpy as np
import pytest
import torch

from read_b200 import ops, synth
from read_b200.scene_edit import SceneComposer
from read_b200.viewer import SceneRenderer
from scene_scale_util import kept_units
from test_gpu_scene_edit import TOL_FP32, _assert_maps_equal, _composed_oracle, _net_and_texture

pytestmark = pytest.mark.gpu
STREET = 60.0                                    # metres of street per stitched scene
N_CARS = 8


def _dev():
    return torch.device("cuda", 0)


def _translate(x, y, z, yaw=0.0):
    M = np.eye(4)
    M[:3, :3] = [[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]]
    M[:3, 3] = [x, y, z]
    return M


def _car(rng, n=300):
    """A compact car-sized cloud (4 x 1.5 x 2 m) centred on the origin."""
    return (rng.uniform(-0.5, 0.5, (n, 3)) * [4.0, 1.5, 2.0] + [0.0, 0.75, 0.0]).astype(np.float32)


def _world(n_segments, rng, n_streets=4, street_points=40_000):
    """Streets + a garage of N_CARS cars carved into objects + instances, n_segments in all; every 5th instance hidden."""
    comp = SceneComposer(_dev())
    streets = [comp.add_scene(synth.street_scene(street_points, depth=STREET, seed=40 + k),
                              torch.rand((1, 8, street_points), generator=torch.Generator().manual_seed(k)),
                              placement=_translate(0, 0, -STREET * k)) for k in range(n_streets)]
    cars = np.concatenate([_car(rng) + [100.0 * (k + 1), 0, 0] for k in range(N_CARS)])
    garage = comp.add_scene(cars, torch.rand((1, 8, cars.shape[0]), generator=torch.Generator().manual_seed(99)))
    depth = STREET * n_streets

    def place(k):
        return _translate(rng.uniform(-12, 12) - 100.0 * (k + 1), -1.6, rng.uniform(-depth + 3, -3), rng.uniform(-np.pi, np.pi))
    objs = [comp.add_object(garage, np.arange(300 * k, 300 * (k + 1)), place(k)) for k in range(N_CARS)]
    n_inst = n_segments - n_streets - 1 - N_CARS
    insts = []
    for k in range(N_CARS):
        cnt = n_inst // N_CARS + (1 if k < n_inst % N_CARS else 0)
        insts += comp.add_instances(objs[k], np.stack([place(k) for _ in range(cnt)]))
    for h in insts[::5]:
        comp.set_visible(h, False)
    assert comp.store.nseg == n_segments
    return comp, streets, garage, objs, insts


def _views(W, H, depth, which):
    """Camera-to-world poses inside the world: mid-street looking along it, across it, back, and from its far end."""
    poses = {"along": _translate(0, 0, -depth / 2), "across": _translate(2, 0, -depth / 2, np.pi / 2),
             "back": _translate(-3, 0.5, -depth / 2, np.pi), "diag": _translate(5, 1, -depth / 4, np.pi / 5),
             "end": _translate(0, 1.0, -depth + 2), "left": _translate(-10, 0, -depth / 3, -np.pi / 2),
             "up": _translate(0, 0, -depth / 2, 0.1), "start": _translate(0, 1.5, -1, np.pi)}
    proj = synth.camera_batch(W, H, [0])[0][0]
    view = np.stack([poses[w] for w in which]).astype(np.float32)
    return synth.total_matrix(np.repeat(proj[None], len(which), 0), view)


def _raster(comp, seg_m, W, H, L, culled):
    pyr = ops.Pyramid(seg_m.shape[1], W, H, L, _dev())
    pyr.clear()
    m = torch.from_numpy(seg_m).to(_dev())
    if culled:
        ops.raster_project_segments_culled(pyr, comp.store, m)
    else:
        ops.raster_project_segments(pyr, comp.store, m)
    return pyr


def _maps(pyr):
    ops.raster_derive(pyr)
    maps = [ops.zbuf_resolve(pyr, l) for l in range(pyr.L)]
    torch.cuda.synchronize()
    return [(i.cpu().numpy(), d.cpu().numpy()) for i, d in maps]


def _check_count(comp, seg_m):
    st = comp.store
    got = ops.last_surviving_units(st)
    want = kept_units(st, seg_m)
    assert got == len(want), (got, len(want))
    return got


# --------------------------------------------------------------------------------- 1. bit-identical to the parameter table
@pytest.mark.parametrize("B", [1, 8])
def test_culled_path_equals_the_parameter_table_path(B):
    W, H, L = 256, 128, 4
    comp, streets, *_ = _world(113, np.random.default_rng(B))
    which = ["along", "across", "back", "diag", "end", "left", "up", "start"]
    groups = [[w] for w in which] if B == 1 else [which]
    total_units, populated = comp.store.nunits, 0
    for ws in groups:
        seg_m = comp.segment_matrices(_views(W, H, STREET * len(streets), ws))
        want = _raster(comp, seg_m, W, H, L, culled=False)
        got = _raster(comp, seg_m, W, H, L, culled=True)
        torch.cuda.synchronize()
        assert torch.equal(got.buf, want.buf), ws
        populated += int((got.level(0) != 0x7FFFFFFFFFFFFFFF).sum())
        n = _check_count(comp, seg_m)
        if B == 1:
            assert n < 0.75 * total_units, (ws, n, total_units)                          # the camera is inside the world
    assert populated > 0.2 * W * H * 4


# ------------------------------------------------------------------------------------ 2. thousands of segments vs the oracle
@pytest.mark.parametrize("nseg", [1000, 4096])
def test_thousands_of_instances_against_the_oracle(oracle_mod, nseg):
    W, H, L = 128, 64, 4
    comp, streets, garage, objs, insts = _world(nseg, np.random.default_rng(nseg), street_points=20_000)
    for ws in (["along"], ["across"], ["back", "diag"]):
        seg_m = comp.segment_matrices(_views(W, H, STREET * len(streets), ws))
        got = _maps(_raster(comp, seg_m, W, H, L, culled=True))
        n = _check_count(comp, seg_m)
        assert n < comp.store.nunits
        _assert_maps_equal(got, _composed_oracle(oracle_mod, comp, seg_m, W, H, L), f"{nseg} segments {ws}")
        assert (got[0][0] != 0).sum() > 0.2 * W * H * len(ws)


# ------------------------------------------------------------------------------------------------ 3. a frame where nothing survives
def test_all_culled_frame_is_empty_and_the_net_sees_empty_inputs(synth_sd):
    W, H = 128, 64
    comp, streets, garage, *_ = _world(200, np.random.default_rng(3), n_streets=2, street_points=10_000)
    proj = synth.camera_batch(W, H, [0])[0][0]
    away = _translate(0, 0, 500.0, np.pi)                              # far beyond the start, looking away from the world
    seg_m = comp.segment_matrices(synth.total_matrix(proj[None], away[None].astype(np.float32)))
    maps = _maps(_raster(comp, seg_m, W, H, 4, culled=True))
    assert ops.last_surviving_units(comp.store) == 0 and len(kept_units(comp.store, seg_m)) == 0
    for idx, dep in maps:
        assert not idx.any() and not dep.any()
    sr = SceneRenderer(comp, synth_sd, (W, H), flip_vertical=True)
    sr.model.net.precision = "fp32"
    got = sr.infer(proj, away)
    ref = _net_and_texture(synth_sd, comp.texture.texture_.detach().cpu(), 1, False, "fp32")
    inputs = {(f"uv_1d_p1_ds{l}" if l else "uv_1d_p1"): torch.zeros((1, 1, H >> l, W >> l), device=_dev()) for l in range(4)}
    inputs["id"] = 0
    with torch.no_grad():
        want = ref(inputs)
    assert float((got['output'][..., :3] - want[0].permute(1, 2, 0).flip(0)).abs().max()) < TOL_FP32
    # hiding everything gives the same empty frame
    for s in streets:
        comp.set_visible(s, False)
    comp.set_visible(garage, False)                                    # with its cars and their instances
    p, v = synth.camera_batch(W, H, [40])
    again = sr.infer(p[0], v[0])
    assert ops.last_surviving_units(comp.store) == 0
    assert float((again['output'][..., :3] - want[0].permute(1, 2, 0).flip(0)).abs().max()) < TOL_FP32


# ------------------------------------------------------------------------------------------------------------ 4. the net path
def test_infer_on_4096_segments_equals_forward_on_oracle_maps(oracle_mod, synth_sd):
    W, H = 128, 64
    comp, streets, *_ = _world(4096, np.random.default_rng(4), street_points=20_000)
    sr = SceneRenderer(comp, synth_sd, (W, H), flip_vertical=True)
    sr.model.net.precision = "fp32"
    ref = _net_and_texture(synth_sd, comp.texture.texture_.detach().cpu(), 1, False, "fp32")
    proj = synth.camera_batch(W, H, [0])[0][0]
    depth = STREET * len(streets)
    for pose in (_translate(0, 0, -depth / 2), _translate(1, 0.5, -depth / 3, np.pi / 2)):
        total = synth.total_matrix(proj[None], pose[None].astype(np.float32))
        seg_m = comp.segment_matrices(total)
        maps = _composed_oracle(oracle_mod, comp, seg_m, W, H, 4)
        inputs = {(f"uv_1d_p1_ds{l}" if l else "uv_1d_p1"): torch.from_numpy(maps[l][0][:, None]).cuda() for l in range(4)}
        inputs["id"] = 0
        got = sr.infer(proj, pose)
        assert ops.last_surviving_units(comp.store) < comp.store.nunits
        with torch.no_grad():
            want = ref(inputs)
        assert float((got['output'][..., :3] - want[0].permute(1, 2, 0).flip(0)).abs().max()) < TOL_FP32


# --------------------------------------------------------------------------------------------- 5. edits show on the next frame
def test_edits_at_scale_take_effect_on_the_next_frame(synth_sd):
    W, H = 128, 64
    rng = np.random.default_rng(5)
    comp, streets, garage, objs, insts = _world(4000, rng, street_points=20_000)
    r = SceneRenderer(comp, synth_sd, (W, H))
    proj = synth.camera_batch(W, H, [0])[0][0]
    pose = _translate(0, 0, -STREET * len(streets) / 2)
    f1 = r.infer(proj, pose)['output'].clone()
    # car k sits at x = 100 (k + 1) in the garage: these transforms put it 8 m in front of the camera
    in_front = [_translate(-100.0 * (k + 1) + 2.0 * (k - 4), -1.6, -STREET * len(streets) / 2 - 8) for k in range(N_CARS)]
    comp.set_transform(insts[1], in_front[0])                          # an instance of car 0
    for h in insts[2:600]:
        comp.set_visible(h, False)
    f2 = r.infer(proj, pose)['output']
    fresh = SceneRenderer(comp, synth_sd, (W, H)).infer(proj, pose)['output']
    torch.cuda.synchronize()
    assert torch.equal(f2, fresh) and not torch.equal(f2, f1)
    comp.add_instances(objs[3], np.stack(in_front[3:4] * 96))             # a layout change: 4096 segments
    assert comp.store.nseg == 4096
    f3 = r.infer(proj, pose)['output']
    fresh = SceneRenderer(comp, synth_sd, (W, H)).infer(proj, pose)['output']
    torch.cuda.synchronize()
    assert torch.equal(f3, fresh) and not torch.equal(f3, f2)
