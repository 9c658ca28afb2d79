"""Scene editing at scale: the culled segmented rasterizer (ops.raster_project_segments_culled, used by SceneRenderer) against the
paths a user has today, at 1920x1088 with the seeded net, arms alternated round by round in one process:
  (a) C3 (one 10M-point synth.street_scene) with K = 16 / 64 objects carved out, everything in view: culled raster vs the
      parameter-table raster (ops.raster_project_segments) on the same store; the culled frame must be bit-identical (asserted);
  (b) a 2 km street: 8 stitched 10M-point scenes, camera in the middle: culled SceneRenderer vs FrameRenderer on the same 80M
      points as one cloud (and the parameter-table raster on the composed store);
  (c) (b) plus 1024 / 4096 segments of instanced cars (16 cars of 3,000 points carved from a garage scene, instances spread
      along the street): culled SceneRenderer vs FrameRenderer on a cloud with the instances baked in.
The arms of one workload alternate round by round; workloads run one after the other (each is freed before the next is built, so
the 80M-point arms fit the card).  Per arm: raster ms (CUDA events around the raster call alone, cull included, on a cleared level-0 pyramid), infer ms (CUDA events
around each infer), the fraction of (segment, chunk) units that survive, the cull kernels' own time and the rasterizer kernel's
(torch.profiler, a separate pass), and the host time of a frame (perf_counter around segment_matrices + the visibility bytes,
and around the whole infer call before its synchronise), with the card and its power limit read in the same run.
   python scripts/bench_scene_scale.py [--rounds R] [--frames F] [--n N] [out.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from read_b200 import _lib as L, ops, synth                       # noqa: E402
from read_b200.scene_edit import SceneComposer                  # noqa: E402
from read_b200.viewer import FrameRenderer, SceneRenderer       # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=3)
ap.add_argument("--frames", type=int, default=10)
ap.add_argument("--n", type=int, default=10_000_000, help="points per street scene")
ap.add_argument("out", nargs="?")
args = ap.parse_args()

L.require_device(0)
dev = torch.device("cuda", 0)
N, W, H = args.n, 1920, 1088
DEPTH = 250.0                                                   # synth.street_scene's length: 8 scenes = 2 km
sd = synth.synth_state_dict(synth.SEED)
cams = [synth.camera_batch(W, H, [7 + f]) for f in range(args.frames)]
totals = [FrameRenderer.total_matrix(p[0], v[0]) for p, v in cams]


def translate(x, y, z, yaw=0.0):
    M = np.eye(4)
    M[:3, :3] = [[np.cos(yaw), 0, np.sin(yaw)], [0, 1, 0], [-np.sin(yaw), 0, np.cos(yaw)]]
    M[:3, 3] = [x, y, z]
    return M


def stats(ts):
    ts = np.asarray(ts)
    return {"median_ms": float(np.median(ts)), "min_ms": float(ts.min()), "max_ms": float(ts.max()), "n": int(ts.size)}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


# ---------------------------------------------------------------- (a) C3 with K objects, everything in view
def workload_a():
    xyz_c3 = synth.street_scene(N)
    tex_c3 = torch.rand((1, 8, N), generator=torch.Generator().manual_seed(synth.SEED))
    clutter0 = int(0.4 * N) + int(0.4 * N)
    per_box = (N - clutter0) // 2000
    arms = {}
    for K in (16, 64):
        comp = SceneComposer(dev)
        s = comp.add_scene(xyz_c3, tex_c3)
        for b in np.linspace(0, 1999 - 3, K).astype(int):
            comp.add_object(s, np.arange(clutter0 + b * per_box, clutter0 + (b + 3) * per_box))
        arms[f"a{K}"] = dict(comp=comp, renderer=SceneRenderer(comp, sd, (W, H)), old=True)
    return arms


# ---------------------------------------------------------------- (b) 8 stitched scenes, camera in the middle
streets = [synth.street_scene(N, seed=synth.SEED + k) for k in range(8)]
offsets = [DEPTH * (4 - k) for k in range(8)]                   # scene k spans z in [offset - 250, offset]; the camera is near 0
tex_b = torch.rand((1, 8, 8 * N), generator=torch.Generator().manual_seed(1))


def street_world():
    comp = SceneComposer(dev)
    for k in range(8):
        comp.add_scene(streets[k], tex_b[:, :, k * N:(k + 1) * N], placement=translate(0, 0, offsets[k]))
    return comp


world_xyz = np.concatenate([s + np.float32([0, 0, o]) for s, o in zip(streets, offsets)])


def workload_b():
    comp_b = street_world()
    return {"b": dict(comp=comp_b, renderer=SceneRenderer(comp_b, sd, (W, H)), old=True),
            "b_frame": dict(renderer=FrameRenderer(world_xyz, sd, tex_b, (W, H), device=dev))}


# ---------------------------------------------------------------- (c) (b) + instanced cars
rng = np.random.default_rng(7)
n_car, n_cars = 3000, 16
cars = np.concatenate([(rng.uniform(-0.5, 0.5, (n_car, 3)) * [4.0, 1.5, 2.0] + [100.0 * (k + 1), 0.75, 0.0]).astype(np.float32)
                       for k in range(n_cars)])
tex_cars = torch.rand((1, 8, cars.shape[0]), generator=torch.Generator().manual_seed(2))


def workload_c(nseg):
    arms = {}
    comp = street_world()
    garage = comp.add_scene(cars, tex_cars)
    objs = [comp.add_object(garage, np.arange(n_car * k, n_car * (k + 1)), np.eye(4)) for k in range(n_cars)]
    n_inst = nseg - 8 - 1 - n_cars
    Ms = [translate(rng.uniform(-12, 12) - 100.0 * (i % n_cars + 1), -1.6, rng.uniform(-4 * DEPTH, 4 * DEPTH),
                    rng.uniform(-np.pi, np.pi)) for i in range(n_inst + n_cars)]
    for k, o in enumerate(objs):
        comp.set_transform(o, Ms[k])
    for k in range(n_cars):
        comp.add_instances(objs[k], np.stack(Ms[n_cars + k::n_cars]))
    assert comp.store.nseg == nseg
    # the baked cloud a user builds today: every car and instance transformed into the world, descriptors copied
    baked, baked_tex = [world_xyz], [tex_b]
    for i, M in enumerate(Ms):
        k = i % n_cars
        p = cars[n_car * k:n_car * (k + 1)].astype(np.float64)
        baked.append((p @ M[:3, :3].T + M[:3, 3]).astype(np.float32))
        baked_tex.append(tex_cars[:, :, n_car * k:n_car * (k + 1)])
    arms[f"c{nseg}"] = dict(comp=comp, renderer=SceneRenderer(comp, sd, (W, H)), old=False)
    arms[f"c{nseg}_frame"] = dict(renderer=FrameRenderer(np.concatenate(baked), sd, torch.cat(baked_tex, 2), (W, H), device=dev))
    return arms


pyr = ops.Pyramid(1, W, H, 1, dev)
ref = ops.Pyramid(1, W, H, 1, dev)


def check(arms):
    """The culled raster equals the parameter-table raster where both apply; the surviving fraction of the last frame."""
    for name, arm in arms.items():
        if "comp" not in arm:
            continue
        for f in (0, args.frames - 1):
            m = torch.from_numpy(arm["comp"].segment_matrices(totals[f])).to(dev)
            pyr.clear()
            ops.raster_project_segments_culled(pyr, arm["comp"].store, m)
            if arm["old"]:
                ref.clear()
                ops.raster_project_segments(ref, arm["comp"].store, m)
                torch.cuda.synchronize()
                assert torch.equal(pyr.buf, ref.buf), f"arm {name}: culled raster differs from the parameter-table raster"
        arm["units"] = arm["comp"].store.nunits
        arm["survive"] = ops.last_surviving_units(arm["comp"].store) / arm["units"]


def raster_fn(arm, f, old):
    if "comp" not in arm:
        m = torch.from_numpy(totals[f]).reshape(1, 4, 4).to(dev)
        return lambda: ops.raster_project_sorted(pyr, arm["renderer"].store, m)
    comp = arm["comp"]
    m = torch.from_numpy(comp.segment_matrices(totals[f])).to(dev)
    vis = comp.store.visible_flags().to(dev)
    if old:
        return lambda: ops.raster_project_segments(pyr, comp.store, m)
    return lambda: ops.raster_project_segments_culled(pyr, comp.store, m, vis)


res, kernels, info, order = {}, {}, {}, []


def measure(arms):
    names = list(arms)
    order.extend(names)
    for k in names:
        res[k] = {"raster": [], "raster_old": [], "infer": [], "host": [], "infer_host": []}
    for rnd in range(args.rounds + 1):                              # round 0 warms every arm up
        for name in (names if rnd % 2 else names[::-1]):
            arm, r = arms[name], arms[name]["renderer"]
            for f in range(args.frames):
                p, v = cams[f]
                t0 = time.perf_counter()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                r.infer(p[0], v[0])
                t1 = time.perf_counter()
                b.record()
                b.synchronize()
                t_infer = a.elapsed_time(b)
                if "comp" in arm:
                    h0 = time.perf_counter()
                    arm["comp"].segment_matrices(totals[f])
                    arm["comp"].store.visible_flags().clone()
                    h1 = time.perf_counter()
                pyr.clear()
                t_raster = timed(raster_fn(arm, f, False))
                if arm.get("old"):
                    pyr.clear()
                    t_old = timed(raster_fn(arm, f, True))
                if rnd:
                    res[name]["infer"].append(t_infer)
                    res[name]["infer_host"].append((t1 - t0) * 1e3)
                    res[name]["raster"].append(t_raster)
                    if "comp" in arm:
                        res[name]["host"].append((h1 - h0) * 1e3)
                    if arm.get("old"):
                        res[name]["raster_old"].append(t_old)

    # ---------------------------------------------------------------- kernel times (a separate, profiled pass)
    for name, arm in arms.items():
        if "comp" not in arm:
            continue
        fns = [raster_fn(arm, f, False) for f in range(args.frames)]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for fn in fns:
                pyr.clear()
                fn()
            torch.cuda.synchronize()
        acc = {}
        for e in prof.events():
            for key in ("seg_cull_kernel", "seg_compact_kernel", "raster_table_kernel"):
                if key in e.name:
                    acc.setdefault(key, []).append(e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3)
        kernels[name] = {k: stats(v) for k, v in acc.items()}

    for name, arm in arms.items():
        info[name] = ({"segments": arm["comp"].store.nseg, "units": arm["units"], "surviving_fraction": arm["survive"]}
                      if "comp" in arm else {"points": int(arm["renderer"].xyz.shape[0])})


for build in (workload_a, workload_b, lambda: workload_c(1024), lambda: workload_c(4096)):
    arms = build()
    check(arms)
    measure(arms)
    del arms
    torch.cuda.synchronize()
    torch.cuda.empty_cache()

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except Exception as e:                                          # noqa: BLE001
    card = f"{torch.cuda.get_device_name(0)} (power limit unavailable: {e})"
out = {"card": card, "points_per_scene": N, "viewport": [W, H], "rounds": args.rounds, "frames_per_round": args.frames, "arms": {}}
for name in order:
    r = res[name]
    row = {"raster": stats(r["raster"]), "infer": stats(r["infer"]), "infer_call_host": stats(r["infer_host"]), **info[name]}
    if r["host"]:
        row.update(host=stats(r["host"]), kernels=kernels[name])
    if r["raster_old"]:
        row["raster_parameter_table"] = stats(r["raster_old"])
    out["arms"][name] = row
print(json.dumps(out, indent=1))
if args.out:
    with open(args.out, "w") as fh:
        json.dump(out, fh, indent=1)
