"""Scene editing and stitching at C3 (10M-point street scene, 1920x1088, the seeded net), arms alternated round by round:
  (a) FrameRenderer on the single sorted store;
  (b) SceneRenderer, the same scene with K objects carved out of the box clutter, all transforms identity - its frame must be
      bit-identical to (a) (asserted);
  (c) as (b), every object moved every frame and a quarter of them hidden;
  (d) two 5M-point scenes stitched with a placement.
Per arm: rasterizer time (CUDA events around the raster launch alone, on a cleared level-0 pyramid) and SceneRenderer /
FrameRenderer.infer frame time (CUDA events around each call), median and range, with the card and its power limit.
   python scripts/bench_scene_edit.py [--rounds R] [--frames F] [out.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from read_b200 import _lib as L, ops, synth                       # noqa: E402
from read_b200.scene_edit import SceneComposer                  # noqa: E402
from read_b200.viewer import FrameRenderer, SceneRenderer       # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--frames", type=int, default=20)
ap.add_argument("--n", type=int, default=10_000_000)
ap.add_argument("out", nargs="?")
args = ap.parse_args()

L.require_device(0)
dev = torch.device("cuda", 0)
N, W, H = args.n, 1920, 1088
xyz = synth.street_scene(N)
tex = torch.rand((1, 8, N), generator=torch.Generator().manual_seed(synth.SEED))
sd = synth.synth_state_dict(synth.SEED)
clutter0 = int(0.4 * N) + int(0.4 * N)                          # street_scene: ground, facades, then 2000 boxes in order
per_box = (N - clutter0) // 2000
cams = [synth.camera_batch(W, H, [7 + f]) for f in range(args.frames)]
totals = [FrameRenderer.total_matrix(p[0], v[0]) for p, v in cams]


def objects_of(k):
    """k objects, each 3 boxes of the clutter spread along the street (their points are contiguous in generation order)."""
    boxes = np.linspace(0, 1999 - 3, k).astype(int)
    return [np.arange(clutter0 + b * per_box, clutter0 + (b + 3) * per_box) for b in boxes]


def moved(i, f):
    M = np.eye(4)
    M[:3, 3] = [0.5 * np.sin(0.3 * f + i), 0.0, 0.7 * np.cos(0.2 * f + i)]
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


fr = FrameRenderer(xyz, sd, tex, (W, H), device=dev)
renderers, comps = {"a": fr}, {}
for K in (16, 64):
    comp = SceneComposer(dev)
    s = comp.add_scene(xyz, tex)
    objs = [comp.add_object(s, ids) for ids in objects_of(K)]
    comps[f"b{K}"] = (comp, objs, False)
    renderers[f"b{K}"] = SceneRenderer(comp, sd, (W, H))
    comp_c = SceneComposer(dev)
    s = comp_c.add_scene(xyz, tex)
    objs_c = [comp_c.add_object(s, ids) for ids in objects_of(K)]
    for o in objs_c[::4]:
        comp_c.set_visible(o, False)
    comps[f"c{K}"] = (comp_c, objs_c, True)
    renderers[f"c{K}"] = SceneRenderer(comp_c, sd, (W, H))
half = N // 2
comp_d = SceneComposer(dev)
comp_d.add_scene(synth.street_scene(half), tex[:, :, :half])
P = np.eye(4)
P[:3, 3] = [0.0, 0.0, -250.0]                                   # the second street continues the first
comp_d.add_scene(synth.street_scene(N - half, seed=synth.SEED + 1), tex[:, :, half:], placement=P)
comps["d"] = (comp_d, [], False)
renderers["d"] = SceneRenderer(comp_d, sd, (W, H))

# (b) must equal (a) bit for bit
for arm in ("b16", "b64"):
    for f in (0, args.frames - 1):
        want = fr.infer(*[c[0] for c in cams[f]])["output"]
        got = renderers[arm].infer(*[c[0] for c in cams[f]])["output"]
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"arm {arm}: composed identity frame differs from FrameRenderer"

pyr = ops.Pyramid(1, W, H, 1, dev)


def raster_fn(arm, f):
    if arm == "a":
        m = torch.from_numpy(totals[f]).reshape(1, 4, 4).to(dev)
        return lambda: ops.raster_project_sorted(pyr, fr.store, m)
    comp = comps[arm][0]
    m = torch.from_numpy(comp.segment_matrices(totals[f])).to(dev)
    return lambda: ops.raster_project_segments(pyr, comp.store, m)


def edit(arm, f):
    comp, objs, move = comps.get(arm, (None, [], False))
    if move:
        for i, o in enumerate(objs):
            comp.set_transform(o, moved(i, f))


order = list(renderers)
raster_t = {k: [] for k in order}
frame_t = {k: [] for k in order}
for rnd in range(args.rounds + 1):                              # round 0 warms every arm up
    for arm in (order if rnd % 2 else order[::-1]):
        r = renderers[arm]
        for f in range(args.frames):
            edit(arm, f)
            p, v = cams[f]
            t_frame = timed(lambda: r.infer(p[0], v[0]))
            pyr.clear()
            t_raster = timed(raster_fn(arm, f))
            if rnd:
                frame_t[arm].append(t_frame)
                raster_t[arm].append(t_raster)

try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except Exception as e:                                          # noqa: BLE001
    card = f"{torch.cuda.get_device_name(0)} (power limit unavailable: {e})"
res = {"card": card, "points": N, "viewport": [W, H], "rounds": args.rounds, "frames_per_round": args.frames,
       "arms": {k: {"segments": (comps[k][0].store.nseg if k in comps else 1),
                    "visible_points": (N if k in ("a", "d") or k.startswith("b") else
                                       N - sum(len(ids) for ids in objects_of(int(k[1:]))[::4])),
                    "raster": stats(raster_t[k]), "infer": stats(frame_t[k])} for k in order}}
print(json.dumps(res, indent=1))
if args.out:
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
