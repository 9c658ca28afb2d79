"""Cost of point sprites on the C3 frame (10 M-point street scene, 1920x1088, L = 4).

    python scripts/bench_point_sprites.py [--reps 5] [--iters 50] [--out DIR]

Arms (alternated, --reps rounds): the input formats _p1 (the existing 1-pixel frame path), _p2, _p3, _ps8, and _p1 keys with
per-point sizes (uniform in [0.5, 4]).  Per arm, per round: the raster time (CUDA events around the rasterizer alone, median of
--iters calls; _p1 = the sorted-store kernel plus the level derive, the others = the sprite kernel, which writes every level) and
the FrameRenderer.infer time (host clock around --iters frames ending in a synchronise).  Prints and writes (summary.json under
--out, default a directory under the system's temporary directory) the median and range over rounds, with the card name and
power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from read_b200 import ops, sprites, synth  # noqa: E402
from read_b200.viewer import FrameRenderer  # noqa: E402

N, W, H, L = 10_000_000, 1920, 1088, 4
ARMS = {
    "p1": "uv_1d, uv_1d_ds1, uv_1d_ds2, uv_1d_ds3",
    "p2": "uv_1d_p2, uv_1d_p2_ds1, uv_1d_p2_ds2, uv_1d_p2_ds3",
    "p3": "uv_1d_p3, uv_1d_p3_ds1, uv_1d_p3_ds2, uv_1d_p3_ds3",
    "ps8": "uv_1d_ps8, uv_1d_ps8_ds1, uv_1d_ps8_ds2, uv_1d_ps8_ds3",
    "sizes": "uv_1d, uv_1d_ds1, uv_1d_ds2, uv_1d_ds3",
}


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def raster_ms(store, m, fmt, sized, iters):
    pyr = ops.Pyramid(1, W, H, L, m.device)
    levels = sprites.sprite_levels(fmt, L)
    one = sprites.one_pixel(levels, store.psize if sized else None)

    def draw():
        if one:
            ops.raster_project_sorted(pyr, store, m)
            ops.raster_derive(pyr)
        else:
            ops.raster_project_sprites(pyr, store, m, levels)
    for _ in range(3):
        pyr.clear()
        draw()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        pyr.clear()
        a.record()
        draw()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def infer_ms(fr, proj, view, iters):
    for _ in range(3):
        fr.infer(proj, view)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fr.infer(proj, view)
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="bench_point_sprites_")
    os.makedirs(out, exist_ok=True)
    dev = torch.device("cuda", 0)
    xyz = synth.street_scene(N, depth=250.0)
    sizes = np.random.default_rng(1).uniform(0.5, 4.0, N).astype(np.float32)
    proj, view = synth.camera_batch(W, H, [0])
    m = torch.from_numpy(synth.total_matrix(proj, view)).to(dev)
    x = torch.from_numpy(xyz).to(dev)
    stores = {False: ops.SortedPoints(x), True: ops.SortedPoints(x, point_sizes=sizes)}
    sd = synth.synth_state_dict(synth.SEED)
    tex = torch.rand((1, 8, N), generator=torch.Generator().manual_seed(2))
    frs = {a: FrameRenderer(xyz, sd, tex, (W, H), input_format=f, point_sizes=sizes if a == "sizes" else None,
                            return_net_input=False) for a, f in ARMS.items()}
    res = {a: {"raster_ms": [], "infer_ms": []} for a in ARMS}
    for _ in range(args.reps):
        for a, f in ARMS.items():
            res[a]["raster_ms"].append(raster_ms(stores[a == "sizes"], m, f, a == "sizes", args.iters))
            res[a]["infer_ms"].append(infer_ms(frs[a], proj[0], view[0], args.iters))
    summary = {"card": card(), "points": N, "size": [W, H], "arms": {}}
    for a, r in res.items():
        summary["arms"][a] = {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in r.items()}
        print(f"{a:6s} raster {summary['arms'][a]['raster_ms']['median']:.3f} ms "
              f"({summary['arms'][a]['raster_ms']['min']:.3f}-{summary['arms'][a]['raster_ms']['max']:.3f})  "
              f"infer {summary['arms'][a]['infer_ms']['median']:.3f} ms "
              f"({summary['arms'][a]['infer_ms']['min']:.3f}-{summary['arms'][a]['infer_ms']['max']:.3f})")
    print(summary["card"])
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
