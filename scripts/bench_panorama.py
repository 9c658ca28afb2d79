"""Cost of a 360-degree panorama against a frame on the C3 scene (10 M-point street scene), and how visible its seam is.

    python scripts/bench_panorama.py [--reps 3] [--iters 20] [--out DIR]

Arms (each with its own FrameRenderer, alternated over --reps rounds):
  frame     FrameRenderer.infer at 1920x1088 (2.09 M px), the camera bench.py uses;
  panorama  FrameRenderer.infer_panorama at 360 degrees, 4096x1024 with margin 128 (4352x1024 = 4.46 M px drawn and refined),
            the camera in the middle of the street.
Per arm, per round: the raster time (CUDA events around the rasterizer and the level derive alone, median of --iters calls) and
the call time (host clock around --iters calls ending in a synchronise).  Then the seam ratio S(M) for M in 0, 64, 128, 256: the
mean |RGB(col 0) - RGB(col W-1)| over the mean |RGB(col j) - RGB(col j+1)| of the interior columns, over three headings; 1 means
the seam is no more visible than any other column boundary.  Prints and writes (summary.json under --out, default a directory
under the system's temporary directory) the median and range over rounds, with the card name and power limit read in the same
run."""
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

from read_b200 import ops, synth  # noqa: E402
from read_b200.panorama import Panorama, raster_panorama_sorted  # noqa: E402
from read_b200.viewer import FrameRenderer  # noqa: E402

N, DEPTH, W, H, L = 10_000_000, 250.0, 1920, 1088, 4
PW, PH, PM = 4096, 1024, 128
MARGINS = (0, 64, 128, 256)


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def street_view(yaw_deg=0.0):
    """Camera-to-world: eye in the middle of the street (z = -DEPTH / 2), turned by yaw_deg about y."""
    a = np.deg2rad(yaw_deg)
    m = np.eye(4)
    m[:3, :3] = [[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]]
    m[:3, 3] = (0.0, 0.0, -DEPTH / 2)
    return m.astype(np.float32)


def events_ms(draw, clear, iters):
    for _ in range(3):
        clear()
        draw()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        clear()
        a.record()
        draw()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def call_ms(call, iters):
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        call()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3 / iters


def seam_ratio(fr, pano, yaws):
    num = den = 0.0
    for y in yaws:
        rgb = fr.infer_panorama(street_view(y), pano)['output'][..., :3].double()
        num += float((rgb[:, 0] - rgb[:, -1]).abs().mean())
        den += float((rgb[:, 1:-1] - rgb[:, 2:]).abs().mean())      # boundaries j | j + 1 for j = 1 .. W - 2
    return num / den


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="bench_panorama_")
    os.makedirs(out, exist_ok=True)
    dev = torch.device("cuda", 0)
    xyz = synth.street_scene(N, depth=DEPTH)
    sd = synth.synth_state_dict(synth.SEED)
    tex = torch.rand((1, 8, N), generator=torch.Generator().manual_seed(2))
    proj, view = synth.camera_batch(W, H, [0])
    pano = Panorama(PW, PH, margin=PM)
    fr_frame = FrameRenderer(xyz, sd, tex, (W, H), return_net_input=False)
    fr_pano = FrameRenderer(xyz, sd, tex, (W, H), return_net_input=False)
    store = fr_frame.store
    m_frame = torch.from_numpy(synth.total_matrix(proj, view)).to(dev)
    m_pano = torch.from_numpy(Panorama.world_to_camera(street_view()[None])).to(dev)
    pyr_frame = ops.Pyramid(1, W, H, L, dev)
    pyr_pano = ops.Pyramid(1, pano.plane_width, PH, L, dev)

    def draw_frame():
        ops.raster_project_sorted(pyr_frame, store, m_frame)
        ops.raster_derive(pyr_frame)

    def draw_pano():
        raster_panorama_sorted(pyr_pano, store, m_pano, pano)
        ops.raster_derive(pyr_pano)

    arms = {
        "frame": (draw_frame, pyr_frame.clear, lambda: fr_frame.infer(proj[0], view[0])),
        "panorama": (draw_pano, pyr_pano.clear, lambda: fr_pano.infer_panorama(street_view(), pano)),
    }
    res = {a: {"raster_ms": [], "call_ms": []} for a in arms}
    for _ in range(args.reps):
        for a, (draw, clear, call) in arms.items():
            res[a]["raster_ms"].append(events_ms(draw, clear, args.iters))
            res[a]["call_ms"].append(call_ms(call, args.iters))
    summary = {"card": card(), "points": N, "frame": [W, H], "panorama": [PW, PH, PM],
               "pixels": {"frame": W * H, "panorama": pano.plane_width * PH}, "arms": {}}
    for a, r in res.items():
        summary["arms"][a] = {k: {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))} for k, v in r.items()}
        s = summary["arms"][a]
        print(f"{a:9s} raster {s['raster_ms']['median']:.3f} ms ({s['raster_ms']['min']:.3f}-{s['raster_ms']['max']:.3f})  "
              f"call {s['call_ms']['median']:.3f} ms ({s['call_ms']['min']:.3f}-{s['call_ms']['max']:.3f})")
    del fr_frame, fr_pano
    torch.cuda.empty_cache()
    summary["seam_ratio"] = {}
    for M in MARGINS:
        fr = FrameRenderer(xyz, sd, tex, (W, H), return_net_input=False)
        summary["seam_ratio"][M] = seam_ratio(fr, Panorama(PW, PH, margin=M), (0.0, 77.0, 200.0))
        print(f"S({M}) = {summary['seam_ratio'][M]:.3f}")
        del fr
        torch.cuda.empty_cache()
    print(summary["card"])
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
