"""Cost of the point-cloud views (FrameRenderer.render_points) on the C3 frame: 10 M points of synth.street_scene, 1920x1088, one view.

    python scripts/bench_point_views.py [--reps 3] [--iters 30] [--k 20] [--out DIR]

Arms, alternated round by round (--reps rounds), each the median of --iters samples per round:
  infer      FrameRenderer.infer (the neural frame): CUDA events around one call, host work included;
  call       render_points in each mode: CUDA events around one call (clear + raster + shade with all its host work: argument
             checks, camera upload, descriptor, output allocation);
  raster     clear + the 1-pixel sorted-store raster of the view's 1-level z-buffer alone: CUDA events around --k back-to-back
             pairs, divided by --k (the device time; the host enqueues far faster than the raster runs);
  shade      the shading kernel alone: --k read_point_view launches with a descriptor and output built once, captured in one
             CUDA graph, CUDA events around its replay, divided by --k (no host work inside the window).
For the shading kernel, the bytes it must move (8 B of key and 16 B of output per pixel, plus per drawn pixel the 32-byte sectors
holding the rows its mode reads) over its time, and that rate's share of the H100 SXM data-sheet 3.35 TB/s.  A separate
torch.profiler pass then reports the median device duration of --k plain point_view_kernel launches (a cross-check of
the shade arm).  Prints
and writes (summary.json under --out, default a directory under the system's temporary directory) the median and range over
rounds, with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from read_b200 import ops, point_views, synth  # noqa: E402
from read_b200.viewer import FrameRenderer  # noqa: E402

N, W, H = 10_000_000, 1920, 1088
PEAK = 3.35e12
MODES = [("color", 0), ("pca", 0), ("normals", 0), ("normals", 1), ("depth", 0), ("uv", 0), ("xyz", 0), ("label", 0)]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name(0)


def call_ms(fn, iters):
    """Median of --iters single calls, CUDA events around each (the stream is idle at the first event: host work counts)."""
    for _ in range(3):
        fn()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def window_ms(fn, iters, k):
    """Median over --iters windows of ``fn()`` (which enqueues k units of work) / k, CUDA events around each window."""
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / k)
    return float(np.median(times))


def shade_bytes(keys, mode, submode):
    """Bytes the shading kernel must move: key + output per pixel, and per drawn pixel the 32-byte sectors of its rows."""
    drawn = keys != 0x7FFFFFFFFFFFFFFF
    ids = (keys[drawn] & 0xFFFFFFFF)
    total = keys.numel() * (8 + 16)
    if mode in ("color", "pca", "label") or (mode == "normals"):
        total += 32 * ids.numel()                                     # one 16-byte row, never across a sector
    if mode in ("depth", "xyz") or (mode == "normals" and submode in (1, 3)):
        first, last = (12 * ids) // 32, (12 * ids + 11) // 32       # a 12-byte position may straddle two sectors
        total += 32 * int((last - first + 1).sum())
    return int(total), int(drawn.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--k", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="bench_point_views_")
    os.makedirs(out, exist_ok=True)
    xyz = synth.street_scene(N, depth=250.0)
    rng = np.random.default_rng(3)
    colors = rng.random((N, 3), dtype=np.float32)
    normals = rng.standard_normal((N, 3)).astype(np.float32)
    normals /= np.linalg.norm(normals, axis=1, keepdims=True)
    proj, view = synth.camera_batch(W, H, [0])
    P, V = proj[0], view[0]
    sd = synth.synth_state_dict(synth.SEED)
    tex = torch.rand((1, 8, N), generator=torch.Generator().manual_seed(2))
    fr = FrameRenderer(xyz, sd, tex, (W, H), colors=colors, normals=normals, return_net_input=False)
    total = FrameRenderer.total_matrix(P, V)
    m = torch.from_numpy(total[None]).to(fr.device)
    fr.render_points(P, V, "pca")                                     # PCA colours: once per texture version, not per frame
    pyr = fr._views.pyr
    keys = pyr.level(0).clone()                                       # the view's z-buffer, shaded alone below
    bounds = (xyz.min(0), xyz.max(0))
    surface = torch.empty((H, W, 4), dtype=torch.float32, device=fr.device)
    graphs, descs = {}, {}
    for mode, sub in MODES:
        table = point_views.table_for(mode, fr.colors, fr.normals, lambda: fr._views.pca(fr.model._texture(0).texture_))
        pts = fr.xyz if mode in ("normals", "depth", "xyz") else None
        d = descs[(mode, sub)] = point_views.view_desc(mode, sub, table, pts, total, V, *bounds, (0., 0., 0., 1.), False)
        point_views.launch(pyr, d, surface)                           # warm-up outside capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(args.k):
                point_views.launch(pyr, d, surface)
        graphs[(mode, sub)] = g

    def raster_k():
        for _ in range(args.k):
            pyr.clear()
            ops.raster_project_sorted(pyr, fr.store, m)

    res = {"infer": [], "raster": []}
    for mode, sub in MODES:
        res[f"call_{mode}{sub}"] = []
        res[f"shade_{mode}{sub}"] = []
    for _ in range(args.reps):
        res["infer"].append(call_ms(lambda: fr.infer(P, V), args.iters))
        res["raster"].append(window_ms(raster_k, args.iters, args.k))
        for mode, sub in MODES:
            res[f"call_{mode}{sub}"].append(call_ms(lambda: fr.render_points(P, V, mode, sub), args.iters))
        pyr.level(0).copy_(keys)
        for mode, sub in MODES:
            res[f"shade_{mode}{sub}"].append(window_ms(graphs[(mode, sub)].replay, args.iters, args.k))
    assert torch.equal(pyr.level(0), keys)                            # the z-buffer the raster arm rewrote is the same one
    # cross-check: device durations of the shading kernel launches (torch.profiler, a pass of its own)
    from torch.profiler import ProfilerActivity, profile
    prof_us = {}
    for mode, sub in MODES:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.k):
                point_views.launch(pyr, descs[(mode, sub)], surface)
            torch.cuda.synchronize()
        ds = [e.device_time for e in prof.events() if "point_view_kernel" in e.name]
        prof_us[f"shade_{mode}{sub}"] = float(np.median(ds)) if ds else None
    cmd = "python scripts/bench_point_views.py " + " ".join(sys.argv[1:])
    summary = {"card": card(), "command": cmd, "points": N, "size": [W, H], "arms": {}}
    for a, v in res.items():
        summary["arms"][a] = {"median_ms": float(np.median(v)), "min_ms": float(min(v)), "max_ms": float(max(v))}
    for mode, sub in MODES:
        nbytes, drawn = shade_bytes(keys, mode, sub)
        s = summary["arms"][f"shade_{mode}{sub}"]
        s["bytes"], s["drawn_pixels"] = nbytes, drawn
        s["GB_per_s"] = nbytes / (s["median_ms"] * 1e-3) / 1e9
        s["share_of_3.35TBps"] = nbytes / (s["median_ms"] * 1e-3) / PEAK
        s["profiler_median_us"] = prof_us[f"shade_{mode}{sub}"]
    for a, s in summary["arms"].items():
        extra = f"  {s['bytes'] / 1e9:.4f} GB  {s['GB_per_s']:.0f} GB/s  {100 * s['share_of_3.35TBps']:.0f}% of 3.35 TB/s" \
            f"  profiler {s['profiler_median_us']} us" if "bytes" in s else ""
        print(f"{a:16s} {s['median_ms']:.4f} ms ({s['min_ms']:.4f}-{s['max_ms']:.4f}){extra}")
    print(summary["card"])
    print(cmd)
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
