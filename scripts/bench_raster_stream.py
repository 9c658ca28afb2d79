"""Sorted-store rasterizer at C3 (10M points, 1920x1088): streaming kernel (TMA ring) vs the round-1 LDG kernel, interleaved
(ABAB) so clock drift cancels; every variant is compared key for key with the unsorted render.
   python scripts/bench_raster_stream.py [out.json]"""
import os, sys, json
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from read_b200 import synth, ops, _lib as L
lib = L.load()
dev = torch.device("cuda", 0)
N, W, H = 10_000_000, 1920, 1088
x0 = torch.from_numpy(synth.street_scene(N)).to(dev)
store = ops.SortedPoints(x0)
mats = []
for t in (7, 23, 40):
    proj, view = synth.camera_batch(W, H, [t])
    mats.append(torch.from_numpy(synth.total_matrix(proj, view)).to(dev))
pyr = ops.Pyramid(1, W, H, 1, dev)


def setopt(**kw):
    for k, v in kw.items():
        L.check(lib.read_set_option(k.encode(), v))


refs = []
for m in mats:
    pyr.clear(); ops.raster_project(pyr, x0, m); torch.cuda.synchronize(); refs.append(pyr.buf.clone())
variants = [("legacy", dict(raster_stream=0, raster_occupancy=0, raster_stages=3, raster_carveout=-1)),
            ("stream 3 stages", dict(raster_stream=1, raster_occupancy=0, raster_stages=3, raster_carveout=-1)),
            ("stream 2 stages", dict(raster_stream=1, raster_occupancy=0, raster_stages=2, raster_carveout=-1)),
            ("stream 2 stages, carveout 45%", dict(raster_stream=1, raster_occupancy=0, raster_stages=2, raster_carveout=45)),
            ("stream 3 stages, carveout 65%", dict(raster_stream=1, raster_occupancy=0, raster_stages=3, raster_carveout=65)),
            ("stream 3 stages, carveout 100%", dict(raster_stream=1, raster_occupancy=0, raster_stages=3, raster_carveout=100))]
times = {k: [] for k, _ in variants}
bad = {k: 0 for k, _ in variants}
for k, o in variants:
    setopt(**o)
    for m, r in zip(mats, refs):
        pyr.clear(); ops.raster_project_sorted(pyr, store, m); torch.cuda.synchronize()
        bad[k] += int((pyr.buf != r).sum())
for rep in range(10):
    for k, o in variants:
        setopt(**o)
        pyr.clear(); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); ops.raster_project_sorted(pyr, store, mats[0]); b.record(); torch.cuda.synchronize()
        times[k].append(a.elapsed_time(b) * 1e3)
setopt(raster_stream=1, raster_occupancy=0, raster_stages=2, raster_carveout=45)
rows = []
for k, _ in variants:
    ts = sorted(times[k][2:])
    med = ts[len(ts) // 2]
    rows.append({"variant": k, "us_median": med, "us_best": ts[0], "store_GBps": 16 * N / (med * 1e-6) / 1e9, "mismatches": bad[k]})
    print(f"{k:32s}: median {med:7.1f} us  best {ts[0]:7.1f} us  {16 * N / (med * 1e-6) / 1e9:7.1f} GB/s of the 16 B/point store  mismatching keys {bad[k]}")
if len(sys.argv) > 1:
    json.dump(rows, open(sys.argv[1], "w"), indent=1)

# resolve + gather (fused) on the state the rasterizer leaves
tex = torch.rand((N, 8), device=dev)
pyr4 = ops.Pyramid(1, W, H, 4, dev)
outs = [torch.empty((1, H >> l, W >> l, 8), dtype=torch.bfloat16, device=dev) for l in range(4)]
pyr4.clear()
gts = []
for rep in range(10):
    ops.raster_project_sorted(pyr4, store, mats[0]); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); ops.pyramid_resolve_gather(tex, pyr4, outs, L.FEAT_NHWC_BF16, reset_level0=True); b.record(); torch.cuda.synchronize()
    gts.append(a.elapsed_time(b) * 1e3)
ts = sorted(gts[2:])
print(f"pyramid_resolve_gather: median {ts[len(ts)//2]:6.1f} us  best {ts[0]:6.1f} us")
