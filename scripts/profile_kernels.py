"""Launch each hot kernel of the C3 workload exactly once (eagerly, no CUDA graph) so that
`ncu --set full -k regex:...` captures one instance of each.  Usage:
    ncu --set full --clock-control none --import-source on -k regex:"raster_project|gather_kernel|gated_conv" \
        -o prof python scripts/profile_kernels.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from read_b200 import synth, ops, _lib as L          # noqa: E402
from read_b200.engine import UNetEngine              # noqa: E402

W, H, LEVELS, N = 1920, 1088, 4, 10_000_000
LAYERS = sys.argv[1].split(",") if len(sys.argv) > 1 else [
    "Encoder.0.layers.0.main.0", "Encoder.1.layers.0.main.0", "Encoder.2.layers.0.main.0", "Encoder.3.layers.0.main.0",
    "AFFs.0.conv.0", "feat_extract.1", "feat_extract.0", "Convs.2"]

dev = torch.device("cuda", 0)
torch.cuda.set_device(0)
lib = L.load()
xyz = torch.from_numpy(synth.street_scene(N)).to(dev)
proj, view = synth.camera_batch(W, H, [7])
m = torch.from_numpy(synth.total_matrix(proj, view)).to(dev)
pyr = ops.Pyramid(1, W, H, LEVELS, dev)
pyr.clear()
tex = torch.rand((N, 8), device=dev)
eng = UNetEngine(synth.synth_state_dict(synth.SEED), 1, H, W, dev, precision="bf16", use_graph=False)
store = ops.SortedPoints(xyz)                     # scene load (torch ops, not profiled kernels of ours)
torch.cuda.synchronize()
ops.raster_project_sorted(pyr, store, m)          # the frame path's rasterizer
ops.pyramid_resolve_gather(tex, pyr, eng.inputs, L.FEAT_NHWC_BF16, reset_level0=True)
torch.cuda.synchronize()
sp = L.stream_ptr()
by_name = {ly.name: ly for ly in eng.layers}
for name in LAYERS:
    L.check(lib.read_conv_plan_launch(by_name[name].plan, sp))
torch.cuda.synchronize()
print("profiled layers:", LAYERS, eng.impl_histogram())
