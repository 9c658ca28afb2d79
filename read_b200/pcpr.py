"""Drop-in for the reference's native module ``pcpr`` (MyRender/CloudProjection/pcpr_cuda.cpp:23-42).

    import read_b200.pcpr as pcpr
    index, depth = pcpr.forward(points[N,3] f32, total_m[B,4,4] f32, w, h, block_size)

Same contract: inputs may live on CPU or CUDA (they are moved, pcpr_cuda.cpp:29-30), they must be float and
contiguous (RuntimeError otherwise, pcpr_cuda.cpp:17-21,32-34), results are CPU float tensors
``[index[B,h,w], depth[B,h,w]]`` (point_render.cu:196-199).  ``block_size`` is accepted and ignored (the
kernel picks its own persistent launch shape).  Output is deterministic: min depth, ties -> lowest id,
empty -> 0 — the sequential semantics of DepthProject, which the reference kernel only approximates under
contention (SURVEY.md §8 a3'').
"""
import torch

from . import ops
from . import _lib as L


def forward_device(in_points, total_m, tar_width, tar_height, block_size=512):
    """Same as ``forward`` but keeps the results on the GPU (no D2H copy, no sync)."""
    L.require_device()
    dev = torch.device("cuda", torch.cuda.current_device())
    in_points = in_points.to(dev)
    total_m = total_m.to(dev)
    for name, t in (("in_points", in_points), ("total_m", total_m)):
        if not t.is_contiguous():
            raise RuntimeError(f"{name} must be contiguous")
        if t.dtype != torch.float32:
            raise RuntimeError(f"{name} must be a float tensor")
    if total_m.dim() != 3:
        raise RuntimeError("batch_size check")
    if in_points.dim() != 2 or in_points.shape[1] != 3:
        raise RuntimeError("in_points must be (num_points,3)")
    return ops.pcpr_forward_device(in_points, total_m, int(tar_width), int(tar_height))


def forward(in_points, total_m, tar_width, tar_height, block_size=512):
    idx, dep = forward_device(in_points, total_m, tar_width, tar_height, block_size)
    return [idx.cpu(), dep.cpu()]
