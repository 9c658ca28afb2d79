"""Record what the reference's own CUDA rasterizer (pcpr.forward, compiled from its unmodified sources into oracle/_ref/ by
oracle/build_ref.py) returns on the two scenes of tests/test_gpu_reference_kernel.py, so that test runs without the reference.

Needs a GPU and oracle/_ref/pcpr*.so:

    python tests/golden/make_ref_pcpr_golden.py [OUT_DIR]      # default: tests/golden

The scenes are regenerated from their seeds by the test; only the reference's outputs are stored.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def collision_free_scene():
    """One point per pixel centre of a 64x48 image (identity matrix: u = W(x+1)/2), random depths, shuffled ids; id 0 off-screen."""
    W, H = 64, 48
    ys, xs = np.mgrid[0:H, 0:W]
    x = (xs.ravel() + 0.5) / W * 2 - 1
    y = 1 - (ys.ravel() + 0.5) / H * 2
    rng = np.random.default_rng(0)
    z = rng.uniform(-0.9, 0.9, x.size)
    xyz = np.stack([x, y, z], 1).astype(np.float32)[rng.permutation(x.size)]
    xyz = np.concatenate([np.full((1, 3), 9, np.float32), xyz])
    return xyz, np.eye(4, dtype=np.float32)[None], W, H


def dense_scene():
    from gpu_util import scene_and_cams
    xyz, M = scene_and_cams(300_000, 128, 96, [0], depth=60.0)
    return xyz, M, 128, 96


SCENES = {"ref_pcpr_collision_free": collision_free_scene, "ref_pcpr_dense": dense_scene}


def main():
    from oracle import build_ref
    ref = build_ref.load()
    assert ref is not None, "oracle/_ref/pcpr*.so not built"
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden")
    os.makedirs(out_dir, exist_ok=True)
    for name, scene in SCENES.items():
        xyz, M, W, H = scene()
        ri, rd = ref.forward(torch.from_numpy(xyz), torch.from_numpy(M), W, H, 512)
        # the dense scene's index map is not stored: the reference's winner there depends on thread timing
        arrays = dict(index=ri.numpy(), depth=rd.numpy()) if name == "ref_pcpr_collision_free" else dict(depth=rd.numpy())
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **arrays)
        print(name, tuple(ri.shape), file=sys.stderr)


if __name__ == "__main__":
    main()
