"""Generate the committed golden fixtures by running THE REFERENCE'S OWN Python modules.

Run once where a checkout of the reference exists (READ_REFERENCE_ROOT, default /root/reference); CPU only:

    python tests/golden/make_golden.py

For each case: a small seeded scene + cameras -> index maps from the sequential z-buffer oracle (the
reference's rasterizer is CUDA-only and cannot execute here) -> the reference's PointTexture / NetAndTexture /
UNet (imported from the reference checkout, top-level copies, `imageio` stubbed — SURVEY.md §8c) -> RGB.
Weights come from read_b200.synth.synth_state_dict(seed) loaded into the reference UNet with strict=True, so
the fixture stores only a seed + a checksum instead of 120 MB of parameters.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ.get("READ_REFERENCE_ROOT", "/root/reference"))
sys.modules.setdefault("imageio", types.ModuleType("imageio"))

from READ.models.unet import UNet as RefUNet                      # noqa: E402
from READ.models.texture import PointTexture as RefPointTexture   # noqa: E402
from READ.models.compose import NetAndTexture as RefNetAndTexture  # noqa: E402

import oracle                                                     # noqa: E402
from read_b200 import synth                                       # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))

CASES = [
    # name, n_points, W, H, L, trajectory steps (batch), scene depth
    ("net_64x64_b1", 6000, 64, 64, 5, [3], 40.0),
    ("net_80x48_b2", 8000, 80, 48, 4, [0, 11], 40.0),
]


def main():
    torch.manual_seed(synth.SEED)
    torch.set_num_threads(os.cpu_count())
    sd = synth.synth_state_dict(synth.SEED)
    net = RefUNet()
    net.load_state_dict(sd, strict=True)
    net.eval()
    for name, n, W, H, L, ts, depth in CASES:
        xyz = synth.street_scene(n, depth=depth, seed=synth.SEED + len(name))
        proj, view = synth.camera_batch(W, H, ts)
        total_m, idx, dep = oracle.render_pyramid(xyz, proj, view, W, H, L)
        assert all(oracle.count_degenerate(xyz, m) == 0 for m in total_m)
        g = torch.Generator().manual_seed(synth.SEED)
        tex = RefPointTexture(8, n, activation='none', init_method='zeros')
        with torch.no_grad():
            tex.texture_.copy_(torch.rand((1, 8, n), generator=g))
        model = RefNetAndTexture(net, {0: tex}, 1)
        model.load_textures([0])
        model.eval()
        inputs = {f"uv_1d_p1_ds{l}" if l else "uv_1d_p1": torch.from_numpy(idx[l]) for l in range(L)}
        inputs["id"] = torch.zeros(len(ts), dtype=torch.long)
        with torch.no_grad():
            out, net_input = model(dict(inputs), return_input=True)
            feats0 = tex(torch.from_numpy(idx[0]))
        np.savez_compressed(
            os.path.join(OUT, name + ".npz"),
            xyz=xyz, proj=proj, view=view, total_m=total_m, W=W, H=H, L=L,
            texture=tex.texture_.detach().numpy(),
            seed=synth.SEED, sd_checksum=synth.state_dict_checksum(sd),
            out=out.numpy(), feat0=feats0.numpy(),
            **{f"index{l}": idx[l] for l in range(L)}, **{f"depth{l}": dep[l] for l in range(L)})
        print(name, "out", tuple(out.shape), "mean|out|", float(out.abs().mean()),
              "covered px l0", int((idx[0] > 0).sum()), "/", idx[0].size)


if __name__ == "__main__":
    main()
