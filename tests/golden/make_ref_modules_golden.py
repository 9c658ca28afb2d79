"""Record the outputs of THE REFERENCE'S OWN Python modules that tests/test_oracle_pin_reference.py compares against
(UNet state-dict layout, UNet forward, PointTexture gather) in tests/golden/ref_modules.npz, so that test runs without the reference.

Needs a checkout of the reference (READ) at READ_REFERENCE_ROOT (default /root/reference); CPU only:

    python tests/golden/make_ref_modules_golden.py

Inputs are regenerated from their seeds by the test; weights come from read_b200.synth.synth_state_dict.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.environ.get("READ_REFERENCE_ROOT", "/root/reference"))
sys.modules.setdefault("imageio", types.ModuleType("imageio"))

from READ.models.unet import UNet                  # noqa: E402
from READ.models.texture import PointTexture       # noqa: E402

from read_b200 import synth                        # noqa: E402


def unet_inputs():
    g = torch.Generator().manual_seed(7)
    return [torch.rand((2, 8, 32 >> l, 48 >> l), generator=g) for l in range(5)]


def train_inputs():
    g = torch.Generator().manual_seed(11)
    return [torch.rand((1, 8, 32 >> l, 32 >> l), generator=g) for l in range(4)]


def gather_ids():
    g = torch.Generator().manual_seed(3)
    return torch.randint(0, 500, (3, 1, 9, 7), generator=g).float()


def main():
    sd = synth.synth_state_dict(synth.SEED)
    net = UNet()
    ref_sd = net.state_dict()
    keys = sorted(ref_sd)
    shapes = np.full((len(keys), 4), -1, np.int64)          # -1 pads the unused trailing dims
    for i, k in enumerate(keys):
        shapes[i, :ref_sd[k].dim()] = list(ref_sd[k].shape)
    net.load_state_dict(sd, strict=True)
    net.eval()
    with torch.no_grad():
        unet_out = net(*unet_inputs()).numpy()
        train_out = net(*train_inputs()).numpy()
    torch.manual_seed(3)
    tex = PointTexture(8, 500, init_method='rand')
    with torch.no_grad():
        gathered = tex(gather_ids()).numpy()
    np.savez_compressed(os.path.join(OUT, "ref_modules.npz"), unet_out=unet_out, train_out=train_out,
                        texture=tex.texture_.detach().numpy(), gathered=gathered, sd_keys=np.array(keys),
                        sd_shapes=shapes, sd_dtypes=np.array([str(ref_sd[k].dtype) for k in keys]))


if __name__ == "__main__":
    main()
