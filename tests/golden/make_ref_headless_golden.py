"""Record THE REFERENCE'S OWN headless-trainer model contract (src/READ/models/compose.py: ModelAndLoss, src/READ/models/unet.py:
UNet) in tests/golden/ref_headless.npz, so that tests/test_headless_host.py can pin read_b200.headless and the step restated in the
tests without the reference:

* src ModelAndLoss on seeded im_out / target / mask, with torch's L1Loss standing in for the VGG loss: the loss dict's keys and
  values, without a mask, with use_mask and a mask, and with use_mask but mask=None;
* the src UNet (weights read_b200.synth.synth_state_dict) on a seeded 64x64 four-level input, in eval mode: the keys of its output
  dict, 'im_out', and its state_dict keys.

Needs a checkout of the reference (READ) at READ_REFERENCE_ROOT (default /root/reference); CPU only, nothing is downloaded.
src/READ/models/compose.py imports imageio without using it; a one-line stub stands in for it:

    python tests/golden/make_ref_headless_golden.py
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.environ.get("READ_REFERENCE_ROOT", "/root/reference"), "src"))
sys.modules.setdefault("imageio", types.ModuleType("imageio"))

from READ.models import compose as ref_compose    # noqa: E402
from READ.models import unet as ref_unet          # noqa: E402

from read_b200 import synth                       # noqa: E402

LOSS_SEED = 31
NET_SEED = 32


def loss_operands():
    """im_out, target [2,3,24,20] and a binary mask [2,1,24,20], the target masked as src/train.py:181-187 masks it."""
    g = torch.Generator().manual_seed(LOSS_SEED)
    im_out = torch.rand((2, 3, 24, 20), generator=g) * 1.2 - 0.1
    target = torch.rand((2, 3, 24, 20), generator=g)
    mask = (torch.rand((2, 1, 24, 20), generator=g) < 0.7).float()
    return im_out, target * mask, mask


def net_inputs():
    g = torch.Generator().manual_seed(NET_SEED)
    return [torch.rand((1, 8, 64 >> l, 64 >> l), generator=g) for l in range(4)]


class _Fixed(torch.nn.Module):
    """A model returning a fixed {'im_out'}: the loss half of ModelAndLoss on its own."""

    def __init__(self, im_out):
        super().__init__()
        self.im_out = im_out

    def forward(self, *inputs, **kwargs):
        return {'im_out': self.im_out}


def main():
    out = {}
    im_out, target, mask = loss_operands()
    cases = {"plain": (False, {}), "mask": (True, {'mask': mask}), "mask_none": (True, {'mask': None})}
    for tag, (use_mask, kw) in cases.items():
        mal = ref_compose.ModelAndLoss(_Fixed(im_out), torch.nn.L1Loss(), use_mask=use_mask)
        output, loss = mal({'id': torch.zeros(2)}, target, label=None, **kw)
        assert output['im_out'] is im_out
        out[f"loss_keys_{tag}"] = np.array(list(loss))
        for k, v in loss.items():
            out[f"loss_{tag}_{k}"] = v.detach().numpy()
            print(tag, k, float(v))
    out["im_out_operand"], out["target_operand"], out["mask_operand"] = im_out.numpy(), target.numpy(), mask.numpy()

    net = ref_unet.UNet(num_input_channels=8, num_output_channels=3, feature_scale=4, num_res=4)
    net.load_state_dict(synth.synth_state_dict(synth.SEED), strict=True)
    net.eval()
    xs = net_inputs()
    with torch.no_grad():
        res = net(*xs)
    out["net_out_keys"] = np.array(list(res))
    out["net_im_out"] = res['im_out'].numpy()
    for l, x in enumerate(xs):
        out[f"net_input_{l}"] = x.numpy()
    out["net_state_dict_keys"] = np.array(list(net.state_dict()))
    print("net", list(res), tuple(res['im_out'].shape), len(out["net_state_dict_keys"]), "state_dict keys")
    np.savez_compressed(os.path.join(OUT, "ref_headless.npz"), **out)


if __name__ == "__main__":
    main()
