"""Pin the oracle's torch restatement and our UNet to the reference's real modules, through their outputs recorded by
tests/golden/make_ref_modules_golden.py (the reference's UNet / PointTexture run on the same seeded inputs and weights)."""
import os

import numpy as np
import torch

from conftest import GOLDEN


def _golden():
    return np.load(os.path.join(GOLDEN, "ref_modules.npz"))


def _ref_layout():
    """{state_dict key: (shape, dtype name)} of the reference UNet."""
    g = _golden()
    return {str(k): (tuple(int(d) for d in s if d >= 0), str(t)) for k, s, t in zip(g["sd_keys"], g["sd_shapes"], g["sd_dtypes"])}


def test_state_dict_keys_identical_to_reference(synth_sd):
    ref = _ref_layout()
    assert set(ref) == set(synth_sd)
    for k, (shape, _) in ref.items():
        assert tuple(shape) == tuple(synth_sd[k].shape), k
    from read_b200.unet import UNet as OurUNet
    ours = OurUNet().state_dict()
    assert list(sorted(ours)) == list(sorted(ref))
    for k, (shape, dtype) in ref.items():
        assert tuple(shape) == tuple(ours[k].shape) and dtype == str(ours[k].dtype), k
    OurUNet().load_state_dict({k: torch.zeros(shape, dtype=getattr(torch, dt.split(".")[1])) for k, (shape, dt) in ref.items()},
                              strict=True)


def test_unet_oracle_equals_reference_module(synth_sd):
    from oracle import unet_ref
    g = torch.Generator().manual_seed(7)
    H, W = 32, 48
    xs = [torch.rand((2, 8, H >> l, W >> l), generator=g) for l in range(5)]
    want = torch.from_numpy(_golden()["unet_out"])
    with torch.no_grad():
        got = unet_ref.unet_forward(synth_sd, xs)
    assert float((want - got).abs().max()) < 2e-5


def test_gather_oracle_equals_reference_module():
    from oracle import unet_ref
    gd = _golden()
    g = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 500, (3, 1, 9, 7), generator=g).float()
    got = unet_ref.point_texture(torch.from_numpy(gd["texture"]), ids)
    assert torch.equal(torch.from_numpy(gd["gathered"]), got)


def test_training_forward_of_our_unet_equals_reference(synth_sd):
    """The library (autograd) path of read_b200.unet.UNet must agree with the reference on CPU."""
    from read_b200.unet import UNet as OurUNet
    ours = OurUNet()
    ours.load_state_dict(synth_sd)
    ours.eval()
    g = torch.Generator().manual_seed(11)
    xs = [torch.rand((1, 8, 32 >> l, 32 >> l), generator=g) for l in range(4)]
    want = torch.from_numpy(_golden()["train_out"])
    got = ours(*xs)                      # grad enabled -> torch path
    assert float((want - got.detach()).abs().max()) < 2e-5
    got.sum().backward()
    assert ours.get_submodule("feat_extract.0").block["conv_f"].weight.grad is not None
