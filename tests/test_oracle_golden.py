"""Oracle vs the committed golden fixtures (generated from the reference's own Python modules by
tests/golden/make_golden.py).  CPU only."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from read_b200 import synth

CASES = ["net_64x64_b1", "net_80x48_b2"]


@pytest.mark.parametrize("name", CASES)
def test_raster_oracle_reproduces_fixture(oracle_mod, name):
    g = load_golden(name)
    W, H, L = int(g["W"]), int(g["H"]), int(g["L"])
    total_m, idx, dep = oracle_mod.render_pyramid(g["xyz"], g["proj"], g["view"], W, H, L)
    np.testing.assert_array_equal(total_m, g["total_m"])
    for l in range(L):
        np.testing.assert_array_equal(idx[l], g[f"index{l}"])
        np.testing.assert_array_equal(dep[l], g[f"depth{l}"])


@pytest.mark.parametrize("name", CASES)
def test_gather_oracle_matches_reference_output(name):
    from oracle import unet_ref
    g = load_golden(name)
    feat = unet_ref.point_texture(torch.from_numpy(g["texture"]), torch.from_numpy(g["index0"]))
    np.testing.assert_array_equal(feat.numpy(), g["feat0"])      # pure gather: bit exact


@pytest.mark.parametrize("name", CASES)
def test_net_oracle_matches_reference_output(synth_sd, name):
    from oracle import unet_ref
    g = load_golden(name)
    assert abs(synth.state_dict_checksum(synth_sd) - float(g["sd_checksum"])) < 1e-6 * float(g["sd_checksum"]), \
        "synthetic weights differ from the ones the fixture was generated with (torch RNG changed?)"
    L = int(g["L"])
    maps = [torch.from_numpy(g[f"index{l}"]) for l in range(L)]
    with torch.no_grad():
        out = unet_ref.net_and_texture(synth_sd, torch.from_numpy(g["texture"]), maps)
    err = float((out - torch.from_numpy(g["out"])).abs().max())
    assert err < 2e-5, err      # same fp32 ops as the reference, only summation-order noise of the conv backend
