"""UNet.train_precision and the pipeline's --net_train_precision (no GPU): the flag parses and defaults to fp32, and the fp32
training path keeps every conv, the residual blocks included, on GatedConv.forward (torch operators)."""
import argparse

import pytest
import torch

from read_b200 import blocks
from read_b200.pipeline import TexturePipeline
from read_b200.unet import UNet, GatedConv


def _parser():
    ap = argparse.ArgumentParser()
    TexturePipeline().export_args(ap)
    return ap


def test_net_train_precision_flag_parses_and_defaults_to_fp32():
    ap = _parser()
    assert ap.parse_args([]).net_train_precision == 'fp32'
    assert ap.parse_args(['--net_train_precision', 'bf16']).net_train_precision == 'bf16'
    with pytest.raises(SystemExit):
        ap.parse_args(['--net_train_precision', 'fp16'])


@pytest.mark.parametrize("flag", [[], ['--net_train_precision', 'bf16']])
def test_create_sets_the_net_train_precision(flag):
    args = _parser().parse_args(['--n_points', '16'] + flag)
    args.inference = True
    p = TexturePipeline()
    p.create(args)
    assert p.net.train_precision == (flag[-1] if flag else 'fp32')
    assert UNet().train_precision == 'fp32'


def _inputs(size=32):
    g = torch.Generator().manual_seed(0)
    return [torch.rand((1, 8, size >> l, size >> l), generator=g) for l in range(4)]


def test_fp32_training_routes_every_block_conv_through_gatedconv_forward(monkeypatch):
    net = UNet().eval()
    called = []
    orig = GatedConv.forward

    def spy(self, x):
        called.append(self)
        return orig(self, x)

    def no_bf16(*a, **kw):
        raise AssertionError("the bf16 block path was taken with train_precision='fp32'")

    monkeypatch.setattr(GatedConv, 'forward', spy)
    monkeypatch.setattr(blocks, 'res_stack', no_bf16)
    net(*_inputs()).mean().backward()
    names = {id(m): n for n, m in net.named_modules()}
    got = [names[id(m)] for m in called]
    block_convs = {f"{s}.{i}.layers.{r}.main.{j}" for s in ("Encoder", "Decoder") for i in range(4) for r in range(4) for j in (0, 1)}
    assert block_convs <= set(got)
    assert len(got) == len(set(got)) == 99                 # the net's 99 convs (not the unused ConvsOut heads), once each
    assert not any(n.startswith("ConvsOut") for n in got)
    assert net.get_submodule("Encoder.0.layers.0.main.0").block['conv_f'].weight.grad is not None


def test_bf16_training_needs_cuda_and_a_known_precision():
    net = UNet().eval()
    net.train_precision = 'bf16'
    with pytest.raises(RuntimeError, match="CUDA"):
        net(*_inputs())
    net.train_precision = 'fp16'
    with pytest.raises(ValueError, match="train_precision"):
        net(*_inputs())
