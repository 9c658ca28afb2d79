"""train_precision='bf16_all' (no GPU): which conv goes where, the flag, the argument checks of the new backward entry points
(weight gradient for 1x1 / stride-2 convs, stride-2 input gradient and its filter packing, 1x1 input-gradient packing), and the
TMA-kernel layers the 21 1x1 and stride-2 convs need for their [f | m] recompute and input gradients."""
import argparse
import ctypes

import pytest
import torch

from read_b200 import _lib, blocks
from read_b200.pipeline import TexturePipeline
from read_b200.unet import UNet, GatedConv, layer_table

SINGLE = ({"feat_extract.0", "feat_extract.5"} | {f"SCM{i}.main.{j}" for i in range(3) for j in (0, 2)}
          | {f"AFFs.{i}.conv.1" for i in range(3)} | {f"FAM{i}.merge" for i in range(3)})
BLOCKS = {f"{s}.{i}.layers.{r}.main.{j}" for s in ("Encoder", "Decoder") for i in range(4) for r in range(4) for j in (0, 1)}
NEW = ({f"feat_extract.{i}" for i in (1, 2, 3, 4, 6, 7)} | {f"Convs.{i}" for i in range(3)}
       | {f"AFFs.{i}.conv.0" for i in range(3)} | {f"SCM{i}.{n}" for i in range(3) for n in ("main.1", "main.3", "conv")})
SOURCES = {**{f"AFFs.{i}.conv.0": 4 for i in range(3)}, **{f"Convs.{i}": 2 for i in range(3)}}


def test_bf16_all_routing_sends_each_conv_through_one_call(monkeypatch):
    """A spy stands in for the CUDA Function: no conv through GatedConv.forward, the 21 1x1 / stride-2 convs through
    gated_conv_srcs (AFFs.*.conv.0 with 4 sources, Convs.* with 2, every other one with 1), the 14 single 3x3 stride-1 convs
    through gated_conv, the 64 block convs through res_stack (8 convs a call); each conv once, and every used parameter gets a
    gradient."""
    assert len(SINGLE) == 14 and len(BLOCKS) == 64 and len(NEW) == 21
    net = UNet().eval()
    net.train_precision = 'bf16_all'
    names = {id(m): n for n, m in net.named_modules()}
    orig = GatedConv.forward
    torch_calls, single_calls, stack_calls, new_calls = [], [], [], {}

    def spy_forward(self, x):
        torch_calls.append(names[id(self)])
        return orig(self, x)

    def spy_apply(mods, n_src, per_item, *tensors):
        xs, residual, params = tensors[:n_src], tensors[n_src], tensors[n_src + 1:]
        assert len(params) == 6 * len(mods) and params[0] is mods[0].block['conv_f'].weight and not per_item
        if len(mods) == 8:
            for m in mods:
                stack_calls.append(names[id(m)])
            x = xs[0]
            for r in range(0, 8, 2):
                x = orig(mods[r + 1], orig(mods[r], x)) + x
            return x
        mod, = mods
        name = names[id(mod)]
        if (mod.k, mod.stride) == (3, 1):
            single_calls.append(name)
        else:
            assert name not in new_calls, name
            new_calls[name] = n_src
        y = orig(mod, torch.cat(xs, 1) if n_src > 1 else xs[0])
        return y if residual is None else y + residual

    monkeypatch.setattr(GatedConv, 'forward', spy_forward)
    monkeypatch.setattr(blocks.ConvChainFn, 'apply', spy_apply)
    g = torch.Generator().manual_seed(0)
    xs = [torch.rand((1, 8, 32 >> l, 32 >> l), generator=g) for l in range(4)]
    out = net(*xs)
    assert out.shape == (1, 3, 32, 32)
    out.mean().backward()
    assert torch_calls == []
    assert set(new_calls) == NEW
    assert new_calls == {n: SOURCES.get(n, 1) for n in NEW}
    assert len(single_calls) == len(set(single_calls)) == 14 and set(single_calls) == SINGLE
    assert len(stack_calls) == len(set(stack_calls)) == 64 and set(stack_calls) == BLOCKS
    for n, p in net.named_parameters():
        if not n.startswith("ConvsOut"):
            assert p.grad is not None, n


def test_bf16_all_flag_parses_and_fp32_stays_the_default():
    ap = argparse.ArgumentParser()
    TexturePipeline().export_args(ap)
    assert ap.parse_args(['--net_train_precision', 'bf16_all']).net_train_precision == 'bf16_all'
    assert ap.parse_args([]).net_train_precision == 'fp32'
    assert UNet().train_precision == 'fp32'
    with pytest.raises(SystemExit):
        ap.parse_args(['--net_train_precision', 'bf16_most'])
    net = UNet().eval()
    net.train_precision = 'bf16_most'
    with pytest.raises(ValueError, match="train_precision"):
        net(*[torch.rand((1, 8, 32 >> l, 32 >> l)) for l in range(4)])


def test_gated_conv_srcs_rejects_what_it_does_not_run():
    with pytest.raises(ValueError, match="feat_extract.1.*even"):
        blocks.gated_conv_srcs(GatedConv(32, 64, 3, 2, True).eval(), [torch.zeros(1, 32, 10, 9)], "feat_extract.1")
    with pytest.raises(ValueError, match="gated_conv"):
        blocks.gated_conv_srcs(GatedConv(32, 64, 3, 1, True).eval(), [torch.zeros(1, 32, 8, 8)])
    with pytest.raises(ValueError, match="multiple of 32"):
        blocks.gated_conv_srcs(GatedConv(72, 64, 1, 1, True).eval(), [torch.zeros(1, 8, 8, 8), torch.zeros(1, 64, 8, 8)])
    with pytest.raises(RuntimeError, match="eval"):
        blocks.gated_conv_srcs(GatedConv(32, 64, 1, 1, True), [torch.zeros(1, 32, 8, 8)])
    with pytest.raises(RuntimeError, match="CUDA"):
        blocks.gated_conv_srcs(GatedConv(32, 64, 4, 2, True).eval(), [torch.zeros(1, 32, 8, 8)])


def test_padded_channels():
    assert [blocks.padded_channels(c) for c in (3, 16, 32, 56, 64, 120, 128, 248, 256)] == [16, 16, 32, 64, 64, 128, 128, 256, 256]
    # every 3x3 conv of the net runs at max(C, 16): the RGB output conv (C = 3) at 16, every other one at its own C
    rows = [(name, cout) for name, cin, cout, k, s, _ in layer_table() if k == 3]
    assert {cout for _, cout in rows} == {3, 16, 32, 64, 128, 256}
    for name, cout in rows:
        assert blocks.padded_channels(cout) == max(cout, 16), name


P, ODD = 0x1000, 0x1008


def _err():
    return _lib.load().read_last_error()


def test_conv_wgrad_arguments():
    lib = _lib.load()
    # every (k, stride) of the 21 convs and every channel pair they have passes to the alignment check, before any launch
    for name, cin, cout, k, s, _ in layer_table():
        if name in NEW:
            C = blocks.padded_channels(cout)
            for cs in _sources(name, cin):
                assert lib.read_conv_wgrad(ODD, P, 2, 8 * s, 6 * s, 8, 6, C, cs, k, s, P, P, None) == -1
                assert b"16B aligned" in _err(), (cin, cout, k, s, _err())
    assert lib.read_conv_wgrad(P, P, 1, 8, 8, 8, 8, 32, 32, 1, 1, None, P, None) == -1 and b"null pointer" in _err()
    assert lib.read_conv_wgrad(P, P, 0, 8, 8, 4, 4, 32, 32, 3, 2, P, P, None) == -1 and b"bad shape" in _err()
    for k, s in ((4, 1), (1, 2), (2, 2), (3, 3), (5, 1)):
        assert lib.read_conv_wgrad(ODD, P, 1, 8, 8, 8 // s, 8 // s, 32, 32, k, s, P, P, None) == -1, (k, s)
        assert b"is not one of" in _err()
    assert lib.read_conv_wgrad(ODD, P, 1, 9, 8, 4, 4, 32, 32, 3, 2, P, P, None) == -1 and b"even input" in _err()
    assert lib.read_conv_wgrad(ODD, P, 1, 8, 8, 8, 8, 32, 32, 3, 2, P, P, None) == -1 and b"even input" in _err()
    assert lib.read_conv_wgrad(ODD, P, 1, 8, 8, 4, 4, 32, 32, 1, 1, P, P, None) == -1 and b"does not match" in _err()
    for cout, cin in ((56, 32), (96, 64), (32, 48), (32, 24)):
        assert lib.read_conv_wgrad(ODD, P, 1, 8, 8, 8, 8, cout, cin, 1, 1, P, P, None) == -1, (cout, cin)
        assert b"Cin must be 8, 16 or a multiple of 32" in _err()


def test_stride2_dgrad_arguments():
    lib = _lib.load()
    for k, cin, cout in ((3, 32, 64), (3, 64, 128), (3, 128, 256), (4, 64, 32), (4, 128, 64), (4, 256, 128)):
        assert lib.read_conv_dgrad_s2(ODD, P, 2, 5, 7, cout, cin, k, P, None) == -1
        assert b"16B aligned" in _err(), (k, cin, cout, _err())
    assert lib.read_conv_dgrad_s2(P, None, 2, 5, 7, 64, 32, 3, P, None) == -1 and b"null pointer" in _err()
    assert lib.read_conv_dgrad_s2(P, P, 2, 0, 7, 64, 32, 3, P, None) == -1 and b"bad shape" in _err()
    for k in (1, 2, 5):
        assert lib.read_conv_dgrad_s2(ODD, P, 2, 5, 7, 64, 32, k, P, None) == -1 and b"k must be 3 or 4" in _err()
    for cin, cout in ((16, 64), (48, 64), (32, 56), (32, 96), (8, 32)):
        assert lib.read_conv_dgrad_s2(ODD, P, 2, 5, 7, cout, cin, 3, P, None) == -1, (cin, cout)
        assert b"Cin must be a multiple of 32" in _err()
    assert lib.read_pack_weights_dgrad_s2(P, None, 64, 32, 3, P, None) == -1 and b"null pointer" in _err()
    assert lib.read_pack_weights_dgrad_s2(P, P, 64, 32, 2, P, None) == -1 and b"k must be 3 or 4" in _err()
    assert lib.read_pack_weights_dgrad_s2(P, P, 64, 48, 3, P, None) == -1 and b"multiple of 32" in _err()


def test_1x1_dgrad_packing_arguments():
    lib = _lib.load()
    f = lib.read_pack_weights_tc_dgrad1x1
    assert f(P, P, 32, 480, 0, 32, None, None) == -1 and b"null pointer" in _err()
    for c0, cn, cin in ((0, 48, 480), (0, 256, 256), (0, 8, 8), (448, 64, 480), (-32, 32, 480), (0, 96, 128)):
        assert f(P, P, 32, cin, c0, cn, P, None) == -1, (c0, cn, cin)
        assert b"the slice must lie in the input" in _err()
    for cout in (56, 120, 8, 96):
        assert f(P, P, cout, 64, 0, 64, P, None) == -1 and b"Cout must be" in _err(), cout


def _desc(srcs, cout, k=1, stride=1, H=40, W=40, raw=True, residual=False):
    d = _lib.ReadConvDesc()
    d.act_dtype, d.n_src = _lib.ACT_BF16, len(srcs)
    for i, c in enumerate(srcs):
        d.src[i].ptr, d.src[i].C, d.src[i].H, d.src[i].W = 0x1000, c, H, W
        d.src[i].mode, d.src[i].factor = _lib.SRC_IDENTITY, 1
    pad = (k - 1) // 2
    d.B, d.Hin, d.Win, d.Cin = 2, H, W, sum(srcs)
    d.Hout, d.Wout, d.Cout = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1, cout
    d.k, d.stride, d.pad = k, stride, pad
    d.out_mode = _lib.OUT_RAW_NHWC if raw else _lib.OUT_NHWC
    if residual:
        d.residual = 0x2000
    return d


def _sources(name, cin):
    if name.startswith("AFFs"):
        return [32, 64, 128, 256]
    if name.startswith("Convs"):
        return [cin // 2, cin // 2]
    return [cin]


def test_tma_kernel_takes_every_layer_of_the_new_convs():
    """For each of the 21 convs: the forward launch, the RAW [f | m] recompute (one plan, or one per 64 output channels for a 1x1
    conv wider than 64) and every 1x1 input-gradient plan (per source, per 128 channels, 16 channels padded to 32)."""
    lib = _lib.load()
    ok = lambda d: lib.read_conv_tc_supported(ctypes.byref(d))
    n = 0
    for name, cin, cout, k, s, _ in layer_table():
        if name not in NEW:
            continue
        n += 1
        C, srcs = blocks.padded_channels(cout), _sources(name, cin)
        assert ok(_desc(srcs, C, k, s, raw=False)) == 1, name
        assert ok(_desc(srcs, C if k != 1 else min(C, 64), k, s)) == 1, name
        if k == 1:
            for cs in srcs:
                for a in range(0, cs, 128):
                    assert ok(_desc([2 * C], max(min(128, cs - a), 32) // 2)) == 1, (name, cs, a)
    assert n == 21
    # a stride-2 RAW plan takes no residual, and a RAW 1x1 plan still stops at Cout 64
    assert ok(_desc([64], 64, 3, 2, residual=True)) == 0
    assert ok(_desc([64], 32, 4, 2, residual=True)) == 0
    assert ok(_desc([128], 128)) == 0
    assert lib.read_tc_weight_elems(16, 64, 1) == 64 * 32          # the padded dgrad plan of SCM2.main.1 (16 channels -> N = 32)
