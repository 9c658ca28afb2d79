"""bf16 training of the gated 3x3 convs outside the residual blocks (no GPU): which conv goes where under
train_precision='bf16', and the argument checks of the newly accepted weight-gradient and input-gradient shapes."""
import ctypes

import pytest
import torch

from read_b200 import _lib, blocks
from read_b200.unet import UNet, GatedConv

SINGLE = ({"feat_extract.0", "feat_extract.5"} | {f"SCM{i}.main.{j}" for i in range(3) for j in (0, 2)}
          | {f"AFFs.{i}.conv.1" for i in range(3)} | {f"FAM{i}.merge" for i in range(3)})
BLOCKS = {f"{s}.{i}.layers.{r}.main.{j}" for s in ("Encoder", "Decoder") for i in range(4) for r in range(4) for j in (0, 1)}
TORCH = ({f"feat_extract.{i}" for i in (1, 2, 3, 4, 6, 7)} | {f"Convs.{i}" for i in range(3)}
         | {f"AFFs.{i}.conv.0" for i in range(3)} | {f"SCM{i}.{n}" for i in range(3) for n in ("main.1", "main.3", "conv")})


def test_bf16_routing_sends_each_conv_through_one_call(monkeypatch):
    """The torch spies stand in for the CUDA Function: 21 convs through GatedConv.forward, the 14 single 3x3 stride-1 convs
    through gated_conv, the 64 block convs through res_stack (8 convs a call), each conv once, in forward and backward."""
    assert len(SINGLE) == 14 and len(BLOCKS) == 64 and len(TORCH) == 21
    net = UNet().eval()
    net.train_precision = 'bf16'
    names = {id(m): n for n, m in net.named_modules()}
    orig = GatedConv.forward
    torch_calls, single_calls, stack_calls = [], [], []

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
        assert (mod.k, mod.stride) == (3, 1) and n_src == 1, names[id(mod)]
        single_calls.append(names[id(mod)])
        y = orig(mod, xs[0])
        return y if residual is None else y + residual

    monkeypatch.setattr(GatedConv, 'forward', spy_forward)
    monkeypatch.setattr(blocks.ConvChainFn, 'apply', spy_apply)
    g = torch.Generator().manual_seed(0)
    xs = [torch.rand((1, 8, 32 >> l, 32 >> l), generator=g) for l in range(4)]
    out = net(*xs)
    assert out.shape == (1, 3, 32, 32)
    out.mean().backward()
    assert len(torch_calls) == len(set(torch_calls)) == 21 and set(torch_calls) == TORCH
    assert len(single_calls) == len(set(single_calls)) == 14 and set(single_calls) == SINGLE
    assert len(stack_calls) == len(set(stack_calls)) == 64 and set(stack_calls) == BLOCKS
    assert net.get_submodule("feat_extract.5").block['conv_f'].weight.grad is not None


def test_gated_conv_takes_3x3_stride_1_eval_convs_only():
    with pytest.raises(ValueError, match="3x3 stride-1"):
        blocks.gated_conv(GatedConv(32, 64, 3, 2, True).eval(), torch.zeros(1, 32, 8, 8))
    with pytest.raises(RuntimeError, match="eval"):
        blocks.gated_conv(GatedConv(8, 32, 3, 1, True), torch.zeros(1, 8, 8, 8))
    with pytest.raises(RuntimeError, match="CUDA"):
        blocks.gated_conv(GatedConv(8, 32, 3, 1, True).eval(), torch.zeros(1, 8, 8, 8))


def test_narrow_weight_gradient_shapes_are_accepted():
    """Cin = 8 / 16 (the descriptor pyramid) and Cout = 16 (SCM2.main.0, the padded RGB conv) pass the channel check: with a
    misaligned pointer the call stops at the alignment check that follows it, before any launch."""
    lib = _lib.load()
    p, odd = 0x1000, 0x1008
    for cout, cin in ((32, 8), (16, 8), (64, 8), (32, 16), (16, 32)):
        assert lib.read_conv3x3_wgrad(odd, p, 1, 8, 8, cout, cin, p, p, None) == -1
        assert b"16B aligned" in lib.read_last_error(), (cout, cin, lib.read_last_error())
    for cout, cin in ((16, 24), (16, 48), (24, 8), (8, 8), (48, 16)):
        assert lib.read_conv3x3_wgrad(odd, p, 1, 8, 8, cout, cin, p, p, None) == -1, (cout, cin)
        assert b"Cin must be 8, 16 or a multiple of 32" in lib.read_last_error()


def test_cin8_input_gradient_arguments():
    lib = _lib.load()
    p, odd = 0x1000, 0x1008
    for cout in (16, 32, 64):
        assert lib.read_conv3x3_dgrad_cin8(odd, p, p, 1, 8, 8, cout, p, None) == -1
        assert b"16B aligned" in lib.read_last_error(), (cout, lib.read_last_error())
    for cout in (8, 48, 128):
        assert lib.read_conv3x3_dgrad_cin8(odd, p, p, 1, 8, 8, cout, p, None) == -1, cout
        assert b"Cout must be 16, 32 or 64" in lib.read_last_error()
    assert lib.read_conv3x3_dgrad_cin8(p, p, None, 1, 8, 8, 32, p, None) == -1
    assert b"null pointer" in lib.read_last_error()
    assert lib.read_conv3x3_dgrad_cin8(p, p, p, 0, 8, 8, 32, p, None) == -1
    # the TMA kernel's dgrad packing still takes no 8-channel input: that gradient has its own kernel
    assert lib.read_pack_weights_tc_dgrad(p, p, 32, 8, p, None) == -1


def test_raw_recompute_of_the_new_shapes_is_a_tma_layer():
    """The RAW [f | m] recompute of every new shape (Cin = 8 with C = 16 / 32 / 64, the RGB conv padded to C = 16) and the input
    gradient of the padded RGB conv (Cin' = 32, Cout' = 16) are layers the TMA kernel accepts."""
    lib = _lib.load()

    def raw(cin, cout):
        d = _lib.ReadConvDesc()
        d.act_dtype, d.n_src = _lib.ACT_BF16, 1
        d.src[0].ptr, d.src[0].C, d.src[0].H, d.src[0].W = 0x1000, cin, 40, 40
        d.src[0].mode, d.src[0].factor = _lib.SRC_IDENTITY, 1
        d.B, d.Hin, d.Win, d.Cin, d.Hout, d.Wout, d.Cout = 2, 40, 40, cin, 40, 40, cout
        d.k, d.stride, d.pad = 3, 1, 1
        d.out_mode = _lib.OUT_RAW_NHWC
        return lib.read_conv_tc_supported(ctypes.byref(d))

    for cin, cout in ((8, 16), (8, 32), (8, 64), (32, 16)):
        assert raw(cin, cout) == 1, (cin, cout)
    assert lib.read_tc_weight_elems(16, 32, 3) == 9 * 32 * 32          # dgrad filters of the padded RGB conv
