"""Per-item train-mode BatchNorm (UNet.train_batchnorm = 'per_item') without a GPU: the semantics in float64 on torch (one batched
call == B single-item calls), which path each conv takes, NetAndTexture's batched train-mode call, the per-item pixel check, the
argument checks of the per-item entry points (all before any launch) and the CLI flag."""
import argparse
import copy

import pytest
import torch
import torch.nn as nn

from read_b200 import _lib, blocks, unet as unet_mod
from read_b200.compose import NetAndTexture
from read_b200.pipeline import TexturePipeline
from read_b200.unet import UNet, GatedConv

from test_train_bn_host import BLOCKS, NEW, SINGLE


def _inputs(B, S, gen, dtype=torch.float32):
    return [torch.rand((B, 8, S >> l, S >> l), generator=gen, dtype=dtype) for l in range(4)]


def _rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300))


def test_per_item_fp32_in_float64_equals_single_item_calls():
    """One batched call of 3 items == 3 calls of one item each (the per-item loop of a deep copy): output, loss, every gradient and
    every running statistic, at 64x64 in float64, where only the convs' rounding at B = 3 against B = 1 differs."""
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(1)
    net = UNet().double().train()
    with torch.no_grad():                                   # non-trivial affine parameters and running statistics
        for m in net.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
                m.running_mean.uniform_(-0.1, 0.1)
                m.running_var.uniform_(0.5, 2.0)
    ref = copy.deepcopy(net)
    net.train_batchnorm = 'per_item'
    xs = [x.requires_grad_() for x in _inputs(3, 64, gen, torch.float64)]
    xr = [x.detach().clone().requires_grad_() for x in xs]
    w = torch.rand((3, 3, 64, 64), generator=gen, dtype=torch.float64)

    out = net(*xs)
    loss = (out * w).sum()
    loss.backward()
    outs = [ref(*[x[i:i + 1] for x in xr]) for i in range(3)]
    out_r = torch.cat(outs)
    loss_r = sum((o * w[i:i + 1]).sum() for i, o in enumerate(outs))
    loss_r.backward()

    assert _rel(out, out_r) < 1e-10
    assert abs(loss.item() - loss_r.item()) / abs(loss_r.item()) < 1e-10
    for x, y in zip(xs, xr):
        assert _rel(x.grad, y.grad) < 1e-10
    pr = dict(ref.named_parameters())
    for n, p in net.named_parameters():
        if pr[n].grad is None:                              # ConvsOut.* are unused by forward
            assert p.grad is None, n
            continue
        assert _rel(p.grad, pr[n].grad) < 1e-10, n
    br = dict(ref.named_buffers())
    for n, b in net.named_buffers():
        if n.endswith("num_batches_tracked"):
            assert int(b) == int(br[n]), n
        else:
            assert _rel(b, br[n]) < 1e-10, n
    assert int(net.get_submodule("Encoder.0.layers.0.main.0.block.norm").num_batches_tracked) == 3


def _spy_run(monkeypatch, tp, tb, B=3):
    """The net in train() under ``tp`` / ``tb``, with spies standing in for the CUDA Function and the per-item torch path; returns
    the convs each path saw and the batch sizes F.batch_norm was called with."""
    net = UNet().train()
    net.train_precision, net.train_batchnorm = tp, tb
    names = {id(m): n for n, m in net.named_modules()}
    orig, orig_item, orig_bn = GatedConv.forward, unet_mod.gated_conv_per_item, torch.nn.functional.batch_norm
    seen = {k: [] for k in ("torch", "torch_item", "single", "multi", "stack", "single_item", "multi_item", "stack_item", "bn")}

    def spy_forward(self, x):
        seen["torch"].append(names[id(self)])
        return orig(self, x)

    def spy_item(mod, x):
        seen["torch_item"].append(names[id(mod)])
        return orig_item(mod, x)

    def spy_bn(x, *a, **kw):
        seen["bn"].append(x.shape[0])
        return orig_bn(x, *a, **kw)

    def spy_apply(mods, n_src, per_item, *tensors):
        xs, residual = tensors[:n_src], tensors[n_src]
        assert all(m.block['norm'].training for m in mods) and len(tensors) == n_src + 1 + 6 * len(mods)
        f, tag = (orig_item, "_item") if per_item else (orig, "")
        if len(mods) == 8:
            for m in mods:
                seen["stack" + tag].append(names[id(m)])
            x = xs[0]
            for r in range(0, 8, 2):
                x = f(mods[r + 1], f(mods[r], x)) + x
            return x
        mod, = mods
        seen[("single" if (mod.k, mod.stride) == (3, 1) else "multi") + tag].append(names[id(mod)])
        y = f(mod, torch.cat(xs, 1) if n_src > 1 else xs[0])
        return y if residual is None else y + residual

    monkeypatch.setattr(GatedConv, 'forward', spy_forward)
    monkeypatch.setattr(unet_mod, 'gated_conv_per_item', spy_item)
    monkeypatch.setattr(torch.nn.functional, 'batch_norm', spy_bn)
    monkeypatch.setattr(blocks.ConvChainFn, 'apply', spy_apply)
    out = net(*_inputs(B, 32, torch.Generator().manual_seed(0)))
    out.mean().backward()
    return seen


def _once(names, want):
    return len(names) == len(set(names)) == len(want) and set(names) == want


def test_per_item_bf16_all_runs_every_conv_with_per_item_statistics(monkeypatch):
    seen = _spy_run(monkeypatch, 'bf16_all', 'per_item')
    assert _once(seen["stack_item"], BLOCKS) and _once(seen["single_item"], SINGLE) and _once(seen["multi_item"], NEW)
    assert not (seen["torch"] or seen["torch_item"] or seen["stack"] or seen["single"] or seen["multi"])


def test_per_item_bf16_normalises_the_21_torch_convs_per_item(monkeypatch):
    seen = _spy_run(monkeypatch, 'bf16', 'per_item')
    assert _once(seen["stack_item"], BLOCKS) and _once(seen["single_item"], SINGLE)
    assert _once(seen["torch_item"], NEW) and seen["torch"] == [] and seen["multi_item"] == []
    assert seen["bn"] == [1] * (3 * 99)         # the spies of the kernels' paths normalise per item on torch too


def test_per_item_fp32_normalises_every_conv_per_item_on_torch(monkeypatch):
    seen = _spy_run(monkeypatch, 'fp32', 'per_item')
    assert _once(seen["torch_item"], BLOCKS | SINGLE | NEW) and seen["torch"] == []     # 99 convs: ConvsOut.* are unused
    assert seen["bn"] == [1] * (3 * 99)


def test_batch_mode_takes_no_per_item_path(monkeypatch):
    seen = _spy_run(monkeypatch, 'bf16_all', 'batch')
    assert _once(seen["stack"], BLOCKS) and _once(seen["single"], SINGLE) and _once(seen["multi"], NEW)
    assert not (seen["torch_item"] or seen["stack_item"] or seen["single_item"] or seen["multi_item"])


def test_eval_mode_ignores_per_item(monkeypatch):
    net = UNet().eval()
    net.train_batchnorm = 'per_item'
    calls = []
    monkeypatch.setattr(unet_mod, 'gated_conv_per_item', lambda m, x: calls.append(1))
    net(*[x.requires_grad_() for x in _inputs(2, 32, torch.Generator().manual_seed(0))])
    assert calls == []


def test_bad_train_batchnorm_raises():
    net = UNet().train()
    net.train_batchnorm = 'items'
    with pytest.raises(ValueError, match="train_batchnorm"):
        net(*_inputs(1, 32, torch.Generator().manual_seed(0)))


class _CountingNet(nn.Module):
    def __init__(self, tb):
        super().__init__()
        self.train_batchnorm, self.calls = tb, []

    def forward(self, *xs, **kwargs):
        self.calls.append(xs[0].shape[0])
        return xs[0][:, :3] * 1.0


class _Tex(nn.Module):
    def forward(self, idx):
        return idx.expand(-1, 8, -1, -1).float()


def _nt_run(tb, ids, temporal_average=False, train=True):
    net = _CountingNet(tb)
    m = NetAndTexture(net, {0: _Tex(), 1: _Tex()}, temporal_average=temporal_average)
    m.load_textures([0, 1])
    m.train(train)
    B = len(ids)
    inp = {("uv_1d_p1" + (f"_ds{l}" if l else "")): torch.rand(B, 1, 16 >> l, 16 >> l) for l in range(4)}
    inp["id"] = torch.tensor(ids)
    out, net_input = m(inp, return_input=True)
    assert out.shape == (B, 3, 16, 16) and net_input[0].shape == (1, 8, 16, 16)
    assert torch.equal(net_input[0], inp["uv_1d_p1"][-1:].expand(-1, 8, -1, -1)) or temporal_average
    return net.calls


def test_net_and_texture_makes_one_net_call_in_per_item_train_mode():
    assert _nt_run('per_item', [0, 0, 0]) == [3]
    assert _nt_run('batch', [0, 0, 0]) == [1, 1, 1]
    assert _nt_run('per_item', [0, 0, 0], temporal_average=True) == [1, 1, 1]
    assert _nt_run('per_item', [0, 1, 0]) == [1, 1, 1]
    assert _nt_run('batch', [0, 0, 0], train=False) == [3]


def test_per_item_needs_two_pixels_per_item():
    """At 16x16 the 1/16 level (feat_extract.7's output) has 1 pixel per item: it passes in batch mode at B >= 2 and raises in
    per-item mode, where the per-item loop raises."""
    x = torch.zeros(4, 256, 2, 2)
    m = GatedConv(256, 128, 4, 2, True)
    with pytest.raises(RuntimeError, match="CUDA"):                        # batch mode: 4 pixels
        blocks.gated_conv_srcs(m, [x], "feat_extract.7", batch_stats=True)
    with pytest.raises(ValueError, match="feat_extract.7.*more than 1 value.*per item"):
        blocks.gated_conv_srcs(m, [x], "feat_extract.7", batch_stats=True, per_item=True)
    with pytest.raises(ValueError, match="SCM1.main.2.*per item"):
        blocks.gated_conv(GatedConv(32, 32, 3, 1, True), torch.zeros(3, 32, 1, 1), batch_stats=True, name="SCM1.main.2",
                          per_item=True)
    with pytest.raises(ValueError, match="per item"):
        blocks.stack_forward([GatedConv(32, 32, 3, 1, True) for _ in range(8)], torch.zeros(3, 32, 1, 1), batch_stats=True,
                             per_item=True)
    # on torch the per-item loop's own check
    net = UNet().train()
    net.train_batchnorm = 'per_item'
    with pytest.raises(ValueError, match="more than 1 value"):
        net(*_inputs(2, 16, torch.Generator().manual_seed(0)))


P, ODD = 0x1000, 0x1008


def _err():
    return _lib.load().read_last_error()


def test_per_item_entry_points_reject_bad_arguments_before_any_launch():
    lib = _lib.load()
    stats = lambda g, it, px, C, n=None, ws=P: lib.read_bn_batch_stats_items(g, it, px, C, n or C, P, P, 1e-5, 0.1, P, P, P, P, P, P,
                                                                             ws, None)
    apply_ = lambda g, it, px, C, y=P: lib.read_bn_apply_items(g, it, px, C, P, P, None, y, None)
    reduce_ = lambda dy, it, px, C: lib.read_bn_backward_reduce_items(dy, P, it, px, C, 1, P, P, P, P, P, P, None)
    gate = lambda dy, it, px, C: lib.read_gate_backward_batch_stats_items(dy, P, it, px, C, 0, P, P, P, P, P, P, P, P, P, P, None)
    for f in (stats, apply_, reduce_, gate):
        for C in (16, 32, 64, 128, 192, 256):                               # accepted: stops at the alignment check
            assert f(ODD, 3, 100, C) == -1 and b"16B aligned" in _err(), (f, C, _err())
        for C in (0, 8, 48, 96, 320, 3):
            assert f(ODD, 3, 100, C) == -1 and b"C must be 16, 32, 64 or a multiple of 64" in _err(), (f, C, _err())
        for px in (1, 0, -5):
            assert f(P, 3, px, 64) == -1 and b"at least 2 pixels per item" in _err(), (f, px, _err())
        for it in (0, -1, 65536):
            assert f(P, it, 100, 64) == -1 and b"items must lie in" in _err(), (f, it, _err())
    assert stats(P, 3, 100, 64, ws=ODD) == -1 and b"16B aligned" in _err()
    assert apply_(P, 3, 100, 64, y=ODD) == -1 and b"16B aligned" in _err()
    assert stats(P, 3, 100, 64, n=65) == -1 and b"n_real" in _err()
    assert lib.read_bn_batch_stats_items(P, 3, 100, 64, 64, P, P, 0.0, 0.1, P, P, P, P, P, P, P, None) == -1 and b"eps" in _err()
    assert lib.read_bn_batch_stats_items(None, 3, 100, 64, 64, P, P, 1e-5, 0.1, P, P, P, P, P, P, P, None) == -1
    assert b"null pointer" in _err()
    assert lib.read_bn_workspace_bytes_items(8, 64) >= 8 * (lib.read_bn_workspace_bytes(64) - 256)
    assert lib.read_bn_workspace_bytes_items(0, 64) == -1 and lib.read_bn_workspace_bytes_items(3, 48) == -1


def test_cli_flag():
    p = argparse.ArgumentParser()
    TexturePipeline().export_args(p)
    assert p.parse_args([]).net_train_batchnorm == 'batch'
    assert p.parse_args(["--net_train_batchnorm", "per_item"]).net_train_batchnorm == 'per_item'
    with pytest.raises(SystemExit):
        p.parse_args(["--net_train_batchnorm", "crop"])
