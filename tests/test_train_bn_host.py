"""Train-mode BatchNorm on the bf16 paths (no GPU): which conv takes the batch-statistics path with the net in train(), the
rejections of what the kernels do not implement, the argument checks of the new entry points (all before any launch) and the key
of the packed-filter cache."""
import pytest
import torch

from read_b200 import _lib, blocks
from read_b200.unet import UNet, GatedConv

SINGLE = ({"feat_extract.0", "feat_extract.5"} | {f"SCM{i}.main.{j}" for i in range(3) for j in (0, 2)}
          | {f"AFFs.{i}.conv.1" for i in range(3)} | {f"FAM{i}.merge" for i in range(3)})
BLOCKS = {f"{s}.{i}.layers.{r}.main.{j}" for s in ("Encoder", "Decoder") for i in range(4) for r in range(4) for j in (0, 1)}
NEW = ({f"feat_extract.{i}" for i in (1, 2, 3, 4, 6, 7)} | {f"Convs.{i}" for i in range(3)}
       | {f"AFFs.{i}.conv.0" for i in range(3)} | {f"SCM{i}.{n}" for i in range(3) for n in ("main.1", "main.3", "conv")})


def _spy_run(monkeypatch, tp):
    """The net in train() under ``tp``, with spies standing in for the CUDA Functions; returns the convs each path saw."""
    net = UNet().train()
    net.train_precision = tp
    names = {id(m): n for n, m in net.named_modules()}
    orig = GatedConv.forward
    seen = {"torch": [], "single": [], "multi": [], "stack": []}

    def spy_forward(self, x):
        seen["torch"].append(names[id(self)])
        return orig(self, x)

    class SpySingle:
        @staticmethod
        def apply(x, residual, mod, *params):
            assert mod.block['norm'].training and len(params) == 6
            seen["single"].append(names[id(mod)])
            y = orig(mod, x)
            return y if residual is None else y + residual

    class SpyMulti:
        @staticmethod
        def apply(mod, n_src, *args):
            assert mod.block['norm'].training
            seen["multi"].append(names[id(mod)])
            xs = args[:n_src]
            return orig(mod, torch.cat(xs, 1) if n_src > 1 else xs[0])

    def spy_stack(net_, prefix, x, batch_stats=False):
        assert batch_stats
        for m in blocks.stack_convs(net_, prefix):
            assert m.block['norm'].training
            seen["stack"].append(names[id(m)])
        for r in range(net_.num_res):
            p = f"{prefix}.layers.{r}"
            x = orig(net_.get_submodule(p + ".main.1"), orig(net_.get_submodule(p + ".main.0"), x)) + x
        return x

    monkeypatch.setattr(GatedConv, 'forward', spy_forward)
    monkeypatch.setattr(blocks, 'GatedConvFn', SpySingle)
    monkeypatch.setattr(blocks, 'MultiSourceConvFn', SpyMulti)
    monkeypatch.setattr(blocks, 'res_stack', spy_stack)
    g = torch.Generator().manual_seed(0)
    out = net(*[torch.rand((1, 8, 32 >> l, 32 >> l), generator=g) for l in range(4)])
    out.mean().backward()
    return seen


def test_bf16_all_in_train_mode_sends_every_conv_through_batch_statistics(monkeypatch):
    seen = _spy_run(monkeypatch, 'bf16_all')
    assert seen["torch"] == []
    assert len(seen["stack"]) == len(set(seen["stack"])) == 64 and set(seen["stack"]) == BLOCKS
    assert len(seen["single"]) == len(set(seen["single"])) == 14 and set(seen["single"]) == SINGLE
    assert len(seen["multi"]) == len(set(seen["multi"])) == 21 and set(seen["multi"]) == NEW


def test_bf16_in_train_mode_keeps_the_21_convs_on_torch(monkeypatch):
    seen = _spy_run(monkeypatch, 'bf16')
    assert len(seen["stack"]) == 64 and len(seen["single"]) == 14 and seen["multi"] == []
    assert len(seen["torch"]) == len(set(seen["torch"])) == 21 and set(seen["torch"]) == NEW


def test_default_still_requires_eval_mode():
    x = torch.zeros(1, 32, 8, 8)
    with pytest.raises(RuntimeError, match="eval"):
        blocks.gated_conv(GatedConv(32, 32, 3, 1, True), x)
    with pytest.raises(RuntimeError, match="eval"):
        blocks.gated_conv_srcs(GatedConv(32, 64, 1, 1, True), [x])
    with pytest.raises(RuntimeError, match="eval"):
        blocks.stack_forward([GatedConv(32, 32, 3, 1, True) for _ in range(8)], x)
    # with batch_stats the checks pass and the call reaches the CUDA check
    with pytest.raises(RuntimeError, match="CUDA"):
        blocks.gated_conv(GatedConv(32, 32, 3, 1, True), x, batch_stats=True)


def _bad_norms():
    m = GatedConv(32, 32, 3, 1, True)
    m.block['norm'].momentum = None
    yield m, "momentum=None"
    m = GatedConv(32, 32, 3, 1, True)
    m.block['norm'] = torch.nn.BatchNorm2d(32, track_running_stats=False)
    yield m, "track_running_stats"
    m = GatedConv(32, 32, 3, 1, True)
    m.block['norm'] = torch.nn.BatchNorm2d(32, affine=False)
    yield m, "affine"


def test_unsupported_batchnorm_settings_raise_naming_the_layer():
    x = torch.zeros(1, 32, 8, 8)
    for m, what in _bad_norms():
        with pytest.raises(ValueError, match=f"SCM1.main.2.*{what}"):
            blocks.gated_conv(m, x, batch_stats=True, name="SCM1.main.2")
        with pytest.raises(ValueError, match=what):
            blocks.stack_forward([m] * 8, x, batch_stats=True)
    net = UNet().train()
    net.get_submodule("Encoder.2.layers.1.main.1").block['norm'].momentum = None
    with pytest.raises(ValueError, match="Encoder.2.layers.1.main.1.*momentum=None"):
        blocks.res_stack(net, "Encoder.2", torch.zeros(1, 128, 8, 8), batch_stats=True)
    # an eval-mode norm is not concerned
    m = GatedConv(32, 32, 3, 1, True).eval()
    m.block['norm'].momentum = None
    with pytest.raises(RuntimeError, match="CUDA"):
        blocks.gated_conv(m, x, batch_stats=True)


def test_one_pixel_per_channel_raises_naming_the_layer():
    with pytest.raises(ValueError, match="feat_extract.0.*more than 1 value"):
        blocks.gated_conv(GatedConv(8, 32, 3, 1, True), torch.zeros(1, 8, 1, 1), batch_stats=True, name="feat_extract.0")
    with pytest.raises(ValueError, match="feat_extract.1.*more than 1 value"):
        blocks.gated_conv_srcs(GatedConv(32, 64, 3, 2, True), [torch.zeros(1, 32, 2, 2)], "feat_extract.1", batch_stats=True)
    with pytest.raises(ValueError, match="more than 1 value"):
        blocks.stack_forward([GatedConv(32, 32, 3, 1, True) for _ in range(8)], torch.zeros(1, 32, 1, 1), batch_stats=True)
    with pytest.raises(RuntimeError, match="CUDA"):                       # 2 pixels are enough
        blocks.gated_conv_srcs(GatedConv(32, 64, 3, 2, True), [torch.zeros(2, 32, 2, 2)], batch_stats=True)


P, ODD = 0x1000, 0x1008


def _err():
    return _lib.load().read_last_error()


def test_bn_entry_points_reject_bad_arguments_before_any_launch():
    lib = _lib.load()
    stats = lambda g, px, C, n=None, ws=P: lib.read_bn_batch_stats(g, px, C, n or C, P, P, 1e-5, 0.1, P, P, P, P, None, P, P, ws, None)
    apply_ = lambda g, px, C, y=P: lib.read_bn_apply(g, px, C, P, P, None, y, None)
    reduce_ = lambda dy, px, C: lib.read_bn_backward_reduce(dy, P, px, C, 1, P, P, P, P, P, P, None)
    gate = lambda dy, px, C: lib.read_gate_backward_batch_stats(dy, P, px, C, 0, P, P, P, P, P, P, P, P, P, P, None)
    for f in (stats, apply_, reduce_, gate):
        for C in (16, 32, 64, 128, 192, 256):                               # accepted: stops at the alignment check
            assert f(ODD, 100, C) == -1 and b"16B aligned" in _err(), (f, C, _err())
        for C in (0, 8, 48, 96, 320, 3):
            assert f(ODD, 100, C) == -1 and b"C must be 16, 32, 64 or a multiple of 64" in _err(), (f, C, _err())
        for px in (1, 0, -5):
            assert f(P, px, 64) == -1 and b"at least 2 pixels" in _err(), (f, px, _err())
    assert stats(P, 100, 64, ws=ODD) == -1 and b"16B aligned" in _err()
    assert apply_(P, 100, 64, y=ODD) == -1 and b"16B aligned" in _err()
    assert stats(P, 100, 64, n=65) == -1 and b"n_real" in _err()
    assert lib.read_bn_batch_stats(P, 100, 64, 64, P, P, 0.0, 0.1, P, P, P, P, None, P, P, P, None) == -1 and b"eps" in _err()
    assert lib.read_bn_batch_stats(None, 100, 64, 64, P, P, 1e-5, 0.1, P, P, P, P, None, P, P, P, None) == -1
    assert b"null pointer" in _err()
    assert lib.read_bn_workspace_bytes(64) > 0 and lib.read_bn_workspace_bytes(48) == -1


def test_filter_cache_key_follows_the_weights():
    m = GatedConv(64, 32, 1, 1, True)
    wf, wm = m.block['conv_f'].weight, m.block['conv_m'].weight
    srcs = [torch.zeros(1, 4, 4, 32), torch.zeros(1, 4, 4, 32)]
    k0 = blocks.filter_key(m, wf, wm, 32, srcs)
    assert blocks.filter_key(m, wf, wm, 32, srcs) == k0
    with torch.no_grad():
        wf.add_(0.0)                                                       # any in-place update bumps the version
    k1 = blocks.filter_key(m, wf, wm, 32, srcs)
    assert k1 != k0
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    m(torch.rand(1, 64, 4, 4)).sum().backward()
    opt.step()
    assert blocks.filter_key(m, wf, wm, 32, srcs) != k1
    assert blocks.filter_key(m, wf, wm, 32, [torch.zeros(1, 4, 4, 64)]) != blocks.filter_key(m, wf, wm, 32, srcs)
    m2 = GatedConv(64, 32, 1, 1, True)
    m2.load_state_dict(m.state_dict())
    assert blocks.filter_key(m2, m2.block['conv_f'].weight, m2.block['conv_m'].weight, 32, srcs) != \
        blocks.filter_key(m, wf, wm, 32, srcs)
