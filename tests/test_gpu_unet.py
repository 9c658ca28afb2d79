"""-m gpu: the refinement-net engine and the full pipeline vs the golden fixtures (generated from the reference's
own modules) and vs the oracle."""
import numpy as np
import pytest
import torch

from conftest import load_golden
from gpu_util import dev, psnr
from read_b200 import ops, synth, _lib as L
from read_b200.engine import UNetEngine
from read_b200.unet import UNet
from read_b200.texture import PointTexture
from read_b200.compose import NetAndTexture

pytestmark = pytest.mark.gpu

# Stated tolerances (SURVEY.md §8c, calibrated on first measurement, then frozen):
TOL_FP32 = 2e-4          # parity mode: fp32 storage + fp32 CUDA-core math vs fp32 CPU reference, max-abs
TOL_BF16 = 3e-2          # production mode: bf16 activations, tensor-core math, max-abs
PSNR_BF16 = 45.0


def _engine_out(sd, feats, precision, conv_impl="auto", graph=False):
    B, _, H, W = feats[0].shape
    eng = UNetEngine(sd, B, H, W, dev(), precision=precision, conv_impl=conv_impl, use_graph=graph)
    eng.set_inputs_nchw([f.to(dev()) for f in feats])
    out = eng.run().clone()
    torch.cuda.synchronize()
    return out.cpu(), eng


def _golden_feats(g):
    from oracle import unet_ref
    tex = torch.from_numpy(g["texture"])
    return [unet_ref.point_texture(tex, torch.from_numpy(g[f"index{l}"])) for l in range(4)]


@pytest.mark.parametrize("name", ["net_64x64_b1", "net_80x48_b2"])
def test_engine_fp32_parity_with_reference_fixture(synth_sd, name):
    g = load_golden(name)
    out, eng = _engine_out(synth_sd, _golden_feats(g), "fp32")
    assert eng.n_launches() == 99                          # one launch per BasicConv
    err = float((out - torch.from_numpy(g["out"])).abs().max())
    assert err < TOL_FP32, err


@pytest.mark.parametrize("name", ["net_64x64_b1", "net_80x48_b2"])
@pytest.mark.parametrize("conv_impl", ["generic", "tma_only", "auto"])
def test_engine_bf16_within_stated_tolerance(synth_sd, name, conv_impl):
    g = load_golden(name)
    out, eng = _engine_out(synth_sd, _golden_feats(g), "bf16", conv_impl)
    hist = eng.impl_histogram()
    if conv_impl == "auto":
        assert hist["wgmma_tma"] >= 70 and hist["generic"] == 0, hist   # every layer on tensor cores
    elif conv_impl == "tma_only":
        assert hist["wgmma_tma"] >= 70 and hist["wgmma_gather"] == 0, hist
    else:
        assert hist["wgmma_tma"] == 0 and hist["wgmma_gather"] == 0
    want = torch.from_numpy(g["out"])
    err = float((out - want).abs().max())
    assert err < TOL_BF16, err
    assert psnr(out.numpy(), want.numpy(), peak=float(want.abs().max())) > PSNR_BF16


def test_engine_graph_replay_equals_eager(synth_sd):
    g = load_golden("net_64x64_b1")
    feats = _golden_feats(g)
    a, _ = _engine_out(synth_sd, feats, "bf16", graph=False)
    b, eng = _engine_out(synth_sd, feats, "bf16", graph=True)
    assert torch.equal(a, b)
    eng.run(); eng.run()
    torch.cuda.synchronize()
    assert torch.equal(eng.output.cpu(), a)


def test_side_chain_schedule_is_bit_identical(synth_sd, monkeypatch):
    """READ_B200_SIDE_CHAIN=1 (SCM1 / SCM0 blocks on a second stream with capped grids, joined by an event; off by default): the
    same kernels in a different schedule - the captured two-stream graph and the eager run equal the single-stream output."""
    g = load_golden("net_64x64_b1")
    feats = _golden_feats(g)
    a, _ = _engine_out(synth_sd, feats, "bf16", graph=True)
    monkeypatch.setenv("READ_B200_SIDE_CHAIN", "1")
    b, eng = _engine_out(synth_sd, feats, "bf16", graph=True)
    assert getattr(eng, "_side_range", None) is not None, "the side chain was not planned"
    assert torch.equal(a, b)
    eng.run(); eng.run()
    torch.cuda.synchronize()
    assert torch.equal(eng.output.cpu(), a)
    c, _ = _engine_out(synth_sd, feats, "bf16", graph=False)
    assert torch.equal(a, c)


def test_engine_vs_oracle_larger_random_input(synth_sd):
    from oracle import unet_ref
    gen = torch.Generator().manual_seed(9)
    H, W = 96, 160
    feats = [torch.rand((1, 8, H >> l, W >> l), generator=gen) for l in range(4)]
    with torch.no_grad():
        want = unet_ref.unet_forward(synth_sd, feats)
    out32, _ = _engine_out(synth_sd, feats, "fp32")
    assert float((out32 - want).abs().max()) < TOL_FP32
    out16, _ = _engine_out(synth_sd, feats, "bf16")
    assert float((out16 - want).abs().max()) < TOL_BF16


def test_module_surface_matches_reference_fixture(synth_sd):
    """NetAndTexture(UNet, PointTexture) driven exactly like READ/gl/nn.py:113-121 (dict of index maps + id)."""
    g = load_golden("net_80x48_b2")
    L_ = int(g["L"])
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    tex = PointTexture(8, g["texture"].shape[-1])
    with torch.no_grad():
        tex.texture_.copy_(torch.from_numpy(g["texture"]))
    model = NetAndTexture(net, {0: tex}, 1)
    model.load_textures(0)
    model.cuda().eval()
    inputs = {f"uv_1d_p1_ds{l}" if l else "uv_1d_p1": torch.from_numpy(g[f"index{l}"]).cuda() for l in range(L_)}
    inputs["id"] = torch.zeros(2, dtype=torch.long)
    want = torch.from_numpy(g["out"])
    for precision, tol in (("fp32", TOL_FP32), ("bf16", TOL_BF16)):
        net.precision = precision
        with torch.no_grad():
            out, net_input = model(dict(inputs), return_input=True)
        assert tuple(out.shape) == (2, 3, 48, 80) and out.is_cuda and len(net_input) == L_
        np.testing.assert_array_equal(net_input[0].cpu().numpy(), g["feat0"][-1:])       # the last item's input, as the reference returns
        assert float((out.cpu() - want).abs().max()) < tol
    # per-item loop (different texture ids in one batch) gives the same frames as the batched pass
    tex2 = PointTexture(8, g["texture"].shape[-1])
    with torch.no_grad():
        tex2.texture_.copy_(torch.from_numpy(g["texture"]))
    model2 = NetAndTexture(net, {0: tex, 1: tex2}, 1)
    model2.load_textures([0, 1])
    model2.cuda().eval()
    inputs["id"] = torch.tensor([0, 1])
    with torch.no_grad():
        out2 = model2(dict(inputs))
    assert float((out2 - out).abs().max()) < 1e-6


def test_fused_render_path_equals_index_map_path(synth_sd):
    g = load_golden("net_64x64_b1")
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    tex = PointTexture(8, g["texture"].shape[-1])
    with torch.no_grad():
        tex.texture_.copy_(torch.from_numpy(g["texture"]))
    model = NetAndTexture(net, {0: tex}, 1)
    model.load_textures(0)
    model.cuda().eval()
    xyz = torch.from_numpy(g["xyz"]).cuda()
    M = torch.from_numpy(g["total_m"]).cuda()
    for precision, tol in (("fp32", TOL_FP32), ("bf16", TOL_BF16)):
        net.precision = precision
        out, maps = model.render(xyz, M, 64, 64, n_levels=4, want_maps=True)
        for l in range(4):
            np.testing.assert_array_equal(maps[l][0].cpu().numpy(), g[f"index{l}"][:, 0])
            np.testing.assert_array_equal(maps[l][1].cpu().numpy(), g[f"depth{l}"][:, 0])
        assert float((out.cpu() - torch.from_numpy(g["out"])).abs().max()) < tol


def test_non_multiple_of_16_is_rejected(synth_sd):
    with pytest.raises(RuntimeError, match="multiples of 16"):
        UNetEngine(synth_sd, 1, 40, 64, dev())


def test_frame_renderer_matches_ogl_infer_contract():
    """read_b200.viewer.FrameRenderer.infer == READ/gl/nn.py:123-124 (permute + alpha) on the fused render, and the
    vertical flip of viewer.py:267."""
    import numpy as np
    from read_b200 import synth
    from read_b200.viewer import FrameRenderer
    W, H, n = 128, 64, 40_000
    xyz = synth.street_scene(n, depth=60.0, seed=5)
    sd = synth.synth_state_dict(synth.SEED)
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(2))
    proj, view = synth.camera_batch(W, H, [3])
    r = FrameRenderer(xyz, sd, tex, (W, H))
    got = r.infer(proj[0], view[0])['output'].clone()
    m = torch.from_numpy(synth.total_matrix(proj, view)).cuda()
    with torch.no_grad():
        ref = r.model.render(r.xyz, m, W, H)[0].permute(1, 2, 0)
    want = torch.cat([ref, ref[:, :, :1] * 0 + 1], 2).contiguous()
    assert tuple(got.shape) == (H, W, 4) and got.is_cuda and got.dtype == torch.float32
    assert torch.equal(got, want)
    rf = FrameRenderer(xyz, sd, tex, (W, H), flip_vertical=True)
    assert torch.equal(rf.infer(proj[0], view[0])['output'], want.flip(0))
    with pytest.raises(AssertionError, match="set width 112"):
        FrameRenderer(xyz, sd, tex, (120, 64))


def _small_scene(n=60_000, W=128, H=64, ss=1):
    from read_b200 import synth
    xyz = synth.street_scene(n, depth=60.0, seed=5)
    sd = synth.synth_state_dict(synth.SEED)
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(2))
    net = UNet()
    net.load_state_dict(sd, strict=True)
    t = PointTexture(8, n)
    with torch.no_grad():
        t.texture_.copy_(tex)
    model = NetAndTexture(net, {0: t}, ss)
    model.load_textures(0)
    model.cuda().eval()
    return xyz, model


def _index_inputs(oracle_mod, xyz, W, H, pose):
    """The reference's input dict (one 'uv' key per level) from the oracle's index maps of one view."""
    from read_b200 import synth
    proj, view = synth.camera_batch(W, H, [pose])
    M, idx, _ = oracle_mod.render_pyramid(xyz, proj, view, W, H, 4)
    d = {(f"uv_1d_p1_ds{l}" if l else "uv_1d_p1"): torch.from_numpy(idx[l]).cuda() for l in range(4)}
    d["id"] = 0
    return torch.from_numpy(M).cuda(), d


@pytest.mark.parametrize("ss", [2, 3])
def test_fused_supersampling_equals_index_map_path(oracle_mod, ss):
    """NetAndTexture.ss > 1 (READ/models/compose.py:162-163, READ/gl/nn.py:100-101): pyramid rendered at ss x the viewport, every
    level reduced with F.interpolate(scale_factor=1/ss, 'bilinear').  The fused path's staging kernel must equal torch's
    interpolate on the index-map path (fp32 parity mode: same net, so the RGB agrees to fp32 rounding)."""
    W, H = 128, 64
    xyz, model = _small_scene(W=W, H=H, ss=ss)
    model.net.precision = "fp32"
    M, inputs = _index_inputs(oracle_mod, xyz, W * ss, H * ss, 3)
    with torch.no_grad():
        want, want_in = model(dict(inputs), return_input=True)
        got, got_in = model.render(torch.from_numpy(xyz).cuda(), M, W, H, return_input=True)
    assert tuple(got.shape) == (1, 3, H, W)
    for a, b in zip(got_in, want_in):
        assert tuple(a.shape) == tuple(b.shape)
        assert float((a - b).abs().max()) < 1e-6
    assert float((got - want).abs().max()) < TOL_FP32
    model.net.precision = "bf16"
    with torch.no_grad():
        got16 = model.render(torch.from_numpy(xyz).cuda(), M, W, H)
    assert float((got16 - want).abs().max()) < TOL_BF16


def test_fused_temporal_average_equals_index_map_path(oracle_mod):
    """temporal_average (compose.py:167-171): the net input of frame t is the mean of its features and frame t-1's (already
    averaged) input.  Three consecutive poses through the fused path and through the index-map path."""
    W, H = 128, 64
    xyz, model = _small_scene(W=W, H=H)
    model.net.precision = "fp32"
    model.temporal_average = True
    x = torch.from_numpy(xyz).cuda()
    outs_f, outs_i = [], []
    for pose in (1, 2, 3):
        M, inputs = _index_inputs(oracle_mod, xyz, W, H, pose)
        with torch.no_grad():
            outs_f.append(model.render(x, M, W, H))
            outs_i.append(model(dict(inputs)))
    for a, b in zip(outs_f, outs_i):
        assert float((a - b).abs().max()) < TOL_FP32
    assert float((outs_f[2] - outs_f[1]).abs().max()) > 1e-5            # the frames do differ
    # switching the option off drops the history
    model.temporal_average = False
    M, inputs = _index_inputs(oracle_mod, xyz, W, H, 3)
    with torch.no_grad():
        plain = model.render(x, M, W, H)
        model.last_input = None
        want = model(dict(inputs))
    assert float((plain - want).abs().max()) < TOL_FP32


def test_frame_renderer_options_and_net_input(oracle_mod):
    """FrameRenderer(supersampling, temporal_average) == OGL(..., supersampling, temporal_average) of READ/gl/nn.py:76-129:
    'net_input' is the list the model saw, 'output' a fresh [H,W,4] tensor per call."""
    from read_b200 import synth
    from read_b200.viewer import FrameRenderer
    W, H, n = 128, 64, 40_000
    xyz = synth.street_scene(n, depth=60.0, seed=5)
    sd = synth.synth_state_dict(synth.SEED)
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(2))
    proj, view = synth.camera_batch(W, H, [3, 4])
    r = FrameRenderer(xyz, sd, tex, (W, H), supersampling=2, temporal_average=True)
    assert r.model.ss == 2 and r.model.temporal_average is True
    a = r.infer(proj[0], view[0])
    b = r.infer(proj[1], view[1])
    assert a['output'].data_ptr() != b['output'].data_ptr()
    assert len(a['net_input']) == 4 and tuple(a['net_input'][0].shape) == (1, 8, H, W) and a['net_input'][0].dtype == torch.float32
    assert tuple(a['net_input'][3].shape) == (1, 8, H // 8, W // 8)
    # frame 0 has no history: equals the plain ss = 2 render
    r2 = FrameRenderer(xyz, sd, tex, (W, H), supersampling=2, return_net_input=False)
    c = r2.infer(proj[0], view[0])
    assert c['net_input'] is None
    assert torch.equal(c['output'], a['output'])
    assert not torch.equal(r2.infer(proj[1], view[1])['output'], b['output'])       # frame 1 is blended with frame 0


def test_index_map_surface_direct_engine_path_equals_module_path(synth_sd):
    """NetAndTexture.forward's inference shortcut (descriptors gathered from the index maps straight into the engine's NHWC inputs)
    returns exactly what the general path returns (PointTexture.forward -> UNet.forward), B = 1 and B = 2, with an activation."""
    from read_b200.compose import NetAndTexture
    from read_b200.texture import PointTexture
    from read_b200.unet import UNet
    n, H, W = 4000, 64, 96
    gen = torch.Generator().manual_seed(9)
    for act, B in (("none", 1), ("sigmoid", 2)):
        net = UNet()
        net.load_state_dict(synth_sd, strict=True)
        tex = PointTexture(8, n, activation=act)
        with torch.no_grad():
            tex.texture_.copy_(torch.rand((1, 8, n), generator=gen) * 2 - 1)
        model = NetAndTexture(net, {0: tex}, 1)
        model.load_textures(0)
        model.cuda().eval()
        inp = {"id": torch.zeros(B, dtype=torch.long)}
        for l in range(4):
            ids = torch.randint(0, n, (B, 1, H >> l, W >> l), generator=gen).float()
            inp["uv_1d_p1" + (f"_ds{l}" if l else "")] = ids.cuda()
        with torch.no_grad():
            fast = model(inp)
            assert model._direct_engine_forward({k: v for k, v in inp.items() if k != "id"}, [0] * B) is not None
            slow, _ = model(inp, return_input=True)              # kwargs -> the general path
        assert fast.shape == (B, 3, H, W)
        assert torch.equal(fast, slow)


def test_sharded_frame_stream_lookahead_single_rank(synth_sd):
    """dist.ShardedFrameStream without a process group (world 1): the rasterizer of step s+1 runs on the side stream under the net of
    step s; every step's frame equals the plain sequence raster -> resolve/gather -> net.  (2 / 4 ranks: scripts/check_sharded_render.py.)"""
    from read_b200 import dist as rdist
    n, W, H = 60_000, 128, 64
    d = dev()
    store = ops.SortedPoints(torch.from_numpy(synth.street_scene(n, depth=60.0, seed=5)).to(d))
    tex_nd = torch.rand((n, 8), device=d)
    eng, eng1 = UNetEngine(synth_sd, 1, H, W, d), UNetEngine(synth_sd, 1, H, W, d)
    sfs = rdist.ShardedFrameStream(store, tex_nd, eng, W, H, 4, L.FEAT_NHWC_BF16)
    mats = [torch.from_numpy(synth.total_matrix(*synth.camera_batch(W, H, [p]))).to(d) for p in (0, 3, 6, 9, 12)]
    one = ops.Pyramid(1, W, H, 4, d)
    for s in range(4):
        nxt = mats[s + 1] if s != 2 else None                     # step 3 arrives without a look-ahead: the stream must cope
        out = sfs.step(mats[s], nxt).clone()
        one.clear()
        ops.raster_project_sorted(one, store, mats[s])
        ops.pyramid_resolve_gather(tex_nd, one, eng1.inputs, L.FEAT_NHWC_BF16)
        ref = eng1.run()
        torch.cuda.synchronize()
        assert torch.equal(out, ref), f"step {s}"
    torch.cuda.current_stream().wait_stream(sfs.side)
    torch.cuda.synchronize()
