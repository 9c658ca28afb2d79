"""-m gpu: parity at the BASELINE sizes themselves (VERDICT r01 weak #1/#2, ADVICE r01 low #1).

* rasterizer at C3 (10 M points, 1920x1072 and 1920x1088), sorted store and unsorted cloud, bit-compared with the
  oracle's sequential z-buffer (oracle.pcpr_forward, 0.1 s per level);
* refinement net at C2 (512x512, the 1 M-point scene) and on a 1024x512 window of the C3 feature pyramid against the
  oracle's fp32 restatement (oracle/unet_ref.py) - the sizes at which every CTA of the persistent kernels walks many
  tiles and the C128 / C256 weight ring wraps;
* the full 1920x1088 bf16 frame against the fp32 CUDA-core engine (which the small-size tests pin to the oracle).
"""
import numpy as np
import pytest
import torch

from gpu_util import dev, psnr
from read_b200 import ops, synth, _lib as L
from read_b200.engine import UNetEngine

pytestmark = pytest.mark.gpu

TOL_FP32 = 2e-4
TOL_BF16 = 3e-2
PSNR_BF16 = 45.0


@pytest.fixture(scope="module")
def c3_scene():
    return synth.street_scene(10_000_000)


@pytest.mark.parametrize("H", [1072, 1088])
def test_c3_raster_bit_exact_vs_oracle(oracle_mod, c3_scene, H):
    """10 M points, L = 4: every level's index and depth map equals the oracle's, for the sorted store (frame path) and
    the unsorted cloud (pcpr.forward / MyRender path).  point_render.cu:125-167."""
    W, Lv = 1920, 4
    xyz = c3_scene
    proj, view = synth.camera_batch(W, H, [7])
    M = synth.total_matrix(proj, view)
    assert oracle_mod.count_degenerate(xyz, M[0]) == 0
    d = dev()
    x = torch.from_numpy(xyz).to(d)
    m = torch.from_numpy(M).to(d)
    a, b = ops.Pyramid(1, W, H, Lv, d), ops.Pyramid(1, W, H, Lv, d)
    a.clear(); b.clear()
    ops.raster_project(a, x, m)
    store = ops.SortedPoints(x)
    ops.raster_project_sorted(b, store, m)
    ops.raster_derive(b)
    torch.cuda.synchronize()
    assert torch.equal(a.buf, b.buf)
    for l, (w, h) in enumerate(oracle_mod.level_sizes(W, H, Lv)):
        oi, od = oracle_mod.pcpr_forward(xyz, M, w, h)
        gi, gd = ops.zbuf_resolve(b, l)
        np.testing.assert_array_equal(gi.cpu().numpy(), oi, err_msg=f"index level {l}")
        np.testing.assert_array_equal(gd.cpu().numpy().view(np.uint32), od.view(np.uint32), err_msg=f"depth level {l}")


def _window_feats(oracle_mod, xyz, tex, W, H, t, win=None):
    """Oracle index maps of one view -> the reference's PointTexture features [1,8,h,w] per level (optionally a window
    (x0, y0, cw, ch) of the frame, aligned to 8 px so every level crops exactly)."""
    from oracle import unet_ref
    proj, view = synth.camera_batch(W, H, [t])
    _, idx, _ = oracle_mod.render_pyramid(xyz, proj, view, W, H, 4, threads=4)
    feats = []
    for l in range(4):
        m = idx[l]
        if win is not None:
            x0, y0, cw, ch = win
            m = m[:, :, y0 >> l:(y0 + ch) >> l, x0 >> l:(x0 + cw) >> l].copy()
        feats.append(unet_ref.point_texture(tex, torch.from_numpy(m)))
    return feats


def _check_net(synth_sd, feats):
    from oracle import unet_ref
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    with torch.no_grad():
        want = unet_ref.unet_forward(synth_sd, feats)
    B, _, H, W = feats[0].shape
    res = {}
    for precision, tol in (("fp32", TOL_FP32), ("bf16", TOL_BF16)):
        eng = UNetEngine(synth_sd, B, H, W, dev(), precision=precision, use_graph=(precision == "bf16"))
        eng.set_inputs_nchw([f.to(dev()) for f in feats])
        out = eng.run().clone()
        torch.cuda.synchronize()
        out = out.cpu()
        assert torch.isfinite(out).all()
        err = float((out - want).abs().max())
        res[precision] = err
        assert err < tol, (precision, err)
        if precision == "bf16":
            assert psnr(out.numpy(), want.numpy(), peak=float(want.abs().max())) > PSNR_BF16
            h = eng.impl_histogram()
            assert h["generic"] == 0, h
        del eng
        torch.cuda.empty_cache()
    return res


def test_c2_net_512x512_vs_oracle(oracle_mod, synth_sd):
    """BASELINE config 2 (1 M points, 512x512): feature pyramid from the oracle's index maps, full net, both precisions.
    READ/models/unet.py:202-285."""
    n, W, H = 1_000_000, 512, 512
    xyz = synth.street_scene(n)
    tex = torch.rand((1, 8, n), generator=torch.Generator().manual_seed(5))
    _check_net(synth_sd, _window_feats(oracle_mod, xyz, tex, W, H, 3))


def test_c3_window_1024x512_net_vs_oracle(oracle_mod, synth_sd, c3_scene):
    """A 1024x512 window of the C3 (10 M points, 1920x1088) feature pyramid: 4096 full-resolution tiles (28 per CTA), the
    C128 layers run 256 tiles x 1 n-tile, the C256 layers 64 tiles x 2 n-tiles through the streamed-weight ring."""
    W, H = 1920, 1088
    tex = torch.rand((1, 8, c3_scene.shape[0]), generator=torch.Generator().manual_seed(synth.SEED))
    win = ((W - 1024) // 2 // 8 * 8, (H - 512) // 2 // 8 * 8, 1024, 512)
    _check_net(synth_sd, _window_feats(oracle_mod, c3_scene, tex, W, H, 7, win))


def test_c3_full_frame_bf16_vs_fp32_engine(synth_sd):
    """The headline frame itself (1920x1088, B = 1): wgmma bf16 engine (CUDA graph) vs the fp32 CUDA-core engine on the same
    feature pyramid.  The fp32 engine is pinned to the oracle / the reference fixtures at small sizes and on the C2 / C3-window
    cases above; here it carries that pin to the full frame (every persistent CTA walks 110 full-resolution tiles)."""
    W, H = 1920, 1088
    g = torch.Generator().manual_seed(11)
    feats = [torch.rand((1, 8, H >> l, W >> l), generator=g) for l in range(4)]
    outs = {}
    for precision in ("fp32", "bf16"):
        eng = UNetEngine(synth_sd, 1, H, W, dev(), precision=precision, use_graph=(precision == "bf16"))
        eng.set_inputs_nchw([f.to(dev()) for f in feats])
        eng.run()
        out = eng.run().clone()                       # second run: graph replay on warm state
        torch.cuda.synchronize()
        outs[precision] = out.cpu()
        del eng
        torch.cuda.empty_cache()
    a, b = outs["bf16"], outs["fp32"]
    assert torch.isfinite(a).all() and torch.isfinite(b).all()
    err = float((a - b).abs().max())
    assert err < TOL_BF16, err
    assert psnr(a.numpy(), b.numpy(), peak=float(b.abs().max())) > PSNR_BF16
