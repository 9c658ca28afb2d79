"""-m gpu: exact checks of every forward descriptor gather entry point (csrc/gather.cu) on seeded inputs.

activation none: bit for bit against index_select on the clamped int64 ids (empty keys read point 0), in every layout; bf16 is the
round-to-nearest of the f32 value.  sigmoid / tanh: every form and layout gives the same bits on the same ids, within the error bound
of the kernel's arithmetic of a float64 reference.  Ids are negative, fractional, >= N, empty keys and keys whose id is >= N; pixel counts are not multiples of 256,
and some exceed one full grid wave (256 threads x 16 blocks x SMs).  The fused pyramid kernel is checked against
read_raster_derive_levels plus one read_gather_from_zbuf per level."""
import ctypes

import numpy as np
import pytest
import torch

from gpu_util import dev
from read_b200 import ops, _lib as L

pytestmark = pytest.mark.gpu

EMPTY = 0x7FFFFFFFFFFFFFFF
LAYOUTS = (L.FEAT_NCHW_F32, L.FEAT_NHWC_F32, L.FEAT_NHWC_BF16)


def _wave():
    return 256 * 16 * torch.cuda.get_device_properties(0).multi_processor_count


def _tex(N, D, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn((N, D), generator=g) * 3).to(dev())


def _raw_ids(B, h, w, N, seed):
    """int64 ids: in range, negative, >= N."""
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-N // 4, N + N // 4, (B, h, w), generator=g)


def _keys(raw, seed):
    """Packed z-buffer keys for int64 ids >= 0: random depth bits, ~1/5 empty, and ids >= 2^31 (low 32 bits) at ~1/20."""
    g = torch.Generator().manual_seed(seed)
    depth = torch.randint(0, 0x3F800000, raw.shape, generator=g)
    u = torch.rand(raw.shape, generator=g)
    ids = torch.where(u < 0.05, torch.full_like(raw, 0xFFFFFFF0), raw.clamp(min=0))
    return torch.where(u > 0.8, torch.full_like(raw, EMPTY), (depth << 32) | ids)


def _key_ids(keys):
    return torch.where(keys == EMPTY, torch.zeros_like(keys), keys & 0xFFFFFFFF)


def _reference(nd, ids64):
    """[B, D, h, w] f32: index_select on the clamped ids."""
    N, D = nd.shape
    B, h, w = ids64.shape
    rows = nd.index_select(0, ids64.clamp(0, N - 1).reshape(-1).to(nd.device))
    return rows.reshape(B, h, w, D).permute(0, 3, 1, 2).contiguous()


def _as_nchw(out, layout):
    return out if layout == L.FEAT_NCHW_F32 else out.permute(0, 3, 1, 2).float()


def _check_layouts(outs, want_nchw):
    """outs: {layout: gather output}; f32 layouts equal want bit for bit, bf16 is its round-to-nearest."""
    for layout, out in outs.items():
        if layout == L.FEAT_NHWC_BF16:
            assert torch.equal(out, want_nchw.permute(0, 2, 3, 1).to(torch.bfloat16)), layout
        else:
            assert torch.equal(_as_nchw(out, layout), want_nchw), layout


def _zbuf_gather(nd, keys, layout, act="none", out=None):
    B, h, w = keys.shape
    pyr = ops.Pyramid(B, w, h, 1, dev())
    pyr.buf[: keys.numel()].copy_(keys.reshape(-1))
    return ops.gather_from_zbuf(nd, pyr, 0, layout, act, out=out)


# (B, h, w): ragged pixel counts, and one above a full grid wave for D = 8
SHAPES = [(1, 1, 1), (3, 37, 29), (2, 17, 255)]


@pytest.mark.parametrize("D", [1, 3, 8, 16])
def test_one_texture_gathers_equal_index_select(D):
    N = 1000
    nd = _tex(N, D, seed=D)
    shapes = SHAPES + ([(2, 600, 457)] if D == 8 else [])
    assert D != 8 or 2 * 600 * 457 > _wave()
    for i, (B, h, w) in enumerate(shapes):
        raw = _raw_ids(B, h, w, N, seed=100 + i)
        frac = torch.rand(raw.shape, generator=torch.Generator().manual_seed(i)) * 0.98 * torch.sign(raw.float() + 0.5)
        fids = raw.float() + frac                                 # .long() truncates toward zero: -0.7 -> 0, 3.9 -> 3
        assert torch.equal(fids.long(), raw)
        keys = _keys(raw, seed=200 + i)
        for ids64, call in ((raw, lambda lay: ops.gather_from_index(nd, fids.to(dev()).contiguous(), lay)),
                            (raw, lambda lay: ops.gather_from_index(nd, raw.to(dev(), torch.int32).contiguous(), lay)),
                            (_key_ids(keys), lambda lay: _zbuf_gather(nd, keys.to(dev()), lay))):
            want = _reference(nd, ids64)
            _check_layouts({lay: call(lay) for lay in LAYOUTS}, want)


def test_table_gathers_equal_index_select_per_item():
    Ns = [700, 1000, 50]
    tex = [_tex(n, 8, seed=10 + s) for s, n in enumerate(Ns)]
    slots = [2, 0, 1, 2, 0]
    for i, (h, w) in enumerate([(1, 1), (37, 29), (300, 400)]):
        if i == 2:
            assert len(slots) * h * w > _wave()
        raw = torch.stack([_raw_ids(1, h, w, Ns[s], seed=300 + 10 * i + b)[0] for b, s in enumerate(slots)])
        want = torch.cat([_reference(tex[s], raw[b:b + 1]) for b, s in enumerate(slots)])
        for ids in (raw.float().to(dev()).contiguous(), raw.to(dev(), torch.int32).contiguous()):
            _check_layouts({lay: ops.gather_from_index_items(tex, slots, ids, lay) for lay in LAYOUTS}, want)


def _ulps(got, ref):
    """|got - ref| in ulps of the float32 nearest ref."""
    return np.abs(got.astype(np.float64) - ref) / np.spacing(np.abs(ref.astype(np.float32))).astype(np.float64)


# tanhf: CUDA's documented bound, 2 ulp.  1 / (1 + expf(-v)): expf is within 2 ulp (relative 2^-22) and the add and the IEEE division
# round once each (relative 2^-24), so the result is within 2^-22 + 2^-23 of the exact value, relatively, up to second-order terms;
# in ulps of the result that reaches 2.6 on these inputs
SIGMOID_REL = 1.5 * 2.0 ** -22 * (1 + 2.0 ** -20)


@pytest.mark.parametrize("act", ["sigmoid", "tanh"])
@pytest.mark.parametrize("D", [1, 3, 8, 16])
def test_activations_agree_across_forms_and_stay_within_their_error_bound(act, D):
    N, B, h, w = 1000, 2, 19, 23
    nd = _tex(N, D, seed=50 + D)
    ids = _raw_ids(B, h, w, N, seed=60).clamp(0, N - 1)
    g = torch.Generator().manual_seed(61)
    keys = (torch.randint(0, 0x3F800000, ids.shape, generator=g) << 32) | ids
    fids, iids = ids.float().to(dev()).contiguous(), ids.to(dev(), torch.int32).contiguous()
    base = ops.gather_from_index(nd, fids, L.FEAT_NCHW_F32, act)
    forms = [lambda lay: ops.gather_from_index(nd, fids, lay, act), lambda lay: ops.gather_from_index(nd, iids, lay, act),
             lambda lay: _zbuf_gather(nd, keys.to(dev()), lay, act)]
    if D == 8:                                                    # the table forms, every item on the same texture
        forms += [lambda lay, i=i: ops.gather_from_index_items([nd], [0] * B, i, lay, act) for i in (fids, iids)]
    for call in forms:
        _check_layouts({lay: call(lay) for lay in LAYOUTS}, base)
    v = _reference(nd, ids).cpu().numpy().astype(np.float64)
    got = base.cpu().numpy().astype(np.float64)
    if act == "sigmoid":
        ref = 1.0 / (1.0 + np.exp(-v))
        assert (np.abs(got - ref) / ref).max() <= SIGMOID_REL
    else:
        assert _ulps(got, np.tanh(v)).max() <= 2.0


def test_zero_size_gathers_write_nothing():
    nd = _tex(100, 8, seed=1)
    sentinel = torch.full((4096,), float("nan"), device=dev())
    src = torch.zeros(64, dtype=torch.int64, device=dev())          # a torch tensor without elements has a null data pointer
    lib, st = L.load(), L.stream_ptr()
    for B, h, w in ((0, 4, 4), (2, 0, 4), (2, 4, 0)):
        for lay in LAYOUTS:
            for name in ("read_gather_from_index", "read_gather_from_index_i32", "read_gather_from_zbuf"):
                L.check(getattr(lib, name)(nd.data_ptr(), 8, 100, src.data_ptr(), B, h, w, lay, 0, sentinel.data_ptr(), st))
            if B:
                t = ops.tex_table([0] * B, [100], tex=[nd])
                for name in ("read_gather_from_index_items", "read_gather_from_index_items_i32"):
                    L.check(getattr(lib, name)(ctypes.byref(t), src.data_ptr(), h, w, lay, 0, sentinel.data_ptr(), st))
    torch.cuda.synchronize()
    assert bool(sentinel.isnan().all())


def _level0_keys(pyr, N, seed):
    B, (w, h) = pyr.B, pyr.sizes[0]
    raw = torch.randint(0, N + N // 10, (B, h, w), generator=torch.Generator().manual_seed(seed))
    return _keys(raw, seed + 1).reshape(-1)


@pytest.mark.parametrize("layout", [L.FEAT_NHWC_BF16, L.FEAT_NHWC_F32])
@pytest.mark.parametrize("B,view0,nviews,W,H", [(1, 0, 1, 40, 24), (3, 0, 3, 40, 24), (3, 1, 1, 56, 8), (3, 1, 2, 200, 136),
                                                (3, 2, 1, 200, 136), (1, 0, 1, 1160, 1000)])
def test_fused_pyramid_resolve_equals_derive_and_per_level_gathers(layout, B, view0, nviews, W, H):
    N = 5000
    d = dev()
    nd = _tex(N, 8, seed=7)
    assert W % 8 == 0 and H % 8 == 0 and (W % 16 or H % 16)
    if W == 1160:
        assert 32 * (W // 8) * (H // 8) > _wave()
    for reset in (False, True):
        pyr = ops.Pyramid(B, W, H, 4, d)
        junk = torch.randint(0, 1 << 62, (pyr.entries,), generator=torch.Generator().manual_seed(W + reset))
        pyr.buf.copy_(junk)
        pyr.level(0).copy_(_level0_keys(pyr, N, seed=H + B))
        before = pyr.buf.clone()
        ref = ops.Pyramid(B, W, H, 4, d)
        ref.buf.copy_(before)
        ops.raster_derive(ref)
        dt = torch.bfloat16 if layout == L.FEAT_NHWC_BF16 else torch.float32
        outs = [torch.full((nviews, h, w, 8), float("nan"), dtype=dt, device=d) for w, h in pyr.sizes]
        ops.pyramid_resolve_gather(nd, pyr, outs, layout, view0=view0, nviews=nviews, reset_level0=reset)
        v = slice(view0, view0 + nviews)
        for l, (w, h) in enumerate(pyr.sizes):
            want = ops.gather_from_zbuf(nd, ref, l, layout)
            assert torch.equal(outs[l], want[v]), l
            got, der = pyr.level(l).view(B, h, w), ref.level(l).view(B, h, w)
            old = before[pyr.offsets[l]: pyr.offsets[l] + B * w * h].view(B, h, w)
            if l == 0:
                assert torch.equal(got[v], torch.full_like(got[v], EMPTY) if reset else old[v]), l
            else:
                assert torch.equal(got[v], der[v]), l
            outside = [b for b in range(B) if not view0 <= b < view0 + nviews]
            assert torch.equal(got[outside], old[outside]), l
