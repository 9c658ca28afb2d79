"""-m gpu: a scene of N = 2^24 + 2^21 points, more than float32 index maps can number (synth.street_scene orders its clutter last, so
many visible points have ids above 2^24; every odd one of them has no float32).

* raster: MyRender returns int32 maps equal to the int32 oracle on every level, depths bit for bit; over 10^4 level-0 pixels show an
  id float32 cannot hold, and the float maps are wrong there;
* gather: int32 maps, every layout and activation, one texture and a texture table, against a float64 index_select on int64 ids
  and against the float gather of the same values under small ids;
* backward: integer-valued gradients, so every sum is exact: the dense, sparse, items and deterministic int32 scatters equal a
  float64 index_add_, the touched flags are the ids present; the deterministic forms repeat their bits and equal the float forms
  on small-id maps;
* inference: NetAndTexture on MyRender's int32 maps is bit-identical to NetAndTexture.render, for this scene and for a batch that
  mixes it with a small one;
* training: one headless step (bf16_all, per_item, VGGLoss, SparseRMSprop): the sparse accumulator against a float64 index_add_ of
  the gradient reaching the net input; the step changes exactly the touched rows with a gradient, odd ids above 2^24 included.
"""
import os
import sys
import types
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import headless_util as hu  # noqa: E402
import oracle_i32  # noqa: E402
import vgg_util  # noqa: E402
from gpu_util import dev  # noqa: E402
from test_gpu_train_deterministic import deterministic  # noqa: E402,F401  (fixture)
from read_b200 import _lib as L, headless, ops, synth, train as rtrain  # noqa: E402
from read_b200.myrender import MyRender  # noqa: E402
from read_b200.texture import PointTexture  # noqa: E402
from read_b200.unet import UNet  # noqa: E402
from read_b200.vgg_loss import VGGLoss  # noqa: E402

pytestmark = pytest.mark.gpu

N = 2 ** 24 + 2 ** 21
W = H = 512
CAMERAS = [0, 4]                        # the CPU oracle finds 58,108 level-0 pixels of ids float32 cannot hold in these two views
FORMAT4 = "uv_1d_p1, uv_1d_p1_ds1, uv_1d_p1_ds2, uv_1d_p1_ds3"
EXACT = 2 ** 24 + 1                     # float32 holds every id up to 2^24 (clouds of up to 2^24 + 1 points)


def _scene(n, fmt, ds_id=0, seed=synth.SEED):
    s = hu.scene(n, W, H, ds_id=ds_id, seed=seed)
    s.input_format = fmt
    return s


@pytest.fixture(scope="module")
def big():
    """The scene, its views and MyRender's five-level maps (device)."""
    s = _scene(N, hu.INPUT_FORMAT)
    r = MyRender(device_outputs=True)
    r.update_ds([s])
    data = hu.batch(W, H, CAMERAS)
    maps, depths = r.render(data)
    keys = [k for k in maps if k != 'id']
    xyz = s.scene_data['pointcloud']['xyz']
    tm = synth.total_matrix(data['proj_matrix'].numpy(), data['view_matrix'].numpy())
    return types.SimpleNamespace(scene=s, renderer=r, data=data, xyz=xyz, total_m=tm, ids=[maps[k][:, 0].contiguous() for k in keys],
                                 depths=[depths[k][:, 0] for k in keys])


def _inexact(ids):
    i = ids.long()
    return (i > EXACT) & (i.float().long() != i)


def test_myrender_int32_maps_equal_the_oracle(big, oracle_mod):
    assert big.renderer.index_dtype == torch.int32
    sizes = ops.level_sizes(W, H, len(big.ids))
    with ThreadPoolExecutor(max_workers=len(sizes)) as ex:
        want = list(ex.map(lambda s: oracle_i32.pcpr_forward_i32(big.xyz, big.total_m, s[0], s[1]), sizes))
    for l, ((wi, wd), gi, gd) in enumerate(zip(want, big.ids, big.depths)):
        assert gi.dtype == torch.int32 and gd.dtype == torch.float32
        assert np.array_equal(gi.cpu().numpy(), wi), f"level {l} index"
        assert np.array_equal(gd.cpu().numpy().view(np.uint32), wd.view(np.uint32)), f"level {l} depth"
    i0 = big.ids[0].cpu()
    bad = _inexact(i0)
    print(f"\nlevel 0: {int((i0 > 2 ** 24).sum())} pixels of ids above 2^24, {int(bad.sum())} of them without a float32")
    assert int(bad.sum()) >= 10_000
    fi, _ = oracle_mod.pcpr_forward(big.xyz, big.total_m, W, H)                 # the float map the parent returns
    assert (torch.from_numpy(fi).long()[bad] != i0.long()[bad]).all()


def _tex(n, seed):
    g = torch.Generator(device=dev()).manual_seed(seed)
    return torch.rand((n, 8), generator=g, device=dev()) * 4 - 2


def _compact(ids):
    """(small-id float32 map, int32 copy of it, the rows they select): the same gather with every id below 2^24."""
    uniq, inv = torch.unique(ids.long(), return_inverse=True)
    small = inv.to(torch.int32).reshape(ids.shape).contiguous()
    return small.float().contiguous(), small, uniq


LAYOUTS = [L.FEAT_NCHW_F32, L.FEAT_NHWC_F32, L.FEAT_NHWC_BF16]


def _ref_gather(tex, ids, layout):
    v = tex.double().index_select(0, ids.long().clamp(0, tex.shape[0] - 1).reshape(-1)).reshape(*ids.shape, 8)
    if layout == L.FEAT_NCHW_F32:
        return v.permute(0, 3, 1, 2).float()
    return v.float() if layout == L.FEAT_NHWC_F32 else v.float().bfloat16()


@pytest.mark.parametrize("act", ["none", "sigmoid", "tanh"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_int32_gather_is_exact(big, layout, act):
    tex, tex2 = _tex(N, 1), _tex(N, 2)
    for ids in big.ids[:2]:
        got = ops.gather_from_index(tex, ids, layout, act)
        small_f, small_i, rows = _compact(ids)
        sub = tex[rows].contiguous()
        assert torch.equal(got, ops.gather_from_index(sub, small_f, layout, act))          # the float path on the same values
        assert torch.equal(ops.gather_from_index(sub, small_i, layout, act), ops.gather_from_index(sub, small_f, layout, act))
        if act == "none":
            assert torch.equal(got, _ref_gather(tex, ids, layout))
        items = ops.gather_from_index_items([tex, tex2], [0, 1], ids, layout, act)
        per = [ops.gather_from_index(t, ids[b:b + 1].contiguous(), layout, act) for b, t in enumerate((tex, tex2))]
        assert torch.equal(items, torch.cat(per, 0))
        sub2 = tex2[rows].contiguous()
        assert torch.equal(ops.gather_from_index_items([sub, sub2], [0, 1], small_i, layout, act),
                           ops.gather_from_index_items([sub, sub2], [0, 1], small_f, layout, act))


def _int_grad(ids, seed):
    g = torch.Generator(device=dev()).manual_seed(seed)
    B, h, w = ids.shape
    return torch.randint(-8, 9, (B, 8, h, w), generator=g, device=dev()).float()


def _ref_scatter(go, ids, n):
    rows = ids.long().clamp(0, n - 1).reshape(-1)
    return torch.zeros((n, 8), dtype=torch.float64, device=dev()).index_add_(0, rows, go.permute(0, 2, 3, 1).reshape(-1, 8).double())


def _present(ids, n):
    t = torch.zeros(n, dtype=torch.uint8, device=dev())
    t[ids.long().clamp(0, n - 1).reshape(-1)] = 1
    return t


def _scatters(go, ids):
    """Dense, sparse, dense items and sparse items scatters of one map (items: item b into texture b, both of N points)."""
    out = {"dense": (ops.gather_backward(go, ids, N), None)}
    acc, touched = torch.zeros((N, 8), device=dev()), torch.zeros(N, dtype=torch.uint8, device=dev())
    ops.gather_backward_sparse(go, ids, N, acc, touched)
    out["sparse"] = (acc, touched)
    grads = [torch.zeros((N, 8), device=dev()) for _ in range(2)]
    ops.gather_backward_items(go, ids, [0, 1], [N, N], grads)
    out["items"] = (grads, None)
    grads = [torch.zeros((N, 8), device=dev()) for _ in range(2)]
    flags = [torch.zeros(N, dtype=torch.uint8, device=dev()) for _ in range(2)]
    ops.gather_backward_items(go, ids, [0, 1], [N, N], grads, flags)
    out["sparse_items"] = (grads, flags)
    return out


def _check_exact(out, go, ids):
    want = _ref_scatter(go, ids, N)
    assert torch.equal(out["dense"][0].double(), want)
    acc, touched = out["sparse"]
    assert torch.equal(acc.double(), want) and torch.equal(touched, _present(ids, N))
    for b in range(2):
        wb = _ref_scatter(go[b:b + 1], ids[b:b + 1], N)
        assert torch.equal(out["items"][0][b].double(), wb), f"items, slot {b}"
        assert torch.equal(out["sparse_items"][0][b].double(), wb), f"sparse items, slot {b}"
        assert torch.equal(out["sparse_items"][1][b], _present(ids[b:b + 1], N)), f"sparse items flags, slot {b}"


def test_int32_scatters_are_exact(big):
    for l, ids in enumerate(big.ids[:2]):
        go = _int_grad(ids, 10 + l)
        _check_exact(_scatters(go, ids), go, ids)
        big_ids = ids.long()[ids.long() > EXACT]
        assert big_ids.numel() > 0 and bool((big_ids % 2 == 1).any())


def test_int32_deterministic_scatters_are_exact_repeat_and_match_the_float_forms(big, deterministic):
    for l, ids in enumerate(big.ids[:2]):
        go = _int_grad(ids, 20 + l)
        first = _scatters(go, ids)
        _check_exact(first, go, ids)
        again = _scatters(go, ids)
        for k in first:
            a, b = first[k], again[k]
            for x, y in zip(a[0] if isinstance(a[0], list) else [a[0]], b[0] if isinstance(b[0], list) else [b[0]]):
                assert torch.equal(x, y), k
    # small-id maps: the float and int32 forms run the same order of additions, so non-integer gradients give the same bits
    small_f, small_i, _ = _compact(big.ids[0])
    g = torch.Generator(device=dev()).manual_seed(3)
    go = torch.randn((small_f.shape[0], 8) + tuple(small_f.shape[1:]), generator=g, device=dev())
    n = int(small_f.max()) + 1
    assert torch.equal(ops.gather_backward(go, small_f, n), ops.gather_backward(go, small_i, n))
    for sparse in (False, True):
        res = []
        for ids in (small_f, small_i):
            grads = [torch.zeros((n, 8), device=dev()) for _ in range(2)]
            flags = [torch.zeros(n, dtype=torch.uint8, device=dev()) for _ in range(2)] if sparse else None
            ops.gather_backward_items(go, ids, [0, 1], [n, n], grads, flags)
            if sparse:
                acc, t = torch.zeros((n, 8), device=dev()), torch.zeros(n, dtype=torch.uint8, device=dev())
                ops.gather_backward_sparse(go, ids, n, acc, t)
                grads += [acc, t]
            res.append(grads)
        assert all(torch.equal(a, b) for a, b in zip(*res)), f"sparse={sparse}"


def _net(synth_sd, **attrs):
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    for k, v in attrs.items():
        setattr(net, k, v)
    return net


def _texture(n, seed):
    t = PointTexture(8, n)
    with torch.no_grad():
        t.texture_.copy_(torch.rand((1, 8, n), generator=torch.Generator().manual_seed(seed)))
    return t


def test_inference_on_int32_maps_is_bit_identical_to_render(big, synth_sd):
    small = _scene(50_000, FORMAT4, ds_id=1, seed=7)
    large = types.SimpleNamespace(**dict(vars(big.scene), input_format=FORMAT4))
    r = MyRender([large, small], device_outputs=True)
    assert r.index_dtype == torch.int32
    model = headless.NetAndTexture(_net(synth_sd), {0: _texture(N, 1), 1: _texture(50_000, 2)})
    model.load_textures([0, 1])
    model.to(dev()).eval()
    tm = torch.from_numpy(big.total_m).to(dev())
    clouds = {0: torch.from_numpy(big.xyz).to(dev()), 1: torch.from_numpy(small.scene_data['pointcloud']['xyz']).to(dev())}
    want = {tid: model.render(clouds[tid], tm, W, H, texture_id=tid, n_levels=4) for tid in (0, 1)}
    for ids in ([0, 0], [0, 1]):
        data = dict(big.data, input={'id': torch.tensor(ids)})
        maps, _ = r.render(data)
        assert all(v.dtype == torch.int32 for k, v in maps.items() if k != 'id')
        with torch.no_grad():
            got = model(maps)['im_out']
        for b, tid in enumerate(ids):
            assert torch.equal(got[b], want[tid][b]), f"batch {ids}, item {b}"
    # render(want_maps=True) hands out int32 maps too, equal to MyRender's
    _, maps = model.render(clouds[0], tm, W, H, n_levels=4, want_maps=True)
    assert all(m[0].dtype == torch.int32 and torch.equal(m[0], i) for m, i in zip(maps, big.ids))


def test_headless_training_step_on_int32_maps(big, synth_sd, monkeypatch):
    net = _net(synth_sd, train_precision='bf16_all', train_batchnorm='per_item')
    tex = _texture(N, 3)
    model = headless.NetAndTexture(net, {0: tex})
    model.load_textures([0])
    model.to(dev()).train()
    opt_net = torch.optim.Adam(net.parameters(), lr=1e-4)
    opt_tex = rtrain.SparseRMSprop([tex], lr=0.1)
    loss_mod = hu.ModelAndLoss(model, VGGLoss(features=vgg_util.seeded_features()).to(dev()))
    target = torch.rand((2, 3, H, W), generator=torch.Generator().manual_seed(7)).to(dev())
    seen = []
    apply = rtrain._GatherSparse.apply

    def recording(texture_, ids, tex_module):
        out = apply(texture_, ids, tex_module)
        rec = [ids, None]
        out.register_hook(lambda g: rec.__setitem__(1, g.detach().clone()))
        seen.append(rec)
        return out

    monkeypatch.setattr(rtrain._GatherSparse, "apply", recording)
    loss = hu.forward_loss(big.renderer, loss_mod, big.data, target, None, dev(), model.reg_loss)
    loss.backward()
    monkeypatch.undo()
    assert len(seen) == len(big.ids) and all(i.dtype == torch.int32 for i, _ in seen)
    seen = [(i, g) for i, g in seen if g is not None]                 # a level the net does not read receives no gradient
    assert len(seen) >= 4
    want = torch.zeros((N, 8), dtype=torch.float64, device=dev())
    for ids, g in seen:
        want += _ref_scatter(g.float(), ids, N)
    sp = tex._sparse
    err = float((sp.grad.double() - want).abs().max())
    scale = float(want.abs().max())
    print(f"\nsparse accumulator: max abs error {err:.3e} of max |grad| {scale:.3e}")
    assert err <= 1e-5 * scale
    touched = sp.touched.clone().bool()
    assert torch.equal(touched, torch.stack([_present(i, N) for i, _ in seen]).amax(0).bool())
    # RMSprop moves a row by about lr * g / (|g| + eps / sqrt(1 - alpha)): above |g| = 1e-10 that is far beyond a float32 ulp of
    # the descriptor, below it the row may keep its bits
    has_grad = (sp.grad.abs() > 1e-10).any(1)
    before = tex.texture_.detach().clone()
    opt_net.step()
    opt_tex.step()
    torch.cuda.synchronize()
    changed = (tex.texture_.detach() != before)[0].any(0)
    assert not bool(changed[~touched].any()), "an untouched row changed"
    assert bool(changed[touched & has_grad].all()), "a touched row with a gradient did not change"
    assert int(has_grad.sum()) > 0.9 * int(touched.sum())
    odd_big = torch.nonzero(changed).reshape(-1)
    odd_big = odd_big[(odd_big > EXACT) & (odd_big % 2 == 1)]
    print(f"rows changed: {int(changed.sum())}, odd ids above 2^24 among them: {odd_big.numel()}")
    assert odd_big.numel() > 1000
