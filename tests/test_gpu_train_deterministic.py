"""Training under torch.use_deterministic_algorithms(True): the *_det entry points (csrc/scatter_det.cu, csrc/conv_bwd.cu) that
texture._Gather, train._GatherSparse and the bf16 gated-conv backward (blocks.py) pick when the flag is on.

* the descriptor-gradient scatter, dense and sparse: bit-identical to a numpy float32 restatement of the order documented in
  include/read_b200.h, bit-identical between calls, and within 1e-5 of float64;
* the gate backward (eval-mode, batch statistics, per item) and the BatchNorm backward reduction (call-wide, per item): two calls
  bit-identical, [df | dm] bit-identical to the default kernels, the sums within fp32 reordering of them and within the
  kernel-level bound (relative L2 1e-3) of float64;
* the weight gradient of every conv kind with many split-K parts, accumulating into a non-zero dW: two calls bit-identical and
  within the conv2d_weight bound;
* the whole net with NetAndTexture, Adam and SparseRMSprop: two 5-step runs bit-identical (losses, parameters, BatchNorm running
  statistics, descriptors, square_avg) for every precision, eval and train() per_item, L1 and VGGLoss; the same bits under
  warn_only=True with no warning; the flag off gives the same first loss within 1e-3;
* one forward + backward of that step with the flag on against the flag off: the parameter gradients, the descriptor gradient
  (dense and sparse) and the running statistics within the bounds of the float64 and whole-net tests;
* the float64 tests of every training Function (stacks, single convs, FAM, 1x1 / stride-2, eval / batch / per-item BatchNorm,
  the per-item whole net, the dense and sparse gather) rerun with the flag on, every reduction routed to a *_det entry point;
* exchange_sparse_grads raises under the flag (warns under warn_only) before it touches torch.distributed.
"""
import functools
import os
import warnings

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import dev
from read_b200 import _lib as L, blocks, ops, train as rtrain
from read_b200.compose import NetAndTexture
from read_b200.texture import PointTexture
from read_b200.unet import UNet
import test_gpu_gather as t_gather
import test_gpu_train as t_train
import test_gpu_train_all as t_all
import test_gpu_train_blocks as t_blocks
import test_gpu_train_bn as t_bn
import test_gpu_train_bn_items as t_items
import test_gpu_train_convs as t_convs

gpu = pytest.mark.gpu
CHUNK = 128                     # include/read_b200.h: read_gather_backward_det


@pytest.fixture
def deterministic():
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
            torch.backends.cudnn.benchmark)
    torch.use_deterministic_algorithms(True)
    torch.backends.cudnn.benchmark = False
    yield
    torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
    torch.backends.cudnn.benchmark = prev[2]


# ------------------------------------------------------------------ descriptor-gradient scatter
def scatter_np(go, ids, N, out):
    """The documented order in numpy float32: stable sort by clamped id, runs summed per 128-position chunk from 0, an id's runs
    added in chunk order, the result added once to its row of ``out``."""
    B, D, h, w = go.shape
    key = np.clip(ids.reshape(-1).astype(np.int64), 0, N - 1)
    order = np.argsort(key, kind="stable")
    sk, rows = key[order], go.transpose(0, 2, 3, 1).reshape(-1, D)[order]
    total = len(sk)
    starts = np.flatnonzero(np.r_[True, sk[1:] != sk[:-1]])
    ends = np.r_[starts[1:], total]
    zero = np.zeros((1, D), np.float32)
    for a, e in zip(starts, ends):
        cuts = [a] + list(range((a // CHUNK + 1) * CHUNK, e, CHUNK)) + [e]
        seg = None
        for i in range(len(cuts) - 1):
            piece = np.cumsum(np.vstack([zero, rows[cuts[i]:cuts[i + 1]]]), axis=0, dtype=np.float32)[-1]
            seg = piece if seg is None else (seg + piece).astype(np.float32)
        out[sk[a]] = (out[sk[a]] + seg).astype(np.float32)
    return out


def _ids(B, h, w, N, seed):
    """At least half the pixels on id 0 (empty), the rest from a pool shared by every item."""
    g = np.random.default_rng(seed)
    pool = g.integers(1, N, size=max(N // 8, 4))
    ids = pool[g.integers(0, len(pool), size=(B, h, w))]
    ids[g.random((B, h, w)) < 0.55] = 0
    return ids.astype(np.float32)


LEVELS = [(96, 64), (48, 32), (24, 16), (12, 8)]


@gpu
@pytest.mark.parametrize("sparse", [False, True])
def test_scatter_matches_the_documented_order(deterministic, sparse):
    lib, B, D, N = L.load(), 8, 8, 3000
    for lvl, (h, w) in enumerate(LEVELS):
        ids = _ids(B, h, w, N, seed=lvl)
        go = np.random.default_rng(10 + lvl).standard_normal((B, D, h, w)).astype(np.float32)
        assert (ids == 0).mean() >= 0.5
        god, idd = torch.from_numpy(go).to(dev()), torch.from_numpy(ids).to(dev())
        runs = []
        for _ in range(2):
            if sparse:
                prefill = np.random.default_rng(99).standard_normal((N, D)).astype(np.float32)
                acc, touched = torch.from_numpy(prefill).to(dev()), torch.zeros(N, dtype=torch.uint8, device=dev())
                ws = ops.det_workspace(lib.read_gather_backward_det_workspace_bytes(B, D, h, w, N), dev(), "test")
                L.check(lib.read_gather_backward_sparse_det(god.data_ptr(), idd.data_ptr(), B, D, h, w, N, acc.data_ptr(),
                                                            touched.data_ptr(), ws.data_ptr(), L.stream_ptr()))
                runs.append((acc.cpu().numpy(), touched.cpu().numpy()))
            else:
                prefill = np.zeros((N, D), np.float32)
                runs.append((ops.gather_backward(god, idd, N).cpu().numpy(), None))
        assert np.array_equal(runs[0][0].view(np.uint32), runs[1][0].view(np.uint32)), "two calls differ"
        want = scatter_np(go, ids, N, prefill.copy())
        assert np.array_equal(runs[0][0].view(np.uint32), want.view(np.uint32)), f"level {lvl}: not the documented order"
        if sparse:
            seen = np.zeros(N, np.uint8)
            seen[np.unique(ids.astype(np.int64))] = 1
            assert np.array_equal(runs[0][1], seen)
        f64 = prefill.astype(np.float64)
        np.add.at(f64, ids.reshape(-1).astype(np.int64), go.transpose(0, 2, 3, 1).reshape(-1, D).astype(np.float64))
        rel = np.linalg.norm(runs[0][0] - f64) / np.linalg.norm(f64)
        assert rel <= 1e-5, (lvl, rel)


@gpu
def test_texture_backward_under_the_flag_is_reproducible(deterministic):
    tex = PointTexture(8, 4000, init_method="rand").to(dev())
    ids = torch.from_numpy(_ids(8, 64, 48, 4000, seed=5)).unsqueeze(1).to(dev())
    grads = []
    for _ in range(2):
        tex.texture_.grad = None
        (tex(ids) * torch.linspace(-1, 1, 64 * 48, device=dev()).view(1, 1, 64, 48)).sum().backward()
        grads.append(tex.texture_.grad.clone())
    assert torch.equal(grads[0], grads[1])


# ------------------------------------------------------------------ gate backward and BatchNorm reduction
def _gate_operands(items, P, C, seed):
    g = torch.Generator().manual_seed(seed)
    dy = (torch.randn((items * P, C), generator=g)).bfloat16().to(dev())
    fm = (torch.randn((items * P, 2 * C), generator=g) * 2).bfloat16().to(dev())
    vec = lambda *s, lo=0.0: (torch.rand(s, generator=g) + lo).to(dev())
    return dict(dy=dy, fm=fm, bf=vec(C) - 0.5, bm=vec(C) - 0.5, scale=vec(items, C, lo=0.5), mean=vec(items, C) - 0.5,
                inv=vec(items, C, lo=0.5), s0=torch.randn((items, C), generator=g).to(dev()) * 50,
                s1=torch.randn((items, C), generator=g).to(dev()) * 50)


def _gate_call(kind, o, items, P, C, elu, det):
    """One call of a gate / BN pass; returns (dfm or None, the fp32 sums)."""
    lib, st = L.load(), L.stream_ptr()
    ws = ops.det_workspace(lib.read_gate_det_workspace_bytes(items, C), dev(), "test") if det else None
    w = [ws.data_ptr()] if det else []
    sfx = "_det" if det else ""
    dfm = torch.empty_like(o["fm"])
    p = lambda t: t.data_ptr()
    if kind == "gate":
        red = torch.ones((4, C), device=dev())                  # accumulate onto 1
        L.check(getattr(lib, "read_gate_backward" + sfx)(p(o["dy"]), p(o["fm"]), P, C, elu, p(o["bf"]), p(o["bm"]), p(o["scale"]),
                                                         p(o["mean"]), p(o["inv"]), p(dfm), p(red[0]), p(red[1]), p(red[2]),
                                                         p(red[3]), *w, st))
        return dfm, red
    if kind == "gate_batch":
        red = torch.ones((2, C), device=dev())
        L.check(getattr(lib, "read_gate_backward_batch_stats" + sfx)(p(o["dy"]), p(o["fm"]), P, C, elu, p(o["bf"]), p(o["bm"]),
                                                                     p(o["scale"]), p(o["mean"]), p(o["inv"]), p(o["s0"]),
                                                                     p(o["s1"]), p(dfm), p(red[0]), p(red[1]), *w, st))
        return dfm, red
    if kind == "gate_items":
        red = torch.ones((2, C), device=dev())
        L.check(getattr(lib, "read_gate_backward_batch_stats_items" + sfx)(p(o["dy"]), p(o["fm"]), items, P, C, elu, p(o["bf"]),
                                                                           p(o["bm"]), p(o["scale"]), p(o["mean"]), p(o["inv"]),
                                                                           p(o["s0"]), p(o["s1"]), p(dfm), p(red[0]), p(red[1]),
                                                                           *w, st))
        return dfm, red
    if kind == "bn":
        red = torch.ones((2, C), device=dev())
        L.check(getattr(lib, "read_bn_backward_reduce" + sfx)(p(o["dy"]), p(o["fm"]), P, C, elu, p(o["bf"]), p(o["bm"]),
                                                              p(o["mean"]), p(o["inv"]), p(red[0]), p(red[1]), *w, st))
        return None, red
    red = torch.ones((2, items, C), device=dev())
    L.check(getattr(lib, "read_bn_backward_reduce_items" + sfx)(p(o["dy"]), p(o["fm"]), items, P, C, elu, p(o["bf"]), p(o["bm"]),
                                                                p(o["mean"]), p(o["inv"]), p(red[0]), p(red[1]), *w, st))
    return None, red


def _gate_fp64(kind, o, n_items, n_px, C, elu):
    """The sums of _gate_call in float64 from the same bf16 / fp32 operands (blocks.fm_columns: the RAW column order)."""
    raw = o["fm"].cpu().double()
    fmcat = torch.empty_like(raw)
    fmcat[:, blocks.fm_columns(C)] = raw
    f, m = fmcat[:, :C] + o["bf"].cpu().double(), fmcat[:, C:] + o["bm"].cpu().double()
    s = torch.sigmoid(m)
    A = F.elu(f) if elu else f
    Ad = torch.where(f > 0, torch.ones_like(f), A + 1) if elu else torch.ones_like(f)
    dy = o["dy"].cpu().double()
    r = torch.arange(dy.shape[0]) // n_px if kind.endswith("items") else torch.zeros(dy.shape[0], dtype=torch.long)
    sc, mu, iv = (o[k].cpu().double()[r] for k in ("scale", "mean", "inv"))
    xh = dy * (A * s - mu) * iv
    if kind == "bn":
        return torch.stack([dy.sum(0), xh.sum(0)])
    if kind == "bn_items":
        return torch.stack([dy.reshape(n_items, n_px, C).sum(1), xh.reshape(n_items, n_px, C).sum(1)])
    if kind == "gate":
        dg = dy * sc
    else:
        s0, s1 = o["s0"].cpu().double()[r], o["s1"].cpu().double()[r]
        dg = dy * sc - sc * iv * s1 / n_px * (A * s - mu) - sc * s0 / n_px
    df, dm = dg * s * Ad, dg * A * s * (1 - s)
    sums = [df.sum(0), dm.sum(0)]
    return torch.stack(sums + [xh.sum(0), dy.sum(0)] if kind == "gate" else sums)


@gpu
@pytest.mark.parametrize("kind", ["gate", "gate_batch", "gate_items", "bn", "bn_items"])
@pytest.mark.parametrize("C", [16, 32, 64, 128, 192, 256])
@pytest.mark.parametrize("items", [2, 3])
def test_gate_and_bn_reductions_are_reproducible(kind, C, items):
    P = 37 * 41 + items                                                     # ragged
    per_item = kind.endswith("items")
    n_items, n_px = (items, P) if per_item else (1, items * P)
    o = _gate_operands(items, P, C, seed=C + items)
    for elu in (0, 1):
        a, b = (_gate_call(kind, o, n_items, n_px, C, elu, True) for _ in range(2))
        ref = _gate_call(kind, o, n_items, n_px, C, elu, False)
        torch.cuda.synchronize()
        assert torch.equal(a[1], b[1]), "two calls differ"
        if a[0] is not None:
            assert torch.equal(a[0], b[0]) and torch.equal(a[0], ref[0]), "[df | dm] differs"
        rel = float((a[1] - ref[1]).norm() / (ref[1] - 1).norm())
        assert rel <= 1e-5, (kind, C, items, elu, rel)
        # against float64 within the kernel-level bound of test_gpu_train_bn / test_gpu_train_bn_items (relative L2 1e-3 per sum)
        want = _gate_fp64(kind, o, n_items, n_px, C, elu)
        got = (a[1].cpu().double() - 1)
        for k in range(want.shape[0]):
            r64 = float((got[k] - want[k]).norm() / want[k].norm())
            assert r64 <= 1e-3, (kind, C, items, elu, k, r64)


# ------------------------------------------------------------------ weight gradient
@gpu
@pytest.mark.parametrize("cin,C,k,stride,B,H,W", [(8, 16, 3, 1, 2, 45, 67), (16, 32, 3, 1, 2, 45, 67), (32, 64, 3, 1, 2, 37, 45),
                                                  (64, 64, 3, 1, 3, 29, 35), (128, 128, 3, 1, 2, 21, 27), (256, 256, 3, 1, 2, 17, 19),
                                                  (16, 32, 1, 1, 2, 37, 45), (64, 128, 1, 1, 2, 21, 27), (32, 64, 3, 2, 2, 86, 70),
                                                  (128, 256, 3, 2, 2, 26, 38), (64, 32, 4, 2, 2, 86, 70), (256, 128, 4, 2, 2, 26, 38)])
def test_wgrad_is_reproducible_and_accumulates(cin, C, k, stride, B, H, W):
    lib = L.load()
    Ho, Wo = H // stride, W // stride
    g = torch.Generator().manual_seed(C + k + cin)
    dcat = torch.randn((B, Ho, Wo, 2 * C), generator=g).bfloat16()
    dfm = dcat[..., blocks.fm_columns(C)].contiguous().to(dev())
    x = torch.randn((B, H, W, cin), generator=g).bfloat16()
    xd = x.to(dev())
    pre = torch.randn((2, C, cin, k, k), generator=g)
    assert lib.read_conv_wgrad_det_workspace_bytes(B, Ho, Wo, C, cin, k, stride) >= 8 * 2 * C * cin * k * k  # >= 2 splits' copies
    outs = []
    for _ in range(2):
        dw = pre.clone().to(dev())
        ws = ops.det_workspace(lib.read_conv_wgrad_det_workspace_bytes(B, Ho, Wo, C, cin, k, stride), dev(), "test")
        L.check(lib.read_conv_wgrad_det(dfm.data_ptr(), xd.data_ptr(), B, H, W, Ho, Wo, C, cin, k, stride, dw[0].data_ptr(),
                                        dw[1].data_ptr(), ws.data_ptr(), L.stream_ptr()))
        outs.append(dw.cpu())
    assert torch.equal(outs[0], outs[1]), "two calls differ"
    want = torch.nn.grad.conv2d_weight(x.double().permute(0, 3, 1, 2), (2 * C, cin, k, k), dcat.double().permute(0, 3, 1, 2),
                                       stride=stride, padding=(k - 1) // 2)
    got = (outs[0] - pre).reshape(2 * C, cin, k, k).double()
    rel = float((got - want).norm() / want.norm())
    assert rel <= 1e-3, rel


# ------------------------------------------------------------------ the whole training step
N_PTS, B, HW = 20000, 2, 256
KEYS = ["uv_1d_p1"] + [f"uv_1d_p1_ds{l}" for l in range(1, 4)]


def _run(synth_sd, tp, train_mode, loss_kind, steps=5):
    torch.manual_seed(0)
    tex = PointTexture(8, N_PTS, init_method="zeros")
    with torch.no_grad():
        tex.texture_.copy_(torch.rand((1, 8, N_PTS), generator=torch.Generator().manual_seed(1)))
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    net.train_precision = tp
    net.train_batchnorm = "per_item"
    model = NetAndTexture(net, {0: tex}, 1)
    model.load_textures(0)
    model.to(dev())
    model.train(train_mode)
    if loss_kind == "vgg":
        import vgg_util
        from read_b200.vgg_loss import VGGLoss
        crit = VGGLoss(net="caffe", features=vgg_util.seeded_features()).to(dev())
    else:
        crit = F.l1_loss
    opt_net, opt_tex = torch.optim.Adam(net.parameters(), lr=1e-3), rtrain.SparseRMSprop(tex, lr=1e-1)
    g = torch.Generator().manual_seed(2)
    target = torch.rand((B, 3, HW, HW), generator=g).to(dev())
    losses = []
    for s in range(steps):
        inputs = {k: torch.from_numpy(_ids(B, HW >> l, HW >> l, N_PTS, seed=100 * s + l)).unsqueeze(1).to(dev())
                  for l, k in enumerate(KEYS)}
        inputs["id"] = torch.zeros(B, dtype=torch.long)
        loss = crit(model(inputs), target)
        loss.backward()
        opt_net.step()
        opt_tex.step()
        opt_net.zero_grad(set_to_none=True)
        losses.append(loss.detach())
    torch.cuda.synchronize()
    bn = [t.detach().cpu() for n, t in net.named_buffers() if "running" in n]
    return dict(loss=torch.stack(losses).cpu(), params=[p.detach().cpu() for p in net.parameters()], bn=bn,
                desc=tex.texture_.detach().cpu(), sq=opt_tex.dense_square_avg(tex).cpu())


def _same(a, b):
    return all(torch.equal(x, y) for k in a for x, y in zip(a[k] if isinstance(a[k], list) else [a[k]],
                                                              b[k] if isinstance(b[k], list) else [b[k]]))


@gpu
@pytest.mark.parametrize("loss_kind", ["l1", "vgg"])
@pytest.mark.parametrize("train_mode", [False, True])
@pytest.mark.parametrize("tp", ["fp32", "bf16", "bf16_all"])
def test_whole_step_is_bit_reproducible(synth_sd, deterministic, tp, train_mode, loss_kind):
    a = _run(synth_sd, tp, train_mode, loss_kind)
    b = _run(synth_sd, tp, train_mode, loss_kind)
    assert _same(a, b), "two runs under the flag differ"
    if tp == "bf16_all" and train_mode:
        torch.use_deterministic_algorithms(True, warn_only=True)
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            c = _run(synth_sd, tp, train_mode, loss_kind)
        assert not [x for x in w if "determinis" in str(x.message)], [str(x.message) for x in w]
        assert _same(a, c), "warn_only changed the bits"
    # With the flag off the first step's loss agrees; later steps do not compare closely: RMSprop's first update of a point is
    # lr * sign(g), so a descriptor whose gradient is a near-zero sum moves by +-lr on reordering noise alone.
    torch.use_deterministic_algorithms(False)
    off = _run(synth_sd, tp, train_mode, loss_kind, steps=1)
    rel = abs(float(off["loss"][0]) - float(a["loss"][0])) / float(a["loss"][0])
    assert rel <= 1e-3, rel


# ------------------------------------------------------------------ the values of the Python wiring
def _one_backward(synth_sd, tp, train_mode, sparse, det):
    """One forward + backward of NetAndTexture (L1 loss) at 2 x 256^2 with the flag ``det``; the net's parameter gradients, the
    descriptor gradient (texture_.grad, or the sparse accumulator of SparseRMSprop) and the BatchNorm running statistics."""
    torch.use_deterministic_algorithms(det)
    tex = PointTexture(8, N_PTS, init_method="zeros")
    with torch.no_grad():
        tex.texture_.copy_(torch.rand((1, 8, N_PTS), generator=torch.Generator().manual_seed(1)))
    net = UNet()
    net.load_state_dict(synth_sd, strict=True)
    net.train_precision = tp
    net.train_batchnorm = "per_item"
    model = NetAndTexture(net, {0: tex}, 1)
    model.load_textures(0)
    model.to(dev())
    model.train(train_mode)
    if sparse:
        rtrain.SparseRMSprop(tex, lr=1e-1)
    target = torch.rand((B, 3, HW, HW), generator=torch.Generator().manual_seed(2)).to(dev())
    inputs = {k: torch.from_numpy(_ids(B, HW >> l, HW >> l, N_PTS, seed=l)).unsqueeze(1).to(dev()) for l, k in enumerate(KEYS)}
    inputs["id"] = torch.zeros(B, dtype=torch.long)
    F.l1_loss(model(inputs), target).backward()
    torch.cuda.synchronize()
    out = {f"grad {n}": p.grad.detach().cpu() for n, p in net.named_parameters() if p.grad is not None}
    out["descriptor grad"] = (tex._sparse.grad if sparse else tex.texture_.grad).detach().cpu()
    out.update({n: t.detach().cpu() for n, t in net.named_buffers() if "running" in n})
    return out


@gpu
@pytest.mark.parametrize("sparse", [False, True], ids=["dense", "sparse"])
@pytest.mark.parametrize("train_mode", [False, True])
@pytest.mark.parametrize("tp", ["fp32", "bf16", "bf16_all"])
def test_one_backward_with_the_flag_agrees_with_the_flag_off(synth_sd, deterministic, tp, train_mode, sparse):
    """Before any optimizer step, so nothing amplifies the reordering, against the flag off.  Eval mode: every gradient and
    running statistic within the per-layer bounds of the float64 tests (relative L2 2e-2, cosine 0.999).  train(): batch
    statistics amplify rounding through the 99 layers (the flag also changes torch's own convolution algorithms), measured here
    up to relative L2 0.14 / cosine 0.990 for single parameters and 0.09 / 0.996 for the descriptor gradient between the two
    arms, so these are held to the bounds of the whole-net train-mode test (test_gpu_train_bn: cosine 0.95 for all parameters
    together and per descriptor gradient, 0.999 for the running statistics), with 0.95 for each parameter as well.  The values
    of each layer under the flag are checked against float64 by the reruns below."""
    on = _one_backward(synth_sd, tp, train_mode, sparse, True)
    off = _one_backward(synth_sd, tp, train_mode, sparse, False)
    assert on.keys() == off.keys()
    rows = {}
    for k in on:
        a, b = on[k].double().flatten(), off[k].double().flatten()
        if b.norm() == 0:
            assert a.norm() == 0, k
            continue
        rows[k] = (float((a - b).norm() / b.norm()), float(torch.dot(a, b) / (a.norm() * b.norm())))
    grads = [k for k in on if k.startswith("grad ")]
    cat = lambda d: torch.cat([d[k].double().flatten() for k in grads])
    a, b = cat(on), cat(off)
    rows["all parameter gradients"] = (float((a - b).norm() / b.norm()), float(torch.dot(a, b) / (a.norm() * b.norm())))
    for what, keys in (("parameters", [k for k in grads if k in rows]), ("others", [k for k in rows if k not in grads])):
        w = max(keys, key=lambda k: rows[k][0])
        print(f"\n{tp} train={train_mode} sparse={sparse} {what}: worst rel L2 {rows[w][0]:.2e} ({w}), worst cosine "
              f"{min(rows[k][1] for k in keys):.8f}")
    for k, (rel, cos) in rows.items():
        if not train_mode or "running" in k:
            assert rel <= 2e-2 and cos >= 0.999, (k, rel, cos)
        else:
            assert cos >= 0.95, (k, rel, cos)


# The float64 tests of the training Functions, rerun with the flag on: the layers' outputs, gradients and running statistics
# through the deterministic entry points, against float64 autograd within the bounds those tests freeze.  warn_only=True, so that
# a torch op of a float64 reference with no deterministic form warns instead of raising; every reduction of ours must go through
# a *_det entry point and none through its default form.
_DEFAULT_REDUCTIONS = ("read_gather_backward", "read_gather_backward_sparse", "read_gate_backward", "read_bn_backward_reduce",
                       "read_gate_backward_batch_stats", "read_bn_backward_reduce_items", "read_gate_backward_batch_stats_items",
                       "read_conv3x3_wgrad", "read_conv_wgrad")
_DET_REDUCTIONS = ("read_gather_backward_det", "read_gather_backward_sparse_det", "read_gate_backward_det",
                   "read_bn_backward_reduce_det", "read_gate_backward_batch_stats_det", "read_bn_backward_reduce_items_det",
                   "read_gate_backward_batch_stats_items_det", "read_conv_wgrad_det")


def _under_the_flag(fn):
    @functools.wraps(fn)
    def run(*args, **kwargs):
        lib, calls = L.load(), []
        saved = {n: getattr(lib, n) for n in _DEFAULT_REDUCTIONS + _DET_REDUCTIONS}
        prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
        try:
            for n, f in saved.items():
                setattr(lib, n, (lambda n, f: lambda *a: calls.append(n) or f(*a))(n, f))
            torch.use_deterministic_algorithms(True, warn_only=True)
            fn(*args, **kwargs)
        finally:
            for n, f in saved.items():
                setattr(lib, n, f)
            torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
        assert calls and set(calls) <= set(_DET_REDUCTIONS), sorted(set(calls))
    return gpu(run)


test_stack_fp64_under_the_flag = _under_the_flag(t_blocks.test_stack_forward_and_grads_match_fp64_autograd)
test_single_conv_fp64_under_the_flag = _under_the_flag(t_convs.test_conv_forward_and_grads_match_fp64_autograd)
test_fam_merge_fp64_under_the_flag = _under_the_flag(t_convs.test_fam_merge_matches_fp64_autograd)
test_1x1_stride2_conv_fp64_under_the_flag = _under_the_flag(t_all.test_conv_forward_and_grads_match_fp64_autograd)
test_train_mode_stack_fp64_under_the_flag = _under_the_flag(t_bn.test_train_mode_stack_matches_fp64)
test_train_mode_single_conv_fp64_under_the_flag = _under_the_flag(t_bn.test_train_mode_single_conv_matches_fp64)
test_train_mode_1x1_stride2_fp64_under_the_flag = _under_the_flag(t_bn.test_train_mode_1x1_and_stride2_conv_matches_fp64)
test_per_item_stack_fp64_under_the_flag = _under_the_flag(t_items.test_per_item_stack_matches_fp64_loop)
test_per_item_single_conv_fp64_under_the_flag = _under_the_flag(t_items.test_per_item_single_conv_matches_fp64_loop)
test_per_item_fam_merge_fp64_under_the_flag = _under_the_flag(t_items.test_per_item_fam_merge_matches_fp64_loop)
test_per_item_1x1_stride2_fp64_under_the_flag = _under_the_flag(t_items.test_per_item_1x1_and_stride2_conv_matches_fp64_loop)
test_full_net_per_item_under_the_flag = _under_the_flag(t_items.test_full_net_batched_per_item_call_equals_the_loop)
test_sparse_gather_backward_under_the_flag = _under_the_flag(t_train.test_sparse_backward_equals_autograd_of_the_oracle)
test_dense_gather_backward_under_the_flag = _under_the_flag(t_gather.test_point_texture_module_forward_backward_vs_oracle)


# ------------------------------------------------------------------ exchange_sparse_grads
def _no_dist(monkeypatch):
    import torch.distributed as dist

    def boom(*a, **k):
        raise AssertionError("torch.distributed touched")
    monkeypatch.setattr(dist, "is_available", boom)
    monkeypatch.setattr(dist, "is_initialized", boom)


def test_exchange_sparse_grads_raises_under_the_flag(deterministic, monkeypatch):
    _no_dist(monkeypatch)
    with pytest.raises(RuntimeError, match="exchange_sparse_grads"):
        rtrain.exchange_sparse_grads(PointTexture(8, 16))


@gpu
def test_exchange_sparse_grads_warns_under_warn_only(deterministic, monkeypatch):
    torch.use_deterministic_algorithms(True, warn_only=True)
    tex = PointTexture(8, 16).to(dev())
    import torch.distributed as dist
    calls = []
    monkeypatch.setattr(dist, "is_initialized", lambda: calls.append(1) or False)
    with pytest.warns(UserWarning, match="exchange_sparse_grads"):
        assert rtrain.exchange_sparse_grads(tex) == 0
    assert calls == [1]
