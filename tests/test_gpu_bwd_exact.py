"""Exact checks of the training backward kernels at every tile, segment and item edge (tests/bwd_exact_util.py states the method).

* weight gradient: read_conv3x3_wgrad, read_conv_wgrad (1x1, 3x3 / 4x4 stride 2) and read_conv_wgrad_det, every (Cin, C) the net
  trains, W across the 32-pixel segments, H in {1, 2, 7}, B in {1, 4, 8} up to 8 x 256^2, both chunk / split regimes: every
  element equal to pre-fill + the exact float64 gradient, the padded rows exactly the pre-fill, nothing written outside dW;
* input gradient: the RAW 3x3 plan under blocks.dgrad (with and without the ResBlock residual), the RAW 1x1 plans under
  blocks.dgrad_1x1 (each source slice of a concat), read_conv3x3_dgrad_cin8 and read_conv_dgrad_s2: every bf16 element the
  round-to-nearest of the exact sum, nothing written outside dx;
* gate / BatchNorm backward (all forms, atomic and _det): dbeta / sum_dy of integer dy exact per item; [df | dm] and the other
  sums within the per-element bounds; an output-gradient impulse gives [df | dm] exactly 0 outside its two columns;
* descriptor scatter (read_gather_backward[_sparse][_det], the multi-texture _items forms): integer grad_out, clamped and heavily
  repeated ids, 16 slots x 64 items: every accumulator element and touched flag exact.
"""
import ctypes
import types
import zlib

import pytest
import torch

import bwd_exact_util as U
from gpu_util import dev
from read_b200 import _lib as L, blocks, ops

gpu = pytest.mark.gpu
WORST = {}


def _gen(*key):
    return torch.Generator().manual_seed(zlib.crc32(repr(key).encode()))


def _worst(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)
    print(f"\nworst err/bound so far: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _ws(nbytes):
    return ops.det_workspace(nbytes, dev(), "test")


# ------------------------------------------------------------------ weight gradient
def _wgrad_case(case):
    cin, C, k, stride, B, H, W = case
    g = _gen("wgrad", case)
    dcat = U.int_tensor((B, H, W, 2 * C), U.WGRAD_AMP, g)
    n_real = U.PADDED.get((k, stride, cin, C))
    if n_real is not None:
        dcat = U.zero_padded_columns(dcat, n_real)
    x = U.int_tensor((B, stride * H, stride * W, cin), U.WGRAD_AMP, g)
    pre = U.int_tensor((2, C, cin, k, k), U.WGRAD_PREFILL, g, zero_frac=0.0)
    return dcat.to(dev()), x.bfloat16().to(dev()), pre.to(dev()), n_real


def _wgrad_run(entry, case, dfm, x, pre):
    cin, C, k, stride, B, H, W = case
    lib, st = L.load(), L.stream_ptr()
    outs = [U.Guarded(pre[i].numel(), torch.float32, dev(), pre[i]) for i in range(2)]
    p = [o.out.data_ptr() for o in outs]
    if entry == "conv3x3_wgrad":
        L.check(lib.read_conv3x3_wgrad(dfm.data_ptr(), x.data_ptr(), B, H, W, C, cin, p[0], p[1], st))
    elif entry == "conv_wgrad":
        L.check(lib.read_conv_wgrad(dfm.data_ptr(), x.data_ptr(), B, stride * H, stride * W, H, W, C, cin, k, stride, p[0], p[1],
                                    st))
    else:
        ws = _ws(lib.read_conv_wgrad_det_workspace_bytes(B, H, W, C, cin, k, stride))
        L.check(lib.read_conv_wgrad_det(dfm.data_ptr(), x.data_ptr(), B, stride * H, stride * W, H, W, C, cin, k, stride, p[0],
                                        p[1], ws.data_ptr(), st))
    torch.cuda.synchronize()
    for o, name in zip(outs, ("dwf", "dwm")):
        o.check(f"{entry} {case} {name}")
    return [o.out.view(C, cin, k, k) for o in outs]


@gpu
@pytest.mark.parametrize("case", U.WGRAD_CASES, ids=lambda c: "cin{}-C{}-k{}s{}-B{}-{}x{}".format(*c))
def test_wgrad_is_exact(case):
    cin, C, k, stride, B, H, W = case
    dcat, x, pre, n_real = _wgrad_case(case)
    dfm = U.to_raw(dcat).bfloat16().contiguous()
    want = U.wgrad_ref(dcat, x, k, stride)
    entries = (["conv3x3_wgrad"] if (k, stride) == (3, 1) else []) + ["conv_wgrad", "conv_wgrad_det"]
    names = ["o", "ci", "ky", "kx"]
    for entry in entries:
        dwf, dwm = _wgrad_run(entry, case, dfm, x, pre)
        U.assert_exact(dwf, pre[0].double() + want[:C], f"{entry} {case} dwf", names)
        U.assert_exact(dwm, pre[1].double() + want[C:], f"{entry} {case} dwm", names)
        if n_real is not None:
            assert torch.equal(dwf[n_real:], pre[0][n_real:]) and torch.equal(dwm[n_real:], pre[1][n_real:]), "padded rows"


# ------------------------------------------------------------------ input gradient: RAW 3x3 and 1x1 plans
def _dgrad_operands(key, B, H, W, C, cin, k, n_real=None):
    g = _gen("dgrad", key)
    dcat = U.int_tensor((B, H, W, 2 * C), U.DGRAD_AMP, g)
    if n_real is not None:
        dcat = U.zero_padded_columns(dcat, n_real)
    wcat = U.int_tensor((2 * C, cin, k, k), U.DGRAD_AMP, g)
    return dcat.to(dev()), wcat.to(dev()), g


def _nonrep_ok(want, what):
    frac = U.bf16_nonrepresentable_fraction(want)
    assert frac >= 0.1, f"{what}: only {frac:.2f} of the exact sums need rounding; the round-to-nearest check would be weak"


@gpu
@pytest.mark.parametrize("case", U.DGRAD3_CASES, ids=lambda c: "cin{}-C{}-B{}-{}x{}".format(*c))
def test_dgrad_raw3x3_is_exact(case):
    cin, C, B, H, W = case
    lib, st = L.load(), L.stream_ptr()
    dcat, wcat, g = _dgrad_operands(case, B, H, W, C, cin, 3, U.PADDED.get((3, 1, cin, C)))
    wf, wm = wcat[:C].contiguous(), wcat[C:].contiguous()
    w_dgrad = torch.empty(lib.read_tc_weight_elems(cin // 2, 2 * C, 3), dtype=torch.bfloat16, device=dev())
    L.check(lib.read_pack_weights_tc_dgrad(wf.data_ptr(), wm.data_ptr(), C, cin, w_dgrad.data_ptr(), st))
    dfm = U.to_raw(dcat).bfloat16().contiguous()
    base = U.dgrad_ref(dcat, wcat, H, W, 1)
    _nonrep_ok(base, f"dgrad {case}")
    conv = types.SimpleNamespace(wf=wf, wm=wm, C=C, w_dgrad=w_dgrad)
    zeros = torch.zeros(cin, dtype=torch.float32, device=dev())
    names = ["b", "y", "x", "c"]
    for res in (None, U.int_tensor((B, H, W, cin), U.DGRAD_RES_AMP, g).bfloat16().to(dev())):
        want = base + (0 if res is None else res.double())
        out = U.Guarded(B * H * W * cin, torch.bfloat16, dev())
        blocks._launch(lib, dfm, cin // 2, w_dgrad, (zeros,) * 4, False, L.OUT_RAW_NHWC, out.out, res)
        torch.cuda.synchronize()
        what = f"RAW 3x3 dgrad {case} residual={res is not None}"
        out.check(what)
        U.assert_bf16_rn(out.out.view(B, H, W, cin), want, what, names)
        assert torch.equal(blocks.dgrad(dfm, conv, residual=res), out.out.view(B, H, W, cin)), what + ": blocks.dgrad"


@gpu
@pytest.mark.parametrize("case", U.DGRAD1_CASES, ids=lambda c: "src{}-C{}-B{}-{}x{}".format("_".join(map(str, c[0])), *c[1:]))
def test_dgrad_raw1x1_plans_are_exact_per_source(case):
    srcs, C, B, H, W = case
    lib = L.load()
    cin = sum(srcs)
    dcat, wcat, _ = _dgrad_operands(case, B, H, W, C, cin, 1, U.PADDED.get((1, 1, srcs[0], C)) if len(srcs) == 1 else None)
    c = types.SimpleNamespace(pk={'wf': wcat[:C].contiguous(), 'wm': wcat[C:].contiguous()}, C=C)
    dfm = U.to_raw(dcat).bfloat16().contiguous()
    want = U.dgrad_ref(dcat, wcat, H, W, 1)
    _nonrep_ok(want, f"dgrad 1x1 {case}")
    names = ["b", "y", "x", "c"]
    c0 = 0
    for cs in srcs:
        for a, cn, w in blocks._dgrad1x1_filters(lib, c.pk, C, c0, cs):
            n_out = max(cn, 32)
            out = U.Guarded(B * H * W * n_out, torch.bfloat16, dev())
            zeros = torch.zeros(n_out // 2, dtype=torch.float32, device=dev())
            blocks._launch(lib, dfm, n_out // 2, w, (zeros,) * 4, False, L.OUT_RAW_NHWC, out.out, k=1)
            torch.cuda.synchronize()
            what = f"RAW 1x1 dgrad {case} channels {a}..{a + cn - 1}"
            out.check(what)
            got = out.out.view(B, H, W, n_out)
            U.assert_bf16_rn(got[..., :cn], want[..., a:a + cn], what, names)
            assert not bool(got[..., cn:].float().any()), what + ": the zero-filter columns"
        U.assert_bf16_rn(blocks.dgrad_1x1(dfm, c, c0, cs), want[..., c0:c0 + cs], f"blocks.dgrad_1x1 {case} source at {c0}", names)
        c0 += cs


@gpu
@pytest.mark.parametrize("case", U.DG8_CASES, ids=lambda c: "C{}-B{}-{}x{}".format(*c))
def test_dgrad_cin8_is_exact(case):
    C, B, H, W = case
    lib = L.load()
    dcat, wcat, _ = _dgrad_operands(case, B, H, W, C, 8, 3)
    dfm = U.to_raw(dcat).bfloat16().contiguous()
    want = U.dgrad_ref(dcat, wcat, H, W, 1)
    _nonrep_ok(want, f"dgrad cin8 {case}")
    out = U.Guarded(B * H * W * 8, torch.bfloat16, dev())
    L.check(lib.read_conv3x3_dgrad_cin8(dfm.data_ptr(), wcat[:C].contiguous().data_ptr(), wcat[C:].contiguous().data_ptr(), B, H,
                                        W, C, out.out.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    out.check(f"dgrad_cin8 {case}")
    U.assert_bf16_rn(out.out.view(B, H, W, 8), want, f"dgrad_cin8 {case}", ["b", "y", "x", "c"])


@gpu
@pytest.mark.parametrize("case", U.DS_CASES, ids=lambda c: "k{}-cin{}-C{}-B{}-{}x{}".format(*c))
def test_dgrad_s2_is_exact(case):
    k, cin, C, B, Hi, Wi = case
    lib, st = L.load(), L.stream_ptr()
    Ho, Wo = Hi // 2, Wi // 2
    dcat, wcat, _ = _dgrad_operands(case, B, Ho, Wo, C, cin, k)
    dfm = U.to_raw(dcat).bfloat16().contiguous()
    wt = torch.empty((k * k, cin, 2 * C), dtype=torch.bfloat16, device=dev())
    L.check(lib.read_pack_weights_dgrad_s2(wcat[:C].contiguous().data_ptr(), wcat[C:].contiguous().data_ptr(), C, cin, k,
                                           wt.data_ptr(), st))
    want = U.dgrad_ref(dcat, wcat, Hi, Wi, 2)
    _nonrep_ok(want, f"dgrad s2 {case}")
    out = U.Guarded(B * Hi * Wi * cin, torch.bfloat16, dev())
    L.check(lib.read_conv_dgrad_s2(dfm.data_ptr(), wt.data_ptr(), B, Ho, Wo, C, cin, k, out.out.data_ptr(), st))
    torch.cuda.synchronize()
    out.check(f"dgrad_s2 {case}")
    U.assert_bf16_rn(out.out.view(B, Hi, Wi, cin), want, f"dgrad_s2 {case}", ["b", "y", "x", "c"])


# ------------------------------------------------------------------ gate / BatchNorm backward
def _gate_operands(items, P, C, seed, int_dy=False, spread=False):
    g = torch.Generator().manual_seed(seed)
    n = items * P
    dy = U.int_tensor((n, C), 8, g) if int_dy else torch.randn((n, C), generator=g) * 4
    fm = U.to_raw(U.gate_fm_values(n, C, g)).bfloat16()
    bias = lambda: torch.where(torch.arange(C) % 2 == 0, torch.zeros(C), torch.rand(C, generator=g) - 0.5)
    # per item statistics a few orders of magnitude apart when ``spread``
    mag = (10.0 ** torch.randint(-2, 3, (items, 1), generator=g).float()) if spread else torch.ones((items, 1))
    vec = lambda lo: (torch.rand((items, C), generator=g) + lo)
    o = dict(dy=dy.bfloat16(), fm=fm, bf=bias(), bm=bias(), scale=vec(0.5) * mag, mean=(vec(0) - 0.5) * mag, inv=vec(0.5) / mag,
             s0=torch.randn((items, C), generator=g) * 50 * mag, s1=torch.randn((items, C), generator=g) * 50 * mag)
    return {k: v.to(dev()).contiguous() for k, v in o.items()}


def _gate_run(kind, o, items, P, C, elu, det, prefill=0.0):
    """One call; returns dfm (or None) and the fp32 sums {name: tensor}, all outputs guard-banded."""
    lib, st = L.load(), L.stream_ptr()
    wst = _ws(lib.read_gate_det_workspace_bytes(items if kind.endswith("items") else 1, C)) if det else None   # alive until the end
    ws = [wst.data_ptr()] if det else []
    sfx = "_det" if det else ""
    p = lambda t: t.data_ptr()
    nsum = {"gate": 4, "gate_batch": 2, "gate_items": 2, "bn": 2, "bn_items": 2}[kind]
    rows = items if kind == "bn_items" else 1
    sums = [U.Guarded(rows * C, torch.float32, dev(), torch.full((rows * C,), prefill)) for _ in range(nsum)]
    sp = [s.out.data_ptr() for s in sums]
    dfm = U.Guarded(o["fm"].numel(), torch.bfloat16, dev()) if kind.startswith("gate") else None
    n = items * P
    if kind == "gate":
        L.check(getattr(lib, "read_gate_backward" + sfx)(p(o["dy"]), p(o["fm"]), n, C, elu, p(o["bf"]), p(o["bm"]), p(o["scale"]),
                                                         p(o["mean"]), p(o["inv"]), p(dfm.out), *sp, *ws, st))
    elif kind == "gate_batch":
        L.check(getattr(lib, "read_gate_backward_batch_stats" + sfx)(p(o["dy"]), p(o["fm"]), n, C, elu, p(o["bf"]), p(o["bm"]),
                                                                     p(o["scale"]), p(o["mean"]), p(o["inv"]), p(o["s0"]),
                                                                     p(o["s1"]), p(dfm.out), *sp, *ws, st))
    elif kind == "gate_items":
        L.check(getattr(lib, "read_gate_backward_batch_stats_items" + sfx)(p(o["dy"]), p(o["fm"]), items, P, C, elu, p(o["bf"]),
                                                                           p(o["bm"]), p(o["scale"]), p(o["mean"]), p(o["inv"]),
                                                                           p(o["s0"]), p(o["s1"]), p(dfm.out), *sp, *ws, st))
    elif kind == "bn":
        L.check(getattr(lib, "read_bn_backward_reduce" + sfx)(p(o["dy"]), p(o["fm"]), n, C, elu, p(o["bf"]), p(o["bm"]),
                                                              p(o["mean"]), p(o["inv"]), *sp, *ws, st))
    else:
        L.check(getattr(lib, "read_bn_backward_reduce_items" + sfx)(p(o["dy"]), p(o["fm"]), items, P, C, elu, p(o["bf"]),
                                                                    p(o["bm"]), p(o["mean"]), p(o["inv"]), *sp, *ws, st))
    torch.cuda.synchronize()
    what = f"{kind}{sfx} items={items} P={P} C={C} elu={elu}"
    for s in sums:
        s.check(what + " sums")
    if dfm is not None:
        dfm.check(what + " dfm")
    names = {"gate": ["dbias_f", "dbias_m", "dgamma", "dbeta"], "bn": ["sum_dy", "sum_dy_xhat"],
             "bn_items": ["sum_dy", "sum_dy_xhat"]}.get(kind, ["dbias_f", "dbias_m"])
    return (None if dfm is None else dfm.out.view(n, 2 * C)), {k: s.out.view(rows, C) for k, s in zip(names, sums)}, what


GATE_EXACT = [(C, 3, P) for C in U.GATE_CS for P in U.gate_item_pixels(C)] + [(C, it, P) for C, it, P in U.GATE_BIG]


@gpu
@pytest.mark.parametrize("C,items,P", GATE_EXACT)
def test_gate_and_bn_dy_sums_are_exact(C, items, P):
    """dbeta (eval gate) and sum_dy (call-wide and per item) of integer dy: the exact sums over each item's pixels, onto a pre-fill."""
    o = _gate_operands(items, P, C, seed=C * 1000 + items + P, int_dy=True)
    dy = o["dy"].double().reshape(items, P, C)
    per_item, total = dy.sum(1), dy.sum((0, 1))
    pre = 7.0
    for det in (False, True):
        for elu in (0, 1):
            _, s, what = _gate_run("gate", o, items, P, C, elu, det, pre)
            U.assert_exact(s["dbeta"][0], pre + total, what + " dbeta", ["c"])
            _, s, what = _gate_run("bn", o, items, P, C, elu, det, pre)
            U.assert_exact(s["sum_dy"][0], pre + total, what + " sum_dy", ["c"])
            if P >= 2:
                _, s, what = _gate_run("bn_items", o, items, P, C, elu, det, pre)
                U.assert_exact(s["sum_dy"], pre + per_item, what + " sum_dy", ["item", "c"])


GATE_BOUND = [(C, 3, P) for C in U.GATE_CS for P in (2, U.ppb(C) + 1, 37 * 41)] + [(64, 64, 64 * 64), (32, 1, 8 * 128 * 128)]


@gpu
@pytest.mark.parametrize("C,items,P", GATE_BOUND)
def test_gate_and_bn_backward_within_per_element_bounds(C, items, P):
    o = _gate_operands(items, P, C, seed=C * 7 + items * 3 + P, spread=True)
    one = {k: (v[:1] if k in ("scale", "mean", "inv", "s0", "s1") else v) for k, v in o.items()}   # call-wide statistics
    for elu in (0, 1):
        for det in (False, True):
            for kind in ("gate", "gate_batch", "gate_items", "bn", "bn_items"):
                per_item = kind.endswith("items")
                if kind != "gate" and P * (1 if per_item else items) < 2:
                    continue
                ops_ = o if per_item else one
                ref = U.gate_ref(ops_, C, elu, {"gate": "eval", "gate_batch": "batch", "gate_items": "items"}.get(kind, "eval"),
                                 items if per_item else 1, P if per_item else items * P)
                dfm, s, what = _gate_run(kind, ops_, items, P, C, elu, det)
                if dfm is not None:
                    _worst("dfm (bf16)", U.assert_bound(dfm, ref["dfm"], ref["T_dfm"], U.TAU, what + " dfm", rel=U.REL_BF16,
                                                        names=["pixel", "column"]))
                    _worst("dfm tau share", U.tau_share(dfm, ref["dfm"], ref["T_dfm"], U.TAU, U.REL_BF16))
                    _worst("dbias sums", U.assert_bound(s["dbias_f"][0], ref["sum_df"], ref["T_sum"], U.TAU_S, what + " dbias_f",
                                                        names=["c"]))
                    _worst("dbias sums", U.assert_bound(s["dbias_m"][0], ref["sum_dm"], ref["T_sum"], U.TAU_S, what + " dbias_m",
                                                        names=["c"]))
                if kind == "gate":
                    _worst("dgamma / sum_dy_xhat", U.assert_bound(s["dgamma"][0], ref["dgamma"], ref["T_dgamma"], U.TAU_S,
                                                                  what + " dgamma", names=["c"]))
                if kind in ("bn", "bn_items"):
                    want = ref["sum_xh"] if per_item else ref["sum_xh"].sum(0, keepdim=True)
                    T = ref["T_xh"] if per_item else ref["T_xh"].sum(0, keepdim=True)
                    _worst("dgamma / sum_dy_xhat", U.assert_bound(s["sum_dy_xhat"], want, T, U.TAU_S, what + " sum_dy_xhat",
                                                                  names=["item", "c"]))


@gpu
@pytest.mark.parametrize("C", U.GATE_CS)
def test_gate_impulse_touches_only_its_two_columns(C):
    """Eval-mode gate backward of a one-element output gradient: [df | dm] is exactly 0 everywhere but that pixel's f and m columns."""
    P = 3 * U.ppb(C) + 5
    o = _gate_operands(1, P, C, seed=C)
    fmcols = U.fm_columns(C)
    for (px, ch) in ((0, 0), (P - 1, C - 1), (U.ppb(C), C // 2 + 1)):
        dy = torch.zeros((P, C))
        dy[px, ch] = 3.0
        o["dy"] = dy.bfloat16().to(dev())
        for det in (False, True):
            dfm, _, what = _gate_run("gate", o, 1, P, C, 1, det)
            nz = dfm.float().nonzero().tolist()
            allowed = {(px, int(j)) for j in range(2 * C) if int(fmcols[j]) in (ch, C + ch)}
            assert {tuple(e) for e in nz} <= allowed, f"{what}: impulse at pixel {px} channel {ch} wrote {nz[:6]}"


# ------------------------------------------------------------------ descriptor scatter
def _ids(B, h, w, N, g, zero_frac=0.5):
    """Half the pixels on point 0, the rest from a small pool (many duplicates) plus ids that clamp: negative and >= N."""
    n = B * h * w
    pool = torch.randint(0, N, (max(N // 16, 3),), generator=g)
    ids = pool[torch.randint(0, len(pool), (n,), generator=g)].float()
    r = torch.rand(n, generator=g)
    ids[r < zero_frac] = 0
    ids[(r >= zero_frac) & (r < zero_frac + 0.03)] = -3.0
    ids[(r >= zero_frac + 0.03) & (r < zero_frac + 0.06)] = float(N + 17)
    ids[(r >= zero_frac + 0.06) & (r < zero_frac + 0.09)] = float(N - 1)
    return ids.reshape(B, h, w)


GATHER_CASES = [(1, 8, 3, 17, 23), (2, 8, 2, 9, 31), (5000, 8, 3, 33, 47), (3000, 5, 2, 16, 16), (200000, 8, 8, 256, 256)]


@gpu
@pytest.mark.parametrize("N,D,B,h,w", GATHER_CASES)
def test_gather_backward_is_exact(N, D, B, h, w):
    lib, st = L.load(), L.stream_ptr()
    g = _gen("gather", N, D, B, h, w)
    go = U.int_tensor((B, D, h, w), 8, g)
    ids = _ids(B, h, w, N, g)
    pre = U.int_tensor((N, D), 100, g, zero_frac=0.2)
    want = torch.from_numpy(U.gather_ref(go.numpy(), ids.numpy(), N, pre.numpy()))
    seen = torch.zeros(N, dtype=torch.uint8)
    seen[ids.long().clamp(0, N - 1).reshape(-1)] = 1
    god, idd = go.to(dev()), ids.to(dev())
    for sparse in (False, True):
        for det in (False, True):
            if sparse and D != 8:
                continue
            out = U.Guarded(N * D, torch.float32, dev(), pre)
            tch = U.Guarded(N, torch.uint8, dev())
            wst = _ws(lib.read_gather_backward_det_workspace_bytes(B, D, h, w, N)) if det else None
            ws = [wst.data_ptr()] if det else []
            name = "read_gather_backward" + ("_sparse" if sparse else "") + ("_det" if det else "")
            extra = [tch.out.data_ptr()] if sparse else []
            L.check(getattr(lib, name)(god.data_ptr(), idd.data_ptr(), B, D, h, w, N, out.out.data_ptr(), *extra, *ws, st))
            torch.cuda.synchronize()
            what = f"{name} N={N} D={D} B={B} {h}x{w}"
            out.check(what)
            tch.check(what + " touched")
            U.assert_exact(out.out.view(N, D), want, what, ["id", "c"])
            if sparse:
                U.assert_exact(tch.out, seen, what + " touched", ["id"])


@gpu
@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
def test_gather_backward_items_is_exact(sparse, det):
    """16 slots x 64 items: slots of 1, 2 and many points, a slot that receives nothing, every item's pixels into its own slot."""
    lib, st = L.load(), L.stream_ptr()
    g = _gen("items", sparse, det)
    n_items, h, w = 64, 24, 20
    NS = [1, 2, 3, 700, 64, 5000, 1, 129, 2, 333, 4096, 7, 50, 2, 999, 17]
    slots = torch.randint(0, len(NS), (n_items,), generator=g).tolist()
    slots[:len(NS)] = range(len(NS))                        # every slot used
    go = U.int_tensor((n_items, 8, h, w), 8, g)
    ids = torch.stack([_ids(1, h, w, NS[s], g)[0] for s in slots])
    receives = [s != 5 for s in range(len(NS))]             # slot 5 has no accumulator
    pre = [U.int_tensor((n, 8), 100, g, zero_frac=0.2) for n in NS]
    outs = [U.Guarded(n * 8, torch.float32, dev(), p) if r else None for n, p, r in zip(NS, pre, receives)]
    tch = [U.Guarded(n, torch.uint8, dev()) for n in NS]
    t = ops.tex_table(slots, NS, grad=[o.out if o is not None else None for o in outs],
                      touched=[x.out for x in tch] if sparse else None)
    god, idd = go.to(dev()), ids.to(dev())
    name = "read_gather_backward" + ("_sparse" if sparse else "") + "_items" + ("_det" if det else "")
    wst = _ws(lib.read_gather_backward_det_workspace_bytes(n_items, 8, h, w, sum(NS))) if det else None
    ws = [wst.data_ptr()] if det else []
    L.check(getattr(lib, name)(god.data_ptr(), idd.data_ptr(), ctypes.byref(t), h, w, *ws, st))
    torch.cuda.synchronize()
    for s, n in enumerate(NS):
        items = [b for b in range(n_items) if slots[b] == s]
        want = U.gather_ref(go[items].numpy(), ids[items].numpy(), n, pre[s].numpy())
        what = f"{name} slot {s} (N={n}, items {items})"
        tch[s].check(what + " touched")
        if outs[s] is None:
            assert not bool(tch[s].out.any()), what + ": a slot without accumulator was touched"
            continue
        outs[s].check(what)
        U.assert_exact(outs[s].out.view(n, 8), torch.from_numpy(want), what, ["id", "c"])
        if sparse:
            seen = torch.zeros(n, dtype=torch.uint8)
            seen[ids[items].long().clamp(0, n - 1).reshape(-1)] = 1
            U.assert_exact(tch[s].out, seen, what + " touched", ["id"])
