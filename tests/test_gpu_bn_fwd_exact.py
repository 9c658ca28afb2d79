"""-m gpu: per-element checks of train-mode BatchNorm's forward (csrc/bn_train.cu) at every CTA, item and stride edge: the
statistics of integer-valued inputs against their exact values within the bounds of bn_fwd_exact_util, the running statistics as a
bit-exact replay of the kernel's update on its own outputs and within a float64 bound, and the apply bit for bit against its fp32
formula.  Every output sits between guard bands that must stay unchanged."""
import numpy as np
import pytest
import torch

import bn_fwd_exact_util as B
from bwd_exact_util import Guarded, assert_exact
from gpu_util import dev
from read_b200 import _lib as L

pytestmark = pytest.mark.gpu

N_STATS = len(B.stats_cases(132))            # the list has the same structure for every SM count
N_APPLY = len(B.apply_cases(132))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nan(n):
    return torch.full((n,), float("nan"), dtype=torch.float32)


def _stats(lib, case, x, gamma, beta, rm, rv, ws=None):
    """One statistics call on x [items, P, C]; returns the outputs (numpy [items, C]), the running statistics and the
    workspace.  Every output is guarded and pre-filled with NaN."""
    items, P, C, nr = case.items, case.P, case.C, case.n_real
    gd = torch.from_numpy(x).to(dev()).bfloat16().contiguous()
    outs = {k: Guarded(items * C, torch.float32, dev(), _nan(items * C)) for k in ("mean", "inv_std", "scale", "shift")}
    var = None if case.per_item else Guarded(C, torch.float32, dev(), _nan(C))
    run = {k: Guarded(nr, torch.float32, dev(), torch.from_numpy(v)) for k, v in (("rm", rm), ("rv", rv))}
    gt, bt = torch.from_numpy(gamma).to(dev()), torch.from_numpy(beta).to(dev())
    if ws is None:
        nbytes = lib.read_bn_workspace_bytes_items(items, C) if case.per_item else lib.read_bn_workspace_bytes(C)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=dev())
    p = lambda k: outs[k].out.data_ptr()
    head = (gd.data_ptr(), items, P) if case.per_item else (gd.data_ptr(), P)
    tail = (run["rm"].out.data_ptr(), run["rv"].out.data_ptr(), p("mean"), p("inv_std"))
    tail += () if case.per_item else (var.out.data_ptr(),)
    fn = lib.read_bn_batch_stats_items if case.per_item else lib.read_bn_batch_stats
    L.check(fn(*head, C, nr, gt.data_ptr(), bt.data_ptr(), B.EPS, case.momentum, *tail, p("scale"), p("shift"), ws.data_ptr(),
               L.stream_ptr()))
    torch.cuda.synchronize()
    for k, gbuf in list(outs.items()) + list(run.items()) + ([("var", var)] if var else []):
        gbuf.check(f"{case.id} {k}")
    got = {k: v.out.cpu().numpy().reshape(items, C) for k, v in outs.items()}
    if var is not None:
        got["var"] = var.out.cpu().numpy().reshape(1, C)
    else:
        off = B.ws_layout(True, items, C)[0]
        got["uvar"] = ws[off:off + items * C * 4].view(torch.float32).cpu().numpy().reshape(items, C)
    return got, run["rm"].out.cpu().numpy(), run["rv"].out.cpu().numpy(), ws


def _check_case(case, got, grm, grv, x, gamma, beta, rm, rv, sms):
    """The statistics within their bounds, the padded channels exact, the running statistics replayed and bounded; returns the
    worst share of each bound."""
    items, P, C, nr = case.items, case.P, case.C, case.n_real
    bnd = B.stats_bounds(x, sms, gamma, beta, nr)
    vk = "uvar" if case.per_item else "var"
    worst = B.check_stats(got, bnd, case.id, ["mean", "inv_std", "scale", "shift", vk])
    pad = slice(nr, C)
    for k in ("mean", "scale", "shift", vk):
        assert_exact(torch.from_numpy(got[k][:, pad]), torch.zeros(got[k][:, pad].shape), f"{case.id} padded {k}")
    rs = np.float32(1.0 / np.sqrt(np.float64(np.float32(B.EPS))))
    assert_exact(torch.from_numpy(got["inv_std"][:, pad]), torch.full(got["inv_std"][:, pad].shape, float(rs)),
                 f"{case.id} padded inv_std")
    # running statistics: bit-exact replay on the kernel's own outputs, and within the float64 bound of the exact update
    if case.per_item:
        wm, wv = B.running_items_replay(rm, rv, got["mean"][:, :nr], got["uvar"][:, :nr], case.momentum)
        assert_exact(torch.from_numpy(grm), torch.from_numpy(wm), f"{case.id} running_mean replay", ["c"])
        assert_exact(torch.from_numpy(grv), torch.from_numpy(wv), f"{case.id} running_var replay", ["c"])
    else:
        wm, _ = B.running_items_replay(rm, rv, got["mean"][:, :nr], got["mean"][:, :nr], case.momentum)
        assert_exact(torch.from_numpy(grm), torch.from_numpy(wm), f"{case.id} running_mean replay", ["c"])
        cand = B.running_call_candidates(rv, got["var"][0, :nr].astype(np.float64), P, case.momentum)
        ok = (grv >= cand.min(0)) & (grv <= cand.max(0))
        assert ok.all(), (f"{case.id} running_var outside the replays of the fp32 values around var * P / (P - 1)",
                          np.nonzero(~ok)[0][:6], grv[~ok][:6], cand[:, ~ok][:, :6])
    (bm, em), (bv, ev) = B.running_bound(rm, rv, tuple(a[:, :nr] for a in bnd["mean"]),
                                         tuple(a[:, :nr] for a in bnd["uvar"]), case.momentum)
    for name, g, w, e in (("running_mean", grm, bm, em), ("running_var", grv, bv, ev)):
        err = np.abs(g.astype(np.float64) - w)
        assert (err <= e).all(), (f"{case.id} {name} beyond its float64 bound", np.nonzero(err > e)[0][:6])
        worst[name] = float(np.max(np.where(e > 0, err / np.where(e > 0, e, 1), 0), initial=0))
    return worst


@pytest.mark.parametrize("i", range(N_STATS), ids=[c.id for c in B.stats_cases(132)])
def test_batch_stats_within_exact_bounds(i):
    sms = _sms()
    case = B.stats_cases(sms)[i]
    x, gamma, beta, rm, rv = B.stats_operands(case)
    a2, a1 = B.sums_precondition(case, x, sms)
    assert a2 < B.EXACT_LIMIT and a1 < B.EXACT_LIMIT
    got, grm, grv, _ = _stats(L.load(), case, x, gamma, beta, rm, rv)
    worst = _check_case(case, got, grm, grv, x, gamma, beta, rm, rv, sms)
    print(f"\n{case.id}: worst err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))


@pytest.mark.parametrize("per_item", [False, True], ids=["call", "items"])
def test_consecutive_calls_share_one_workspace(per_item):
    """A call over many pixels (a full grid of partials), then one over few on the same workspace: the second must read none of
    the first's partials or counters."""
    sms, lib = _sms(), L.load()
    items = 3 if per_item else 1
    C = 64
    big = B.Case(per_item, items, 3 * B.stats_cap(sms) * B.ppb(C) + 11, C, 56, momentum=0.1, seed=200)
    small = B.Case(per_item, items, 37, C, 56, momentum=0.1, seed=201)
    ws = None
    for case in (big, small, big):
        x, gamma, beta, rm, rv = B.stats_operands(case)
        got, grm, grv, ws = _stats(lib, case, x, gamma, beta, rm, rv, ws)
        _check_case(case, got, grm, grv, x, gamma, beta, rm, rv, sms)


@pytest.mark.parametrize("i", range(N_APPLY), ids=[f"B{c[0]}-P{c[1]}-C{c[2]}" for c in B.apply_cases(132)])
def test_apply_bit_exact(i):
    sms, lib = _sms(), L.load()
    items, P, C = B.apply_cases(sms)[i]
    n = items * P * C
    for k, residual in enumerate((False, True)):
        g, scale, shift, r = B.apply_operands(items, P, C, residual, seed=i * 2 + k)
        want = torch.from_numpy(B.apply_replay(g, scale, shift, r).reshape(-1))
        gd = torch.from_numpy(g).to(dev()).bfloat16().reshape(-1)
        rd = torch.from_numpy(r).to(dev()).bfloat16().reshape(-1) if residual else None
        sd, hd = torch.from_numpy(scale).to(dev()), torch.from_numpy(shift).to(dev())
        for in_place in (False, True):
            what = f"apply B{items} P{P} C{C} residual={residual} in_place={in_place}"
            yb = Guarded(n, torch.bfloat16, dev(), gd if in_place else None)
            src = yb.out if in_place else gd
            if items > 1:
                L.check(lib.read_bn_apply_items(src.data_ptr(), items, P, C, sd.data_ptr(), hd.data_ptr(), L.ptr(rd),
                                                yb.out.data_ptr(), L.stream_ptr()))
            else:
                L.check(lib.read_bn_apply(src.data_ptr(), P, C, sd.data_ptr(), hd.data_ptr(), L.ptr(rd), yb.out.data_ptr(),
                                          L.stream_ptr()))
            torch.cuda.synchronize()
            yb.check(what)
            assert_exact(yb.out.view(torch.int16).cpu().reshape(items, P, C), want.reshape(items, P, C), what,
                         ["item", "p", "c"])
