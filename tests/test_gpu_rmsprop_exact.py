"""-m gpu: per-element checks of the sparse descriptor optimizer's kernels (csrc/train.cu) called through their entry points on
prepared state: the step (both instances, the vector D = 8 path and the generic loop, gaps up to 10^5 steps, alpha 0.99 / 0.9 / 0,
past one pass of the grid) bit for bit where it is correctly rounded and within powf's documented error where it is not; the dense
square_avg; the compaction of touched rows under a short capacity; the scatter of (id, row) pairs with repeated and out-of-range
ids; and SparseRMSprop with weight decay against torch.optim.RMSprop.  Every output sits between guard bands."""
import numpy as np
import pytest
import torch

import rmsprop_exact_util as R
from bwd_exact_util import Guarded, assert_exact
from gpu_util import dev
from read_b200 import _lib as L, train
from read_b200.texture import PointTexture

pytestmark = pytest.mark.gpu

LR, EPS, WD, K = 0.1, 1e-8, 1e-2, 0.37
N_CASES = len(R.cases(132))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _g(a, dtype):
    t = torch.from_numpy(np.ascontiguousarray(a).reshape(-1))
    return Guarded(t.numel(), dtype, dev(), t)


def _bits(a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32))


def _step(lib, state, D, N, variant, alpha, step, shadow=True):
    """One call on the guarded state (dict of Guarded); returns the outputs as numpy."""
    wd = WD if variant in ("wd", "reg0") else 0.0
    args = [state["param"].out.data_ptr(), state["shadow"].out.data_ptr() if shadow else None, state["grad"].out.data_ptr(),
            state["touched"].out.data_ptr(), state["sq"].out.data_ptr(), state["last"].out.data_ptr(), N, D, step, LR, alpha, EPS,
            wd]
    if variant in ("reg", "reg0"):
        coef = torch.tensor(K if variant == "reg" else 0.0, dtype=torch.float32, device=dev())
        L.check(lib.read_sparse_rmsprop_step_reg(*args, coef.data_ptr(), L.stream_ptr()))
    else:
        L.check(lib.read_sparse_rmsprop_step(*args, L.stream_ptr()))
    torch.cuda.synchronize()
    for k, v in state.items():
        v.check(f"{variant} D{D} N{N} {k}")
    get = lambda k: state[k].out.cpu().numpy()
    return {"param": get("param").reshape(D, N), "shadow": get("shadow").reshape(N, D), "grad": get("grad").reshape(N, D),
            "sq": get("sq").reshape(N, D), "last": get("last"), "touched": get("touched")}


def _check(got, p, g, q, touched, last, D, N, variant, alpha, step, what, shadow_p=None):
    wd = WD if variant in ("wd", "reg0") else 0.0
    k = K if variant == "reg" else 0.0 if variant == "reg0" else None
    want = R.step_replay(p, g, q, touched, last, LR, alpha, EPS, wd, k, step=step, q_kernel=got["sq"])
    lo, hi = want["sq_lo"], want["sq_hi"]
    ok = (got["sq"] >= lo) & (got["sq"] <= hi)
    if not ok.all():
        i, c = np.argwhere(~ok)[0]
        raise AssertionError(f"{what} square_avg: {int((~ok).sum())} elements outside the replay range, e.g. [i={i}, c={c}] got "
                             f"{got['sq'][i, c]!r} range [{lo[i, c]!r}, {hi[i, c]!r}] dt {step - int(last[i])}")
    assert_exact(_bits(got["param"]), _bits(want["param"]), f"{what} param bits", ["c", "i"])
    shadow_want = want["shadow"] if shadow_p is None else shadow_p
    assert_exact(_bits(got["shadow"]), _bits(shadow_want), f"{what} shadow bits", ["i", "c"])
    assert_exact(_bits(got["grad"]), _bits(want["grad"]), f"{what} grad bits", ["i", "c"])
    assert_exact(torch.from_numpy(got["last"]), torch.from_numpy(want["last"]), f"{what} last_step", ["i"])
    assert_exact(torch.from_numpy(got["touched"]), torch.from_numpy(want["touched"]), f"{what} touched", ["i"])
    # the share of powf's range the kernel used: |got - mid| over the distance from mid to the range's end on that side
    mid, g64 = want["sq_mid"].astype(np.float64), got["sq"].astype(np.float64)
    end = np.where(g64 >= mid, hi, lo).astype(np.float64)
    share = np.where(end != mid, np.abs(g64 - mid) / np.where(end != mid, np.abs(end - mid), 1), 0)
    return int(want["proc"].sum()), float(share.max(initial=0))


@pytest.mark.parametrize("i", range(N_CASES), ids=[f"D{d}-N{n}-{v}-a{a}" for d, n, v, a in R.cases(132)])
def test_step_replayed_per_element(i):
    lib = L.load()
    D, N, variant, alpha = R.cases(_sms())[i]
    p, g, q, touched, last = R.operands(D, N, seed=i)
    state = {"param": _g(p, torch.float32), "shadow": _g(p.T, torch.float32), "grad": _g(g, torch.float32),
             "touched": _g(touched, torch.uint8), "sq": _g(q, torch.float32), "last": _g(last, torch.int32)}
    what = f"D{D} N{N} {variant} alpha {alpha}"
    got = _step(lib, state, D, N, variant, alpha, R.STEP)
    n_proc, share = _check(got, p, g, q, touched, last, D, N, variant, alpha, R.STEP, what)
    assert n_proc > 0 or N == 1
    print(f"\n{what}: {n_proc} points updated, worst share of the powf range {share:.3g}")
    # a second step on the state the first left: new gradients on a new touched set, dt = 1 for the points just updated
    rng = np.random.default_rng(100 + i)
    t2 = (rng.random(N) < 0.5).astype(np.uint8)
    g2 = got["grad"].copy()
    g2[t2.astype(bool)] = np.float32(rng.standard_normal((int(t2.sum()), D)) * 0.3)
    state["grad"].out.copy_(torch.from_numpy(g2.reshape(-1)))
    state["touched"].out.copy_(torch.from_numpy(t2))
    got2 = _step(lib, state, D, N, variant, alpha, R.STEP + 1)
    _check(got2, got["param"], g2, got["sq"], t2, got["last"], D, N, variant, alpha, R.STEP + 1, what + " second step")


@pytest.mark.parametrize("D", [8, 3])
def test_step_without_shadow(D):
    lib, N = L.load(), 1000
    p, g, q, touched, last = R.operands(D, N, seed=77)
    state = {"param": _g(p, torch.float32), "shadow": _g(p.T, torch.float32), "grad": _g(g, torch.float32),
             "touched": _g(touched, torch.uint8), "sq": _g(q, torch.float32), "last": _g(last, torch.int32)}
    got = _step(lib, state, D, N, "plain", 0.99, R.STEP, shadow=False)
    _check(got, p, g, q, touched, last, D, N, "plain", 0.99, R.STEP, f"no shadow D{D}", shadow_p=np.ascontiguousarray(p.T))


@pytest.mark.parametrize("D", [8, 3])
@pytest.mark.parametrize("alpha", R.ALPHAS)
def test_square_avg_dense(D, alpha):
    lib, N = L.load(), 4099
    _, _, q, _, last = R.operands(D, N, seed=9)
    step = R.STEP
    rng = np.random.default_rng(11)
    last[rng.random(N) < 0.2] = step                          # dt = 0
    last[rng.random(N) < 0.1] = step + 5                      # dt < 0: no decay either
    qd, ld = torch.from_numpy(q).to(dev()), torch.from_numpy(last).to(dev())
    out = Guarded(D * N, torch.float32, dev(), torch.full((D * N,), float("nan")))
    L.check(lib.read_square_avg_dense(qd.data_ptr(), ld.data_ptr(), N, D, step, alpha, out.out.data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    out.check("square_avg_dense")
    got = out.out.cpu().numpy().reshape(D, N)
    lo, hi = R.dense_replay(q, last, step, alpha)
    keep = (step - last.astype(np.int64)) <= 0
    assert_exact(_bits(got[:, keep]), _bits(np.ascontiguousarray(q.T[:, keep])), "dense square_avg, dt <= 0", ["c", "i"])
    ok = (got >= lo) & (got <= hi)
    assert ok.all(), ("dense square_avg outside powf's bound", np.argwhere(~ok)[:6])


@pytest.mark.parametrize("N", [1, 31, 33, 1000, 16 * 132 * 256 + 1])
@pytest.mark.parametrize("cap_kind", ["zero", "half", "exact", "more"])
def test_compact_touched(N, cap_kind):
    lib, D = L.load(), 3
    rng = np.random.default_rng(N)
    touched = (rng.random(N) < 0.4).astype(np.uint8)
    touched[-1] = 1
    n_t = int(touched.sum())
    cap = {"zero": 0, "half": n_t // 2, "exact": n_t, "more": n_t + 5}[cap_kind]
    g = np.float32(rng.standard_normal((N, D)))
    gd, td = torch.from_numpy(g).to(dev()), torch.from_numpy(touched).to(dev())
    cnt = torch.zeros(1, dtype=torch.int32, device=dev())
    ids = Guarded(cap, torch.int32, dev(), torch.full((cap,), -7, dtype=torch.int32))
    rows = Guarded(cap * D, torch.float32, dev(), torch.full((cap * D,), -7.0))
    # the interiors' addresses taken from the buffers: an empty view (capacity 0) has no data pointer of its own
    L.check(lib.read_compact_touched(gd.data_ptr(), td.data_ptr(), N, D, cnt.data_ptr(), cap, ids.buf[ids.guard:].data_ptr(),
                                     rows.buf[rows.guard:].data_ptr(), L.stream_ptr()))
    torch.cuda.synchronize()
    ids.check("compact ids")
    rows.check("compact rows")
    assert int(cnt.item()) == n_t
    got_ids, got_rows = ids.out.cpu().numpy(), rows.out.cpu().numpy().reshape(cap, D)
    m = min(cap, n_t)
    sel = got_ids[:m]
    assert len(set(sel.tolist())) == m and (touched[sel] == 1).all(), "compacted ids: not distinct touched rows"
    assert_exact(_bits(got_rows[:m]), _bits(g[sel]), "compacted rows", ["k", "c"])
    assert (got_ids[m:] == -7).all() and (got_rows[m:] == -7).all(), "written past the touched count"
    if cap >= n_t:
        assert sorted(sel.tolist()) == np.nonzero(touched)[0].tolist()


@pytest.mark.parametrize("D", [8, 3])
def test_scatter_pairs(D):
    lib, N, n = L.load(), 5000, 40000
    rng = np.random.default_rng(D)
    ids = rng.integers(0, 300, n).astype(np.int32) * 16 % N        # few distinct ids, each repeated many times
    ids[rng.random(n) < 0.05] = -1
    ids[rng.random(n) < 0.05] = N
    vals = np.float32(rng.integers(-64, 65, (n, D)))
    pre = np.float32(rng.integers(-1000, 1001, (N, D)))
    pre_t = (rng.random(N) < 0.1).astype(np.uint8)
    gbuf, tbuf = _g(pre, torch.float32), _g(pre_t, torch.uint8)
    idd, vd = torch.from_numpy(ids).to(dev()), torch.from_numpy(vals).to(dev())
    L.check(lib.read_scatter_pairs(idd.data_ptr(), vd.data_ptr(), n, D, N, gbuf.out.data_ptr(), tbuf.out.data_ptr(),
                                   L.stream_ptr()))
    torch.cuda.synchronize()
    gbuf.check("scatter grad")
    tbuf.check("scatter touched")
    want = pre.astype(np.float64)
    ok = (ids >= 0) & (ids < N)
    np.add.at(want, ids[ok], vals[ok].astype(np.float64))
    assert np.abs(want).max() < 2 ** 24
    assert_exact(gbuf.out.cpu().reshape(N, D), torch.from_numpy(want), "scatter sums", ["i", "c"])
    wt = pre_t.copy()
    wt[ids[ok]] = 1
    assert_exact(tbuf.out.cpu(), torch.from_numpy(wt), "scatter touched", ["i"])


def test_weight_decay_matches_dense_rmsprop():
    """SparseRMSprop(weight_decay) against torch.optim.RMSprop(weight_decay) over steps that touch few points: weight decay gives
    every point a gradient, so the untouched ones must move as the dense optimizer moves them."""
    D, N, steps = 8, 20000, 6
    gen = torch.Generator().manual_seed(5)
    t = PointTexture(D, N)
    with torch.no_grad():
        t.texture_.copy_(torch.rand((1, D, N), generator=gen) * 2 - 1)
    t = t.to(dev())
    ref = t.texture_.detach().clone().requires_grad_(True)
    opt = train.SparseRMSprop(t, lr=1e-2, weight_decay=1e-2)
    opt_ref = torch.optim.RMSprop([ref], lr=1e-2, weight_decay=1e-2)
    for s in range(steps):
        sp = train.enable_sparse_grad(t)
        ids = torch.randperm(N - 1, generator=gen)[:300] + 1
        rows = torch.randn((300, D), generator=gen)
        sp.grad[ids.to(dev())] = rows.to(dev())
        sp.touched[ids.to(dev())] = 1
        dense = torch.zeros((1, D, N))
        dense[0, :, ids] = rows.t()
        ref.grad = dense.to(dev())
        opt.step()
        opt_ref.step()
        torch.cuda.synchronize()
        err = (t.texture_.detach() - ref.detach()).abs().max().item()
        assert err <= 2e-5, (s, err)
        assert torch.equal(t.point_major(), t.texture_.detach()[0].t().contiguous())
    sq = opt.dense_square_avg(t)
    sq_ref = opt_ref.state[ref]["square_avg"]
    # the kernel takes 1 - alpha in fp32, torch in float64 before rounding it: 1e-6 relative apart at alpha = 0.99
    assert ((sq - sq_ref).abs() <= 1e-5 * sq_ref.abs() + 1e-12).all()
