"""Host checks (no GPU) of rmsprop_exact_util, the replays of test_gpu_rmsprop_exact.py: the case list reaches every path and
edge, the replay of one dense step agrees with torch.optim.RMSprop's on the CPU to 2^-18 relative, and the checks reject
a decay of alpha^(dt - 1), a missing shadow write and a cleared gradient row of an untouched point."""
import numpy as np
import pytest
import torch

import rmsprop_exact_util as R
from bwd_exact_util import assert_exact

SMS_LIST = (132, 114)


@pytest.mark.parametrize("sms", SMS_LIST)
def test_cases_reach_every_path(sms):
    seen = set().union(*(R.case_classes(c, sms) for c in R.cases(sms)))
    want = {f"D={d}" for d in R.DS} | {f"alpha={a}" for a in R.ALPHAS} | {f"variant={v}" for v in ("plain", "wd", "reg", "reg0")}
    want |= {"vector path", "generic loop", "grid-stride tail", "N=1", "N=255", "N=257", "N=2^24+1"}
    assert want <= seen, want - seen
    assert {c[1] for c in R.cases(sms)} >= {R.big_n(sms) - 1, R.big_n(sms) + 1}


def test_operands_cover_every_gap_and_the_eps_regime():
    p, g, q, touched, last = R.operands(8, 5000, seed=1)
    dts = set((R.STEP - last).tolist())
    assert dts == set(R.GAPS) and (last >= 0).all()
    zero_q = (q == 0).all(1)
    assert zero_q.any() and (np.abs(g[zero_q]) < 1e-7).all()
    # the denominator of those rows is eps's: sqrt((1 - alpha) g^2) << eps
    assert (np.sqrt(np.float32(0.01) * g[zero_q] ** 2) < 1e-9).all()
    assert 0.25 < touched.mean() < 0.45 and (g[touched == 0] != 0).any()


def test_gap_of_1e5_underflows_and_bounds_hold():
    lo, hi = R.decay_range(0.99, np.array([100_000, 1000, 2]))
    assert lo[0] == 0 and hi[0] < 1e-44                           # 0.99^1e5 underflows fp32
    assert lo[1] < np.float32(0.99) ** 1000 < hi[1] or abs(lo[1] - 0.99 ** 1000) < 1e-9
    assert lo[2] <= np.float32(0.99) * np.float32(0.99) <= hi[2]
    lo, hi = R.decay_range(0.0, np.array([2, 7]))
    assert (lo == 0).all() and (hi < 1e-44).all()


def test_dt1_replay_equals_torch_rmsprop_on_cpu():
    """All points touched at dt = 1: the replay is torch's dense step up to its roundings.  torch rounds alpha * q and
    g * g * (1 - alpha) separately, and takes 1 - alpha in float64 before rounding it to fp32, while the kernel uses
    1.f - alpha (1e-6 relative apart at alpha = 0.99): the two agree to 2^-18 relative."""
    D, N = 8, 3000
    p, g, q, touched, last = R.operands(D, N, seed=3, all_touched=True)
    last[:] = R.STEP - 1
    want = R.step_replay(p, g, q, touched, last, 0.1, 0.99, 1e-8, 0.0)
    ref = torch.from_numpy(p.copy()[None]).requires_grad_(True)
    opt = torch.optim.RMSprop([ref], lr=0.1, alpha=0.99, eps=1e-8)
    opt.state[ref]["step"] = torch.tensor(1.0)
    opt.state[ref]["square_avg"] = torch.from_numpy(q.T.copy()[None])
    ref.grad = torch.from_numpy(g.T.copy()[None])
    opt.step()
    sq = opt.state[ref]["square_avg"][0].numpy()
    assert np.allclose(sq, want["sq_lo"].T, rtol=2.0 ** -18, atol=0)
    assert np.allclose(ref.detach()[0].numpy(), want["param"], rtol=2.0 ** -18, atol=2e-6)


def _planted(D, N, variant):
    p, g, q, touched, last = R.operands(D, N, seed=D * 7 + N)
    k = 0.37 if variant == "reg" else None
    wd = 1e-2 if variant == "wd" else 0.0
    good = R.step_replay(p, g, q, touched, last, 0.1, 0.9, 1e-8, wd, k)
    return p, g, q, touched, last, k, wd, good


@pytest.mark.parametrize("D", [8, 3])
@pytest.mark.parametrize("variant", ["plain", "wd", "reg"])
def test_checks_reject_planted_defects(D, variant):
    N = 3000
    p, g, q, touched, last, k, wd, good = _planted(D, N, variant)
    proc = good["proc"]
    # alpha^(dt - 1) for alpha^dt: square_avg leaves the powf range at the processed points with dt = 2 or 7 (at 1000 and 10^5
    # both powers of 0.9 underflow to the same few denormals)
    bad = R.step_replay(p, g, q, touched, last + 1, 0.1, 0.9, 1e-8, wd, k)["sq_lo"]
    dt = R.STEP - last
    sel = proc & np.isin(dt, (2, 7)) & (q > 0).all(1)
    assert sel.any()
    out = (bad[sel] < good["sq_lo"][sel]) | (bad[sel] > good["sq_hi"][sel])
    assert out.all(1).mean() > 0.9
    # the parameter replayed on a square_avg that is off by one ulp differs somewhere
    q_off = np.nextafter(good["sq_lo"], np.float32(np.inf))
    off = R.step_replay(p, g, q, touched, last, 0.1, 0.9, 1e-8, wd, k, q_kernel=q_off)["param"]
    with pytest.raises(AssertionError):
        assert_exact(torch.from_numpy(off.view(np.int32)), torch.from_numpy(good["param"].view(np.int32)), "param")
    # a missing shadow write on the last channel (the D != 8 loop's last iteration)
    sh = good["shadow"].copy()
    sh[proc, D - 1] = p.T[proc, D - 1]
    with pytest.raises(AssertionError):
        assert_exact(torch.from_numpy(sh.view(np.int32)), torch.from_numpy(good["shadow"].view(np.int32)), "shadow")
    # a cleared gradient row of an untouched point
    gr = good["grad"].copy()
    untouched = np.nonzero((touched == 0) & (g != 0).any(1))[0]
    gr[untouched[0]] = 0
    with pytest.raises(AssertionError):
        assert_exact(torch.from_numpy(gr.view(np.int32)), torch.from_numpy(good["grad"].view(np.int32)), "grad")
    # non-REG steps leave every untouched point unchanged; REG steps update them all
    if k is None:
        assert (good["param"][:, ~proc].view(np.int32) == p[:, ~proc].view(np.int32)).all()
        assert (good["last"][~proc] == last[~proc]).all()
    else:
        assert proc.all() and (good["param"][:, touched == 0] != p[:, touched == 0]).any()


def test_integer_cases_stay_exact():
    """The scatter test's sums stay below 2^24 whatever the order of the atomics: the largest |prefill| + n * |value|."""
    assert 1000 + 40000 * 64 < 2 ** 24
