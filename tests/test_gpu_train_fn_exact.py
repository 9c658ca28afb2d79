"""-m gpu: per-element checks of the bf16 training autograd Function of read_b200/blocks.py against the float64 replay of its
launches (tests/train_fn_exact_util.py states the method).

* exact tier, eval-mode BatchNorm: block stacks at C = 32 / 64 / 128 / 256 (the role-swapped streamed-weight body with R = 16
  and R = 17 tiles), B = 1 / 2 / 3, one pixel wide, a frozen stack and one whose input needs no gradient; single convs on every
  3x3 stride-1 row of unet.layer_table outside the stacks (FAM*.merge with its residual); gated_conv_srcs on every 1x1 and
  stride-2 row.  Every element of the output, the input gradients, dwf, dbias_f, dgamma and dbeta equals the replay; dwm and
  dbias_m are exactly 0; a residual's gradient is the output gradient bit for bit; the folded scale / shift are the intended
  values.  Under torch.use_deterministic_algorithms(True) the same call gives the same bits.
* train-mode BatchNorm (batch and per-item statistics), single convs and gated_conv_srcs on the same operands: the output is a
  bit-exact replay of bn_apply with the Function's own statistics, and dbeta (a sum of integer output gradients over every
  item) is exact, with and without the deterministic entry points.
* bounded tier, single convs and gated_conv_srcs in eval, batch and per-item modes, with and without the deterministic entry
  points: unpinned gates (saturated and cancelling sigmoid, nonzero m filters) and ELU's negative branch; every element of the
  output, the input gradients, dwf, dwm, dbias_f, dbias_m and dgamma within its bound, dbeta exact.  The worst err / bound of
  each output is printed.
"""
import copy
import types

import pytest
import torch

import train_fn_exact_util as T
from gpu_util import dev
from read_b200 import blocks

pytestmark = pytest.mark.gpu
_OPS = {}


def _operands(case):
    if case not in _OPS:
        _OPS[case] = T.exact_operands(case)
    return _OPS[case]


def _function_node(out):
    """The autograd node of the Function behind ``out`` (through the slice a padded conv's output takes)."""
    todo, seen = [out.grad_fn], set()
    while todo:
        n = todo.pop()
        if n is None or id(n) in seen:
            continue
        seen.add(id(n))
        if hasattr(n, "convs"):
            return n
        todo += [f for f, _ in n.next_functions]
    raise AssertionError("no blocks Function in the graph")


def _call(case, mods, xs, res, gout, mode, det):
    """Run the case's Function on the GPU; returns (out, dxs, dres, grads (6 per conv), FoldedConvs)."""
    ms = [copy.deepcopy(m).to(dev()) for m in mods]
    for m in ms:
        m.train(mode != "eval")
        if mode != "eval":
            m.block['norm'].eps = 1e-5      # the statistics kernels take eps > 0; the checks read the statistics the call used
        if case.need == "frozen":
            m.requires_grad_(False)
    xd = [x.to(dev()).requires_grad_(case.need != "no_x") for x in xs]
    rd = None if res is None else res.to(dev()).requires_grad_(True)
    bs = dict(batch_stats=mode != "eval", per_item=mode == "items")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        if case.family == "stack":
            out = blocks.stack_forward(ms, xd[0], **bs)
        elif case.family == "single":
            out = blocks.gated_conv(ms[0], xd[0], residual=rd, name=case.name, **bs)
        else:
            out = blocks.gated_conv_srcs(ms[0], xd, case.name, **bs)
        node = _function_node(out)
        g = gout.to(dev())
        out.backward(g)
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev)
    convs = node.convs
    grads = []
    for m in ms:
        b = m.block
        for p in (b['conv_f'].weight, b['conv_f'].bias, b['conv_m'].weight, b['conv_m'].bias, b['norm'].weight, b['norm'].bias):
            assert p.grad is None or p.grad.shape == p.shape, (case.id, tuple(p.grad.shape), tuple(p.shape))
            grads.append(p.grad)
    dres = None if rd is None else rd.grad
    if dres is not None:
        assert torch.equal(dres.view(torch.int32), g.view(torch.int32)), f"{case.id}: the residual's gradient is not the output gradient"
    return out.detach(), [x.grad for x in xd], dres, grads, convs


def _bits(t):
    return t.detach().float().cpu().view(torch.int32)


NAMES = T.NAMES


def _check_exact(case, got, r, mods):
    out, dxs, _, grads, convs = got
    T.U.assert_exact(out, r["out"], f"{case.id} output", ["b", "c", "h", "w"])
    for j, (g, w) in enumerate(zip(dxs, r["dxs"])):
        if case.need == "no_x":
            assert g is None, f"{case.id}: an input that needs no gradient got one"
            continue
        T.U.assert_exact(g, w, f"{case.id} input gradient {j}", ["b", "c", "h", "w"])
    for i in range(len(mods)):
        for k, name in enumerate(NAMES):
            g, w = grads[6 * i + k], r["grads"][6 * i + k]
            if case.need == "frozen":
                assert g is None, f"{case.id} conv {i} {name}: a frozen parameter got a gradient"
                continue
            what = f"{case.id} conv {i} {name}"
            if name in ("dwm", "dbias_m"):
                assert bool((g == 0).all()), f"{what}: not exactly 0 with the gate pinned open"
            T.U.assert_exact(g, w, what)
    # the folded BatchNorm the Function used: scale = gamma, shift = beta - running_mean * gamma (eps = 0, running_var = 1)
    for c, m in zip(convs, mods):
        p = T.params64(m)
        n = p["gamma"].numel()
        T.U.assert_exact(c.scale[:n], p["gamma"], f"{case.id} folded scale")
        T.U.assert_exact(c.shift[:n], p["beta"] - p["mean"] * p["gamma"], f"{case.id} folded shift")
        assert bool((c.scale[n:] == 0).all() and (c.shift[n:] == 0).all()), f"{case.id}: padded channels' scale / shift"


@pytest.fixture(scope="module")
def gate_pinned_bwd():
    """Does the gate backward see sigmoid(m + b_m) = 1 exactly at m + b_m = 64?  One conv with f = b_f = 1 (wf = 0), scale 1:
    [df | dm] = [dy | 0] exactly, so dbias_f = sum dy and dbias_m = 0 on integer dy."""
    case = T.Case("pin", "single", (32,), 32, 3, 1, 1, 5, 7, elu=False)
    m = T.make_mods(case)[0]
    with torch.no_grad():
        m.block['conv_f'].weight.zero_()
        m.block['conv_f'].bias.fill_(1.0)
        m.block['conv_m'].weight.zero_()
        m.block['conv_m'].bias.fill_(T.PIN_BIAS_M)
        n = m.block['norm']
        n.eps = 0.0
        n.weight.fill_(1.0)
        n.bias.zero_()
        n.running_mean.zero_()
        n.running_var.fill_(1.0)
    m.eval()
    x = torch.zeros((1, 32, 5, 7))
    gy = torch.randint(-100, 101, (1, 32, 5, 7), generator=torch.Generator().manual_seed(1)).float()
    _, _, _, grads, _ = _call(case, [m], [x], None, gy, "eval", False)
    ok = bool((grads[3] == 0).all()) and torch.equal(grads[1].cpu(), gy.sum((0, 2, 3)))
    print(f"\ngate backward at m + b_m = 64: dbias_m {'== 0' if bool((grads[3] == 0).all()) else '!= 0'}, dbias_f "
          f"{'== sum dy' if ok else '!= sum dy'}")
    assert ok, "the gate backward's sigmoid(64) is not exactly 1: the exact tier's premise fails"
    return ok


def _stack_r(case):
    from test_gpu_fwd_exact_wss import wss_rows
    c = types.SimpleNamespace(hout=case.H, wout=case.W, B=case.B, cout=case.cout)
    return wss_rows(c, torch.cuda.get_device_properties(0).multi_processor_count)


@pytest.mark.parametrize("case", T.EXACT_CASES, ids=lambda c: c.id)
def test_function_is_exact(case, gate_pinned_bwd):
    mods, xs, res, gout = _operands(case)
    r = T.replay(case, mods, xs, res, gout)
    if case.family == "stack" and case.cout >= 128:
        R = _stack_r(case)
        want = T.STACK_R.get((case.cout, case.B, case.H, case.W))
        print(f"\n{case.id}: the streamed-weight body runs R = {R} tiles")
        if torch.cuda.get_device_properties(0).multi_processor_count == 132 and want is not None:
            assert R == want, (case.id, R, want)
    got = _call(case, mods, xs, res, gout, "eval", False)
    _check_exact(case, got, r, mods)
    det = _call(case, mods, xs, res, gout, "eval", True)
    _check_exact(case, det, r, mods)
    for a, b in zip([got[0]] + got[1] + got[3], [det[0]] + det[1] + det[3]):
        if a is not None:
            assert torch.equal(_bits(a), _bits(b)), f"{case.id}: deterministic mode gives other bits"


@pytest.mark.parametrize("mode", ["batch", "items"])
@pytest.mark.parametrize("case", T.SINGLE_CASES + T.MULTI_CASES, ids=lambda c: c.id)
def test_train_mode_output_and_dbeta(case, mode, gate_pinned_bwd):
    mods, xs, res, gout = _operands(case)
    r = T.replay(case, mods, xs, res, gout)
    out, dxs, dres, grads, convs = _call(case, mods, xs, res, gout, mode, False)
    c, n = convs[0], case.cout
    p = T.params64(mods[0])
    fw = r["fwd"][-1]
    g = T.rnd(fw["accf"] + p["bf"][:, None, None]).float()                       # identity epilogue, gate pinned open
    sc, sh = c.scale.cpu(), c.shift.cpu()
    if mode == "items":
        sc, sh = sc[:, :n, None, None], sh[:, :n, None, None]
    else:
        sc, sh = sc[:n, None, None], sh[:n, None, None]
    y = (g * sc) + sh
    if fw["res"] is not None:
        y = y + fw["res"].float()
    T.U.assert_exact(out, y.bfloat16().double(), f"{case.id} {mode} output (bn_apply with the Function's statistics)",
                     ["b", "c", "h", "w"])
    T.U.assert_exact(grads[5], r["grads"][5], f"{case.id} {mode} dbeta")
    # the _det statistics and gate-backward entry points give the same output and dbeta
    det = _call(case, mods, xs, res, gout, mode, True)
    assert torch.equal(_bits(det[0]), _bits(out)), f"{case.id} {mode}: deterministic mode changes the output"
    assert torch.equal(_bits(det[3][5]), _bits(grads[5])), f"{case.id} {mode}: deterministic mode changes dbeta"


# ------------------------------------------------------------------ bounded tier
WORST = {}


def _stats(c, n, mode):
    """The statistics the call used, from its FoldedConv, as float64 [items, n]."""
    rows = lambda t: (t[:, :n] if t.dim() == 2 else t[:n][None]).double().cpu()
    return {k: rows(getattr(c, k)) for k in ("mean", "inv", "scale", "shift")}


@pytest.mark.parametrize("det", [False, True], ids=["atomic", "det"])
@pytest.mark.parametrize("mode", T.BOUNDED_MODES)
@pytest.mark.parametrize("case", T.BOUNDED_CASES, ids=lambda c: c.id)
def test_bounded_tier_within_per_element_bounds(case, mode, det):
    """Unpinned gates, ELU's negative branch, every BatchNorm mode, with and without torch.use_deterministic_algorithms: every
    element of the output, the input gradients, dwf, dwm, dbias_f, dbias_m and dgamma within its propagated bound
    (tests/train_fn_exact_util.py), dbeta exact."""
    mods, xs, res, gout = T.bounded_operands(case)
    out, dxs, _, grads, convs = _call(case, mods, xs, res, gout, mode, det)
    r = T.bounded_ref(case, mods, xs, res, gout, mode, _stats(convs[0], case.cout, mode))
    got = {"out": out, "dwf": grads[0], "dbias_f": grads[1], "dwm": grads[2], "dbias_m": grads[3], "dgamma": grads[4],
           "dbeta": grads[5]}
    got.update({f"dx{j}": g for j, g in enumerate(dxs)})
    for name, g in got.items():
        want, bound = r[name]
        if name == "dbeta":
            T.U.assert_exact(g, want, f"{case.id} {mode} dbeta")
            continue
        worst = T.U.assert_bound(g, want, bound, 1.0, f"{case.id} {mode} {name}")
        key = name if not name.startswith("dx") else "dx"
        WORST[key] = max(WORST.get(key, 0.0), worst)
    print("\nworst err/bound so far: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))
