"""Host-side checks (no GPU) of the argument validation of the weight-gradient entry points and of the stride-2 / 8-channel input
gradients that share their channel rules: for a fixed grid of rejected arguments, each must return READ_ERR_INVALID with the exact
message of the first check that fails in that entry point's own order.  Every case is rejected before any launch: a case that
would pass every check also carries a misaligned pointer, and read_pack_weights_dgrad_s2, which checks no alignment, is only
called with cases it rejects.  Also the deterministic workspace size, which must hold the split count the launch uses."""
import itertools

import pytest
import torch

import bwd_exact_util as U
from read_b200 import _lib

P, ODD = 0x1000, 0x1008                  # 16-byte aligned / 8-byte aligned stand-in device pointers; nothing is dereferenced
NO_DEVICE_SMS = 148                      # num_sms() when the library sees no device


def _cin_wgrad(Cin):
    return Cin in (8, 16) or (Cin % 32 == 0 and Cin > 0)


def _cin_s2(Cin):
    return Cin % 32 == 0 and Cin > 0


def _cout_ok(Cout):                      # the [df | dm] column order: 16, 32, 64 or a multiple of 64
    return Cout == 16 or (Cout % 32 == 0 and Cout > 0 and (Cout <= 64 or Cout % 64 == 0))


def _geom_ok(k, s):
    return (k, s) in ((1, 1), (3, 1), (3, 2), (4, 2))


WGRAD_CH = "Cin must be 8, 16 or a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got {Cin}, {Cout})"
S2_CH = "Cin must be a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got {Cin}, {Cout})"
SHAPE = lambda c: c["B"] >= 1 and c["H"] >= 1 and c["W"] >= 1
MATCH = lambda c: c["Hin"] == c["stride"] * c["H"] and c["Win"] == c["stride"] * c["W"]


# Each entry point: its name in messages, pointer arguments, the pointers its alignment check covers, the argument list of a case,
# its checks in order as (predicate over the case and its pointer values, message template), and the fault kinds it takes.
ENTRIES = {
    "read_conv3x3_wgrad": dict(
        name="conv3x3_wgrad", ptrs=("dfm", "x", "dwf", "dwm"), aligned=("dfm", "x"),
        args=lambda c, v: [v["dfm"], v["x"], c["B"], c["H"], c["W"], c["Cout"], c["Cin"], v["dwf"], v["dwm"], None],
        checks=[(SHAPE, "bad shape"),
                (lambda c: _cin_wgrad(c["Cin"]) and _cout_ok(c["Cout"]), WGRAD_CH),
                ("aligned", "tensors must be 16B aligned")],
        faults=("null", "shape", "cin", "cout", "odd")),
    "read_conv_wgrad": dict(
        name="conv_wgrad", ptrs=("dfm", "x", "dwf", "dwm"), aligned=("dfm", "x"),
        args=lambda c, v: [v["dfm"], v["x"], c["B"], c["Hin"], c["Win"], c["H"], c["W"], c["Cout"], c["Cin"], c["k"], c["stride"],
                           v["dwf"], v["dwm"], None],
        checks=[(SHAPE, "bad shape"),
                (lambda c: _geom_ok(c["k"], c["stride"]),
                 "k={k} stride={stride} is not one of 1x1 / 3x3 stride 1, 3x3 / 4x4 stride 2"),
                (MATCH, "input {Hin}x{Win} does not match output {H}x{W} at stride {stride} (stride 2 needs an even input)"),
                (lambda c: _cin_wgrad(c["Cin"]) and _cout_ok(c["Cout"]), WGRAD_CH),
                ("aligned", "tensors must be 16B aligned")],
        faults=("null", "shape", "cin", "cout", "geom", "match", "odd")),
    "read_conv_wgrad_det": dict(
        name="conv_wgrad_det", ptrs=("dfm", "x", "dwf", "dwm", "workspace"), aligned=("dfm", "x", "workspace"),
        args=lambda c, v: [v["dfm"], v["x"], c["B"], c["Hin"], c["Win"], c["H"], c["W"], c["Cout"], c["Cin"], c["k"], c["stride"],
                           v["dwf"], v["dwm"], v["workspace"], None],
        checks=[(SHAPE, "bad shape"),
                (lambda c: _geom_ok(c["k"], c["stride"]) and MATCH(c),
                 "k={k} stride={stride} input {Hin}x{Win} output {H}x{W} is not 1x1 / 3x3 stride 1 or 3x3 / 4x4 stride 2 "
                 "(input = stride x output)"),
                (lambda c: _cin_wgrad(c["Cin"]) and _cout_ok(c["Cout"]), WGRAD_CH),
                ("aligned", "tensors and workspace must be 16B aligned")],
        faults=("null", "shape", "cin", "cout", "geom", "match", "odd")),
    "read_pack_weights_dgrad_s2": dict(
        name="pack_dgrad_s2", ptrs=("wf", "wm", "out"), aligned=(),
        args=lambda c, v: [v["wf"], v["wm"], c["Cout"], c["Cin"], c["k"], v["out"], None],
        checks=[(lambda c: c["k"] in (3, 4), "k must be 3 or 4 (got {k})"),
                (lambda c: _cin_s2(c["Cin"]) and _cout_ok(c["Cout"]), S2_CH)],
        faults=("null", "cin", "cout", "geom")),
    "read_conv_dgrad_s2": dict(
        name="conv_dgrad_s2", ptrs=("dfm", "wt", "dx"), aligned=("dfm", "wt", "dx"),
        args=lambda c, v: [v["dfm"], v["wt"], c["B"], c["H"], c["W"], c["Cout"], c["Cin"], c["k"], v["dx"], None],
        checks=[(SHAPE, "bad shape"),
                (lambda c: c["k"] in (3, 4), "k must be 3 or 4 (got {k})"),
                (lambda c: _cin_s2(c["Cin"]) and _cout_ok(c["Cout"]), S2_CH),
                ("aligned", "tensors must be 16B aligned")],
        faults=("null", "shape", "cin", "cout", "geom", "odd")),
    "read_conv3x3_dgrad_cin8": dict(
        name="conv3x3_dgrad_cin8", ptrs=("dfm", "wf", "wm", "dx"), aligned=("dfm", "dx"),
        args=lambda c, v: [v["dfm"], v["wf"], v["wm"], c["B"], c["H"], c["W"], c["Cout"], v["dx"], None],
        checks=[(SHAPE, "bad shape"),
                (lambda c: c["Cout"] in (16, 32, 64), "Cout must be 16, 32 or 64 (got {Cout})"),
                ("aligned", "tensors must be 16B aligned")],
        faults=("null", "shape", "cout", "odd")),
}

# an accepted geometry: 3x3 stride 2, output 5x7 from a 10x14 input; 32 -> 64 channels
BASE = dict(B=2, H=5, W=7, Cin=32, Cout=64, k=3, stride=2, dH=0, dW=0, null=None, odd=frozenset())


def _faults(e):
    """kind -> the case updates of that kind this entry point takes (some are accepted values for some entry points)."""
    f = dict(null=[dict(null=p) for p in e["ptrs"]],
             shape=[{d: v} for d in ("B", "H", "W") for v in (0, -1)],
             cin=[dict(Cin=v) for v in (0, 8, 16, 24, 48, 64)],
             cout=[dict(Cout=v) for v in (0, 8, 16, 32, 48, 96, 128, 192)],
             geom=[dict(k=k, stride=s) for k, s in ((1, 1), (3, 1), (3, 2), (4, 2), (2, 1), (1, 2), (4, 1), (3, 3))],
             match=[dict(dH=1), dict(dW=2), dict(dW=-7)],      # an odd input at stride 2, an even mismatch, the stride-1 size
             odd=[dict(odd=frozenset({p})) for p in e["aligned"]])
    return {kind: f[kind] for kind in e["faults"]}


def _case(*updates):
    c = dict(BASE)
    for u in updates:
        c.update(u)
    c["Hin"], c["Win"] = c["stride"] * c["H"] + c["dH"], c["stride"] * c["W"] + c["dW"]
    return c


def _values(e, c):
    return {p: None if p == c["null"] else ODD if p in c["odd"] else P for p in e["ptrs"]}


def _expected(e, c):
    """The message of the first check the case fails, or None when it passes every check."""
    v = _values(e, c)
    if any(v[p] is None for p in e["ptrs"]):
        return f"{e['name']}: null pointer"
    for ok, msg in e["checks"]:
        passed = all(v[p] == P for p in e["aligned"]) if ok == "aligned" else ok(c)
        if not passed:
            return f"{e['name']}: " + msg.format(**c)
    return None


def _cases(e):
    """Every single fault and every pair of faults of different kinds; a case otherwise accepted gets a misaligned pointer last."""
    kinds = _faults(e)
    singles = [(u,) for us in kinds.values() for u in us]
    pairs = [(a, b) for k1, k2 in itertools.combinations(kinds, 2) for a, b in itertools.product(kinds[k1], kinds[k2])]
    for updates in singles + pairs:
        c = _case(*updates)
        if _expected(e, c) is None and e["aligned"]:
            c = _case(*updates, dict(odd=c["odd"] | {e["aligned"][-1]}))
        yield c


@pytest.mark.parametrize("entry", list(ENTRIES))
def test_rejected_arguments_give_the_entry_points_code_and_message(entry):
    lib, e = _lib.load(), ENTRIES[entry]
    n = 0
    for c in _cases(e):
        want = _expected(e, c)
        if want is None:                 # read_pack_weights_dgrad_s2 accepts the case and would launch
            assert not e["aligned"], c
            continue
        assert getattr(lib, entry)(*e["args"](c, _values(e, c))) == -1, (entry, c)
        assert lib.read_last_error().decode() == want, (entry, c)
        n += 1
    assert n >= 100, n


@pytest.mark.parametrize("entry", ["read_conv3x3_wgrad", "read_conv_wgrad", "read_conv_wgrad_det"])
def test_too_large_is_rejected_before_the_launch(entry):
    """Cout = 2^22 gives 131072 column blocks, above the 65535 a grid dimension holds; every pointer is aligned."""
    lib, e = _lib.load(), ENTRIES[entry]
    c = _case(dict(B=1, H=1, W=1, Cin=8, Cout=2 ** 22, k=1, stride=1))
    assert _expected(e, c) is None
    assert getattr(lib, entry)(*e["args"](c, _values(e, c))) == -1
    assert lib.read_last_error().decode() == f"{e['name']}: too large"


def _lib_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count if torch.cuda.is_available() \
        else NO_DEVICE_SMS


def test_det_workspace_rejects_what_the_launch_rejects():
    ws = _lib.load().read_conv_wgrad_det_workspace_bytes
    for B, H, W in ((0, 4, 4), (-1, 4, 4), (1, 0, 4), (1, -1, 4), (1, 4, 0), (1, 4, -1)):
        assert ws(B, H, W, 64, 32, 3, 1) == -1, (B, H, W)
    for Cout, Cin in ((0, 32), (8, 32), (48, 32), (96, 32), (160, 32), (64, 0), (64, 24), (64, 48)):
        assert ws(1, 4, 4, Cout, Cin, 3, 1) == -1, (Cout, Cin)
    for k, s in ((2, 1), (1, 2), (4, 1), (3, 3), (0, 1), (3, 0)):
        assert ws(1, 4, 4, 64, 32, k, s) == -1, (k, s)


def test_det_workspace_holds_one_copy_per_split():
    ws = _lib.load().read_conv_wgrad_det_workspace_bytes
    geoms = ((1, 1), (3, 1), (3, 2), (4, 2))
    # one 32-pixel segment: one split whatever the SM count
    for (k, s), (Cout, Cin), W in itertools.product(geoms, ((16, 8), (32, 16), (64, 32), (128, 64), (256, 96)), (1, 17, 32)):
        assert ws(1, 1, W, Cout, Cin, k, s) == 2 * Cout * Cin * k * k * 4, (k, s, Cout, Cin, W)
    # no limit on the size; the launch would reject this grid
    assert ws(1, 1, 1, 2 ** 22, 8, 1, 1) == 2 * 2 ** 22 * 8 * 4
    sms = _lib_sms()
    for (k, s), (Cout, Cin), (B, H, W) in itertools.product(
            geoms, ((16, 8), (32, 32), (64, 64), (128, 128), (256, 256)), ((1, 3, 33), (4, 17, 100), (8, 128, 128))):
        _, splits, _, _, _ = U.wgrad_grid(B, H, W, Cout, Cin, k, sms)
        assert ws(B, H, W, Cout, Cin, k, s) == splits * 2 * Cout * Cin * k * k * 4, (k, s, Cout, Cin, B, H, W, sms)
