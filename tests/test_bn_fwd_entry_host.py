"""Host-side checks (no GPU) of the train-mode BatchNorm forward's entry points: for a fixed grid of rejected arguments, each of the
four launch functions must return READ_ERR_INVALID with the exact message of the first check that fails in its own order, before
any launch; and the two workspace queries must return the sizes the statistics pass lays its workspace out in."""
import ctypes
import itertools

import pytest

from read_b200 import _lib

P, ODD = 0x1000, 0x1008                  # 16-byte aligned / 8-byte aligned stand-in device pointers; nothing is dereferenced

# the pointers each pass's first null check covers, its second one (the statistics' affine and running parameters), and the ones
# its alignment check covers; var (call-wide statistics) and residual (apply) may be null
STATS_NULL = ("g", "mean", "inv_std", "scale", "shift", "workspace")
STATS_PARAMS = ("gamma", "beta", "running_mean", "running_var")
STATS_ALIGNED = ("g", "workspace")
APPLY_NULL = ("g", "scale", "shift", "y")
APPLY_ALIGNED = ("g", "residual", "y", "scale", "shift")

# (entry point, statistics pass, per item)
ENTRIES = [
    ("read_bn_batch_stats", True, False),
    ("read_bn_batch_stats_items", True, True),
    ("read_bn_apply", False, False),
    ("read_bn_apply_items", False, True),
]

BASE = dict(items=3, pixels=100, C=64, n_real="C", eps=1e-5, momentum=0.1, g=P, gamma=P, beta=P, running_mean=P, running_var=P,
            mean=P, inv_std=P, var=P, scale=P, shift=P, workspace=P, residual=P, y=P)


def _call(lib, entry, stats, per_item, a):
    C = a["C"]
    n_real = C if a["n_real"] == "C" else C + 1 if a["n_real"] == "C+1" else a["n_real"]
    head = [a["g"]] + ([a["items"]] if per_item else []) + [a["pixels"], C]
    if stats:
        args = head + [n_real, a["gamma"], a["beta"], a["eps"], a["momentum"], a["running_mean"], a["running_var"], a["mean"],
                       a["inv_std"]] + ([] if per_item else [a["var"]]) + [a["scale"], a["shift"], a["workspace"]]
    else:
        args = head + [a["scale"], a["shift"], a["residual"], a["y"]]
    return getattr(lib, entry)(*args, None)


def _g(x):                  # a float argument as the library prints it: its fp32 value with %g
    return f"{ctypes.c_float(x).value:g}"


def _expected(entry, stats, per_item, a):
    """The message of the first check ``a`` fails, or None when every check passes: the entry point's checks in its order."""
    C, px, items = a["C"], a["pixels"], a["items"]
    n_real = C if a["n_real"] == "C" else C + 1 if a["n_real"] == "C+1" else a["n_real"]
    set_ = lambda names: all(a[p] is not None for p in names)
    checks = [(set_(STATS_NULL if stats else APPLY_NULL), "null pointer")]
    if per_item:
        checks.append((1 <= items <= 65535, f"items must lie in 1..65535 (got {items})"))
    checks.append((C in (16, 32, 64, 128, 192, 256), f"C must be 16, 32, 64 or a multiple of 64 up to 256 (got {C})"))
    if stats:
        checks += [(1 <= n_real <= C, f"n_real must lie in 1..C (got {n_real}, C = {C})"), (set_(STATS_PARAMS), "null pointer")]
    checks.append((px >= 2, f"batch statistics need at least 2 pixels{' per item' if per_item else ''} (got {px})"))
    if stats:
        checks.append((a["eps"] > 0 and 0 <= a["momentum"] <= 1, f"bad eps / momentum ({_g(a['eps'])}, {_g(a['momentum'])})"))
    checks.append((all(a[p] is None or a[p] % 16 == 0 for p in (STATS_ALIGNED if stats else APPLY_ALIGNED)),
                   "tensors must be 16B aligned"))
    for ok, msg in checks:
        if not ok:
            return f"{entry[len('read_'):]}: {msg}"
    return None


def _faults(stats, per_item):
    """(check, argument overrides) of every rejected value of the grid, one check failing each."""
    yield from (("null", {p: None}) for p in (STATS_NULL if stats else APPLY_NULL))
    if per_item:
        yield from (("items", {"items": it}) for it in (-1, 0, 65536))
    yield from (("C", {"C": C}) for C in (0, 3, 8, 48, 96, 320))
    if stats:
        yield from (("n_real", {"n_real": n}) for n in (0, "C+1"))
        yield from (("params", {p: None}) for p in STATS_PARAMS)
    yield from (("pixels", {"pixels": px}) for px in (-5, 0, 1))
    if stats:
        yield from (("eps", d) for d in ({"eps": 0.0}, {"momentum": -0.1}, {"momentum": 1.5}))
    yield from (("aligned", {p: ODD}) for p in (STATS_ALIGNED if stats else APPLY_ALIGNED))


def _cases(stats, per_item):
    """Every fault alone at each accepted C, and every pair of faults of two different checks (which one is reported is the
    order under test)."""
    faults = list(_faults(stats, per_item))
    for C, (k, f) in itertools.product((16, 32, 64, 128, 192, 256), faults):
        if k != "C":
            yield {**BASE, "C": C, **f}
    for (k1, f1), (k2, f2) in itertools.combinations(faults, 2):
        if k1 != k2 and not f1.keys() & f2.keys():
            yield {**BASE, **f1, **f2}


@pytest.mark.parametrize("entry,stats,per_item", ENTRIES, ids=[e[0] for e in ENTRIES])
def test_rejected_arguments_give_the_entry_points_code_and_message(entry, stats, per_item):
    lib = _lib.load()
    for case in _cases(stats, per_item):
        want = _expected(entry, stats, per_item, case)
        assert want is not None, (entry, case)   # the grid holds rejected arguments only
        assert _call(lib, entry, stats, per_item, case) == -1, (entry, case)
        assert lib.read_last_error().decode() == want, (entry, case)


# bytes of the statistics workspace: call-wide, 256 (the counter) + the partials (count, mean, M2 fp64 of 512 CTAs); per item,
# the 1 + items counters and uvar [items, C] fp32, each rounded up to 256 bytes, + the partials of every item
WORKSPACE_BYTES = {16: 196864, 32: 393472, 64: 786688, 128: 1573120, 256: 3145984}
WORKSPACE_BYTES_ITEMS = {
    (1, 16): 197120, (3, 16): 590336, (8, 16): 1573632, (64, 16): 12587520, (65535, 16): 12889161728,
    (1, 32): 393728, (3, 32): 1180416, (8, 32): 3147008,
    (1, 64): 786944, (3, 64): 2360320, (8, 64): 6293760,
    (1, 128): 1573632, (3, 128): 4720384, (8, 128): 12587264,
    (1, 256): 3147008, (3, 256): 9440512, (8, 256): 25174272,
}


def test_workspace_bytes():
    lib = _lib.load()
    assert {C: lib.read_bn_workspace_bytes(C) for C in WORKSPACE_BYTES} == WORKSPACE_BYTES
    assert {k: lib.read_bn_workspace_bytes_items(*k) for k in WORKSPACE_BYTES_ITEMS} == WORKSPACE_BYTES_ITEMS
    for C in (0, 3, 8, 48, 96, 320):
        assert lib.read_bn_workspace_bytes(C) == -1, C
        assert lib.read_bn_workspace_bytes_items(3, C) == -1, C
    for items in (-1, 0, 65536):
        assert lib.read_bn_workspace_bytes_items(items, 64) == -1, items
