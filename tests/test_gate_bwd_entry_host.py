"""Host-side checks (no GPU) of the argument validation of the ten gate-backward and BatchNorm-backward-reduction entry points:
for a fixed grid of rejected arguments, each must return READ_ERR_INVALID with the exact message, from the first check that fails
in that entry point's own order.  Every case is rejected before any launch; the eval-mode forms accept pixels == 0 as a no-op."""
import itertools

import pytest

from read_b200 import _lib

P, ODD = 0x1000, 0x1008                  # 16-byte aligned / 8-byte aligned stand-in device pointers; nothing is dereferenced

EVAL_PTRS = ("bias_f", "bias_m", "bn_scale", "bn_mean", "bn_inv_std", "dfm", "dbias_f", "dbias_m", "dgamma", "dbeta")
REDUCE_PTRS = ("bias_f", "bias_m", "bn_mean", "bn_inv_std", "sum_dy", "sum_dy_xhat")
BATCH_PTRS = ("bias_f", "bias_m", "bn_scale", "bn_mean", "bn_inv_std", "sum_dy", "sum_dy_xhat", "dfm", "dbias_f", "dbias_m")

# (entry point, its pointer arguments after elu, per item, deterministic)
ENTRIES = [
    ("read_gate_backward", EVAL_PTRS, False, False),
    ("read_bn_backward_reduce", REDUCE_PTRS, False, False),
    ("read_gate_backward_batch_stats", BATCH_PTRS, False, False),
    ("read_bn_backward_reduce_items", REDUCE_PTRS, True, False),
    ("read_gate_backward_batch_stats_items", BATCH_PTRS, True, False),
    ("read_gate_backward_det", EVAL_PTRS, False, True),
    ("read_bn_backward_reduce_det", REDUCE_PTRS, False, True),
    ("read_gate_backward_batch_stats_det", BATCH_PTRS, False, True),
    ("read_bn_backward_reduce_items_det", REDUCE_PTRS, True, True),
    ("read_gate_backward_batch_stats_items_det", BATCH_PTRS, True, True),
]


def _pointers(ptrs, det):
    return ("dy", "fm") + ptrs + (("workspace",) if det else ())


def _call(lib, entry, ptrs, per_item, det, case):
    v = {p: None if p == case["null"] else ODD if p in case["odd"] else P for p in _pointers(ptrs, det)}
    args = [v["dy"], v["fm"]] + ([case["items"]] if per_item else []) + [case["pixels"], case["C"], 1]
    args += [v[p] for p in ptrs] + ([v["workspace"]] if det else []) + [None]
    return getattr(lib, entry)(*args)


def _gate_c_ok(C):          # the channel counts with the RAW [f | m] column order
    return 16 <= C <= 256 and C % 16 == 0 and (C <= 64 or C % 64 == 0)


def _bn_c_ok(C):            # the train-mode BatchNorm counts: the above without 48
    return C in (16, 32, 64) or (C % 64 == 0 and 0 < C <= 256)


def _expected(entry, ptrs, per_item, det, case):
    """The message of the first check ``case`` fails, or None when every check passes: each entry point's checks in its order."""
    name, eval_ = entry[len("read_"):], "dgamma" in ptrs
    C, px, items, odd = case["C"], case["pixels"], case["items"], case["odd"]
    c_msg = (f"C must be 16, 32, 48, 64 or a multiple of 64 up to 256 (got {C})" if eval_ else
             f"C must be 16, 32, 64 or a multiple of 64 up to 256 (got {C})")
    c_ok = _gate_c_ok(C) if eval_ else _bn_c_ok(C)
    aligned = "tensors must be 16B aligned"
    checks = [(case["null"] is None, "null pointer")]
    if per_item:
        checks.append((1 <= items <= 65535, f"items must lie in 1..65535 (got {items})"))
    if det:
        minpx = 0 if eval_ else 2
        checks += [(px >= minpx, f"needs at least {minpx} pixels (got {px})"),
                   (not odd & {"dy", "fm", "workspace"}, "tensors and workspace must be 16B aligned"),
                   (c_ok, c_msg),
                   ("dfm" not in odd, aligned)]
    elif eval_:                                  # a negative pixel count is reported with the channel message
        checks += [(c_ok and px >= 0, c_msg), (not odd & {"dy", "fm", "dfm"}, aligned)]
    else:
        per = " per item" if per_item else ""
        checks += [(c_ok, c_msg), (px >= 2, f"batch statistics need at least 2 pixels{per} (got {px})"),
                   (not odd & {"dy", "fm", "dfm"}, aligned)]
    for ok, msg in checks:
        if not ok:
            return f"{name}: {msg}"
    return None


def _cases(ptrs, per_item, det):
    base = dict(C=64, pixels=100, items=3, null=None, odd=frozenset())
    stop = frozenset({"dfm"} if "dfm" in ptrs else ())    # keeps accepted channel / pixel counts from reaching a launch
    yield from (dict(base, null=p) for p in _pointers(ptrs, det))
    for C, odd in itertools.product((0, 3, 8, 48, 96, 320), (frozenset({"dy"}), stop)):
        yield dict(base, C=C, odd=odd)
    for px, odd in itertools.product((-5, 0, 1), (frozenset({"dy"}), stop)):
        yield dict(base, pixels=px, odd=odd)
    if per_item:
        yield from (dict(base, items=it) for it in (-1, 0, 65536))
    yield from (dict(base, odd=frozenset({p})) for p in ("dy", "fm", "dfm", "workspace") if p in _pointers(ptrs, det))


@pytest.mark.parametrize("entry,ptrs,per_item,det", ENTRIES, ids=[e[0] for e in ENTRIES])
def test_rejected_arguments_give_the_entry_points_code_and_message(entry, ptrs, per_item, det):
    lib = _lib.load()
    for case in _cases(ptrs, per_item, det):
        want = _expected(entry, ptrs, per_item, det, case)
        assert want is not None, (entry, case)   # the grid holds rejected arguments only
        assert _call(lib, entry, ptrs, per_item, det, case) == -1, (entry, case)
        assert lib.read_last_error().decode() == want, (entry, case)


@pytest.mark.parametrize("entry", ["read_gate_backward", "read_gate_backward_det"])
def test_eval_forms_accept_zero_pixels(entry):
    lib = _lib.load()
    case = dict(C=48, pixels=0, items=1, null=None, odd=frozenset())
    assert _call(lib, entry, EVAL_PTRS, False, entry.endswith("_det"), case) == 0
