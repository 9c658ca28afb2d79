"""Host-side checks (no GPU) of the descriptor gather's entry points (csrc/gather.cu): for a fixed grid of rejected arguments, each of
the nine entry points must return READ_ERR_INVALID with the exact message of the first check that fails in its own order, before
any launch; a zero-size gather must return READ_OK before its layout is looked at; and read_set_option must accept every documented
option and reject the retired "gather_variant"."""
import ctypes
import itertools

from read_b200 import _lib

P, ODD = 0x1000, 0x1008                  # 16-byte aligned / 8-byte aligned stand-in device pointers; nothing is dereferenced


def _first_failure(checks):
    """checks: (predicate, message) in the entry point's order; a predicate runs only when every earlier one held."""
    for ok, msg in checks:
        if not ok():
            return msg
    return None


def _cases(base, faults):
    """Every fault alone, and every pair of faults of two different checks on disjoint arguments (which one is reported is the
    order under test)."""
    for _, f in faults:
        yield {**base, **f}
    for (k1, f1), (k2, f2) in itertools.combinations(faults, 2):
        if k1 != k2 and not f1.keys() & f2.keys():
            yield {**base, **f1, **f2}


def _run(lib, call, expected, total, base, faults):
    """Every case must be rejected with its expected message, or be a zero-size call that returns READ_OK; a case that would launch
    is not part of the grid."""
    n = 0
    for a in _cases(base, faults):
        want = expected(a)
        if want is None and total(a) != 0:
            continue
        rc = call(lib, a)
        if want is None:
            assert rc == 0, a
        else:
            assert rc == -1, a
            assert lib.read_last_error().decode() == want, a
        n += 1
    return n


# ---- read_gather_from_index / _i32 / read_gather_from_zbuf: check_gather, then the zero-size return, then the layout
ONE = dict(tex=P, D=8, N=1000, src=P, B=2, h=5, w=7, layout=0, act=0, out=P)
ONE_FAULTS = ([("null", {p: None}) for p in ("tex", "src", "out")]
              + [("shape", {"D": d}) for d in (0, -1)] + [("shape", {"N": n}) for n in (0, -5)]
              + [("shape", {p: -1}) for p in ("B", "h", "w")]
              + [("tex_align", {"tex": ODD}), ("out_align", {"out": ODD})]
              + [("layout", {"layout": v}) for v in (3, -1, 99)]
              + [("zero", {p: 0}) for p in ("B", "h", "w")]
              + [("d3", {"D": 3, "tex": ODD})])                   # a D != 8 texture needs no alignment


def _one_expected(a):
    return _first_failure([
        (lambda: a["tex"] is not None and a["src"] is not None and a["out"] is not None, "gather: null pointer"),
        (lambda: a["D"] >= 1 and a["N"] >= 1 and a["B"] >= 0 and a["h"] >= 0 and a["w"] >= 0, "gather: bad shape"),
        (lambda: a["D"] != 8 or a["tex"] % 16 == 0, "gather: descriptors must be 16B aligned"),
        (lambda: a["out"] % 16 == 0, "gather: output must be 16B aligned"),
    ]) or (None if a["B"] * a["h"] * a["w"] == 0 or a["layout"] in (0, 1, 2) else f"gather: unknown layout {a['layout']}")


def _one_call(name):
    def call(lib, a):
        return getattr(lib, name)(a["tex"], a["D"], a["N"], a["src"], a["B"], a["h"], a["w"], a["layout"], a["act"], a["out"], None)
    return call


def test_one_texture_gathers_reject_with_the_first_failing_check():
    lib = _lib.load()
    for name in ("read_gather_from_index", "read_gather_from_index_i32", "read_gather_from_zbuf"):
        n = _run(lib, _one_call(name), _one_expected, lambda a: a["B"] * a["h"] * a["w"], ONE, ONE_FAULTS)
        assert n == 150, (name, n)


# ---- read_gather_from_index_items / _i32: check_tex_table, ids / output, then the zero-size return, then the layout
ITEMS = dict(table=True, n_slots=2, n_items=3, slot=(0, 1, 1), N=(100, 50), tex=(P, P), h=5, w=7, ids=P, out=P, layout=0)
ITEMS_FAULTS = ([("table", {"table": None})]
                + [("n_slots", {"n_slots": v}) for v in (0, -1, 17)]
                + [("n_items", {"n_items": v}) for v in (0, -1, 65)]
                + [("shape", {p: -1}) for p in ("h", "w")]
                + [("slot", {"slot": s}) for s in ((0, 2, 1), (0, 1, 5))]
                + [("N", {"N": n}) for n in ((100, 0), (-3, 50))]
                + [("tex", {"tex": t}) for t in ((None, P), (P, ODD))]
                + [("io", {p: v}) for p, v in (("ids", None), ("out", None), ("out", ODD))]
                + [("layout", {"layout": v}) for v in (3, -1)]
                + [("zero", {p: 0}) for p in ("h", "w")])


def _items_expected(a):
    what = "gather (items)"
    if a["table"] is None:
        return f"{what}: null table"
    checks = [(lambda: 1 <= a["n_slots"] <= 16, f"{what}: n_slots {a['n_slots']} not in 1..16"),
              (lambda: 1 <= a["n_items"] <= 64, f"{what}: n_items {a['n_items']} not in 1..64"),
              (lambda: a["h"] >= 0 and a["w"] >= 0, f"{what}: bad shape")]
    msg = _first_failure(checks)
    if msg:
        return msg
    slot = list(a["slot"]) + [0] * (a["n_items"] - len(a["slot"]))
    for b in range(a["n_items"]):
        if slot[b] >= a["n_slots"]:
            return f"{what}: item {b} maps to slot {slot[b]}"
    for s in range(a["n_slots"]):
        if a["N"][s] < 1:
            return f"{what}: slot {s} has no points"
        if a["tex"][s] is None or a["tex"][s] % 16:
            return f"{what}: slot {s}: descriptors must be non-null and 16B aligned"
    if a["ids"] is None or a["out"] is None or a["out"] % 16:
        return f"{what}: null or unaligned ids / output"
    if a["n_items"] * a["h"] * a["w"] == 0 or a["layout"] in (0, 1, 2):
        return None
    return f"{what}: unknown layout {a['layout']}"


def _items_call(name):
    def call(lib, a):
        t = None
        if a["table"] is not None:
            t = _lib.ReadTexTable()
            t.n_slots, t.n_items = a["n_slots"], a["n_items"]
            for s in range(min(len(a["N"]), _lib.MAX_TEX_SLOTS)):
                t.N[s], t.tex_nd[s] = a["N"][s], a["tex"][s]
            for b, s in enumerate(a["slot"]):
                t.slot[b] = s
            t = ctypes.byref(t)
        return getattr(lib, name)(t, a["ids"], a["h"], a["w"], a["layout"], 0, a["out"], None)
    return call


def test_table_gathers_reject_with_the_first_failing_check():
    lib = _lib.load()
    for name in ("read_gather_from_index_items", "read_gather_from_index_items_i32"):
        n = _run(lib, _items_call(name), _items_expected, lambda a: a["n_items"] * a["h"] * a["w"], ITEMS, ITEMS_FAULTS)
        assert n == 236, (name, n)


# ---- read_pyramid_resolve_gather: every accepted call launches, so the grid holds rejected calls only
PYR = dict(tex=P, D=8, N=1000, zbuf=P, B=2, view0=0, nviews=2, W=64, H=48, L=4, layout=2, outs=True, out0=P, out1=P, out2=P,
           out3=P)
PYR_FAULTS = ([("view", {"view0": -1}), ("view", {"nviews": 0}), ("view", {"view0": 1}), ("view", {"B": 1}), ("view", {"B": 0})]
              + [("null", {p: None}) for p in ("tex", "zbuf", "outs")]
              + [("D", {"D": d}) for d in (3, 16)] + [("L", {"L": v}) for v in (3, 5)]
              + [("WH", {p: v}) for p, v in (("W", 60), ("H", 44), ("W", 0), ("H", -8))]
              + [("layout", {"layout": v}) for v in (0, 3, -1)]
              + [("align", {p: ODD}) for p in ("tex", "zbuf")]
              + [("out", {f"out{l}": None}) for l in range(4)] + [("out", {"out2": ODD})])


def _pyr_expected(a):
    msg = _first_failure([
        (lambda: a["view0"] >= 0 and a["nviews"] >= 1 and a["view0"] + a["nviews"] <= a["B"], "pyramid resolve: bad view range"),
        (lambda: a["tex"] is not None and a["zbuf"] is not None and a["outs"] is not None, "pyramid resolve: null pointer"),
        (lambda: a["D"] == 8 and a["L"] == 4, "pyramid resolve: fused path needs D == 8 and L == 4"),
        (lambda: a["B"] >= 1 and a["W"] >= 8 and a["H"] >= 8 and a["W"] % 8 == 0 and a["H"] % 8 == 0,
         "pyramid resolve: W and H must be multiples of 8"),
        (lambda: a["layout"] in (1, 2), "pyramid resolve: NHWC layouts only"),
        (lambda: a["tex"] % 16 == 0 and a["zbuf"] % 16 == 0, "pyramid resolve: descriptors / z-buffer must be 16B aligned"),
    ])
    if msg:
        return msg
    for l in range(4):
        o = a[f"out{l}"]
        if o is None or o % 16:
            return f"pyramid resolve: bad output {l}"
    return None


def _pyr_call(lib, a):
    outs = None if a["outs"] is None else (_lib.c_vp * 4)(*[a[f"out{l}"] for l in range(4)])
    return lib.read_pyramid_resolve_gather(a["tex"], a["D"], a["N"], a["zbuf"], a["B"], a["view0"], a["nviews"], a["W"], a["H"],
                                           a["L"], a["layout"], outs, 1, None)


def test_pyramid_resolve_gather_rejects_with_the_first_failing_check():
    n = _run(_lib.load(), _pyr_call, _pyr_expected, lambda a: 1, PYR, PYR_FAULTS)
    assert n == 314, n


# ---- the texture transposes and read_stage_net_inputs: every accepted call launches
TR = dict(cn=P, nd=P, D=8, N=1000)
TR_FAULTS = [("null", {"cn": None}), ("null", {"nd": None}), ("shape", {"D": 0}), ("shape", {"N": 0}), ("shape", {"N": -2}),
             ("align", {"nd": ODD})]


def _tr_expected(point_major):
    def expected(a):
        return _first_failure([
            (lambda: a["cn"] is not None and a["nd"] is not None and a["D"] >= 1 and a["N"] >= 1, "texture transpose: bad arguments"),
            (lambda: not point_major or a["D"] != 8 or a["nd"] % 16 == 0, "texture transpose: output must be 16B aligned"),
        ])
    return expected


def test_texture_transposes_reject_with_the_first_failing_check():
    lib = _lib.load()
    pm = lambda lib, a: lib.read_texture_to_point_major(a["cn"], a["D"], a["N"], a["nd"], None)
    cm = lambda lib, a: lib.read_texture_to_channel_major(a["nd"], a["D"], a["N"], a["cn"], None)
    assert _run(lib, pm, _tr_expected(True), lambda a: 1, TR, TR_FAULTS) == 16
    assert _run(lib, cm, _tr_expected(False), lambda a: 1, TR, TR_FAULTS) == 15


STAGE = dict(src=P, B=1, hs=64, ws=48, C=8, factor=2, act=1, dst=P)
STAGE_FAULTS = ([("null", {p: None}) for p in ("src", "dst")]
                + [("shape", {p: v}) for p, v in (("B", 0), ("B", -1), ("C", 0), ("factor", 0), ("factor", -1), ("hs", 1), ("ws", 1))]
                + [("multiple", {p: v}) for p, v in (("hs", 63), ("ws", 47))]
                + [("act", {"act": v}) for v in (2, -1)])


def _stage_expected(a):
    f = a["factor"]
    return _first_failure([
        (lambda: a["src"] is not None and a["dst"] is not None, "stage_net_inputs: null pointer"),
        (lambda: a["B"] >= 1 and a["C"] >= 1 and f >= 1 and a["hs"] >= f and a["ws"] >= f, "stage_net_inputs: bad shape"),
        (lambda: a["hs"] % f == 0 and a["ws"] % f == 0,
         "stage_net_inputs: the render size must be a multiple of the supersampling factor"),
        (lambda: a["act"] in (0, 1), "stage_net_inputs: bad act_dtype"),
    ])


def test_stage_net_inputs_rejects_with_the_first_failing_check():
    call = lambda lib, a: lib.read_stage_net_inputs(a["src"], a["B"], a["hs"], a["ws"], a["C"], a["factor"], None, 0, a["act"],
                                                    a["dst"], None)
    assert _run(_lib.load(), call, _stage_expected, lambda a: 1, STAGE, STAGE_FAULTS) == 65


# ---- options: the documented names (include/read_b200.h) at their documented defaults, and the retired gather_variant
DOCUMENTED_OPTIONS = {"raster_pipelined": 1, "raster_bulk_tma": 1, "raster_mode": 2, "raster_occupancy": 0, "raster_stream": 1,
                      "raster_dedup": 0, "raster_run": 0, "raster_nbr_filter": 0, "raster_stages": 2, "raster_carveout": 45,
                      "tc_pdl": 1}


def test_set_option_accepts_the_documented_options_and_rejects_gather_variant():
    lib = _lib.load()
    for name, value in DOCUMENTED_OPTIONS.items():
        assert lib.read_set_option(name.encode(), value) == 0, (name, lib.read_last_error())
    for value in (0, 3):
        assert lib.read_set_option(b"gather_variant", value) == -1
        assert lib.read_last_error().decode() == "set_option: unknown option 'gather_variant'"
