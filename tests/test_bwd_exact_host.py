"""Without a GPU: the checkers of test_gpu_bwd_exact.py reject the defects a kernel could have (and accept the exact result), the
shape lists cover the edge classes of each kernel, and every integer case keeps its partial sums exact in fp32."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import bwd_exact_util as U


def _rejects(check, *args, **kw):
    with pytest.raises(AssertionError) as e:
        check(*args, **kw)
    print(f"\nrejected: {str(e.value)[:200]}")
    return str(e.value)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------ checker self-tests: weight gradient
@pytest.mark.parametrize("k,stride", [(3, 1), (1, 1), (3, 2), (4, 2)])
def test_wgrad_checker_rejects_a_dropped_segment_pixel(k, stride):
    g = _gen(1)
    B, H, W, C, cin = 2, 3, 33, 16, 16
    dcat, x = U.int_tensor((B, H, W, 2 * C), 2, g), U.int_tensor((B, stride * H, stride * W, cin), 2, g)
    want = U.wgrad_ref(dcat, x, k, stride)
    U.assert_exact(want.clone(), want, "unmodified")
    bad = dcat.clone()
    bad[1, 2, U.WG_PX - 1] = 0                      # the last pixel of the first 32-pixel segment of one row
    assert "differ" in _rejects(U.assert_exact, U.wgrad_ref(bad, x, k, stride), want, "drop", ["o", "ci", "ky", "kx"])


@pytest.mark.parametrize("k", [3, 4])
def test_wgrad_checker_rejects_the_next_items_row_in_the_pad(k):
    g = _gen(2)
    stride = 1 if k == 3 else 2
    B, H, W, C, cin = 2, 4, 9, 16, 8
    dcat, x = U.int_tensor((B, H, W, 2 * C), 2, g), U.int_tensor((B, stride * H, stride * W, cin), 2, g, zero_frac=0.0)
    want = U.wgrad_ref(dcat, x, k, stride)
    xp = F.pad(x.double().permute(0, 3, 1, 2), (1, 1, 1, 1))
    xp[0, :, -1, 1:-1] = x[1, 0].double().t()       # item 0's bottom pad row read from item 1's first row
    bad = torch.nn.grad.conv2d_weight(xp, (2 * C, cin, k, k), dcat.double().permute(0, 3, 1, 2), stride=stride, padding=0)
    _rejects(U.assert_exact, bad, want, "next item's row")


@pytest.mark.parametrize("C", [16, 128])
def test_wgrad_checker_rejects_swapped_f_m_halves_in_one_column_block(C):
    g = _gen(3)
    dcat, x = U.int_tensor((2, 3, 7, 2 * C), 2, g), U.int_tensor((2, 3, 7, 32), 2, g)
    want = U.wgrad_ref(dcat, x, 3, 1)
    half = min(C, 64)
    bad = want.clone()
    bad[:half], bad[C:C + half] = want[C:C + half], want[:half]       # block 0's conv_f and conv_m rows exchanged
    _rejects(U.assert_exact, bad, want, "swap")


# ------------------------------------------------------------------ input gradients
def _dgrad_case(seed, B=2, H=9, W=17, C=32, cin=32, k=3, stride=1):
    g = _gen(seed)
    dcat = U.int_tensor((B, H, W, 2 * C), U.DGRAD_AMP, g)
    wcat = U.int_tensor((2 * C, cin, k, k), U.DGRAD_AMP, g)
    return dcat, wcat, U.dgrad_ref(dcat, wcat, stride * H, stride * W, stride)


def test_dgrad_checker_rejects_an_off_by_one_tap_flip():
    dcat, wcat, want = _dgrad_case(4)
    U.assert_bf16_rn(want.float().bfloat16(), want, "unmodified")
    wbad = wcat.clone()
    wbad[:, :, 0, 0], wbad[:, :, 0, 1] = wcat[:, :, 0, 1], wcat[:, :, 0, 0]    # one tap read one column off
    _rejects(U.assert_bf16_rn, U.dgrad_ref(dcat, wbad, 9, 17, 1).float().bfloat16(), want, "flip", ["b", "y", "x", "c"])


def test_dgrad_checker_rejects_truncation_instead_of_round_to_nearest():
    _, _, want = _dgrad_case(5)
    assert U.bf16_nonrepresentable_fraction(want) > 0.3
    trunc = (want.float().view(torch.int32) & ~0xFFFF).view(torch.float32).bfloat16()
    _rejects(U.assert_bf16_rn, trunc, want, "truncation", ["b", "y", "x", "c"])


def test_dgrad_cin8_checker_rejects_a_missing_halo_column_at_a_segment_start():
    dcat, wcat, want = _dgrad_case(6, W=65, cin=8)
    bad_in = dcat.clone()
    bad_in[:, :, U.DG8_PX - 1] = 0                 # the pixel left of the second segment, missing from its halo
    bad = want.clone()
    bad[:, :, U.DG8_PX] = U.dgrad_ref(bad_in, wcat, 9, 65, 1)[:, :, U.DG8_PX]
    _rejects(U.assert_bf16_rn, bad.float().bfloat16(), want, "halo", ["b", "y", "x", "c"])


@pytest.mark.parametrize("k", [3, 4])
def test_dgrad_s2_checker_rejects_a_tap_of_the_wrong_parity(k):
    dcat, wcat, want = _dgrad_case(7, H=3, W=33, k=k, stride=2)
    wbad = wcat.clone()
    wbad[:, :, :, 1] = wcat[:, :, :, 0]            # even input columns read filter column 0 instead of 1
    bad = want.clone()
    bad[:, :, 0::2] = U.dgrad_ref(dcat, wbad, 6, 66, 2)[:, :, 0::2]
    _rejects(U.assert_bf16_rn, bad.float().bfloat16(), want, "parity", ["b", "y", "x", "c"])


# ------------------------------------------------------------------ gate / BatchNorm
def _gate_ops(items, P, C, seed, int_dy=False):
    g = _gen(seed)
    n = items * P
    dy = U.int_tensor((n, C), 8, g) if int_dy else torch.randn((n, C), generator=g) * 4
    vec = lambda lo: torch.rand((items, C), generator=g) + lo
    return dict(dy=dy.bfloat16(), fm=U.to_raw(U.gate_fm_values(n, C, g)).bfloat16(), bf=torch.rand(C, generator=g) - 0.5,
                bm=torch.zeros(C), scale=vec(0.5), mean=vec(0) - 0.5, inv=vec(0.5), s0=torch.randn((items, C), generator=g) * 50,
                s1=torch.randn((items, C), generator=g) * 50)


def test_gate_sum_checker_rejects_a_pixel_moved_to_the_neighbouring_item():
    items, P, C = 3, 33, 32
    o = _gate_ops(items, P, C, 8, int_dy=True)
    ref = U.gate_ref(o, C, 1, "items", items, P)
    U.assert_exact(ref["sum_dy"].float(), ref["sum_dy"], "unmodified")
    dy = o["dy"].double()
    p = max(i for i in range(P) if bool(dy[i].any()))          # item 0's last pixel with a non-zero gradient
    bad = ref["sum_dy"].clone()
    bad[0] -= dy[p]
    bad[1] += dy[p]
    _rejects(U.assert_exact, bad, ref["sum_dy"], "moved pixel", ["item", "c"])


@pytest.mark.parametrize("kind", ["eval", "items"])
def test_gate_bound_checker_rejects_a_2ulp_error_in_dm(kind):
    items, P, C = 2, 40, 64
    o = _gate_ops(items, P, C, 9)
    ref = U.gate_ref(o, C, 1, kind, items, P)
    got = ref["dfm"].float().bfloat16()
    U.assert_bound(got, ref["dfm"], ref["T_dfm"], U.TAU, "unmodified", rel=U.REL_BF16)
    mcols = [j for j in range(2 * C) if int(U.fm_columns(C)[j]) >= C]
    dm = ref["dfm"][:, mcols]
    e = np.unravel_index(int(torch.argmax(dm.abs() / (ref["T_dfm"][:, mcols] + 1e-300))), tuple(dm.shape))
    bits = got.view(torch.int16)
    bits[e[0], mcols[e[1]]] += 2                                 # two bf16 ulps away from the round-to-nearest value
    _rejects(U.assert_bound, got, ref["dfm"], ref["T_dfm"], U.TAU, "2 ulp", rel=U.REL_BF16, names=["pixel", "column"])


def test_sum_bound_checker_rejects_an_error_beyond_tau_s():
    o = _gate_ops(1, 300, 16, 10)
    ref = U.gate_ref(o, 16, 0, "eval", 1, 300)
    got = ref["sum_dm"].float()
    U.assert_bound(got, ref["sum_dm"], ref["T_sum"], U.TAU_S, "unmodified")
    got[3] += 2 * U.TAU_S * float(ref["T_sum"][3])
    _rejects(U.assert_bound, got, ref["sum_dm"], ref["T_sum"], U.TAU_S, "sum", names=["c"])


# ------------------------------------------------------------------ gather
def test_gather_checker_rejects_a_pixel_credited_to_the_neighbouring_slot():
    g = _gen(11)
    N, h, w = 50, 6, 7
    go = U.int_tensor((2, 8, h, w), 8, g, zero_frac=0.0)
    ids = torch.randint(-2, N + 3, (2, h, w), generator=g).float()
    pre = [np.zeros((N, 8)), np.zeros((N, 8))]
    want = [U.gather_ref(go[i:i + 1].numpy(), ids[i:i + 1].numpy(), N, pre[i]) for i in range(2)]
    got = [x.copy() for x in want]
    row = int(np.clip(ids[0, 2, 3], 0, N - 1))
    got[0][row] -= go[0, :, 2, 3].numpy()              # item 0 (slot 0) pixel (2, 3) added to slot 1's row instead
    got[1][row] += go[0, :, 2, 3].numpy()
    U.assert_exact(torch.from_numpy(want[1]), torch.from_numpy(want[1]), "unmodified")
    for s in range(2):
        _rejects(U.assert_exact, torch.from_numpy(got[s]), torch.from_numpy(want[s]), f"slot {s}", ["id", "c"])


def test_guard_band_sees_a_write_past_the_end():
    gb = U.Guarded(100, torch.bfloat16, "cpu")
    gb.check("clean")
    gb.buf[gb.guard + 100] = 0.0
    assert "after" in _rejects(gb.check, "tail write")
    gb = U.Guarded(10, torch.float32, "cpu", torch.arange(10.0))
    gb.buf[gb.guard - 1] = 1.0
    assert "before" in _rejects(gb.check, "head write")


# ------------------------------------------------------------------ edge-class coverage
def test_wgrad_cases_cover_every_edge_class_per_geometry():
    for (k, stride), pairs in U.TRAINED.items():
        cases = [c for c in U.WGRAD_CASES if (c[2], c[3]) == (k, stride)]
        cls = set().union(*(U.wgrad_classes(c) for c in cases))
        print(f"\nwgrad {k}x{k} stride {stride}: {sorted(cls)}")
        assert U.WGRAD_REQUIRED <= cls, (k, stride, sorted(U.WGRAD_REQUIRED - cls))
        assert set(pairs) <= {(c[0], c[1]) for c in cases}, (k, stride)
        if k == 4:
            assert "4x4 row groups" in cls
    allc = set().union(*(U.wgrad_classes(c) for c in U.WGRAD_CASES))
    assert {"partial column block", "partial channel block"} <= allc
    assert any(c[4] == 8 and c[5] == 256 and c[6] == 256 for c in U.WGRAD_CASES)
    assert {(k, s, cin, C) for (k, s, cin, C) in U.PADDED} <= {(c[2], c[3], c[0], c[1]) for c in U.WGRAD_CASES}


def test_dgrad_cases_cover_every_edge_class():
    cls = set().union(*(U.tma_classes(c[3], c[4]) for c in U.DGRAD3_CASES + U.DGRAD1_CASES))
    print(f"\nTMA RAW dgrad: {sorted(cls)}")
    assert {"W%8==0", "W%8==1", "W<8", "H%16==0", "H%16==1", "H%16==8", "H%16==9", "H<16"} <= cls
    assert all(c[2] >= 2 for c in U.DGRAD3_CASES + U.DGRAD1_CASES)
    assert {(cin, C) for cin, C in U.TRAINED[(3, 1)] if cin != 8} <= {(c[0], c[1]) for c in U.DGRAD3_CASES}
    widths = {w for c in U.DGRAD1_CASES for w in c[0]}
    assert {16, 32, 64, 128, 256} <= widths and any(len(c[0]) == 4 for c in U.DGRAD1_CASES)
    for C in (16, 32, 64):
        cls = set().union(*(U.dg8_classes(B, H, W, C2) for C2, B, H, W in U.DG8_CASES if C2 == C))
        print(f"dgrad_cin8 C={C}: {sorted(cls)}")
        assert {"W%64==1", "W%64==63", "W%64==0", "W<64"} <= cls
    assert "CTA walks several segments" in set().union(*(U.dg8_classes(B, H, W, C) for C, B, H, W in U.DG8_CASES))
    for k in (3, 4):
        cases = [c for c in U.DS_CASES if c[0] == k]
        cls = set().union(*(U.ds_classes(c[5], c[2]) for c in cases))
        print(f"dgrad_s2 k={k}: {sorted(cls)}")
        assert {"Wi%64==2", "Wi%64==62", "Wi%64==0", "Wi<64", "several K chunks"} <= cls
        assert {2, 4, 6} <= {c[4] for c in cases} and {32, 128, 256} & {c[1] for c in cases}
    assert "one K chunk" in set().union(*(U.ds_classes(c[5], c[2]) for c in U.DS_CASES))
    assert {32, 128, 256} <= {c[1] for c in U.DS_CASES}


def test_gate_cases_cover_the_pixel_step_edges():
    import test_gpu_bwd_exact as T
    for C in U.GATE_CS:
        ps = {P for C2, it, P in T.GATE_EXACT if C2 == C}
        assert set(U.gate_item_pixels(C)) <= ps, C
    assert (64, 64 * 64) in {(it, P) for _, it, P in T.GATE_EXACT}
    assert (1, 8 * 256 * 256) in {(it, P) for _, it, P in T.GATE_EXACT}
    assert {1, 2} <= {c[0] for c in T.GATHER_CASES} and max(c[0] for c in T.GATHER_CASES) >= 100000


# ------------------------------------------------------------------ exactness of the integer cases
def test_integer_cases_stay_below_2_24():
    import test_gpu_bwd_exact as T
    worst = {}
    for c in U.WGRAD_CASES:
        worst["wgrad"] = max(worst.get("wgrad", 0), U.max_partial(U.wgrad_terms(c), U.WGRAD_AMP, U.WGRAD_AMP, U.WGRAD_PREFILL))
    for cin, C, B, H, W in U.DGRAD3_CASES:
        worst["dgrad 3x3"] = max(worst.get("dgrad 3x3", 0), U.max_partial(9 * 2 * C, U.DGRAD_AMP, U.DGRAD_AMP, U.DGRAD_RES_AMP))
    for srcs, C, B, H, W in U.DGRAD1_CASES:
        worst["dgrad 1x1"] = max(worst.get("dgrad 1x1", 0), U.max_partial(2 * C, U.DGRAD_AMP, U.DGRAD_AMP))
    for C, B, H, W in U.DG8_CASES:
        worst["dgrad cin8"] = max(worst.get("dgrad cin8", 0), U.max_partial(9 * 2 * C, U.DGRAD_AMP, U.DGRAD_AMP))
    for k, cin, C, B, Hi, Wi in U.DS_CASES:
        worst["dgrad s2"] = max(worst.get("dgrad s2", 0), U.max_partial(k * k * 2 * C, U.DGRAD_AMP, U.DGRAD_AMP))
    for C, items, P in T.GATE_EXACT:
        worst["dy sums"] = max(worst.get("dy sums", 0), U.max_partial(items * P, 8, 1, 7))
    for N, D, B, h, w in T.GATHER_CASES:
        worst["gather"] = max(worst.get("gather", 0), U.max_partial(B * h * w, 8, 1, 100))
    worst["gather items"] = U.max_partial(64 * 24 * 20, 8, 1, 100)
    print("\nworst-case partial sums:", {k: f"{v} (2^{np.log2(v):.1f})" for k, v in worst.items()})
    assert all(v < U.EXACT_LIMIT for v in worst.values()), worst
