"""Host-side checks of the residual-block backward entry points (no GPU): which RAW 3x3 layers the TMA kernel accepts, and the
argument validation of the packing, gate-backward and weight-gradient calls."""
import ctypes

from read_b200 import _lib


def _raw3x3(cin, cout, residual=True):
    d = _lib.ReadConvDesc()
    d.act_dtype, d.n_src = _lib.ACT_BF16, 1
    d.src[0].ptr, d.src[0].C, d.src[0].H, d.src[0].W = 0x1000, cin, 40, 40
    d.src[0].mode, d.src[0].factor = _lib.SRC_IDENTITY, 1
    d.B, d.Hin, d.Win, d.Cin, d.Hout, d.Wout, d.Cout = 2, 40, 40, cin, 40, 40, cout
    d.k, d.stride, d.pad = 3, 1, 1
    d.out_mode = _lib.OUT_RAW_NHWC
    if residual:
        d.residual = 0x2000
    return d


def test_tc_predicate_for_raw_3x3_with_residual():
    lib = _lib.load()
    ok = lambda d: lib.read_conv_tc_supported(ctypes.byref(d))
    assert ok(_raw3x3(32, 32, residual=False)) == 1          # recomputed [f | m] of a C=32 block conv
    assert ok(_raw3x3(512, 128, residual=False)) == 1        # ... of C=256 (four n tiles)
    assert ok(_raw3x3(64, 16)) == 1                           # input gradient of a C=32 conv, skip added
    assert ok(_raw3x3(512, 128)) == 1                         # ... of C=256 (two n tiles)
    d = _raw3x3(64, 16)
    d.out2, d.out2_mul = 0x3000, 0x4000
    assert ok(d) == 0                                         # RAW takes no FAM output
    d = _raw3x3(64, 16)
    d.stride, d.Hout, d.Wout = 2, 20, 20
    assert ok(d) == 0
    d = _raw3x3(64, 16)
    d.k, d.pad = 1, 0
    assert ok(d) == 0                                         # 1x1 RAW terms still take no residual


def test_backward_entry_points_reject_unsupported_shapes():
    lib = _lib.load()
    p = 0x1000
    assert lib.read_pack_weights_tc_dgrad(p, p, 32, 48, p, None) == -1           # Cin not a multiple of 32
    assert b"pack_tc_dgrad" in lib.read_last_error()
    assert lib.read_pack_weights_tc_dgrad(p, p, 96, 96, p, None) == -1
    assert lib.read_gate_backward(p, p, 100, 8, 1, p, p, p, p, p, p, p, p, p, p, None) == -1
    assert lib.read_gate_backward(p, p, 100, 512, 1, p, p, p, p, p, p, p, p, p, p, None) == -1
    # channel counts without the RAW column order (blocks of 2*min(C, 64) columns): indexing would run past the tensors
    for C in (80, 96, 160, 224):
        assert lib.read_gate_backward(p, p, 100, C, 1, p, p, p, p, p, p, p, p, p, p, None) == -1, C
    for C in (96, 160, 224):
        assert lib.read_conv3x3_wgrad(p, p, 1, 8, 8, C, 32, p, p, None) == -1, C
    assert lib.read_conv3x3_wgrad(p, p, 1, 8, 8, 48, 32, p, p, None) == -1
    assert lib.read_conv3x3_wgrad(p, p, 1, 8, 8, 32, 32, None, p, None) == -1
    assert lib.read_tc_weight_elems(16, 64, 3) == 9 * 64 * 32                   # dgrad filters of a C=32 conv
