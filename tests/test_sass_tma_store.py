"""The TMA conv kernel stores its NHWC outputs with TMA (UTMASTG) out of the epilogue stage in shared memory (no GPU needed)."""
from test_sass_evidence import _has, _kernels, sass  # noqa: F401  (sass is the module fixture)


def test_conv_kernel_stores_through_tma(sass):
    ks = _kernels(sass, "gated_conv_tc_kernel")
    for name, ops in ks.items():
        if "ELi16EE" in name:             # N = 16: the final NCHW fp32 layer stores from registers
            continue
        assert _has(ops, "UTMASTG") > 0, name
