// C-ABI glue: error state, device checks, conv plan dispatch.
#include "common.cuh"
#include "conv_common.cuh"
#include <mutex>
#include <new>

namespace rb {

static thread_local char g_err[1024] = "";
std::atomic<long long> g_launches{0};

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int num_sms()
{
    // per-device cache (DataParallel drives several devices from one process)
    static std::mutex mu;
    static int cache[64];
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 148;
    std::lock_guard<std::mutex> lk(mu);
    if (cache[dev] == 0) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
        cache[dev] = n;
    }
    return cache[dev];
}

}  // namespace rb

using namespace rb;

struct read_conv_plan {
    read_conv_desc d;
    int impl;
    TcPlan *tc;
    TcgPlan *tcg;
    int max_ctas;            // 0 = one CTA per SM; > 0 caps the persistent grid (read_conv_plan_set_max_ctas)
};

static int validate_conv(const read_conv_desc &d)
{
    RB_CHECK_ARG(d.act_dtype == READ_ACT_F32 || d.act_dtype == READ_ACT_BF16, "conv: bad act_dtype");
    RB_CHECK_ARG(d.n_src >= 1 && d.n_src <= READ_MAX_SRC, "conv: 1..%d sources", READ_MAX_SRC);
    RB_CHECK_ARG(d.k == 1 || d.k == 3 || d.k == 4, "conv: kernel size must be 1, 3 or 4");
    RB_CHECK_ARG(d.stride == 1 || d.stride == 2, "conv: stride must be 1 or 2");
    RB_CHECK_ARG(d.B >= 1 && d.Hin >= 1 && d.Win >= 1 && d.Cout >= 1, "conv: bad shape");
    int csum = 0;
    for (int i = 0; i < d.n_src; ++i) {
        const read_src &s = d.src[i];
        RB_CHECK_ARG(s.ptr != nullptr, "conv: source %d is null", i);
        RB_CHECK_ARG(s.C >= 8 && s.C % 8 == 0, "conv: source channels must be a multiple of 8 (got %d)", s.C);
        RB_CHECK_ARG((reinterpret_cast<uintptr_t>(s.ptr) & 15) == 0, "conv: source %d must be 16B aligned", i);
        int eh = s.H, ew = s.W;
        switch (s.mode) {
        case READ_SRC_IDENTITY: break;
        case READ_SRC_NEAREST_DOWN:
            RB_CHECK_ARG(s.factor >= 2, "conv: bad resample factor");
            eh = s.H / s.factor; ew = s.W / s.factor; break;
        case READ_SRC_NEAREST_UP:
            RB_CHECK_ARG(s.factor >= 2, "conv: bad resample factor");
            eh = s.H * s.factor; ew = s.W * s.factor; break;
        case READ_SRC_BILINEAR_UP4: eh = s.H * 4; ew = s.W * 4; break;
        default: RB_CHECK_ARG(false, "conv: unknown source mode %d", s.mode);
        }
        RB_CHECK_ARG(eh == d.Hin && ew == d.Win, "conv: source %d resamples to %dx%d, expected %dx%d", i, eh, ew, d.Hin, d.Win);
        csum += s.C;
    }
    RB_CHECK_ARG(csum == d.Cin, "conv: sources hold %d channels, Cin is %d", csum, d.Cin);
    RB_CHECK_ARG(d.mul == nullptr || (d.n_src == 1 && d.src[0].mode == READ_SRC_IDENTITY), "conv: mul needs one identity source");
    const int eh = (d.Hin + 2 * d.pad - d.k) / d.stride + 1, ew = (d.Win + 2 * d.pad - d.k) / d.stride + 1;
    RB_CHECK_ARG(eh == d.Hout && ew == d.Wout, "conv: output is %dx%d, expected %dx%d", d.Hout, d.Wout, eh, ew);
    RB_CHECK_ARG(d.bias_f && d.bias_m && d.bn_scale && d.bn_shift && d.out, "conv: null parameter pointer");
    RB_CHECK_ARG(d.out_mode == READ_OUT_NHWC || d.out_mode == READ_OUT_NCHW_F32 || d.out_mode == READ_OUT_RAW_NHWC, "conv: bad out_mode");
    RB_CHECK_ARG(d.out_mode != READ_OUT_RAW_NHWC || d.out2 == nullptr, "conv: RAW output takes no out2");
    RB_CHECK_ARG(d.out_mode != READ_OUT_RAW_NHWC || d.residual == nullptr || d.k == 3, "conv: RAW output takes a residual only for 3x3 convs");
    RB_CHECK_ARG(d.addin == nullptr || (d.addin_H == (d.Hout + 1) / 2 && d.addin_W == (d.Wout + 1) / 2),
                 "conv: addin must be [B, ceil(Hout/2), ceil(Wout/2), 2*Cout]");
    RB_CHECK_ARG((d.out_mode != READ_OUT_RAW_NHWC && d.addin == nullptr) || d.impl == READ_CONV_TCGEN05,
                 "conv: RAW output / addin are served by the TMA tensor-core kernel only");
    RB_CHECK_ARG((d.out2 == nullptr) == (d.out2_mul == nullptr), "conv: out2 and out2_mul come together");
    RB_CHECK_ARG(d.out2 == nullptr || d.out_mode == READ_OUT_NHWC, "conv: out2 needs NHWC output");
    return READ_OK;
}

extern "C" {

int read_version(void) { return 100; }
const char *read_last_error(void) { return g_err; }
int64_t read_launch_count(void) { return g_launches.load(); }

int read_device_ok(void)
{
    int dev = 0, major = 0, minor = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
    return (major == 9 && minor == 0) ? 1 : 0;
}

int read_conv_tc_supported(const read_conv_desc *d)
{
    if (!d) return 0;
    return tc_supported(*d) ? 1 : 0;
}

int read_conv_tcg_supported(const read_conv_desc *d)
{
    if (!d) return 0;
    return tcg_supported(*d) ? 1 : 0;
}

int64_t read_tcg_weight_elems(int Cout, int Cin, int k) { return tcg_weight_elems(Cout, Cin, k); }

int read_pack_weights_tcg(const float *wf, const float *wm, int Cout, int Cin, int k, void *out_bf16, void *stream)
{
    RB_CHECK_ARG(wf && wm && out_bf16, "pack_tc_gather: null pointer");
    return tcg_pack(wf, wm, Cout, Cin, k, out_bf16, (cudaStream_t)stream);
}

int read_conv_plan_create(const read_conv_desc *d, read_conv_plan **out)
{
    RB_CHECK_ARG(d && out, "conv plan: null argument");
    int rc = validate_conv(*d);
    if (rc) return rc;
    int impl = d->impl;
    RB_CHECK_ARG(impl != READ_CONV_AUTO, "conv plan: choose impl explicitly (the weight packing differs per kernel)");
    if (impl == READ_CONV_TCGEN05) {
        RB_CHECK_ARG(d->w_tc != nullptr, "conv plan: tensor-core kernel requested without packed bf16 weights");
        if (!tc_supported(*d)) { set_error("conv plan: layer shape not supported by the TMA tensor-core kernel"); return READ_ERR_UNSUPPORTED; }
    } else if (impl == READ_CONV_TCGEN05_GATHER) {
        RB_CHECK_ARG(d->w_tc != nullptr, "conv plan: tensor-core kernel requested without packed bf16 weights");
        if (!tcg_supported(*d)) { set_error("conv plan: layer not supported by the gather tensor-core kernel"); return READ_ERR_UNSUPPORTED; }
    } else {
        RB_CHECK_ARG(impl == READ_CONV_GENERIC, "conv plan: unknown impl %d", impl);
        RB_CHECK_ARG(d->w_generic != nullptr, "conv plan: generic kernel needs w_generic");
        RB_CHECK_ARG((reinterpret_cast<uintptr_t>(d->w_generic) & 15) == 0, "conv plan: w_generic must be 16B aligned");
    }
    read_conv_plan *p = new (std::nothrow) read_conv_plan{*d, impl, nullptr, nullptr, 0};
    RB_CHECK_ARG(p != nullptr, "conv plan: out of host memory");
    if (impl == READ_CONV_TCGEN05) {
        rc = tc_plan_create(*d, &p->tc);
        if (rc) { delete p; return rc; }
    } else if (impl == READ_CONV_TCGEN05_GATHER) {
        rc = tcg_plan_create(*d, &p->tcg);
        if (rc) { delete p; return rc; }
    }
    *out = p;
    return READ_OK;
}

int read_conv_plan_launch(const read_conv_plan *p, void *stream)
{
    RB_CHECK_ARG(p != nullptr, "conv plan: null plan");
    if (p->impl == READ_CONV_TCGEN05) return tc_plan_launch(p->tc, (cudaStream_t)stream, p->max_ctas);
    if (p->impl == READ_CONV_TCGEN05_GATHER) return tcg_plan_launch(p->tcg, (cudaStream_t)stream, p->max_ctas);
    return launch_generic(p->d, (cudaStream_t)stream);
}

int read_conv_plan_impl(const read_conv_plan *p) { return p ? p->impl : 0; }

int read_conv_plan_set_tile_order(read_conv_plan *p, int reversed)
{
    RB_CHECK_ARG(p != nullptr, "conv plan: set_tile_order needs a plan");
    if (p->tc) tc_plan_set_reverse(p->tc, reversed);        // the gather / CUDA-core kernels keep their order
    return READ_OK;
}

int read_conv_plan_set_max_ctas(read_conv_plan *p, int max_ctas)
{
    RB_CHECK_ARG(p != nullptr && max_ctas >= 0, "conv plan: set_max_ctas needs a plan and a count >= 0");
    p->max_ctas = max_ctas;
    return READ_OK;
}

void read_conv_plan_destroy(read_conv_plan *p)
{
    if (!p) return;
    if (p->tc) tc_plan_destroy(p->tc);
    if (p->tcg) tcg_plan_destroy(p->tcg);
    delete p;
}

}  // extern "C"
