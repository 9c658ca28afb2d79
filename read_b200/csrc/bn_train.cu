// Train-mode BatchNorm of the gated convs (read_b200/blocks.py, batch_stats=True): the conv launch writes g = A(f + b_f) *
// sigmoid(m + b_m) with an identity epilogue (scale 1, shift 0, no residual), then
//   bn_stats_kernel<PER_ITEM>   per-channel mean and biased variance of g over the P pixels of the call, inv_std, the folded
//                               scale / shift, and the in-place running-statistics update (torch.nn.BatchNorm2d's train-mode
//                               semantics), all on the device
//   bn_apply_kernel<PER_ITEM>   y = bf16(g * scale + shift [+ residual]), in place over g when the caller wants
// PER_ITEM = true: the same per batch item (UNet.train_batchnorm = 'per_item': item i of a call is normalised with its own
// statistics, and the running statistics end as B single-item calls would leave them).
// The backward's reduction and corrected gate backward live next to the eval-mode gate backward (conv_bwd.cu).
// The statistics are not fused into the TMA conv kernel's epilogue: its instances render every inference frame.
#include "common.cuh"
#include "conv_common.cuh"

namespace rb {

// ------------------------------------------------------------------ batch statistics
// A thread owns 8 channels (one 16-byte vector) of one pixel per step, like the gate backward, and sums g - K and (g - K)^2 in
// fp32, K = the first value the thread reads of each channel: its sums stay small for a channel whose mean is far above its
// spread, and a pixel far from the mean spoils only the few pixels of the thread that starts on it.  Each thread turns its sums
// into (count, mean, M2 = sum of squared deviations from its mean); a CTA combines its threads' in fp64 in a fixed order, in two
// passes (the pooled mean, then M2 = sum of M2_t + n_t (mean_t - mean)^2: deviations from the pooled mean, nothing cancels), into
// the workspace, and the last CTA to finish (counter + fence) combines the CTAs' the same way in CTA order: the result does not
// depend on scheduling and is the same run to run.
constexpr int BN_THREADS = 256, BN_MAX_C = 256, BN_MAX_CTAS = 512, BN_PART = 3;   // workspace: (count, mean, M2) per CTA, channel

// The body of both bn_stats_kernel instances (PER_ITEM: the caller points g, the outputs, part and counter at one item; var
// receives the unbiased variance var * P / (P - 1) for the running update and the running statistics are not touched).  Returns
// whether this CTA was the last one, the one that wrote the outputs.
template <bool PER_ITEM>
__device__ __forceinline__ bool
bn_stats_body(const __nv_bfloat16 *__restrict__ g, long long P, int C, int n_real, const float *__restrict__ gamma,
              const float *__restrict__ beta, float eps, float momentum, float *__restrict__ running_mean,
              float *__restrict__ running_var, float *__restrict__ mean, float *__restrict__ inv_std, float *__restrict__ var,
              float *__restrict__ scale, float *__restrict__ shift, double *__restrict__ part, unsigned int *__restrict__ counter)
{
    __shared__ float sk[BN_THREADS * 8], s1[BN_THREADS * 8], s2[BN_THREADS * 8];
    __shared__ int sn[BN_THREADS];
    __shared__ bool last;
    const int G = C / 8, ppb = BN_THREADS / G;
    const int cg = threadIdx.x % G, co0 = 8 * cg;
    const long long p0 = blockIdx.x * (long long)ppb + threadIdx.x / G;
    float k[8], a1[8], a2[8];
    int n = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) k[j] = a1[j] = a2[j] = 0.f;
    if (threadIdx.x < ppb * G && p0 < P) {
        {
            const uint4 v = *reinterpret_cast<const uint4 *>(g + p0 * C + co0);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 f = bf16x2_val(w[q]);
                k[2 * q] = f.x; k[2 * q + 1] = f.y;
            }
        }
        for (long long p = p0; p < P; p += (long long)gridDim.x * ppb, ++n) {
            const uint4 v = *reinterpret_cast<const uint4 *>(g + p * C + co0);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 f = bf16x2_val(w[q]);
                const float d0 = f.x - k[2 * q], d1 = f.y - k[2 * q + 1];
                a1[2 * q] += d0; a2[2 * q] = fmaf(d0, d0, a2[2 * q]);
                a1[2 * q + 1] += d1; a2[2 * q + 1] = fmaf(d1, d1, a2[2 * q + 1]);
            }
        }
    }
    const float rn = n ? 1.f / (float)n : 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) {                                 // the thread's mean - K and M2
        const float d = a1[j] * rn;
        sk[threadIdx.x * 8 + j] = k[j];
        s1[threadIdx.x * 8 + j] = d;
        s2[threadIdx.x * 8 + j] = fmaxf(fmaf(-a1[j], d, a2[j]), 0.f);
    }
    sn[threadIdx.x] = n;
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += BN_THREADS) {          // channel c: threads c / 8 + G * i, in order
        double cn = 0.0, sum = 0.0, m2 = 0.0;
        for (int i = 0; i < ppb; ++i) {
            const int t = c / 8 + G * i, e = t * 8 + c % 8;
            cn += (double)sn[t];
            sum += (double)sn[t] * ((double)sk[e] + (double)s1[e]);
        }
        const double cm = cn > 0.0 ? sum / cn : 0.0;
        for (int i = 0; i < ppb; ++i) {
            const int t = c / 8 + G * i, e = t * 8 + c % 8;
            const double d = (double)sk[e] + (double)s1[e] - cm;
            m2 += (double)s2[e] + (double)sn[t] * d * d;           // a thread without pixels adds 0
        }
        double *pc = part + (long long)blockIdx.x * BN_PART * C;
        pc[c] = cn;
        pc[C + c] = cm;
        pc[2 * C + c] = m2;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return false;
    __threadfence();
    // the last CTA: lanes = BN_THREADS / C threads per channel (C <= 128), lane l takes CTAs l, l + lanes, ...; the lanes'
    // partials are added in lane order, so the order of every addition is fixed
    __shared__ double red[BN_THREADS];
    const int lanes = C <= BN_THREADS / 2 ? BN_THREADS / C : 1;
    const int c = threadIdx.x % C, lane = threadIdx.x / C;
    const bool active = threadIdx.x < lanes * C;
    double sum = 0.0, m2 = 0.0;
    if (active)
        for (unsigned b = lane; b < gridDim.x; b += lanes) {
            const double *pc = part + (long long)b * BN_PART * C;
            sum += __ldcg(pc + c) * __ldcg(pc + C + c);
        }
    red[threadIdx.x] = sum;
    __syncthreads();
    double mu = 0.0;
    for (int l = 0; l < lanes; ++l) mu += red[l * C + c];
    mu /= (double)P;
    __syncthreads();
    if (active)
        for (unsigned b = lane; b < gridDim.x; b += lanes) {
            const double *pc = part + (long long)b * BN_PART * C, d = __ldcg(pc + C + c) - mu;
            m2 += __ldcg(pc + 2 * C + c) + __ldcg(pc + c) * d * d;
        }
    red[threadIdx.x] = m2;
    __syncthreads();
    m2 = 0.0;
    for (int l = 0; l < lanes; ++l) m2 += red[l * C + c];
    if (active && lane == 0) {
        const double v = m2 / (double)P;
        const double is = 1.0 / sqrt(v + (double)eps);
        const bool real = c < n_real;                            // padded channels: gamma = beta = 0, no running statistics
        const double sc = real ? (double)gamma[c] * is : 0.0;
        mean[c] = (float)mu;
        inv_std[c] = (float)is;
        if constexpr (!PER_ITEM) {
            if (var) var[c] = (float)v;
        }
        scale[c] = (float)sc;
        shift[c] = real ? (float)((double)beta[c] - mu * sc) : 0.f;
        if constexpr (PER_ITEM) {
            var[c] = (float)(v * (double)P / (double)(P - 1));
        } else {
            if (real) {
                running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
                running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)(v * (double)P / (double)(P - 1));
            }
        }
    }
    if (threadIdx.x == 0) *counter = 0u;
    return true;
}

// The per-item pass's running-statistics update (bn_stats_kernel<true>).  Not a template: a template instance's flag would be laid
// out after the statistics body's arrays and cost the kernel a byte more of shared memory.
__device__ __forceinline__ void
bn_items_running_update(int C, int n_real, float momentum, float *__restrict__ running_mean, float *__restrict__ running_var,
                        const float *__restrict__ mean, const float *__restrict__ uvar, unsigned int *__restrict__ counter)
{
    __shared__ bool all_done;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) all_done = atomicAdd(counter, 1u) == gridDim.y - 1;
    __syncthreads();
    if (!all_done) return;
    __threadfence();
    // the call-wide (1 - momentum) * r + momentum * x compiles to fma(x, momentum, (1 - momentum) * r); written out here so that
    // the compiler cannot contract the other product
    for (int c = threadIdx.x; c < n_real; c += BN_THREADS) {      // padded channels have no running statistics
        float rm = running_mean[c], rv = running_var[c];
        for (unsigned i = 0; i < gridDim.y; ++i) {
            rm = fmaf(__ldcg(mean + (long long)i * C + c), momentum, __fmul_rn(1.f - momentum, rm));
            rv = fmaf(__ldcg(uvar + (long long)i * C + c), momentum, __fmul_rn(1.f - momentum, rv));
        }
        running_mean[c] = rm;
        running_var[c] = rv;
    }
    if (threadIdx.x == 0) *counter = 0u;
}

// PER_ITEM: item i = blockIdx.y of a call of gridDim.y items, its P pixels the rows [i * P, (i + 1) * P): the same CTA partition
// (gridDim.x CTAs) and the same combine as the call-wide pass on those rows alone, so its mean / inv_std / scale / shift
// ([items, C]) are bit-identical to a single-item call.  var is uvar (workspace): each item's unbiased variance.  counter[1 + i] is
// item i's CTA counter and counter[0] counts the items that finished; the last CTA of the last one applies every item's running
// update in item order with the call-wide expression, so the running statistics end bit-identical to B single-item calls in a
// row.  A second counter rather than a follow-up launch: one launch per norm is what a batched call saves.
template <bool PER_ITEM>
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(const __nv_bfloat16 *__restrict__ g, long long P, int C, int n_real, const float *__restrict__ gamma,
                const float *__restrict__ beta, float eps, float momentum, float *__restrict__ running_mean,
                float *__restrict__ running_var, float *__restrict__ mean, float *__restrict__ inv_std, float *__restrict__ var,
                float *__restrict__ scale, float *__restrict__ shift, double *__restrict__ part, unsigned int *__restrict__ counter)
{
    const long long it = PER_ITEM ? blockIdx.y : 0, o = it * C;
    const bool last = bn_stats_body<PER_ITEM>(g + it * P * C, P, C, n_real, gamma, beta, eps, momentum, running_mean, running_var,
                                              mean + o, inv_std + o, var + o, scale + o, shift + o,
                                              part + it * gridDim.x * BN_PART * C, counter + (PER_ITEM ? 1 + it : 0));
    if constexpr (PER_ITEM)
        if (last) bn_items_running_update(C, n_real, momentum, running_mean, running_var, mean, var, counter);
}

// ------------------------------------------------------------------ apply
// y = bf16(g * scale + shift [+ residual]) per 16-byte vector of 8 channels; y may be g (no __restrict__ on either).  Without a
// residual, and with one, the result is the bf16 rounding of torch's fp32 evaluation of the same formula.
constexpr int BA_THREADS = 256;

__device__ __forceinline__ void
bn_apply_body(const __nv_bfloat16 *g, long long P, int C, const float *__restrict__ scale, const float *__restrict__ shift,
              const __nv_bfloat16 *__restrict__ residual, __nv_bfloat16 *y)
{
    const int G = C / 8;
    const long long n = P * G;
    for (long long v = blockIdx.x * (long long)BA_THREADS + threadIdx.x; v < n; v += (long long)gridDim.x * BA_THREADS) {
        const int co0 = 8 * (int)(v % G);
        const uint4 vg = *reinterpret_cast<const uint4 *>(g + 8 * v);
        const uint4 vr = residual ? *reinterpret_cast<const uint4 *>(residual + 8 * v) : make_uint4(0u, 0u, 0u, 0u);
        const float4 sa = __ldg(reinterpret_cast<const float4 *>(scale + co0)), sb = __ldg(reinterpret_cast<const float4 *>(scale + co0 + 4));
        const float4 ha = __ldg(reinterpret_cast<const float4 *>(shift + co0)), hb = __ldg(reinterpret_cast<const float4 *>(shift + co0 + 4));
        const float sc[8] = {sa.x, sa.y, sa.z, sa.w, sb.x, sb.y, sb.z, sb.w}, sh[8] = {ha.x, ha.y, ha.z, ha.w, hb.x, hb.y, hb.z, hb.w};
        const uint32_t wg[4] = {vg.x, vg.y, vg.z, vg.w}, wr[4] = {vr.x, vr.y, vr.z, vr.w};
        uint32_t o[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 a = bf16x2_val(wg[q]), r = bf16x2_val(wr[q]);
            // the fp32 formula as torch evaluates it (g * scale, + shift, + residual: separately rounded, no contraction to FMA)
            o[q] = bf16x2_bits(__fadd_rn(__fadd_rn(__fmul_rn(a.x, sc[2 * q]), sh[2 * q]), r.x),
                               __fadd_rn(__fadd_rn(__fmul_rn(a.y, sc[2 * q + 1]), sh[2 * q + 1]), r.y));
        }
        *reinterpret_cast<uint4 *>(y + 8 * v) = make_uint4(o[0], o[1], o[2], o[3]);
    }
}

// PER_ITEM: item blockIdx.y's P rows with its own scale / shift (row blockIdx.y of [items, C])
template <bool PER_ITEM>
__global__ void __launch_bounds__(BA_THREADS)
bn_apply_kernel(const __nv_bfloat16 *g, long long P, int C, const float *__restrict__ scale, const float *__restrict__ shift,
                const __nv_bfloat16 *__restrict__ residual, __nv_bfloat16 *y)
{
    const long long it = PER_ITEM ? blockIdx.y : 0, o = it * P * C;
    bn_apply_body(g + o, P, C, scale + it * C, shift + it * C, residual ? residual + o : nullptr, y + o);
}

// ------------------------------------------------------------------ launchers: the call-wide forms pass items = 1
// The statistics workspace, from its start: the counters (call-wide 1, per item 1 + items), then per item uvar [items, C], then
// the CTA partials (count, mean, M2 per CTA and channel) of every item; each block before the partials is rounded up to 256 bytes.
struct BnWorkspace { int64_t counters, uvar, part, bytes; };     // the number of counters, byte offsets, total bytes
static BnWorkspace bn_ws_layout(bool per_item, int items, int C)
{
    const auto round = [](int64_t b) { return (b + 255) / 256 * 256; };
    const int64_t counters = per_item ? 1 + items : 1, uvar = round(counters * 4);
    const int64_t part = uvar + (per_item ? round((int64_t)items * C * 4) : 0);
    return {counters, uvar, part, part + (int64_t)items * BN_MAX_CTAS * BN_PART * C * (int64_t)sizeof(double)};
}

// CTAs per item of the statistics pass: at most 2 per SM and BN_MAX_CTAS, so an item's partition is a single-item call's
static long long bn_stats_grid(int64_t pixels, int C)
{
    const int ppb = BN_THREADS / (C / 8);
    const long long blocks = (pixels + ppb - 1) / ppb, cap = 2ll * num_sms() < BN_MAX_CTAS ? 2ll * num_sms() : BN_MAX_CTAS;
    return blocks > cap ? cap : blocks;
}

// CTAs per item of the apply pass: the call's CTAs capped at 16 per SM, as for one call
static long long bn_apply_grid(int items, int64_t pixels, int C)
{
    long long blocks = (pixels * (C / 8) + BA_THREADS - 1) / BA_THREADS, cap = 16ll * num_sms() / items;
    if (cap < 1) cap = 1;
    return blocks > cap ? cap : blocks;
}

// The checks after the first null-pointer check, in each entry point's order: [items], C, for the statistics n_real and its
// parameter pointers (params: none is null), pixels, for the statistics eps / momentum, then the alignment of the or-ed addr.
static int bn_pass_checks(const char *name, bool stats, bool per_item, int items, int64_t pixels, int C, int n_real, bool params,
                          float eps, float momentum, uintptr_t addr)
{
    if (per_item) RB_CHECK_ARG(items >= 1 && items <= 65535, "%s: items must lie in 1..65535 (got %d)", name, items);
    RB_CHECK_ARG(bn_channels_ok(C), "%s: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)", name, BN_MAX_C, C);
    if (stats) {
        RB_CHECK_ARG(n_real >= 1 && n_real <= C, "%s: n_real must lie in 1..C (got %d, C = %d)", name, n_real, C);
        RB_CHECK_ARG(params, "%s: null pointer", name);
    }
    RB_CHECK_ARG(pixels >= 2, "%s: batch statistics need at least 2 pixels%s (got %lld)", name, per_item ? " per item" : "",
                 (long long)pixels);
    if (stats)
        RB_CHECK_ARG(eps > 0.f && momentum >= 0.f && momentum <= 1.f, "%s: bad eps / momentum (%g, %g)", name, eps, momentum);
    RB_CHECK_ARG((addr & 15) == 0, "%s: tensors must be 16B aligned", name);
    return READ_OK;
}

// var: the call-wide pass's optional output; per item the kernel's var is uvar in the workspace
template <bool PER_ITEM>
static int bn_stats_launch(const char *name, const void *g, int items, int64_t pixels, int C, int n_real, const float *gamma,
                           const float *beta, float eps, float momentum, float *running_mean, float *running_var, float *mean,
                           float *inv_std, float *var, float *scale, float *shift, void *workspace, void *stream)
{
    RB_CHECK_ARG(g && mean && inv_std && scale && shift && workspace, "%s: null pointer", name);
    if (const int rc = bn_pass_checks(name, true, PER_ITEM, items, pixels, C, n_real, gamma && beta && running_mean && running_var,
                                      eps, momentum, reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(workspace)))
        return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    const BnWorkspace ws = bn_ws_layout(PER_ITEM, items, C);
    char *w = (char *)workspace;
    RB_CUDA(cudaMemsetAsync(w, 0, (size_t)ws.counters * sizeof(unsigned int), st));
    bn_stats_kernel<PER_ITEM><<<dim3((unsigned)bn_stats_grid(pixels, C), (unsigned)items), BN_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)g, (long long)pixels, C, n_real, gamma, beta, eps, momentum, running_mean, running_var, mean, inv_std,
        PER_ITEM ? (float *)(w + ws.uvar) : var, scale, shift, (double *)(w + ws.part), (unsigned int *)w);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

template <bool PER_ITEM>
static int bn_apply_launch(const char *name, const void *g, int items, int64_t pixels, int C, const float *scale, const float *shift,
                           const void *residual, void *y, void *stream)
{
    RB_CHECK_ARG(g && scale && shift && y, "%s: null pointer", name);
    const uintptr_t addr = reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(residual) | reinterpret_cast<uintptr_t>(y) |
                           reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift);
    if (const int rc = bn_pass_checks(name, false, PER_ITEM, items, pixels, C, 0, true, 0.f, 0.f, addr)) return rc;
    bn_apply_kernel<PER_ITEM><<<dim3((unsigned)bn_apply_grid(items, pixels, C), (unsigned)items), BA_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)g, (long long)pixels, C, scale, shift, (const __nv_bfloat16 *)residual, (__nv_bfloat16 *)y);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb

using namespace rb;

extern "C" {

int64_t read_bn_workspace_bytes(int C) { return bn_channels_ok(C) ? bn_ws_layout(false, 1, C).bytes : -1; }

int64_t read_bn_workspace_bytes_items(int items, int C)
{
    return bn_channels_ok(C) && items >= 1 && items <= 65535 ? bn_ws_layout(true, items, C).bytes : -1;
}

int read_bn_batch_stats(const void *g, int64_t pixels, int C, int n_real, const float *gamma, const float *beta, float eps,
                        float momentum, float *running_mean, float *running_var, float *mean, float *inv_std, float *var,
                        float *scale, float *shift, void *workspace, void *stream)
{
    return bn_stats_launch<false>("bn_batch_stats", g, 1, pixels, C, n_real, gamma, beta, eps, momentum, running_mean, running_var,
                                  mean, inv_std, var, scale, shift, workspace, stream);
}

int read_bn_apply(const void *g, int64_t pixels, int C, const float *scale, const float *shift, const void *residual, void *y,
                  void *stream)
{
    return bn_apply_launch<false>("bn_apply", g, 1, pixels, C, scale, shift, residual, y, stream);
}

int read_bn_batch_stats_items(const void *g, int items, int64_t pixels, int C, int n_real, const float *gamma, const float *beta,
                              float eps, float momentum, float *running_mean, float *running_var, float *mean, float *inv_std,
                              float *scale, float *shift, void *workspace, void *stream)
{
    return bn_stats_launch<true>("bn_batch_stats_items", g, items, pixels, C, n_real, gamma, beta, eps, momentum, running_mean,
                                 running_var, mean, inv_std, nullptr, scale, shift, workspace, stream);
}

int read_bn_apply_items(const void *g, int items, int64_t pixels, int C, const float *scale, const float *shift, const void *residual,
                        void *y, void *stream)
{
    return bn_apply_launch<true>("bn_apply_items", g, items, pixels, C, scale, shift, residual, y, stream);
}

}  // extern "C"
