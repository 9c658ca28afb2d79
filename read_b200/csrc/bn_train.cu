// Train-mode BatchNorm of the gated convs (read_b200/blocks.py, batch_stats=True): the conv launch writes g = A(f + b_f) *
// sigmoid(m + b_m) with an identity epilogue (scale 1, shift 0, no residual), then
//   bn_stats   per-channel mean and biased variance of g over the P pixels of the call, inv_std, the folded scale / shift, and the
//              in-place running-statistics update (torch.nn.BatchNorm2d's train-mode semantics), all on the device
//   bn_apply   y = bf16(g * scale + shift [+ residual]), in place over g when the caller wants
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

__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(const __nv_bfloat16 *__restrict__ g, long long P, int C, int n_real, const float *__restrict__ gamma,
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
    if (!last) return;
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
        if (var) var[c] = (float)v;
        scale[c] = (float)sc;
        shift[c] = real ? (float)((double)beta[c] - mu * sc) : 0.f;
        if (real) {
            running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * (float)mu;
            running_var[c] = (1.f - momentum) * running_var[c] + momentum * (float)(v * (double)P / (double)(P - 1));
        }
    }
    if (threadIdx.x == 0) *counter = 0u;
}

// ------------------------------------------------------------------ apply
// y = bf16(g * scale + shift [+ residual]) per 16-byte vector of 8 channels; y may be g (no __restrict__ on either).  Without a
// residual, and with one, the result is the bf16 rounding of torch's fp32 evaluation of the same formula.
constexpr int BA_THREADS = 256;

__global__ void __launch_bounds__(BA_THREADS)
bn_apply_kernel(const __nv_bfloat16 *g, long long P, int C, const float *__restrict__ scale, const float *__restrict__ shift,
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

}  // namespace rb

using namespace rb;

extern "C" {

int64_t read_bn_workspace_bytes(int C)
{
    if (!bn_channels_ok(C)) return -1;
    return 256 + (int64_t)BN_MAX_CTAS * BN_PART * C * (int64_t)sizeof(double);
}

int read_bn_batch_stats(const void *g, int64_t pixels, int C, int n_real, const float *gamma, const float *beta, float eps,
                        float momentum, float *running_mean, float *running_var, float *mean, float *inv_std, float *var,
                        float *scale, float *shift, void *workspace, void *stream)
{
    RB_CHECK_ARG(g && mean && inv_std && scale && shift && workspace, "bn_batch_stats: null pointer");
    RB_CHECK_ARG(bn_channels_ok(C), "bn_batch_stats: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)", BN_MAX_C, C);
    RB_CHECK_ARG(n_real >= 1 && n_real <= C, "bn_batch_stats: n_real must lie in 1..C (got %d, C = %d)", n_real, C);
    RB_CHECK_ARG(gamma && beta && running_mean && running_var, "bn_batch_stats: null pointer");
    RB_CHECK_ARG(pixels >= 2, "bn_batch_stats: batch statistics need at least 2 pixels (got %lld)", (long long)pixels);
    RB_CHECK_ARG(eps > 0.f && momentum >= 0.f && momentum <= 1.f, "bn_batch_stats: bad eps / momentum (%g, %g)", eps, momentum);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
                 "bn_batch_stats: tensors must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    const int ppb = BN_THREADS / (C / 8);
    long long blocks = (pixels + ppb - 1) / ppb;
    const long long cap = 2ll * num_sms() < BN_MAX_CTAS ? 2ll * num_sms() : BN_MAX_CTAS;
    if (blocks > cap) blocks = cap;
    unsigned int *counter = (unsigned int *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), st));
    bn_stats_kernel<<<(unsigned)blocks, BN_THREADS, 0, st>>>((const __nv_bfloat16 *)g, (long long)pixels, C, n_real, gamma, beta,
                                                            eps, momentum, running_mean, running_var, mean, inv_std, var, scale,
                                                            shift, (double *)((char *)workspace + 256), counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_bn_apply(const void *g, int64_t pixels, int C, const float *scale, const float *shift, const void *residual, void *y,
                  void *stream)
{
    RB_CHECK_ARG(g && scale && shift && y, "bn_apply: null pointer");
    RB_CHECK_ARG(bn_channels_ok(C), "bn_apply: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)", BN_MAX_C, C);
    RB_CHECK_ARG(pixels >= 2, "bn_apply: batch statistics need at least 2 pixels (got %lld)", (long long)pixels);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(residual) | reinterpret_cast<uintptr_t>(y) |
                   reinterpret_cast<uintptr_t>(scale) | reinterpret_cast<uintptr_t>(shift)) & 15) == 0,
                 "bn_apply: tensors must be 16B aligned");
    const long long n = pixels * (C / 8);
    long long blocks = (n + BA_THREADS - 1) / BA_THREADS;
    if (blocks > 16ll * num_sms()) blocks = 16ll * num_sms();
    bn_apply_kernel<<<(unsigned)blocks, BA_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)g, (long long)pixels, C, scale, shift, (const __nv_bfloat16 *)residual, (__nv_bfloat16 *)y);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"
