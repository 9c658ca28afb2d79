// Backward of the gated 3x3 stride-1 convs (the residual blocks EBlock / DBlock, READ/models/unet.py:56-76, and the single convs
// around them) for bf16 training (read_b200/blocks.py: ResStackFn, GatedConvFn).  Per conv, last to first:
//   gate backward    one elementwise pass over dY and the recomputed pre-activation [f | m] -> [df | dm] (bf16) and the fp32
//                    per-channel sums dbias_f, dbias_m, dgamma, dbeta of the eval-mode BatchNorm
//   input gradient   the TMA wgmma conv kernel in RAW mode over [df | dm] with flipped, transposed filters
//                    (conv_tc.cu: read_pack_weights_tc_dgrad); the ResBlock skip enters through its residual operand.  An
//                    8-channel input (the descriptor pyramid) has its own kernel in this file (dgrad_cin8_kernel)
//   weight gradient  dW[2C][9][Cin] = sum over pixels of [df | dm]^T x im2col(x): the tensor-core kernel of this file
// The 1x1 and stride-2 3x3 / 4x4 convs of train_precision 'bf16_all' (blocks.py: MultiSourceConvFn) use the same gate backward,
// the weight-gradient kernel's other instances (read_conv_wgrad) and, for a stride-2 conv, the input-gradient kernel
// dgrad_s2_kernel of this file; a 1x1 conv's input gradient is a RAW 1x1 plan of the TMA kernel.
// Both kernels read [f | m] / [df | dm] rows in the column order of the forward RAW output: blocks of 2*half columns
// (half = min(C, 64), the forward plan's n_tile / 2), the conv_f half of a block first.
#include "common.cuh"
#include "conv_common.cuh"
#include "ptx.cuh"

namespace rb {

__device__ __forceinline__ int fm_col(int co, int half) { return (co / half) * 2 * half + co % half; }

// ------------------------------------------------------------------ gate backward
// y = scale * A(f + b_f) * sigmoid(m + b_m) + shift, scale = gamma * inv_std, shift = beta - mean * scale:
//   dg = dy * scale, df = dg * sigmoid * A', dm = dg * A * sigmoid * (1 - sigmoid),
//   dgamma = sum dy * (g - mean) * inv_std, dbeta = sum dy.
// A thread owns 8 channels (one 16-byte vector) of one pixel per step and keeps its channel group across pixels; its sums are
// reduced per CTA in shared memory and leave with one atomic per channel and CTA.
// BATCH: train-mode BatchNorm (mean / inv_std are this batch's statistics over the P pixels).  Its backward adds the terms through
// the statistics: dg = scale * (dy - sum_dy / P - xhat * sum_dy_xhat / P) = scale * dy + k1 * (g - mean) + k0 with
// k1 = -scale * inv_std * sum_dy_xhat / P, k0 = -scale * sum_dy / P; the two sums (= dgamma, dbeta) come from bn_bwd_reduce_kernel,
// so this instance accumulates no dgamma / dbeta.  BATCH = false compiles to the eval-mode kernel unchanged (the appended
// parameters are never read).
constexpr int GB_THREADS = 256, GB_MAX_C = 256;

// ---- deterministic reduction (DET instances, torch.use_deterministic_algorithms): no atomics on the sums.
// A CTA adds the per-thread sums of channel c in thread order (threads c / 8, c / 8 + G, ...) and stores them as its row of the
// caller's workspace part[cta][NS][C] (cta = blockIdx.y * gridDim.x + blockIdx.x); the last CTA to finish (counter + fence, the
// counter zeroed by the entry point and again by that CTA) combines the rows in a fixed order, see gate_det_combine.
__device__ __forceinline__ void gate_det_cta_sum(const float (&v)[8], int C, int G, int ppb, float *__restrict__ row)
{
    __shared__ float buf[GB_THREADS * 8];
#pragma unroll
    for (int j = 0; j < 8; ++j) buf[threadIdx.x * 8 + j] = v[j];
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += GB_THREADS) {
        float s = 0.f;
        for (int r = 0; r < ppb; ++r) s += buf[(r * G + c / 8) * 8 + c % 8];
        row[c] = s;
    }
    __syncthreads();
}

__device__ __forceinline__ bool gate_det_last(unsigned *counter)
{
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x * gridDim.y - 1;
    __syncthreads();
    if (last) __threadfence();
    return last;
}

// The last CTA: output e = (row r, sum k, channel c), r = an item when PER_ITEM (blockIdx.y's CTAs only), else 0 (every CTA).  Its
// n CTA rows are split over `lanes` threads (lane l adds CTAs l, l + lanes, ... in order, lanes = GB_THREADS / outputs when there
// are fewer outputs than threads, else 1) and the lanes' sums are added in lane order; the result is added to dst[k][r * C + c].
template <int NS, bool PER_ITEM>
__device__ __forceinline__ void gate_det_combine(const float *part, int C, float *d0, float *d1, float *d2, float *d3,
                                                 unsigned *counter)
{
    __shared__ float lred[GB_THREADS];
    const int gx = gridDim.x, rows = PER_ITEM ? gridDim.y : 1, n = PER_ITEM ? gx : gx * gridDim.y, O = rows * NS * C;
    const int lanes = O < GB_THREADS ? GB_THREADS / O : 1;
    for (int e0 = 0; e0 < O; e0 += GB_THREADS / lanes) {
        const int e = e0 + threadIdx.x % (GB_THREADS / lanes), l = threadIdx.x / (GB_THREADS / lanes);
        const int c = e % C, k = (e / C) % NS, r = e / (NS * C);
        float s = 0.f;
        if (e < O && l < lanes)
            for (int i = l; i < n; i += lanes) s += __ldcg(part + ((long long)(r * gx + i) * NS + k) * C + c);
        lred[threadIdx.x] = s;
        __syncthreads();
        if (threadIdx.x < GB_THREADS / lanes && e < O) {
            float t = 0.f;
            for (int q = 0; q < lanes; ++q) t += lred[q * (GB_THREADS / lanes) + threadIdx.x];
            float *d = k == 0 ? d0 : k == 1 ? d1 : k == 2 ? d2 : d3;
            d[(long long)r * C + c] += t;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *counter = 0u;
}

template <bool ELU, bool BATCH, bool DET = false>
__device__ __forceinline__ void
gate_bwd_body(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
              const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ scale,
              const float *__restrict__ mean, const float *__restrict__ inv_std, __nv_bfloat16 *__restrict__ dfm,
              float *__restrict__ dbf, float *__restrict__ dbm, float *__restrict__ dgamma, float *__restrict__ dbeta,
              const float *__restrict__ sum_dy, const float *__restrict__ sum_dy_xhat, float *__restrict__ part = nullptr,
              unsigned *__restrict__ counter = nullptr)
{
    __shared__ float red[4][GB_MAX_C];
    if constexpr (!DET) {
        for (int i = threadIdx.x; i < 4 * GB_MAX_C; i += GB_THREADS) (&red[0][0])[i] = 0.f;
        __syncthreads();
    }
    const int G = C / 8, ppb = GB_THREADS / G;
    const int cg = threadIdx.x % G, co0 = 8 * cg, fcol = fm_col(co0, half);
    float bf[8], bm[8], sc[8], mu[8], is[8];
    float s_bf[8], s_bm[8], s_g[8], s_b[8];
    float k1[8], k0[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        bf[j] = bias_f[co0 + j]; bm[j] = bias_m[co0 + j]; sc[j] = scale[co0 + j]; mu[j] = mean[co0 + j]; is[j] = inv_std[co0 + j];
        s_bf[j] = s_bm[j] = s_g[j] = s_b[j] = 0.f;
        if constexpr (BATCH) {
            const float rp = 1.f / (float)P;
            k1[j] = -sc[j] * is[j] * sum_dy_xhat[co0 + j] * rp;
            k0[j] = -sc[j] * sum_dy[co0 + j] * rp;
        }
    }
    if (threadIdx.x < ppb * G) {
        for (long long p = blockIdx.x * (long long)ppb + threadIdx.x / G; p < P; p += (long long)gridDim.x * ppb) {
            const uint4 vy = *reinterpret_cast<const uint4 *>(dy + p * C + co0);
            const uint4 vf = *reinterpret_cast<const uint4 *>(fm + p * 2 * C + fcol);
            const uint4 vm = *reinterpret_cast<const uint4 *>(fm + p * 2 * C + fcol + half);
            const uint32_t wy[4] = {vy.x, vy.y, vy.z, vy.w}, wf[4] = {vf.x, vf.y, vf.z, vf.w}, wm[4] = {vm.x, vm.y, vm.z, vm.w};
            uint32_t odf[4], odm[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 y2 = bf16x2_val(wy[q]), f2 = bf16x2_val(wf[q]), m2 = bf16x2_val(wm[q]);
                float df[2], dm[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = 2 * q + h;
                    const float y = h ? y2.y : y2.x;
                    const float f = (h ? f2.y : f2.x) + bf[j], m = (h ? m2.y : m2.x) + bm[j];
                    const float s = 1.f / (1.f + expf(-m));
                    float A = f, Ad = 1.f;
                    if (ELU && f <= 0.f) { A = expm1f(f); Ad = A + 1.f; }
                    const float g = A * s;
                    float dg;
                    if constexpr (BATCH) dg = fmaf(y, sc[j], fmaf(k1[j], g - mu[j], k0[j]));
                    else dg = y * sc[j];
                    df[h] = dg * s * Ad;
                    dm[h] = dg * A * s * (1.f - s);
                    s_bf[j] += df[h];
                    s_bm[j] += dm[h];
                    if constexpr (!BATCH) {
                        s_g[j] = fmaf(y, (g - mu[j]) * is[j], s_g[j]);
                        s_b[j] += y;
                    }
                }
                odf[q] = bf16x2_bits(df[0], df[1]);
                odm[q] = bf16x2_bits(dm[0], dm[1]);
            }
            *reinterpret_cast<uint4 *>(dfm + p * 2 * C + fcol) = make_uint4(odf[0], odf[1], odf[2], odf[3]);
            *reinterpret_cast<uint4 *>(dfm + p * 2 * C + fcol + half) = make_uint4(odm[0], odm[1], odm[2], odm[3]);
        }
        if constexpr (!DET) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                atomicAdd(&red[0][co0 + j], s_bf[j]);
                atomicAdd(&red[1][co0 + j], s_bm[j]);
                if constexpr (!BATCH) {
                    atomicAdd(&red[2][co0 + j], s_g[j]);
                    atomicAdd(&red[3][co0 + j], s_b[j]);
                }
            }
        }
    }
    if constexpr (DET) {
        constexpr int NS = BATCH ? 2 : 4;
        float *row = part + (long long)(blockIdx.y * gridDim.x + blockIdx.x) * NS * C;
        gate_det_cta_sum(s_bf, C, G, ppb, row);
        gate_det_cta_sum(s_bm, C, G, ppb, row + C);
        if constexpr (!BATCH) {
            gate_det_cta_sum(s_g, C, G, ppb, row + 2 * C);
            gate_det_cta_sum(s_b, C, G, ppb, row + 3 * C);
        }
        if (gate_det_last(counter)) gate_det_combine<NS, false>(part, C, dbf, dbm, dgamma, dbeta, counter);
        return;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += GB_THREADS) {
        atomicAdd(dbf + c, red[0][c]);
        atomicAdd(dbm + c, red[1][c]);
        if constexpr (!BATCH) {
            atomicAdd(dgamma + c, red[2][c]);
            atomicAdd(dbeta + c, red[3][c]);
        }
    }
}

template <bool ELU, bool BATCH>
__global__ void __launch_bounds__(GB_THREADS)
gate_bwd_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ scale,
                const float *__restrict__ mean, const float *__restrict__ inv_std, __nv_bfloat16 *__restrict__ dfm,
                float *__restrict__ dbf, float *__restrict__ dbm, float *__restrict__ dgamma, float *__restrict__ dbeta,
                const float *__restrict__ sum_dy, const float *__restrict__ sum_dy_xhat)
{
    gate_bwd_body<ELU, BATCH>(dy, fm, P, C, half, bias_f, bias_m, scale, mean, inv_std, dfm, dbf, dbm, dgamma, dbeta, sum_dy,
                              sum_dy_xhat);
}

// Per-item train-mode BatchNorm (UNet.train_batchnorm = 'per_item'): item i = blockIdx.y is the P rows [i * P, (i + 1) * P) with
// its own statistics (row i of the [items, C] scale / mean / inv_std / sums), so k1 / k0 come from item i's sums and P; dbias_f /
// dbias_m accumulate over every item.
template <bool ELU>
__global__ void __launch_bounds__(GB_THREADS)
gate_bwd_items_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                      const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ scale,
                      const float *__restrict__ mean, const float *__restrict__ inv_std, __nv_bfloat16 *__restrict__ dfm,
                      float *__restrict__ dbf, float *__restrict__ dbm, const float *__restrict__ sum_dy,
                      const float *__restrict__ sum_dy_xhat)
{
    const long long it = blockIdx.y, o = it * C;
    gate_bwd_body<ELU, true>(dy + it * P * C, fm + it * P * 2 * C, P, C, half, bias_f, bias_m, scale + o, mean + o, inv_std + o,
                             dfm + it * P * 2 * C, dbf, dbm, nullptr, nullptr, sum_dy + o, sum_dy_xhat + o);
}

// ------------------------------------------------------------------ train-mode BatchNorm: backward reduction
// sum_dy += sum dy, sum_dy_xhat += sum dy * (g - mean) * inv_std over the P pixels, with g = A(f + b_f) * sigmoid(m + b_m)
// recomputed from the RAW [f | m] (mean / inv_std: the batch statistics of the forward).  These are dbeta and dgamma, and the
// two terms the corrected gate backward (gate_bwd_kernel<ELU, true>) needs.  Same thread layout and reduction as the gate backward.
// DET: the deterministic reduction above; PER_ITEM: the last CTA writes item r's sums to row r (sum_dy / sum_dy_xhat [items, C]).
template <bool ELU, bool DET = false, bool PER_ITEM = false>
__device__ __forceinline__ void
bn_bwd_reduce_body(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                   const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ mean,
                   const float *__restrict__ inv_std, float *__restrict__ sum_dy, float *__restrict__ sum_dy_xhat,
                   float *__restrict__ part = nullptr, unsigned *__restrict__ counter = nullptr)
{
    __shared__ float red[2][GB_MAX_C];
    if constexpr (!DET) {
        for (int i = threadIdx.x; i < 2 * GB_MAX_C; i += GB_THREADS) (&red[0][0])[i] = 0.f;
        __syncthreads();
    }
    const int G = C / 8, ppb = GB_THREADS / G;
    const int cg = threadIdx.x % G, co0 = 8 * cg, fcol = fm_col(co0, half);
    float bf[8], bm[8], mu[8], is[8], s_b[8], s_g[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        bf[j] = bias_f[co0 + j]; bm[j] = bias_m[co0 + j]; mu[j] = mean[co0 + j]; is[j] = inv_std[co0 + j];
        s_b[j] = s_g[j] = 0.f;
    }
    if (threadIdx.x < ppb * G) {
        for (long long p = blockIdx.x * (long long)ppb + threadIdx.x / G; p < P; p += (long long)gridDim.x * ppb) {
            const uint4 vy = *reinterpret_cast<const uint4 *>(dy + p * C + co0);
            const uint4 vf = *reinterpret_cast<const uint4 *>(fm + p * 2 * C + fcol);
            const uint4 vm = *reinterpret_cast<const uint4 *>(fm + p * 2 * C + fcol + half);
            const uint32_t wy[4] = {vy.x, vy.y, vy.z, vy.w}, wf[4] = {vf.x, vf.y, vf.z, vf.w}, wm[4] = {vm.x, vm.y, vm.z, vm.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float2 y2 = bf16x2_val(wy[q]), f2 = bf16x2_val(wf[q]), m2 = bf16x2_val(wm[q]);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = 2 * q + h;
                    const float y = h ? y2.y : y2.x;
                    const float f = (h ? f2.y : f2.x) + bf[j], m = (h ? m2.y : m2.x) + bm[j];
                    const float s = 1.f / (1.f + expf(-m));
                    const float A = (ELU && f <= 0.f) ? expm1f(f) : f;
                    s_g[j] = fmaf(y, (A * s - mu[j]) * is[j], s_g[j]);
                    s_b[j] += y;
                }
            }
        }
        if constexpr (!DET) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                atomicAdd(&red[0][co0 + j], s_b[j]);
                atomicAdd(&red[1][co0 + j], s_g[j]);
            }
        }
    }
    if constexpr (DET) {
        float *row = part + (long long)(blockIdx.y * gridDim.x + blockIdx.x) * 2 * C;
        gate_det_cta_sum(s_b, C, G, ppb, row);
        gate_det_cta_sum(s_g, C, G, ppb, row + C);
        if (gate_det_last(counter)) gate_det_combine<2, PER_ITEM>(part, C, sum_dy, sum_dy_xhat, nullptr, nullptr, counter);
        return;
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += GB_THREADS) {
        atomicAdd(sum_dy + c, red[0][c]);
        atomicAdd(sum_dy_xhat + c, red[1][c]);
    }
}

template <bool ELU>
__global__ void __launch_bounds__(GB_THREADS)
bn_bwd_reduce_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                     const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ mean,
                     const float *__restrict__ inv_std, float *__restrict__ sum_dy, float *__restrict__ sum_dy_xhat)
{
    bn_bwd_reduce_body<ELU>(dy, fm, P, C, half, bias_f, bias_m, mean, inv_std, sum_dy, sum_dy_xhat);
}

// per item: the sums of item blockIdx.y (its P rows, its mean / inv_std) into row blockIdx.y of [items, C]
template <bool ELU>
__global__ void __launch_bounds__(GB_THREADS)
bn_bwd_reduce_items_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C,
                           int half, const float *__restrict__ bias_f, const float *__restrict__ bias_m,
                           const float *__restrict__ mean, const float *__restrict__ inv_std, float *__restrict__ sum_dy,
                           float *__restrict__ sum_dy_xhat)
{
    const long long it = blockIdx.y, o = it * C;
    bn_bwd_reduce_body<ELU>(dy + it * P * C, fm + it * P * 2 * C, P, C, half, bias_f, bias_m, mean + o, inv_std + o, sum_dy + o,
                            sum_dy_xhat + o);
}

// Deterministic instances (torch.use_deterministic_algorithms): the bodies above with DET, the CTA partials in part / counter.
// The per-item forms take the unshifted pointers: the body's last CTA combines every item (gate: into one dbias_f / dbias_m; BN
// reduce: item r into row r).
template <bool ELU, bool BATCH>
__global__ void __launch_bounds__(GB_THREADS)
gate_bwd_det_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                    const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ scale,
                    const float *__restrict__ mean, const float *__restrict__ inv_std, __nv_bfloat16 *__restrict__ dfm,
                    float *__restrict__ dbf, float *__restrict__ dbm, float *__restrict__ dgamma, float *__restrict__ dbeta,
                    const float *__restrict__ sum_dy, const float *__restrict__ sum_dy_xhat, float *__restrict__ part,
                    unsigned *__restrict__ counter)
{
    gate_bwd_body<ELU, BATCH, true>(dy, fm, P, C, half, bias_f, bias_m, scale, mean, inv_std, dfm, dbf, dbm, dgamma, dbeta, sum_dy,
                                    sum_dy_xhat, part, counter);
}

template <bool ELU>
__global__ void __launch_bounds__(GB_THREADS)
gate_bwd_items_det_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                          const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ scale,
                          const float *__restrict__ mean, const float *__restrict__ inv_std, __nv_bfloat16 *__restrict__ dfm,
                          float *__restrict__ dbf, float *__restrict__ dbm, const float *__restrict__ sum_dy,
                          const float *__restrict__ sum_dy_xhat, float *__restrict__ part, unsigned *__restrict__ counter)
{
    const long long it = blockIdx.y, o = it * C;
    gate_bwd_body<ELU, true, true>(dy + it * P * C, fm + it * P * 2 * C, P, C, half, bias_f, bias_m, scale + o, mean + o,
                                   inv_std + o, dfm + it * P * 2 * C, dbf, dbm, nullptr, nullptr, sum_dy + o, sum_dy_xhat + o, part,
                                   counter);
}

template <bool ELU>
__global__ void __launch_bounds__(GB_THREADS)
bn_bwd_reduce_det_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C, int half,
                         const float *__restrict__ bias_f, const float *__restrict__ bias_m, const float *__restrict__ mean,
                         const float *__restrict__ inv_std, float *__restrict__ sum_dy, float *__restrict__ sum_dy_xhat,
                         float *__restrict__ part, unsigned *__restrict__ counter)
{
    bn_bwd_reduce_body<ELU, true>(dy, fm, P, C, half, bias_f, bias_m, mean, inv_std, sum_dy, sum_dy_xhat, part, counter);
}

template <bool ELU>
__global__ void __launch_bounds__(GB_THREADS)
bn_bwd_reduce_items_det_kernel(const __nv_bfloat16 *__restrict__ dy, const __nv_bfloat16 *__restrict__ fm, long long P, int C,
                               int half, const float *__restrict__ bias_f, const float *__restrict__ bias_m,
                               const float *__restrict__ mean, const float *__restrict__ inv_std, float *__restrict__ sum_dy,
                               float *__restrict__ sum_dy_xhat, float *__restrict__ part, unsigned *__restrict__ counter)
{
    const long long it = blockIdx.y, o = it * C;
    bn_bwd_reduce_body<ELU, true, true>(dy + it * P * C, fm + it * P * 2 * C, P, C, half, bias_f, bias_m, mean + o, inv_std + o,
                                        sum_dy, sum_dy_xhat, part, counter);
}

// ------------------------------------------------------------------ weight gradient
// GEMM  dW[M = 2C columns of [df | dm]][N = 9 taps x Cin] += A[M][K = pixels] * B[K][N], bf16 in, fp32 accumulators in
// registers (mma.sync m16n8k16).  A CTA owns a 64-column x 32-input-channel block for all 9 taps and walks a strided share of
// the image's 32-pixel row segments (split K): per segment it loads the [32 px][64] slice of [df | dm] and the [3 rows][34 px][32]
// halo of x once (cp.async, double-buffered, zero-filled outside the image, which is the forward conv's zero padding) and
// reads every tap's B operand out of that halo with ldmatrix.trans at a shifted pixel offset.  Split-K partials leave through fp32
// atomics into the torch-layout gradients [C][Cin][3][3].
// Warps: 8 = 2 (32 columns each) x 4 (8 input channels each); a warp holds 2 x 9 m16n8 tiles = 72 accumulators per thread.
// Narrow convs (Cin = 8 or 16: the descriptor pyramid; 2C = 32 columns: the RGB output conv padded to C = 16) run in one
// partial block: its loads are zero-filled beyond Cin and beyond 2C, and only real (column, channel) pairs are stored.
// The kernel is a template over the filter size KS and the stride (pad (KS - 1) / 2 rounded up: 0 for 1x1, 1 otherwise):
// 32 output pixels read the x halo of KR filter rows x (STRIDE * 31 + KS) input pixels, tap (ky, kx) of output pixel p sits at
// halo pixel STRIDE * p + kx.  A CTA holds the taps of KR filter rows; a 4x4 filter is split into two groups of two rows over
// blockIdx.z (16 taps would take 128 accumulators per thread), the other sizes keep all rows (KR = KS).
constexpr int WG_THREADS = 256, WG_PX = 32, WG_M = 64, WG_N = 32;
constexpr uint32_t WG_A_BYTES = WG_PX * WG_M * 2;                  // 128-byte rows
__host__ __device__ constexpr int wg_halo(int KS, int STRIDE) { return STRIDE * (WG_PX - 1) + KS; }
__host__ __device__ constexpr uint32_t wg_x_bytes(int KS, int STRIDE, int KR)          // 64-byte rows, rounded up to 128 bytes
{
    return ((uint32_t)KR * wg_halo(KS, STRIDE) * WG_N * 2u + 127u) & ~127u;
}
__host__ __device__ constexpr uint32_t wg_stage(int KS, int STRIDE, int KR) { return WG_A_BYTES + wg_x_bytes(KS, STRIDE, KR); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, bool valid)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t (&r)[4])
{
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(addr)
                 : "memory");
}

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                 "{%0, %1, %2, %3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// H, W: the output (= [df | dm]) size; the input x is [B][STRIDE * H][STRIDE * W][Cin] (the callers check Hin == STRIDE * Hout).
// DET (torch.use_deterministic_algorithms): instead of the atomics, split blockIdx.x stores its partial sums to its own copy of
// the gradients, part[split][2][C][Cin][KS][KS] (conv_f, then conv_m); wgrad_split_sum_kernel adds the copies in split order.
template <int KS, int STRIDE, int KR, bool DET>
__device__ __forceinline__ void
wgrad_body(const __nv_bfloat16 *__restrict__ dfm, const __nv_bfloat16 *__restrict__ x, int B, int H, int W, int C, int Cin, int half,
           float *__restrict__ dwf, float *__restrict__ dwm, float *__restrict__ part)
{
    constexpr int HALO = wg_halo(KS, STRIDE), TAPS = KR * KS, GROUPS = KS / KR, PAD = KS == 1 ? 0 : 1;
    constexpr uint32_t STAGE = wg_stage(KS, STRIDE, KR);
    __shared__ __align__(128) uint8_t sm[2 * STAGE];
    const int ky0 = (blockIdx.z % GROUPS) * KR;
    const int m0 = blockIdx.y * WG_M, n0 = (blockIdx.z / GROUPS) * WG_N;
    const int segs = (W + WG_PX - 1) / WG_PX;
    const long long chunks = (long long)B * H * segs;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp & 1, wq = warp >> 1;
    const uint32_t s0 = s_u32(sm);
    const int twoC = 2 * C;

    auto load = [&](long long ch, int st) {
        const int seg = (int)(ch % segs);
        const long long r = ch / segs;
        const int y = (int)(r % H), b = (int)(r / H), x0 = seg * WG_PX;
        const uint32_t base = s0 + (uint32_t)st * STAGE;
        {   // [df | dm]: 32 pixels x 8 16-byte chunks, one per thread
            const int k = tid >> 3, q = tid & 7;
            const bool ok = x0 + k < W && m0 + 8 * q < twoC;
            const __nv_bfloat16 *src = ok ? dfm + (((long long)b * H + y) * W + x0 + k) * twoC + m0 + 8 * q : dfm;
            cp_async16(base + swz((uint32_t)k * 128u + 16u * q, 128u), src, ok);
        }
        for (int i = tid; i < KR * HALO * 4; i += WG_THREADS) {   // x halo: KR filter rows x HALO pixels, 4 chunks
            const int hp = i >> 2, q = i & 3;
            const int gy = STRIDE * y + ky0 + hp / HALO - PAD, gx = STRIDE * x0 + hp % HALO - PAD;
            const bool ok = gy >= 0 && gy < STRIDE * H && gx >= 0 && gx < STRIDE * W && n0 + 8 * q < Cin;
            const __nv_bfloat16 *src = ok ? x + (((long long)b * (STRIDE * H) + gy) * (STRIDE * W) + gx) * Cin + n0 + 8 * q : x;
            cp_async16(base + WG_A_BYTES + swz((uint32_t)hp * 64u + 16u * q, 64u), src, ok);
        }
    };

    float acc[2][TAPS][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int t = 0; t < TAPS; ++t)
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[mi][t][i] = 0.f;

    const int j = lane >> 3;
    int st = 0;
    if (blockIdx.x < chunks) load(blockIdx.x, 0);
    cp_async_commit();
    for (long long ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        if (ch + gridDim.x < chunks) load(ch + gridDim.x, st ^ 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        const uint32_t sa = s0 + (uint32_t)st * STAGE, sx = sa + WG_A_BYTES;
        // A fragments (columns x pixels) of the warp's two m16 tiles and the segment's two k16 steps, from the [pixel][column] tile
        uint32_t af[2][2][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi)
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
                const int k = 16 * ks + (lane & 7) + 8 * (j >> 1);
                const int col = 32 * wm + 16 * mi + 8 * (j & 1);
                ldmatrix_x4_trans(sa + swz((uint32_t)k * 128u + (uint32_t)col * 2u, 128u), af[mi][ks]);
            }
#pragma unroll
        for (int tap = 0; tap < TAPS; ++tap) {
            // B fragments of both k16 steps: matrix j = pixels 8j..8j+7 of the segment, read at halo (ky, STRIDE * pixel + kx)
            const int hp = (tap / KS) * HALO + tap % KS + STRIDE * (8 * j + (lane & 7));
            uint32_t bfr[4];
            ldmatrix_x4_trans(sx + swz((uint32_t)hp * 64u + 16u * wq, 64u), bfr);
#pragma unroll
            for (int mi = 0; mi < 2; ++mi) {
                mma_16816(acc[mi][tap], af[mi][0], bfr[0], bfr[1]);
                mma_16816(acc[mi][tap], af[mi][1], bfr[2], bfr[3]);
            }
        }
        __syncthreads();
        st ^= 1;
    }
    cp_async_wait<0>();

    // accumulator (row g [+8], columns 2t, 2t+1) -> dW[o][ci][ky][kx] of conv_f or conv_m
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int col = m0 + 32 * wm + 16 * mi + g + 8 * (i >> 1);
            const int ci = n0 + 8 * wq + 2 * t4 + (i & 1);
            if (col >= twoC || ci >= Cin) continue;
            const int rr = col % (2 * half);
            const int o = (col / (2 * half)) * half + rr % half;
            if constexpr (DET) {
                const long long nw = (long long)C * Cin * (KS * KS);
                float *dw = part + ((long long)blockIdx.x * 2 + (rr >= half)) * nw + ((long long)o * Cin + ci) * (KS * KS) + ky0 * KS;
#pragma unroll
                for (int tap = 0; tap < TAPS; ++tap) dw[tap] = acc[mi][tap][i];
            } else {
                float *dw = (rr >= half ? dwm : dwf) + ((long long)o * Cin + ci) * (KS * KS) + ky0 * KS;
#pragma unroll
                for (int tap = 0; tap < TAPS; ++tap) atomicAdd(dw + tap, acc[mi][tap][i]);
            }
        }
}

template <int KS, int STRIDE, int KR>
__global__ void __launch_bounds__(WG_THREADS)
wgrad_kernel(const __nv_bfloat16 *__restrict__ dfm, const __nv_bfloat16 *__restrict__ x, int B, int H, int W, int C, int Cin,
             int half, float *__restrict__ dwf, float *__restrict__ dwm)
{
    wgrad_body<KS, STRIDE, KR, false>(dfm, x, B, H, W, C, Cin, half, dwf, dwm, nullptr);
}

template <int KS, int STRIDE, int KR>
__global__ void __launch_bounds__(WG_THREADS)
wgrad_det_kernel(const __nv_bfloat16 *__restrict__ dfm, const __nv_bfloat16 *__restrict__ x, int B, int H, int W, int C, int Cin,
                 int half, float *__restrict__ part)
{
    wgrad_body<KS, STRIDE, KR, true>(dfm, x, B, H, W, C, Cin, half, nullptr, nullptr, part);
}

// dwf[e] / dwm[e] += the splits' copies of element e added in split order, from 0
__global__ void wgrad_split_sum_kernel(const float *__restrict__ part, int splits, long long nw, float *__restrict__ dwf,
                                       float *__restrict__ dwm)
{
    for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < 2 * nw; e += (long long)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < splits; ++k) s += __ldcg(part + k * 2 * nw + e);
        (e < nw ? dwf : dwm)[e < nw ? e : e - nw] += s;
    }
}

// the launch geometry of wgrad_kernel<KS, STRIDE, KR>: splits (blockIdx.x), column blocks, input-channel blocks x filter-row groups
template <int KS, int KR>
static void wgrad_grid(int B, int H, int W, int Cout, int Cin, long long &s, int &mb, int &nz)
{
    const long long chunks = (long long)B * H * ((W + WG_PX - 1) / WG_PX);
    mb = (2 * Cout + WG_M - 1) / WG_M;
    nz = ((Cin + WG_N - 1) / WG_N) * (KS / KR);
    s = (2ll * num_sms() + mb * nz - 1) / (mb * nz);
    if (s > chunks) s = chunks;
}

template <int KS, int STRIDE, int KR>
static int launch_wgrad_det(const void *dfm, const void *x, int B, int H, int W, int Cout, int Cin, float *dwf, float *dwm,
                            void *workspace, cudaStream_t st)
{
    long long s;
    int mb, nz;
    wgrad_grid<KS, KR>(B, H, W, Cout, Cin, s, mb, nz);
    RB_CHECK_ARG(s <= 0x7FFFFFFF && nz <= 65535 && mb <= 65535, "conv_wgrad_det: too large");
    float *part = (float *)workspace;
    wgrad_det_kernel<KS, STRIDE, KR><<<dim3((unsigned)s, mb, nz), WG_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dfm, (const __nv_bfloat16 *)x, B, H, W, Cout, Cin, Cout < 64 ? Cout : 64, part);
    RB_LAUNCH_CHECK();
    const long long nw = (long long)Cout * Cin * KS * KS;
    long long blocks = (2 * nw + 255) / 256;
    if (blocks > 16ll * num_sms()) blocks = 16ll * num_sms();
    wgrad_split_sum_kernel<<<(unsigned)blocks, 256, 0, st>>>(part, (int)s, nw, dwf, dwm);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

template <int KS, int STRIDE, int KR>
static int launch_wgrad(const void *dfm, const void *x, int B, int H, int W, int Cout, int Cin, float *dwf, float *dwm,
                        cudaStream_t st)
{
    const long long chunks = (long long)B * H * ((W + WG_PX - 1) / WG_PX);
    const int mb = (2 * Cout + WG_M - 1) / WG_M, nz = ((Cin + WG_N - 1) / WG_N) * (KS / KR);
    long long s = (2ll * num_sms() + mb * nz - 1) / (mb * nz);
    if (s > chunks) s = chunks;
    RB_CHECK_ARG(s <= 0x7FFFFFFF && nz <= 65535 && mb <= 65535, "conv_wgrad: too large");
    wgrad_kernel<KS, STRIDE, KR><<<dim3((unsigned)s, mb, nz), WG_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dfm, (const __nv_bfloat16 *)x, B, H, W, Cout, Cin, Cout < 64 ? Cout : 64, dwf, dwm);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

// ------------------------------------------------------------------ input gradient of an 8-channel input
// The convs that read the descriptor pyramid (feat_extract.0, SCM*.main.0: Cin = 8, C = 16 / 32 / 64) need
//   dX[p][n] = sum over taps (ty, tx) and columns k of [df | dm] of dfm[p + (ty - 1, tx - 1)][k] * w_k[n][2 - ty][2 - tx],
// an implicit GEMM with N = 8: exactly one mma.sync m16n8k16 tile, where the TMA kernel's smallest N is 16.  A persistent CTA
// converts the flipped, transposed filters to bf16 in shared memory once ([tap][n][k]), then walks a strided share of the
// image's 64-pixel row segments: per segment it loads the 3-row [df | dm] halo (cp.async, zero-filled outside the image, which
// is the transposed conv's zero padding) and each warp computes 16 pixels x 8 channels over all 9 taps.  Shared-memory rows
// are padded by 16 bytes, so the ldmatrix reads of A and the 32-bit reads of B touch 32 distinct banks.
constexpr int DG8_THREADS = 128, DG8_PX = 64, DG8_HALO = DG8_PX + 2;

__host__ __device__ constexpr uint32_t dg8_row_bytes(int K2) { return (uint32_t)K2 * 2u + 16u; }
__host__ __device__ constexpr uint32_t dg8_smem_bytes(int K2) { return (9u * 8u + 3u * DG8_HALO) * dg8_row_bytes(K2); }

template <int K2>       // columns of [df | dm] = 2C
__global__ void __launch_bounds__(DG8_THREADS)
dgrad_cin8_kernel(const __nv_bfloat16 *__restrict__ dfm, const float *__restrict__ wf, const float *__restrict__ wm, int B, int H,
                  int W, __nv_bfloat16 *__restrict__ dx)
{
    extern __shared__ __align__(16) uint8_t dg_sm[];
    constexpr uint32_t ROW = dg8_row_bytes(K2);
    constexpr int HALF = K2 / 2 < 64 ? K2 / 2 : 64;          // the RAW column order's block: 2*HALF columns, conv_f half first
    const uint32_t sw = s_u32(dg_sm), sx = sw + 9u * 8u * ROW;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 9 * 8 * K2; i += DG8_THREADS) {
        const int k = i % K2, n = (i / K2) % 8, tap = i / (8 * K2);
        const int rr = k % (2 * HALF), o = (k / (2 * HALF)) * HALF + rr % HALF;
        const float *w = rr >= HALF ? wm : wf;
        const int ky = 2 - tap / 3, kx = 2 - tap % 3;
        *reinterpret_cast<__nv_bfloat16 *>(dg_sm + (tap * 8 + n) * ROW + 2 * k) = __float2bfloat16_rn(w[((o * 8 + n) * 3 + ky) * 3 + kx]);
    }
    const int segs = (W + DG8_PX - 1) / DG8_PX;
    const long long chunks = (long long)B * H * segs;
    const int pr = 16 * warp + (lane & 7) + 8 * ((lane >> 3) & 1);   // this lane's ldmatrix row: pixel of the segment
    const uint32_t a_lane = sx + (uint32_t)pr * ROW + (uint32_t)(lane >> 4) * 16u;
    const uint32_t b_lane = sw + (uint32_t)(lane >> 2) * ROW + 4u * (lane & 3);
    const int g = lane >> 2, t4 = lane & 3;
    for (long long ch = blockIdx.x; ch < chunks; ch += gridDim.x) {
        const int seg = (int)(ch % segs);
        const long long r = ch / segs;
        const int y = (int)(r % H), b = (int)(r / H), x0 = seg * DG8_PX;
        __syncthreads();                      // the previous segment's halo is read (and, the first time, the filters stored)
        for (int i = tid; i < 3 * DG8_HALO * (K2 / 8); i += DG8_THREADS) {
            const int hp = i / (K2 / 8), q = i % (K2 / 8);
            const int gy = y + hp / DG8_HALO - 1, gx = x0 + hp % DG8_HALO - 1;
            const bool ok = gy >= 0 && gy < H && gx >= 0 && gx < W;
            const __nv_bfloat16 *src = ok ? dfm + (((long long)b * H + gy) * W + gx) * K2 + 8 * q : dfm;
            cp_async16(sx + (uint32_t)hp * ROW + 16u * q, src, ok);
        }
        cp_async_commit();
        cp_async_wait<0>();
        __syncthreads();
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const uint32_t a_tap = a_lane + (uint32_t)((tap / 3) * DG8_HALO + tap % 3) * ROW, b_tap = b_lane + tap * 8u * ROW;
#pragma unroll
            for (int ks = 0; ks < K2 / 16; ++ks) {
                uint32_t af[4], b0, b1;
                ldmatrix_x4(a_tap + 32u * ks, af);
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b0) : "r"(b_tap + 32u * ks));
                asm volatile("ld.shared.b32 %0, [%1];" : "=r"(b1) : "r"(b_tap + 32u * ks + 16u));
                mma_16816(acc, af, b0, b1);
            }
        }
        // accumulator rows g, g + 8 = pixels, columns 2t, 2t + 1 = input channels
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int px = x0 + 16 * warp + g + 8 * i;
            if (px < W)
                *reinterpret_cast<uint32_t *>(dx + (((long long)b * H + y) * W + px) * 8 + 2 * t4) = bf16x2_bits(acc[2 * i], acc[2 * i + 1]);
        }
    }
}

template <int K2>
static int launch_dgrad_cin8(const void *dfm, const float *wf, const float *wm, int B, int H, int W, void *dx, cudaStream_t st)
{
    constexpr uint32_t smem = dg8_smem_bytes(K2);
    RB_CUDA(cudaFuncSetAttribute(dgrad_cin8_kernel<K2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long chunks = (long long)B * H * ((W + DG8_PX - 1) / DG8_PX);
    long long per_sm = (200u * 1024u) / smem;              // CTAs that fit one SM's shared memory
    if (per_sm > 8) per_sm = 8;
    long long grid = per_sm * num_sms();
    if (grid > chunks) grid = chunks;
    dgrad_cin8_kernel<K2><<<(unsigned)grid, DG8_THREADS, smem, st>>>((const __nv_bfloat16 *)dfm, wf, wm, B, H, W, (__nv_bfloat16 *)dx);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

// ------------------------------------------------------------------ input gradient of a stride-2 conv
// A stride-2 pad-1 conv (3x3 / 4x4) reads input pixel i = 2o - 1 + k with tap k of output pixel o, so its input gradient is a
// transposed conv: input pixel i = 2a + p receives dfm[o] * w[k] for every k = 2(a - o) + p + 1 in [0, KS), i.e. from output
// pixel o = a + (p + 1 - k) / 2 with k of the parity of p + 1 (p = 0: k = 1 [, 3]; p = 1: k = 0, 2).  Rows and columns are
// independent, so per input row the kernel needs at most two rows of [df | dm] (slot s: filter row ky = 2s + 1 - p) and per
// column phase at most two filter columns.  A CTA (4 warps) owns one input row, a 64-pixel segment of it (32 pixels of each
// column phase) and 32 input channels: warp w computes the 16 pixels 16 * (w >> 1) + 0..15 of column phase w & 1 with
// mma.sync m16n8k16 (bf16 in, fp32 accumulators), K = the 2C columns of [df | dm] in chunks of 32 times its <= 4 taps.  Per chunk
// a stage holds the two 34-pixel [df | dm] rows and the row phase's <= 8 taps of the packed filters ([tap][Cin][2C] bf16,
// read_pack_weights_dgrad_s2), loaded with cp.async (zero-filled outside the output image: the conv's zero padding), double
// buffered across the CTA's sequence of (row segment, chunk) items.  The interleaved NHWC dx is written straight from the
// accumulators.  64-byte shared-memory rows with the 64-byte swizzle: the ldmatrix reads touch 32 distinct banks.
constexpr int DS_THREADS = 128, DS_PX = 64, DS_OX = DS_PX / 2 + 2, DS_K = 32, DS_N = 32;
constexpr uint32_t DS_A_BYTES = 2u * DS_OX * DS_K * 2u;             // two [df | dm] rows
constexpr uint32_t DS_B_BYTES = 8u * DS_N * DS_K * 2u;              // <= 2 filter rows x 4 filter columns
constexpr uint32_t DS_STAGE = DS_A_BYTES + DS_B_BYTES;

template <int KS>
__global__ void __launch_bounds__(DS_THREADS)
dgrad_s2_kernel(const __nv_bfloat16 *__restrict__ dfm, const __nv_bfloat16 *__restrict__ wt, int B, int Ho, int Wo, int K2,
                int Cin, __nv_bfloat16 *__restrict__ dx)
{
    __shared__ __align__(128) uint8_t sm[2 * DS_STAGE];
    const int Hi = 2 * Ho, Wi = 2 * Wo;
    const int n0 = blockIdx.y * DS_N;
    const int segs = (Wi + DS_PX - 1) / DS_PX, kchunks = K2 / DS_K;
    const long long rows = (long long)B * Hi * segs;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int px = warp & 1, grp = warp >> 1;
    const uint32_t s0 = s_u32(sm);

    auto load = [&](long long rw, int kc, int st) {
        const int seg = (int)(rw % segs);
        const long long r = rw / segs;
        const int i = (int)(r % Hi), b = (int)(r / Hi);
        const int py = i & 1, a = i >> 1, c0 = seg * (DS_PX / 2);
        const uint32_t base = s0 + (uint32_t)st * DS_STAGE;
        for (int q = tid; q < 2 * DS_OX * 4; q += DS_THREADS) {      // [df | dm] rows: slot s = filter row 2s + 1 - py
            const int hp = q >> 2, ch = q & 3, s = hp / DS_OX, ox = c0 - 1 + hp % DS_OX;
            const int ky = 2 * s + 1 - py, oy = a + (py + 1 - ky) / 2;
            const bool ok = ky < KS && oy >= 0 && oy < Ho && ox >= 0 && ox < Wo;
            const __nv_bfloat16 *src = ok ? dfm + (((long long)b * Ho + oy) * Wo + ox) * K2 + kc * DS_K + 8 * ch : dfm;
            cp_async16(base + swz((uint32_t)hp * 64u + 16u * ch, 64u), src, ok);
        }
        for (int q = tid; q < 2 * KS * DS_N * 4; q += DS_THREADS) {  // filters: [slot s][kx][n][k]
            const int row = q >> 2, ch = q & 3, t = row / DS_N, n = row % DS_N, ky = 2 * (t / KS) + 1 - py, kx = t % KS;
            const bool ok = ky < KS;
            const __nv_bfloat16 *src = ok ? wt + ((long long)(ky * KS + kx) * Cin + n0 + n) * K2 + kc * DS_K + 8 * ch : wt;
            cp_async16(base + DS_A_BYTES + swz((uint32_t)row * 64u + 16u * ch, 64u), src, ok);
        }
    };

    const int arow = (lane & 7) + 8 * ((lane >> 3) & 1);              // this lane's ldmatrix row of the A tile: pixel
    const uint32_t a_k = (uint32_t)(lane >> 4) * 16u;
    const int brow = (lane & 7) + 8 * (lane >> 4);                    // ... of the B tiles: input channel
    const uint32_t b_k = (uint32_t)((lane >> 3) & 1) * 16u;
    const int g = lane >> 2, t4 = lane & 3;
    float acc[4][4];
    long long rw = blockIdx.x;
    int kc = 0, st = 0;
    if (rw < rows) load(rw, 0, 0);
    cp_async_commit();
    while (rw < rows) {
        long long nrw = rw;
        int nkc = kc + 1;
        if (nkc == kchunks) { nkc = 0; nrw += gridDim.x; }
        if (nrw < rows) load(nrw, nkc, st ^ 1);
        cp_async_commit();
        cp_async_wait<1>();
        __syncthreads();
        if (kc == 0) {
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[nt][e] = 0.f;
        }
        const long long r = rw / segs;
        const int py = (int)(r % Hi) & 1;
        const uint32_t sa = s0 + (uint32_t)st * DS_STAGE, sb = sa + DS_A_BYTES;
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            if (2 * s + 1 - py >= KS) continue;                           // 3x3, even rows: one filter row
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int kx = 2 * u + 1 - px;
                if (kx >= KS) continue;                                   // 3x3, even columns: one filter column
                const int hp = s * DS_OX + 16 * grp + 1 + (px + 1 - kx) / 2 + arow;     // dfm pixel c + (px + 1 - kx) / 2
                const uint32_t bt = sb + (uint32_t)(s * KS + kx) * DS_N * 64u;
#pragma unroll
                for (int ks = 0; ks < DS_K / 16; ++ks) {
                    uint32_t af[4];
                    ldmatrix_x4(sa + swz((uint32_t)hp * 64u + 32u * ks + a_k, 64u), af);
#pragma unroll
                    for (int np = 0; np < 2; ++np) {
                        uint32_t bf[4];
                        ldmatrix_x4(bt + swz((uint32_t)(16 * np + brow) * 64u + 32u * ks + b_k, 64u), bf);
                        mma_16816(acc[2 * np], af, bf[0], bf[1]);
                        mma_16816(acc[2 * np + 1], af, bf[2], bf[3]);
                    }
                }
            }
        }
        if (kc == kchunks - 1) {
            // accumulator rows g, g + 8 = the warp's pixels, columns 2t, 2t + 1 = input channels of an n8 tile
            const int seg = (int)(rw % segs), i = (int)(r % Hi), b = (int)(r / Hi);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = seg * DS_PX + 2 * (16 * grp + g + 8 * h) + px;
                if (j >= Wi) continue;
                __nv_bfloat16 *o = dx + (((long long)b * Hi + i) * Wi + j) * Cin + n0 + 2 * t4;
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
                    *reinterpret_cast<uint32_t *>(o + 8 * nt) = bf16x2_bits(acc[nt][2 * h], acc[nt][2 * h + 1]);
            }
        }
        __syncthreads();
        st ^= 1;
        rw = nrw;
        kc = nkc;
    }
    cp_async_wait<0>();
}

// wt[ky * KS + kx][n][c] = w(c)[o(c)][n][ky][kx] in bf16: c = a column of [df | dm] in the RAW column order (blocks of 2*half)
__global__ void pack_dgrad_s2_kernel(const float *__restrict__ wf, const float *__restrict__ wm, int Cout, int Cin, int KS, int half,
                                     __nv_bfloat16 *__restrict__ out)
{
    const long long total = (long long)KS * KS * Cin * 2 * Cout;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % (2 * Cout));
        const long long r = i / (2 * Cout);
        const int n = (int)(r % Cin), tap = (int)(r / Cin);
        const int rr = c % (2 * half), o = (c / (2 * half)) * half + rr % half;
        out[i] = __float2bfloat16_rn((rr >= half ? wm : wf)[((long long)o * Cin + n) * KS * KS + tap]);
    }
}

template <int KS>
static int launch_dgrad_s2(const void *dfm, const void *wt, int B, int Ho, int Wo, int Cout, int Cin, void *dx, cudaStream_t st)
{
    const long long rows = (long long)B * (2 * Ho) * ((2 * Wo + DS_PX - 1) / DS_PX);
    const int nb = Cin / DS_N;
    long long grid = (6ll * num_sms() + nb - 1) / nb;                 // 41.5 KB of shared memory: 5 CTAs per SM
    if (grid > rows) grid = rows;
    RB_CHECK_ARG(grid <= 0x7FFFFFFF && nb <= 65535, "conv_dgrad_s2: too large");
    dgrad_s2_kernel<KS><<<dim3((unsigned)grid, nb), DS_THREADS, 0, st>>>((const __nv_bfloat16 *)dfm, (const __nv_bfloat16 *)wt, B, Ho,
                                                                        Wo, 2 * Cout, Cin, (__nv_bfloat16 *)dx);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb

using namespace rb;

extern "C" {

int read_gate_backward(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f, const float *bias_m,
                       const float *bn_scale, const float *bn_mean, const float *bn_inv_std, void *dfm, float *dbias_f,
                       float *dbias_m, float *dgamma, float *dbeta, void *stream)
{
    RB_CHECK_ARG(dy && fm && dfm && bias_f && bias_m && bn_scale && bn_mean && bn_inv_std && dbias_f && dbias_m && dgamma && dbeta,
                 "gate_backward: null pointer");
    // the [f | m] column order (blocks of 2*min(C, 64)) exists only for C <= 64 or C % 64 == 0, as in the forward RAW plan
    RB_CHECK_ARG(C >= 16 && C <= GB_MAX_C && C % 16 == 0 && (C <= 64 || C % 64 == 0) && pixels >= 0,
                 "gate_backward: C must be 16, 32, 48, 64 or a multiple of 64 up to %d (got %d)", GB_MAX_C, C);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(fm) | reinterpret_cast<uintptr_t>(dfm)) & 15) == 0,
                 "gate_backward: tensors must be 16B aligned");
    if (pixels == 0) return READ_OK;
    const int half = C < 64 ? C : 64, ppb = GB_THREADS / (C / 8);
    long long blocks = (pixels + ppb - 1) / ppb;
    if (blocks > 8ll * num_sms()) blocks = 8ll * num_sms();
    auto k = elu ? gate_bwd_kernel<true, false> : gate_bwd_kernel<false, false>;
    k<<<(unsigned)blocks, GB_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, half, bias_f, bias_m, bn_scale, bn_mean,
        bn_inv_std, (__nv_bfloat16 *)dfm, dbias_f, dbias_m, dgamma, dbeta, nullptr, nullptr);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

static long long gate_grid(int64_t pixels, int C)
{
    const int ppb = GB_THREADS / (C / 8);
    long long blocks = (pixels + ppb - 1) / ppb;
    return blocks > 8ll * num_sms() ? 8ll * num_sms() : blocks;
}

int read_bn_backward_reduce(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f, const float *bias_m,
                            const float *bn_mean, const float *bn_inv_std, float *sum_dy, float *sum_dy_xhat, void *stream)
{
    RB_CHECK_ARG(dy && fm && bias_f && bias_m && bn_mean && bn_inv_std && sum_dy && sum_dy_xhat, "bn_backward_reduce: null pointer");
    RB_CHECK_ARG(bn_channels_ok(C), "bn_backward_reduce: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)", GB_MAX_C, C);
    RB_CHECK_ARG(pixels >= 2, "bn_backward_reduce: batch statistics need at least 2 pixels (got %lld)", (long long)pixels);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(fm)) & 15) == 0,
                 "bn_backward_reduce: tensors must be 16B aligned");
    auto k = elu ? bn_bwd_reduce_kernel<true> : bn_bwd_reduce_kernel<false>;
    k<<<(unsigned)gate_grid(pixels, C), GB_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_mean,
        bn_inv_std, sum_dy, sum_dy_xhat);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_gate_backward_batch_stats(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f,
                                   const float *bias_m, const float *bn_scale, const float *bn_mean, const float *bn_inv_std,
                                   const float *sum_dy, const float *sum_dy_xhat, void *dfm, float *dbias_f, float *dbias_m,
                                   void *stream)
{
    RB_CHECK_ARG(dy && fm && dfm && bias_f && bias_m && bn_scale && bn_mean && bn_inv_std && sum_dy && sum_dy_xhat && dbias_f &&
                     dbias_m,
                 "gate_backward_batch_stats: null pointer");
    RB_CHECK_ARG(bn_channels_ok(C), "gate_backward_batch_stats: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)",
                 GB_MAX_C, C);
    RB_CHECK_ARG(pixels >= 2, "gate_backward_batch_stats: batch statistics need at least 2 pixels (got %lld)", (long long)pixels);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(fm) | reinterpret_cast<uintptr_t>(dfm)) & 15) == 0,
                 "gate_backward_batch_stats: tensors must be 16B aligned");
    auto k = elu ? gate_bwd_kernel<true, true> : gate_bwd_kernel<false, true>;
    k<<<(unsigned)gate_grid(pixels, C), GB_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_scale,
        bn_mean, bn_inv_std, (__nv_bfloat16 *)dfm, dbias_f, dbias_m, nullptr, nullptr, sum_dy, sum_dy_xhat);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

// CTAs per item of the per-item gate passes: the call's CTAs are capped as for a single call of all the items' pixels
static long long gate_grid_items(int items, int64_t pixels, int C)
{
    const int ppb = GB_THREADS / (C / 8);
    long long blocks = (pixels + ppb - 1) / ppb, cap = 8ll * num_sms() / items;
    if (cap < 1) cap = 1;
    return blocks > cap ? cap : blocks;
}

int read_bn_backward_reduce_items(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu, const float *bias_f,
                                  const float *bias_m, const float *bn_mean, const float *bn_inv_std, float *sum_dy,
                                  float *sum_dy_xhat, void *stream)
{
    RB_CHECK_ARG(dy && fm && bias_f && bias_m && bn_mean && bn_inv_std && sum_dy && sum_dy_xhat,
                 "bn_backward_reduce_items: null pointer");
    RB_CHECK_ARG(items >= 1 && items <= 65535, "bn_backward_reduce_items: items must lie in 1..65535 (got %d)", items);
    RB_CHECK_ARG(bn_channels_ok(C), "bn_backward_reduce_items: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)",
                 GB_MAX_C, C);
    RB_CHECK_ARG(pixels >= 2, "bn_backward_reduce_items: batch statistics need at least 2 pixels per item (got %lld)",
                 (long long)pixels);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(fm)) & 15) == 0,
                 "bn_backward_reduce_items: tensors must be 16B aligned");
    auto k = elu ? bn_bwd_reduce_items_kernel<true> : bn_bwd_reduce_items_kernel<false>;
    k<<<dim3((unsigned)gate_grid_items(items, pixels, C), (unsigned)items), GB_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_mean,
        bn_inv_std, sum_dy, sum_dy_xhat);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_gate_backward_batch_stats_items(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu,
                                         const float *bias_f, const float *bias_m, const float *bn_scale, const float *bn_mean,
                                         const float *bn_inv_std, const float *sum_dy, const float *sum_dy_xhat, void *dfm,
                                         float *dbias_f, float *dbias_m, void *stream)
{
    RB_CHECK_ARG(dy && fm && dfm && bias_f && bias_m && bn_scale && bn_mean && bn_inv_std && sum_dy && sum_dy_xhat && dbias_f &&
                     dbias_m,
                 "gate_backward_batch_stats_items: null pointer");
    RB_CHECK_ARG(items >= 1 && items <= 65535, "gate_backward_batch_stats_items: items must lie in 1..65535 (got %d)", items);
    RB_CHECK_ARG(bn_channels_ok(C), "gate_backward_batch_stats_items: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)",
                 GB_MAX_C, C);
    RB_CHECK_ARG(pixels >= 2, "gate_backward_batch_stats_items: batch statistics need at least 2 pixels per item (got %lld)",
                 (long long)pixels);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(fm) | reinterpret_cast<uintptr_t>(dfm)) & 15) == 0,
                 "gate_backward_batch_stats_items: tensors must be 16B aligned");
    auto k = elu ? gate_bwd_items_kernel<true> : gate_bwd_items_kernel<false>;
    k<<<dim3((unsigned)gate_grid_items(items, pixels, C), (unsigned)items), GB_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_scale,
        bn_mean, bn_inv_std, (__nv_bfloat16 *)dfm, dbias_f, dbias_m, sum_dy, sum_dy_xhat);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_conv3x3_wgrad(const void *dfm, const void *x, int B, int H, int W, int Cout, int Cin, float *dwf, float *dwm, void *stream)
{
    RB_CHECK_ARG(dfm && x && dwf && dwm, "conv3x3_wgrad: null pointer");
    RB_CHECK_ARG(B >= 1 && H >= 1 && W >= 1, "conv3x3_wgrad: bad shape");
    RB_CHECK_ARG((Cin == 8 || Cin == 16 || (Cin % 32 == 0 && Cin > 0)) &&
                     (Cout == 16 || (Cout % 32 == 0 && Cout > 0 && (Cout <= 64 || Cout % 64 == 0))),
                 "conv3x3_wgrad: Cin must be 8, 16 or a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got %d, %d)", Cin,
                 Cout);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dfm) | reinterpret_cast<uintptr_t>(x)) & 15) == 0,
                 "conv3x3_wgrad: tensors must be 16B aligned");
    const long long chunks = (long long)B * H * ((W + WG_PX - 1) / WG_PX);
    const int mb = (2 * Cout + WG_M - 1) / WG_M, nb = (Cin + WG_N - 1) / WG_N;
    long long s = (2ll * num_sms() + mb * nb - 1) / (mb * nb);
    if (s > chunks) s = chunks;
    RB_CHECK_ARG(s <= 0x7FFFFFFF && nb <= 65535 && mb <= 65535, "conv3x3_wgrad: too large");
    wgrad_kernel<3, 1, 3><<<dim3((unsigned)s, mb, nb), WG_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dfm, (const __nv_bfloat16 *)x, B, H, W, Cout, Cin, Cout < 64 ? Cout : 64, dwf, dwm);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_conv3x3_dgrad_cin8(const void *dfm, const float *wf, const float *wm, int B, int H, int W, int Cout, void *dx, void *stream)
{
    RB_CHECK_ARG(dfm && wf && wm && dx, "conv3x3_dgrad_cin8: null pointer");
    RB_CHECK_ARG(B >= 1 && H >= 1 && W >= 1, "conv3x3_dgrad_cin8: bad shape");
    RB_CHECK_ARG(Cout == 16 || Cout == 32 || Cout == 64, "conv3x3_dgrad_cin8: Cout must be 16, 32 or 64 (got %d)", Cout);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dfm) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0,
                 "conv3x3_dgrad_cin8: tensors must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    if (Cout == 16) return launch_dgrad_cin8<32>(dfm, wf, wm, B, H, W, dx, st);
    if (Cout == 32) return launch_dgrad_cin8<64>(dfm, wf, wm, B, H, W, dx, st);
    return launch_dgrad_cin8<128>(dfm, wf, wm, B, H, W, dx, st);
}

static bool wgrad_channels_ok(int Cout, int Cin)
{
    return (Cin == 8 || Cin == 16 || (Cin % 32 == 0 && Cin > 0)) && (Cout == 16 || (Cout % 32 == 0 && Cout > 0 && (Cout <= 64 || Cout % 64 == 0)));
}

int read_conv_wgrad(const void *dfm, const void *x, int B, int Hin, int Win, int Hout, int Wout, int Cout, int Cin, int k,
                    int stride, float *dwf, float *dwm, void *stream)
{
    RB_CHECK_ARG(dfm && x && dwf && dwm, "conv_wgrad: null pointer");
    RB_CHECK_ARG(B >= 1 && Hout >= 1 && Wout >= 1, "conv_wgrad: bad shape");
    RB_CHECK_ARG((stride == 1 && (k == 1 || k == 3)) || (stride == 2 && (k == 3 || k == 4)),
                 "conv_wgrad: k=%d stride=%d is not one of 1x1 / 3x3 stride 1, 3x3 / 4x4 stride 2", k, stride);
    RB_CHECK_ARG(Hin == stride * Hout && Win == stride * Wout,
                 "conv_wgrad: input %dx%d does not match output %dx%d at stride %d (stride 2 needs an even input)", Hin, Win, Hout,
                 Wout, stride);
    RB_CHECK_ARG(wgrad_channels_ok(Cout, Cin),
                 "conv_wgrad: Cin must be 8, 16 or a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got %d, %d)", Cin, Cout);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dfm) | reinterpret_cast<uintptr_t>(x)) & 15) == 0,
                 "conv_wgrad: tensors must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    if (k == 1) return launch_wgrad<1, 1, 1>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, st);
    if (stride == 1) return launch_wgrad<3, 1, 3>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, st);
    if (k == 3) return launch_wgrad<3, 2, 3>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, st);
    return launch_wgrad<4, 2, 2>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, st);
}

int read_pack_weights_dgrad_s2(const float *wf, const float *wm, int Cout, int Cin, int k, void *out_bf16, void *stream)
{
    RB_CHECK_ARG(wf && wm && out_bf16, "pack_dgrad_s2: null pointer");
    RB_CHECK_ARG(k == 3 || k == 4, "pack_dgrad_s2: k must be 3 or 4 (got %d)", k);
    RB_CHECK_ARG(Cin % 32 == 0 && Cin > 0 && (Cout == 16 || (Cout % 32 == 0 && Cout > 0 && (Cout <= 64 || Cout % 64 == 0))),
                 "pack_dgrad_s2: Cin must be a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got %d, %d)", Cin, Cout);
    const long long total = (long long)k * k * Cin * 2 * Cout;
    long long blocks = (total + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    pack_dgrad_s2_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(wf, wm, Cout, Cin, k, Cout < 64 ? Cout : 64,
                                                                             (__nv_bfloat16 *)out_bf16);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_conv_dgrad_s2(const void *dfm, const void *wt, int B, int Hout, int Wout, int Cout, int Cin, int k, void *dx, void *stream)
{
    RB_CHECK_ARG(dfm && wt && dx, "conv_dgrad_s2: null pointer");
    RB_CHECK_ARG(B >= 1 && Hout >= 1 && Wout >= 1, "conv_dgrad_s2: bad shape");
    RB_CHECK_ARG(k == 3 || k == 4, "conv_dgrad_s2: k must be 3 or 4 (got %d)", k);
    RB_CHECK_ARG(Cin % 32 == 0 && Cin > 0 && (Cout == 16 || (Cout % 32 == 0 && Cout > 0 && (Cout <= 64 || Cout % 64 == 0))),
                 "conv_dgrad_s2: Cin must be a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got %d, %d)", Cin, Cout);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dfm) | reinterpret_cast<uintptr_t>(wt) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0,
                 "conv_dgrad_s2: tensors must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    if (k == 3) return launch_dgrad_s2<3>(dfm, wt, B, Hout, Wout, Cout, Cin, dx, st);
    return launch_dgrad_s2<4>(dfm, wt, B, Hout, Wout, Cout, Cin, dx, st);
}

// ------------------------------------------------------------------ deterministic entry points
// CTAs of the deterministic gate passes: at most 2 per SM (the last CTA reads every CTA's row), per item for the per-item forms
static long long gate_det_grid(int items, int64_t pixels, int C)
{
    const int ppb = GB_THREADS / (C / 8);
    long long blocks = (pixels + ppb - 1) / ppb, cap = 2ll * num_sms() / items;
    if (cap < 1) cap = 1;
    return blocks > cap ? cap : blocks;
}

static bool gate_det_ok(int C) { return C >= 16 && C <= GB_MAX_C && C % 16 == 0 && (C <= 64 || C % 64 == 0); }

int64_t read_gate_det_workspace_bytes(int items, int C)
{
    if (!gate_det_ok(C) || items < 1 || items > 65535) return -1;
    const long long ctas = items > 2ll * num_sms() ? items : 2ll * num_sms();
    return 256 + ctas * 4 * C * (int64_t)sizeof(float);
}

#define GATE_DET_CHECKS(name, items, pixels, minpx, ...)                                                                        \
    RB_CHECK_ARG(__VA_ARGS__, name ": null pointer");                                                                          \
    RB_CHECK_ARG(items >= 1 && items <= 65535, name ": items must lie in 1..65535 (got %d)", items);                            \
    RB_CHECK_ARG(pixels >= minpx, name ": needs at least %d pixels (got %lld)", minpx, (long long)pixels);                      \
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(fm) | reinterpret_cast<uintptr_t>(workspace)) & \
                  15) == 0,                                                                                                    \
                 name ": tensors and workspace must be 16B aligned")

int read_gate_backward_det(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f, const float *bias_m,
                           const float *bn_scale, const float *bn_mean, const float *bn_inv_std, void *dfm, float *dbias_f,
                           float *dbias_m, float *dgamma, float *dbeta, void *workspace, void *stream)
{
    GATE_DET_CHECKS("gate_backward_det", 1, pixels, 0, dy && fm && dfm && bias_f && bias_m && bn_scale && bn_mean && bn_inv_std &&
                                                           dbias_f && dbias_m && dgamma && dbeta && workspace);
    RB_CHECK_ARG(gate_det_ok(C), "gate_backward_det: C must be 16, 32, 48, 64 or a multiple of 64 up to %d (got %d)", GB_MAX_C, C);
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(dfm) & 15) == 0, "gate_backward_det: tensors must be 16B aligned");
    if (pixels == 0) return READ_OK;
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned *counter = (unsigned *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
    auto k = elu ? gate_bwd_det_kernel<true, false> : gate_bwd_det_kernel<false, false>;
    k<<<(unsigned)gate_det_grid(1, pixels, C), GB_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_scale, bn_mean,
        bn_inv_std, (__nv_bfloat16 *)dfm, dbias_f, dbias_m, dgamma, dbeta, nullptr, nullptr, (float *)((char *)workspace + 256),
        counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_bn_backward_reduce_det(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f,
                                const float *bias_m, const float *bn_mean, const float *bn_inv_std, float *sum_dy, float *sum_dy_xhat,
                                void *workspace, void *stream)
{
    GATE_DET_CHECKS("bn_backward_reduce_det", 1, pixels, 2, dy && fm && bias_f && bias_m && bn_mean && bn_inv_std && sum_dy &&
                                                                sum_dy_xhat && workspace);
    RB_CHECK_ARG(bn_channels_ok(C), "bn_backward_reduce_det: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)", GB_MAX_C, C);
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned *counter = (unsigned *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
    auto k = elu ? bn_bwd_reduce_det_kernel<true> : bn_bwd_reduce_det_kernel<false>;
    k<<<(unsigned)gate_det_grid(1, pixels, C), GB_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_mean,
        bn_inv_std, sum_dy, sum_dy_xhat, (float *)((char *)workspace + 256), counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_gate_backward_batch_stats_det(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f,
                                       const float *bias_m, const float *bn_scale, const float *bn_mean, const float *bn_inv_std,
                                       const float *sum_dy, const float *sum_dy_xhat, void *dfm, float *dbias_f, float *dbias_m,
                                       void *workspace, void *stream)
{
    GATE_DET_CHECKS("gate_backward_batch_stats_det", 1, pixels, 2, dy && fm && dfm && bias_f && bias_m && bn_scale && bn_mean &&
                                                                       bn_inv_std && sum_dy && sum_dy_xhat && dbias_f && dbias_m &&
                                                                       workspace);
    RB_CHECK_ARG(bn_channels_ok(C), "gate_backward_batch_stats_det: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)",
                 GB_MAX_C, C);
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(dfm) & 15) == 0, "gate_backward_batch_stats_det: tensors must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned *counter = (unsigned *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
    auto k = elu ? gate_bwd_det_kernel<true, true> : gate_bwd_det_kernel<false, true>;
    k<<<(unsigned)gate_det_grid(1, pixels, C), GB_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_scale,
        bn_mean, bn_inv_std, (__nv_bfloat16 *)dfm, dbias_f, dbias_m, nullptr, nullptr, sum_dy, sum_dy_xhat,
        (float *)((char *)workspace + 256), counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_bn_backward_reduce_items_det(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu,
                                      const float *bias_f, const float *bias_m, const float *bn_mean, const float *bn_inv_std,
                                      float *sum_dy, float *sum_dy_xhat, void *workspace, void *stream)
{
    GATE_DET_CHECKS("bn_backward_reduce_items_det", items, pixels, 2, dy && fm && bias_f && bias_m && bn_mean && bn_inv_std &&
                                                                          sum_dy && sum_dy_xhat && workspace);
    RB_CHECK_ARG(bn_channels_ok(C), "bn_backward_reduce_items_det: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)",
                 GB_MAX_C, C);
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned *counter = (unsigned *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
    auto k = elu ? bn_bwd_reduce_items_det_kernel<true> : bn_bwd_reduce_items_det_kernel<false>;
    k<<<dim3((unsigned)gate_det_grid(items, pixels, C), (unsigned)items), GB_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_mean,
        bn_inv_std, sum_dy, sum_dy_xhat, (float *)((char *)workspace + 256), counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_gate_backward_batch_stats_items_det(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu,
                                             const float *bias_f, const float *bias_m, const float *bn_scale, const float *bn_mean,
                                             const float *bn_inv_std, const float *sum_dy, const float *sum_dy_xhat, void *dfm,
                                             float *dbias_f, float *dbias_m, void *workspace, void *stream)
{
    GATE_DET_CHECKS("gate_backward_batch_stats_items_det", items, pixels, 2, dy && fm && dfm && bias_f && bias_m && bn_scale &&
                                                                                 bn_mean && bn_inv_std && sum_dy && sum_dy_xhat &&
                                                                                 dbias_f && dbias_m && workspace);
    RB_CHECK_ARG(bn_channels_ok(C), "gate_backward_batch_stats_items_det: C must be 16, 32, 64 or a multiple of 64 up to %d (got %d)",
                 GB_MAX_C, C);
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(dfm) & 15) == 0, "gate_backward_batch_stats_items_det: tensors must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned *counter = (unsigned *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
    auto k = elu ? gate_bwd_items_det_kernel<true> : gate_bwd_items_det_kernel<false>;
    k<<<dim3((unsigned)gate_det_grid(items, pixels, C), (unsigned)items), GB_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)dy, (const __nv_bfloat16 *)fm, (long long)pixels, C, C < 64 ? C : 64, bias_f, bias_m, bn_scale,
        bn_mean, bn_inv_std, (__nv_bfloat16 *)dfm, dbias_f, dbias_m, sum_dy, sum_dy_xhat, (float *)((char *)workspace + 256),
        counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

#undef GATE_DET_CHECKS

static bool wgrad_geom_ok(int Hin, int Win, int Hout, int Wout, int k, int stride)
{
    return ((stride == 1 && (k == 1 || k == 3)) || (stride == 2 && (k == 3 || k == 4))) && Hin == stride * Hout &&
           Win == stride * Wout;
}

int64_t read_conv_wgrad_det_workspace_bytes(int B, int Hout, int Wout, int Cout, int Cin, int k, int stride)
{
    if (B < 1 || Hout < 1 || Wout < 1 || !wgrad_channels_ok(Cout, Cin) || !wgrad_geom_ok(stride * Hout, stride * Wout, Hout, Wout, k, stride))
        return -1;
    long long s;
    int mb, nz;
    if (k == 4) wgrad_grid<4, 2>(B, Hout, Wout, Cout, Cin, s, mb, nz);
    else if (k == 3) wgrad_grid<3, 3>(B, Hout, Wout, Cout, Cin, s, mb, nz);
    else wgrad_grid<1, 1>(B, Hout, Wout, Cout, Cin, s, mb, nz);
    return s * 2 * (int64_t)Cout * Cin * k * k * (int64_t)sizeof(float);
}

int read_conv_wgrad_det(const void *dfm, const void *x, int B, int Hin, int Win, int Hout, int Wout, int Cout, int Cin, int k,
                        int stride, float *dwf, float *dwm, void *workspace, void *stream)
{
    RB_CHECK_ARG(dfm && x && dwf && dwm && workspace, "conv_wgrad_det: null pointer");
    RB_CHECK_ARG(B >= 1 && Hout >= 1 && Wout >= 1, "conv_wgrad_det: bad shape");
    RB_CHECK_ARG(wgrad_geom_ok(Hin, Win, Hout, Wout, k, stride),
                 "conv_wgrad_det: k=%d stride=%d input %dx%d output %dx%d is not 1x1 / 3x3 stride 1 or 3x3 / 4x4 stride 2 "
                 "(input = stride x output)", k, stride, Hin, Win, Hout, Wout);
    RB_CHECK_ARG(wgrad_channels_ok(Cout, Cin),
                 "conv_wgrad_det: Cin must be 8, 16 or a multiple of 32 and Cout 16, 32, 64 or a multiple of 64 (got %d, %d)", Cin, Cout);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(dfm) | reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
                 "conv_wgrad_det: tensors and workspace must be 16B aligned");
    const cudaStream_t st = (cudaStream_t)stream;
    if (k == 1) return launch_wgrad_det<1, 1, 1>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, workspace, st);
    if (stride == 1) return launch_wgrad_det<3, 1, 3>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, workspace, st);
    if (k == 3) return launch_wgrad_det<3, 2, 3>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, workspace, st);
    return launch_wgrad_det<4, 2, 2>(dfm, x, B, Hout, Wout, Cout, Cin, dwf, dwm, workspace, st);
}

}  // extern "C"
