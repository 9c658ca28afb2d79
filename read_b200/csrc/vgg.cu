// The glue of the VGG19 perceptual loss (read_b200/vgg_loss.py, the reference's READ/criterions/vgg_loss.py): everything but the
// convolutions, which are RAW 3x3 plans of the TMA wgmma kernel (conv_tc.cu) and, for the 3-channel image, dgrad_cin8 (conv_bwd.cu).
// A call runs the output images and the target images as one batch of 2n: images 0 .. n-1 are the output, n .. 2n-1 the target.
//   vgg_normalize   NCHW f32 -> (x - mean) / std -> NHWC bf16 with 8 channels (3 real, 5 zero), both halves in one launch
//   vgg_post        per conv: y = ReLU(raw + bias) over the RAW accumulators of both halves; on a loss layer the sum of
//                   |y_out - y_tgt| (fixed combine order: a CTA's threads, then the CTAs in CTA order, added to a double);
//                   the backward's per-element code of the output half (0 = ReLU closed, else 2 + sign(y_out - y_tgt)); the next
//                   conv's input: y itself, or its 2x2 average (AvgPool2d(2, 2), odd rows / columns dropped) written directly
//   vgg_dgrad_in    backward, per conv: dY = [code != 0] * (U + (code - 2) * g * coef), U the gradient of the ReLU output from
//                   the next conv's input gradient (read through the pool's backward: a quarter of the pooled gradient, 0 on the
//                   dropped rows / columns), coef = 1 / numel of the layer's L1 term (0 off the loss layers)
//   vgg_image_grad  NHWC bf16 8-channel input gradient -> NCHW f32 3 channels, divided by std
// partialconv=True (the mask-aware loss) runs VGG's first conv as a partial convolution over the validity mask M of the target
// (M = [sum of the target's channels > 1e-9]), the same M for both halves.  Four variants, each used at conv1_1 only:
//   vgg_normalize_masked   vgg_normalize, both halves' channels times M, and M as one byte per pixel [n, H, W]
//   vgg_post_partial       vgg_post (no pool) with y = ReLU((raw * ratio + bias) * upd): upd = [the 3x3 window of M holds a valid
//                          pixel], ratio = upd * 9 / (valid pixels in it), both recomputed from the byte mask
//   vgg_dgrad_in_partial   vgg_dgrad_in (no pool) times ratio
//   vgg_image_grad_masked  vgg_image_grad times M
#include "common.cuh"
#include "conv_common.cuh"

namespace rb {

constexpr int VG_THREADS = 256;
constexpr int VG_MAX_CTAS = 1024;        // the grid depends on the shape only, so the loss's combine order does too

__device__ __forceinline__ uint4 ld8(const __nv_bfloat16 *p) { return *reinterpret_cast<const uint4 *>(p); }

__device__ __forceinline__ void unpack8(uint4 v, float (&f)[8])
{
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 t = bf16x2_val(w[q]);
        f[2 * q] = t.x;
        f[2 * q + 1] = t.y;
    }
}

__device__ __forceinline__ uint4 pack8(const float (&f)[8])
{
    return make_uint4(bf16x2_bits(f[0], f[1]), bf16x2_bits(f[2], f[3]), bf16x2_bits(f[4], f[5]), bf16x2_bits(f[6], f[7]));
}

static unsigned vg_blocks(long long units)
{
    const long long b = (units + VG_THREADS - 1) / VG_THREADS;
    return (unsigned)(b < 1 ? 1 : b > VG_MAX_CTAS ? VG_MAX_CTAS : b);
}

// Valid pixels in the 3x3 window at (y, x) of one H x W byte mask, zero padding outside: the partial conv's 0 .. 9 count
__device__ __forceinline__ int vg_window(const uint8_t *__restrict__ m, int H, int W, int y, int x)
{
    int c = 0;
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
        const int yy = y + dy;
        if (yy < 0 || yy >= H) continue;
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) {
            const int xx = x + dx;
            if (xx >= 0 && xx < W) c += m[(long long)yy * W + xx];
        }
    }
    return c;
}

// The partial conv's ratio 9 / (c + 1e-8) * clamp(c, 0, 1) as torch evaluates it in fp32: 1e-8 is below half an ulp of c >= 1, and
// 9 / t is reciprocal(t) * 9, two roundings (it differs from a correctly rounded 9 / c at c = 5 and 7)
__device__ __forceinline__ float vg_ratio(int c) { return c ? __fmul_rn(__frcp_rn((float)c), 9.f) : 0.f; }

// ------------------------------------------------------------------ 1. normalise
__global__ void __launch_bounds__(VG_THREADS)
vgg_normalize_kernel(const float *__restrict__ in, const float *__restrict__ tgt, int n, int H, int W, const float *__restrict__ mean,
                     const float *__restrict__ stdv, __nv_bfloat16 *__restrict__ out)
{
    const long long HW = (long long)H * W, total = 2ll * n * HW;
    const float m0 = mean[0], m1 = mean[1], m2 = mean[2], s0 = stdv[0], s1 = stdv[1], s2 = stdv[2];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i - b * HW;
        const float *src = b < n ? in + b * 3 * HW + p : tgt + (b - n) * 3 * HW + p;
        // torch's (x - mean) / std: two separately rounded fp32 operations
        const float v0 = __fdiv_rn(__fsub_rn(src[0], m0), s0);
        const float v1 = __fdiv_rn(__fsub_rn(src[HW], m1), s1);
        const float v2 = __fdiv_rn(__fsub_rn(src[2 * HW], m2), s2);
        *reinterpret_cast<uint4 *>(out + i * 8) = make_uint4(bf16x2_bits(v0, v1), bf16x2_bits(v2, 0.f), 0u, 0u);
    }
}

// One thread per pixel of image b: reads the pixel of output b and of target b, writes both halves and the mask byte.
__global__ void __launch_bounds__(VG_THREADS)
vgg_normalize_masked_kernel(const float *__restrict__ in, const float *__restrict__ tgt, int n, int H, int W,
                            const float *__restrict__ mean, const float *__restrict__ stdv, __nv_bfloat16 *__restrict__ out,
                            uint8_t *__restrict__ mask)
{
    const long long HW = (long long)H * W, total = (long long)n * HW;
    const float m0 = mean[0], m1 = mean[1], m2 = mean[2], s0 = stdv[0], s1 = stdv[1], s2 = stdv[2];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i - b * HW;
        const float *x = in + b * 3 * HW + p, *t = tgt + b * 3 * HW + p;
        const float t0 = t[0], t1 = t[HW], t2 = t[2 * HW];
        // target.sum(1) > 1e-9 in fp32
        const float m = __fadd_rn(__fadd_rn(t0, t1), t2) > 1e-9f ? 1.f : 0.f;
        // ((x - mean) / std) * M, each operation rounded as torch rounds it
        const float x0 = __fmul_rn(__fdiv_rn(__fsub_rn(x[0], m0), s0), m), x1 = __fmul_rn(__fdiv_rn(__fsub_rn(x[HW], m1), s1), m),
                    x2 = __fmul_rn(__fdiv_rn(__fsub_rn(x[2 * HW], m2), s2), m);
        const float y0 = __fmul_rn(__fdiv_rn(__fsub_rn(t0, m0), s0), m), y1 = __fmul_rn(__fdiv_rn(__fsub_rn(t1, m1), s1), m),
                    y2 = __fmul_rn(__fdiv_rn(__fsub_rn(t2, m2), s2), m);
        *reinterpret_cast<uint4 *>(out + i * 8) = make_uint4(bf16x2_bits(x0, x1), bf16x2_bits(x2, 0.f), 0u, 0u);
        *reinterpret_cast<uint4 *>(out + (total + i) * 8) = make_uint4(bf16x2_bits(y0, y1), bf16x2_bits(y2, 0.f), 0u, 0u);
        mask[i] = (uint8_t)(m != 0.f);
    }
}

// ------------------------------------------------------------------ 2. bias, ReLU, L1 term, backward code, pool
// A work unit is 8 channels (16 bytes) of one P x P pixel block (P = 2 before a pool, else 1) of output image b and of target
// image b + n.  Threads sum |y_out - y_tgt| in fp32; a CTA adds its threads' sums in double in a fixed tree, the last CTA to
// finish (counter + fence) adds the CTAs' in CTA order and adds the result, times scale (1 / numel of the term), to *term.
// PARTIAL (P = 1 only): the partial conv of conv1_1 over the byte mask [n, H, W] before the ReLU, (raw * ratio + bias) * upd.
template <int P, bool PARTIAL>
__device__ __forceinline__ void vgg_post_body(const __nv_bfloat16 *raw, const uint8_t *__restrict__ mask, int n, int H, int W, int C,
                                              const float *__restrict__ bias, __nv_bfloat16 *out, int8_t *__restrict__ code,
                                              double *__restrict__ term, double scale, double *__restrict__ part,
                                              unsigned int *__restrict__ counter)
{
    static_assert(!PARTIAL || P == 1, "the partial conv is VGG's first, which no pool follows");
    __shared__ double red[VG_THREADS];
    __shared__ bool last;
    const int G = C / 8;
    const int Hb = (H + P - 1) / P, Wb = (W + P - 1) / P;
    const int Ho = H / P, Wo = W / P;                               // the next conv's input (floor, as AvgPool2d)
    const long long img = (long long)H * W * C, units = (long long)n * Hb * Wb * G;
    float acc = 0.f;
    for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(u % G);
        long long r = u / G;
        const int bx = (int)(r % Wb);
        r /= Wb;
        const int by = (int)(r % Hb);
        const int b = (int)(r / Hb);
        float bs[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) bs[j] = bias[8 * cg + j];
        float pin[8], ptg[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) pin[j] = ptg[j] = 0.f;
#pragma unroll
        for (int dy = 0; dy < P; ++dy)
#pragma unroll
            for (int dx = 0; dx < P; ++dx) {
                const int y = by * P + dy, x = bx * P + dx;
                if (y >= H || x >= W) continue;
                const long long o = (long long)b * img + ((long long)y * W + x) * C + 8 * cg;
                float fi[8], ft[8];
                unpack8(ld8(raw + o), fi);
                unpack8(ld8(raw + o + (long long)n * img), ft);
                float ratio = 1.f;
                bool upd = true;
                if (PARTIAL) {
                    const int c = vg_window(mask + (long long)b * H * W, H, W, y, x);
                    upd = c != 0;
                    ratio = vg_ratio(c);
                }
                uint32_t cw[2] = {0u, 0u};
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (PARTIAL) {
                        fi[j] = upd ? fmaxf(fi[j] * ratio + bs[j], 0.f) : 0.f;
                        ft[j] = upd ? fmaxf(ft[j] * ratio + bs[j], 0.f) : 0.f;
                    } else {
                        fi[j] = fmaxf(fi[j] + bs[j], 0.f);
                        ft[j] = fmaxf(ft[j] + bs[j], 0.f);
                    }
                    const float d = fi[j] - ft[j];
                    if (term) acc += fabsf(d);
                    const int s = term ? (d > 0.f) - (d < 0.f) : 0;
                    const uint32_t c = fi[j] > 0.f ? (uint32_t)(2 + s) : 0u;
                    cw[j / 4] |= c << (8 * (j % 4));
                    pin[j] += fi[j];
                    ptg[j] += ft[j];
                }
                if (code) *reinterpret_cast<uint2 *>(code + o) = make_uint2(cw[0], cw[1]);
                if (P == 1 && out) {
                    *reinterpret_cast<uint4 *>(out + o) = pack8(fi);
                    *reinterpret_cast<uint4 *>(out + o + (long long)n * img) = pack8(ft);
                }
            }
        if (P == 2 && out && by < Ho && bx < Wo) {
            const long long oimg = (long long)Ho * Wo * C, o = (long long)b * oimg + ((long long)by * Wo + bx) * C + 8 * cg;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                pin[j] *= 0.25f;
                ptg[j] *= 0.25f;
            }
            *reinterpret_cast<uint4 *>(out + o) = pack8(pin);
            *reinterpret_cast<uint4 *>(out + o + (long long)n * oimg) = pack8(ptg);
        }
    }
    if (!term) return;
    red[threadIdx.x] = (double)acc;
    __syncthreads();
    for (int s = VG_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = red[0];
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (unsigned i = 0; i < gridDim.x; ++i) s += __ldcg(part + i);
        *term += s * scale;
        *counter = 0u;
    }
}

template <int P>
__global__ void __launch_bounds__(VG_THREADS)
vgg_post_kernel(const __nv_bfloat16 *raw, int n, int H, int W, int C, const float *__restrict__ bias, __nv_bfloat16 *out,
                int8_t *__restrict__ code, double *__restrict__ term, double scale, double *__restrict__ part,
                unsigned int *__restrict__ counter)
{
    vgg_post_body<P, false>(raw, nullptr, n, H, W, C, bias, out, code, term, scale, part, counter);
}

__global__ void __launch_bounds__(VG_THREADS)
vgg_post_partial_kernel(const __nv_bfloat16 *raw, const uint8_t *__restrict__ mask, int n, int H, int W, int C,
                        const float *__restrict__ bias, __nv_bfloat16 *out, int8_t *__restrict__ code, double *__restrict__ term,
                        double scale, double *__restrict__ part, unsigned int *__restrict__ counter)
{
    vgg_post_body<1, true>(raw, mask, n, H, W, C, bias, out, code, term, scale, part, counter);
}

// ------------------------------------------------------------------ 3. gradient into a conv's RAW output
// PARTIAL (no pool): times the partial conv's ratio at the pixel, recomputed from the byte mask [n, H, W].
template <bool POOL, bool PARTIAL>
__device__ __forceinline__ void vgg_dgrad_in_body(const __nv_bfloat16 *__restrict__ up, const int8_t *__restrict__ code,
                                                  const uint8_t *__restrict__ mask, int n, int H, int W, int C,
                                                  const float *__restrict__ g, float coef, __nv_bfloat16 *__restrict__ dy)
{
    static_assert(!(PARTIAL && POOL), "the partial conv is VGG's first, which no pool follows");
    const int G = C / 8, Hu = POOL ? H / 2 : H, Wu = POOL ? W / 2 : W;
    const long long units = (long long)n * H * W * G;
    const float l1 = g[0] * coef;
    for (long long u = blockIdx.x * (long long)blockDim.x + threadIdx.x; u < units; u += (long long)gridDim.x * blockDim.x) {
        const int cg = (int)(u % G);
        long long r = u / G;
        const int x = (int)(r % W);
        r /= W;
        const int y = (int)(r % H);
        const int b = (int)(r / H);
        float uf[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) uf[j] = 0.f;
        const int yu = POOL ? y >> 1 : y, xu = POOL ? x >> 1 : x;
        if (up && yu < Hu && xu < Wu) {
            unpack8(ld8(up + (((long long)b * Hu + yu) * Wu + xu) * C + 8 * cg), uf);
            if (POOL)
#pragma unroll
                for (int j = 0; j < 8; ++j) uf[j] *= 0.25f;
        }
        const uint2 cv = *reinterpret_cast<const uint2 *>(code + u * 8);
        float d[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = (int)(((j < 4 ? cv.x : cv.y) >> (8 * (j % 4))) & 0xFFu);
            d[j] = c ? uf[j] + (float)(c - 2) * l1 : 0.f;
        }
        if (PARTIAL) {
            const float ratio = vg_ratio(vg_window(mask + (long long)b * H * W, H, W, y, x));
#pragma unroll
            for (int j = 0; j < 8; ++j) d[j] *= ratio;
        }
        *reinterpret_cast<uint4 *>(dy + u * 8) = pack8(d);
    }
}

template <bool POOL>
__global__ void __launch_bounds__(VG_THREADS)
vgg_dgrad_in_kernel(const __nv_bfloat16 *__restrict__ up, const int8_t *__restrict__ code, int n, int H, int W, int C,
                    const float *__restrict__ g, float coef, __nv_bfloat16 *__restrict__ dy)
{
    vgg_dgrad_in_body<POOL, false>(up, code, nullptr, n, H, W, C, g, coef, dy);
}

__global__ void __launch_bounds__(VG_THREADS)
vgg_dgrad_in_partial_kernel(const __nv_bfloat16 *__restrict__ up, const int8_t *__restrict__ code, const uint8_t *__restrict__ mask,
                            int n, int H, int W, int C, const float *__restrict__ g, float coef, __nv_bfloat16 *__restrict__ dy)
{
    vgg_dgrad_in_body<false, true>(up, code, mask, n, H, W, C, g, coef, dy);
}

// ------------------------------------------------------------------ 4. image gradient
__global__ void __launch_bounds__(VG_THREADS)
vgg_image_grad_kernel(const __nv_bfloat16 *__restrict__ dx, int n, int H, int W, const float *__restrict__ stdv, float *__restrict__ out)
{
    const long long HW = (long long)H * W, total = (long long)n * HW;
    const float s0 = stdv[0], s1 = stdv[1], s2 = stdv[2];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i - b * HW;
        float f[8];
        unpack8(ld8(dx + i * 8), f);
        float *o = out + b * 3 * HW + p;
        o[0] = __fdiv_rn(f[0], s0);
        o[HW] = __fdiv_rn(f[1], s1);
        o[2 * HW] = __fdiv_rn(f[2], s2);
    }
}

__global__ void __launch_bounds__(VG_THREADS)
vgg_image_grad_masked_kernel(const __nv_bfloat16 *__restrict__ dx, const uint8_t *__restrict__ mask, int n, int H, int W,
                             const float *__restrict__ stdv, float *__restrict__ out)
{
    const long long HW = (long long)H * W, total = (long long)n * HW;
    const float s0 = stdv[0], s1 = stdv[1], s2 = stdv[2];
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / HW, p = i - b * HW;
        float f[8];
        unpack8(ld8(dx + i * 8), f);
        const float m = mask[i] ? 1.f : 0.f;
        float *o = out + b * 3 * HW + p;
        // (dx * M) / std, the backward of ((x - mean) / std) * M
        o[0] = __fdiv_rn(__fmul_rn(f[0], m), s0);
        o[HW] = __fdiv_rn(__fmul_rn(f[1], m), s1);
        o[2 * HW] = __fdiv_rn(__fmul_rn(f[2], m), s2);
    }
}

}  // namespace rb

using namespace rb;

static bool vg_aligned(const void *p, unsigned a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; }

extern "C" {

int64_t read_vgg_workspace_bytes(void) { return 256 + (int64_t)VG_MAX_CTAS * (int64_t)sizeof(double); }

int read_vgg_normalize(const float *input, const float *target, int n, int H, int W, const float *mean, const float *std_, void *out,
                       void *stream)
{
    RB_CHECK_ARG(input && target && mean && std_ && out, "vgg_normalize: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0, "vgg_normalize: empty batch (n = %d, %d x %d)", n, H, W);
    RB_CHECK_ARG(vg_aligned(out, 16), "vgg_normalize: output must be 16B aligned");
    vgg_normalize_kernel<<<vg_blocks(2ll * n * H * W), VG_THREADS, 0, (cudaStream_t)stream>>>(input, target, n, H, W, mean, std_,
                                                                                           (__nv_bfloat16 *)out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_post(const void *raw, int n, int H, int W, int C, const float *bias, int pool, void *out, void *code, double *term,
                  double scale, void *workspace, void *stream)
{
    RB_CHECK_ARG(raw && bias, "vgg_post: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "vgg_post: bad shape (n = %d, %d x %d x %d)", n, H, W, C);
    RB_CHECK_ARG(pool == 0 || pool == 1, "vgg_post: pool must be 0 or 1");
    RB_CHECK_ARG(!term || workspace, "vgg_post: a loss layer needs the workspace");
    RB_CHECK_ARG(vg_aligned(raw, 16) && vg_aligned(out, 16) && vg_aligned(code, 8) && vg_aligned(workspace, 16),
                 "vgg_post: tensors must be 16B aligned (code 8B)");
    RB_CHECK_ARG(!(pool && out == raw), "vgg_post: the pooled output cannot overwrite the RAW input");
    const cudaStream_t st = (cudaStream_t)stream;
    const int P = pool ? 2 : 1;
    const long long units = (long long)n * ((H + P - 1) / P) * ((W + P - 1) / P) * (C / 8);
    unsigned int *counter = (unsigned int *)workspace;
    double *part = workspace ? (double *)((char *)workspace + 256) : nullptr;
    if (term) RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), st));
    if (pool)
        vgg_post_kernel<2><<<vg_blocks(units), VG_THREADS, 0, st>>>((const __nv_bfloat16 *)raw, n, H, W, C, bias, (__nv_bfloat16 *)out,
                                                                   (int8_t *)code, term, scale, part, counter);
    else
        vgg_post_kernel<1><<<vg_blocks(units), VG_THREADS, 0, st>>>((const __nv_bfloat16 *)raw, n, H, W, C, bias, (__nv_bfloat16 *)out,
                                                                   (int8_t *)code, term, scale, part, counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_dgrad_in(const void *up, int pool, const void *code, int n, int H, int W, int C, const float *g, float coef, void *dy,
                      void *stream)
{
    RB_CHECK_ARG(code && g && dy, "vgg_dgrad_in: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "vgg_dgrad_in: bad shape (n = %d, %d x %d x %d)", n, H, W, C);
    RB_CHECK_ARG(pool == 0 || pool == 1, "vgg_dgrad_in: pool must be 0 or 1");
    RB_CHECK_ARG(vg_aligned(up, 16) && vg_aligned(code, 8) && vg_aligned(dy, 16), "vgg_dgrad_in: tensors must be 16B aligned (code 8B)");
    const unsigned blocks = vg_blocks((long long)n * H * W * (C / 8));
    const cudaStream_t st = (cudaStream_t)stream;
    if (pool)
        vgg_dgrad_in_kernel<true><<<blocks, VG_THREADS, 0, st>>>((const __nv_bfloat16 *)up, (const int8_t *)code, n, H, W, C, g, coef,
                                                               (__nv_bfloat16 *)dy);
    else
        vgg_dgrad_in_kernel<false><<<blocks, VG_THREADS, 0, st>>>((const __nv_bfloat16 *)up, (const int8_t *)code, n, H, W, C, g, coef,
                                                                (__nv_bfloat16 *)dy);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_image_grad(const void *dx, int n, int H, int W, const float *std_, float *out, void *stream)
{
    RB_CHECK_ARG(dx && std_ && out, "vgg_image_grad: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0, "vgg_image_grad: empty batch (n = %d, %d x %d)", n, H, W);
    RB_CHECK_ARG(vg_aligned(dx, 16), "vgg_image_grad: input must be 16B aligned");
    vgg_image_grad_kernel<<<vg_blocks((long long)n * H * W), VG_THREADS, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)dx, n, H, W,
                                                                                                  std_, out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_normalize_masked(const float *input, const float *target, int n, int H, int W, const float *mean, const float *std_,
                              void *out, void *mask, void *stream)
{
    RB_CHECK_ARG(input && target && mean && std_ && out && mask, "vgg_normalize_masked: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0, "vgg_normalize_masked: empty batch (n = %d, %d x %d)", n, H, W);
    RB_CHECK_ARG(vg_aligned(out, 16), "vgg_normalize_masked: output must be 16B aligned");
    vgg_normalize_masked_kernel<<<vg_blocks((long long)n * H * W), VG_THREADS, 0, (cudaStream_t)stream>>>(
        input, target, n, H, W, mean, std_, (__nv_bfloat16 *)out, (uint8_t *)mask);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_post_partial(const void *raw, const void *mask, int n, int H, int W, int C, const float *bias, void *out, void *code,
                          double *term, double scale, void *workspace, void *stream)
{
    RB_CHECK_ARG(raw && mask && bias, "vgg_post_partial: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "vgg_post_partial: bad shape (n = %d, %d x %d x %d)", n, H, W, C);
    RB_CHECK_ARG(!term || workspace, "vgg_post_partial: a loss layer needs the workspace");
    RB_CHECK_ARG(vg_aligned(raw, 16) && vg_aligned(out, 16) && vg_aligned(code, 8) && vg_aligned(workspace, 16),
                 "vgg_post_partial: tensors must be 16B aligned (code 8B)");
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned int *counter = (unsigned int *)workspace;
    double *part = workspace ? (double *)((char *)workspace + 256) : nullptr;
    if (term) RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), st));
    vgg_post_partial_kernel<<<vg_blocks((long long)n * H * W * (C / 8)), VG_THREADS, 0, st>>>(
        (const __nv_bfloat16 *)raw, (const uint8_t *)mask, n, H, W, C, bias, (__nv_bfloat16 *)out, (int8_t *)code, term, scale, part,
        counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_dgrad_in_partial(const void *up, const void *mask, const void *code, int n, int H, int W, int C, const float *g,
                              float coef, void *dy, void *stream)
{
    RB_CHECK_ARG(mask && code && g && dy, "vgg_dgrad_in_partial: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0, "vgg_dgrad_in_partial: bad shape (n = %d, %d x %d x %d)", n, H, W,
                 C);
    RB_CHECK_ARG(vg_aligned(up, 16) && vg_aligned(code, 8) && vg_aligned(dy, 16),
                 "vgg_dgrad_in_partial: tensors must be 16B aligned (code 8B)");
    vgg_dgrad_in_partial_kernel<<<vg_blocks((long long)n * H * W * (C / 8)), VG_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)up, (const int8_t *)code, (const uint8_t *)mask, n, H, W, C, g, coef, (__nv_bfloat16 *)dy);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_vgg_image_grad_masked(const void *dx, const void *mask, int n, int H, int W, const float *std_, float *out, void *stream)
{
    RB_CHECK_ARG(dx && mask && std_ && out, "vgg_image_grad_masked: null pointer");
    RB_CHECK_ARG(n > 0 && H > 0 && W > 0, "vgg_image_grad_masked: empty batch (n = %d, %d x %d)", n, H, W);
    RB_CHECK_ARG(vg_aligned(dx, 16), "vgg_image_grad_masked: input must be 16B aligned");
    vgg_image_grad_masked_kernel<<<vg_blocks((long long)n * H * W), VG_THREADS, 0, (cudaStream_t)stream>>>(
        (const __nv_bfloat16 *)dx, (const uint8_t *)mask, n, H, W, std_, out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"
