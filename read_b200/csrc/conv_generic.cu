// Generic fused gated convolution on CUDA cores (fp32 accumulate) for sm_90a.
//
// Covers EVERY BasicConv shape of the refinement net (READ/models/unet.py:22-53): k in {1,3,4},
// stride in {1,2}, any channel count that is a multiple of 8, with the surrounding graph ops fused
// into the operand loader / epilogue:
//   * virtual concat of up to 4 sources (torch.cat, unet.py:88,105,263,271,279)
//   * nearest resample of a source by an integer factor (F.interpolate, unet.py:239-250)
//   * bilinear x4 upsample, align_corners=False (nn.Upsample, unet.py:200)
//   * elementwise product of the input with a second tensor (FAM x1*x2, unet.py:115)
//   * bias, ELU / identity, sigmoid gate, eval-mode BatchNorm affine (unet.py:44-51)
//   * residual add (ResBlock unet.py:20, FAM unet.py:116)
// This is the shape-complete kernel and the fp32 "parity mode" of the net; the dominant 3x3 layers run on
// the wgmma kernel in conv_tc.cu when activations are bf16.
#include "common.cuh"
#include "conv_common.cuh"

namespace rb {

constexpr int GC_BM = 64;     // 8x8 output pixels
constexpr int GC_BN = 64;     // 32 output channels x {f, m}
constexpr int GC_BK = 16;
constexpr int GC_THREADS = 256;

struct SrcView {
    const void *ptr;
    int C, H, W, mode, factor, c_begin;
};

struct GenericArgs {
    SrcView src[READ_MAX_SRC];
    int n_src;
    const void *mul;
    int B, Hin, Win, Cin, Hout, Wout, Cout;
    int k, stride, pad, elu;
    const float *w;
    int Npad, K, Kpad;
    const float *bias_f, *bias_m, *bn_scale, *bn_shift;
    const void *residual;
    void *out;
    int out_mode;
    void *out2;
    const void *out2_mul;
    int tiles_x, tiles_y;
};

template <typename T> struct Vec8;
template <> struct Vec8<float> {
    static __device__ __forceinline__ void load(const float *p, float *v)
    {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(p));
        const float4 b = __ldg(reinterpret_cast<const float4 *>(p) + 1);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
    }
    static __device__ __forceinline__ void store(float *p, const float *v)
    {
        reinterpret_cast<float4 *>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
        reinterpret_cast<float4 *>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
};
template <> struct Vec8<__nv_bfloat16> {
    static __device__ __forceinline__ void load(const __nv_bfloat16 *p, float *v)
    {
        const uint4 r = __ldg(reinterpret_cast<const uint4 *>(p));
        const __nv_bfloat162 *h = reinterpret_cast<const __nv_bfloat162 *>(&r);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float2 f = __bfloat1622float2(h[i]);
            v[2 * i] = f.x;
            v[2 * i + 1] = f.y;
        }
    }
    static __device__ __forceinline__ void store(__nv_bfloat16 *p, const float *v)
    {
        __nv_bfloat162 h[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
        *reinterpret_cast<uint4 *>(p) = *reinterpret_cast<uint4 *>(h);
    }
};

// Fetch 8 consecutive channels [c, c+8) of the logical input at (b, iy, ix); (iy, ix) is in range.
template <typename T>
__device__ __forceinline__ void fetch8(const GenericArgs &a, int b, int iy, int ix, int c, float *v)
{
    int s = 0;
#pragma unroll
    for (int i = 1; i < READ_MAX_SRC; ++i)
        if (i < a.n_src && c >= a.src[i].c_begin) s = i;
    const SrcView &sv = a.src[s];
    const int cl = c - sv.c_begin;
    const T *base = static_cast<const T *>(sv.ptr) + (long long)b * sv.H * sv.W * sv.C + cl;
    if (sv.mode == READ_SRC_BILINEAR_UP4) {
        // torch upsample_bilinear2d, align_corners=False, scale 1/4: src = max(0.25*(dst+0.5)-0.5, 0)
        float sy = 0.25f * ((float)iy + 0.5f) - 0.5f;
        float sx = 0.25f * ((float)ix + 0.5f) - 0.5f;
        sy = sy < 0.f ? 0.f : sy;
        sx = sx < 0.f ? 0.f : sx;
        const int y0 = (int)sy, x0 = (int)sx;
        const int yp = (y0 < sv.H - 1) ? 1 : 0, xp = (x0 < sv.W - 1) ? 1 : 0;
        const float ly = sy - (float)y0, lx = sx - (float)x0;
        const float hy = 1.f - ly, hx = 1.f - lx;
        float v00[8], v01[8], v10[8], v11[8];
        const T *p = base + ((long long)y0 * sv.W + x0) * sv.C;
        Vec8<T>::load(p, v00);
        Vec8<T>::load(p + (long long)xp * sv.C, v01);
        Vec8<T>::load(p + (long long)yp * sv.W * sv.C, v10);
        Vec8<T>::load(p + ((long long)yp * sv.W + xp) * sv.C, v11);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = hy * (hx * v00[i] + lx * v01[i]) + ly * (hx * v10[i] + lx * v11[i]);
        return;
    }
    int yy = iy, xx = ix;
    if (sv.mode == READ_SRC_NEAREST_DOWN) { yy = iy * sv.factor; xx = ix * sv.factor; }
    else if (sv.mode == READ_SRC_NEAREST_UP) { yy = iy / sv.factor; xx = ix / sv.factor; }
    yy = yy < sv.H ? yy : sv.H - 1;   // torch nearest clamps to in-1
    xx = xx < sv.W ? xx : sv.W - 1;
    Vec8<T>::load(base + ((long long)yy * sv.W + xx) * sv.C, v);
}

template <typename T>
__global__ void __launch_bounds__(GC_THREADS) gated_conv_generic_kernel(const __grid_constant__ GenericArgs a)
{
    __shared__ __align__(16) float As[GC_BK][GC_BM + 4];
    __shared__ __align__(16) float Bs[GC_BK][GC_BN];

    const int t = threadIdx.x;
    const int tile = blockIdx.x;
    const int tx_tile = tile % a.tiles_x;
    const int ty_tile = (tile / a.tiles_x) % a.tiles_y;
    const int b = tile / (a.tiles_x * a.tiles_y);
    const int ngrp = blockIdx.y;                 // 32-channel output group

    // A loader role: threads 0..127 -> (pixel, 8-channel group)
    const int lp = t & 63, lg = (t >> 6) & 1;
    const int loy = ty_tile * 8 + (lp >> 3), lox = tx_tile * 8 + (lp & 7);
    // compute role
    const int tx = t & 15, ty = t >> 4;

    float accf[4][2], accm[4][2];
#pragma unroll
    for (int i = 0; i < 4; ++i) { accf[i][0] = accf[i][1] = accm[i][0] = accm[i][1] = 0.f; }

    const int nchunks = a.Kpad / GC_BK;
    for (int kc = 0; kc < nchunks; ++kc) {
        if (t < 128) {
            float v[8];
            const int kidx = kc * GC_BK + lg * 8;
            bool valid = (kidx < a.K) && (loy < a.Hout) && (lox < a.Wout);
            int iy = 0, ix = 0, c = 0;
            if (valid) {
                const int tap = kidx / a.Cin;
                c = kidx - tap * a.Cin;
                const int ky = tap / a.k, kx = tap - ky * a.k;
                iy = loy * a.stride - a.pad + ky;
                ix = lox * a.stride - a.pad + kx;
                valid = (iy >= 0) && (iy < a.Hin) && (ix >= 0) && (ix < a.Win);
            }
            if (valid) {
                fetch8<T>(a, b, iy, ix, c, v);
                if (a.mul) {
                    float m8[8];
                    Vec8<T>::load(static_cast<const T *>(a.mul) + (((long long)b * a.Hin + iy) * a.Win + ix) * a.Cin + c, m8);
#pragma unroll
                    for (int i = 0; i < 8; ++i) v[i] *= m8[i];
                }
            } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = 0.f;
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) As[lg * 8 + i][lp] = v[i];
        }
        {
            const int row = t >> 4, col = (t & 15) * 4;
            const float4 wv = __ldg(reinterpret_cast<const float4 *>(a.w + (long long)(kc * GC_BK + row) * a.Npad + ngrp * GC_BN + col));
            *reinterpret_cast<float4 *>(&Bs[row][col]) = wv;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < GC_BK; ++kk) {
            const float4 av = *reinterpret_cast<const float4 *>(&As[kk][ty * 4]);
            const float2 bf = *reinterpret_cast<const float2 *>(&Bs[kk][tx * 2]);
            const float2 bm = *reinterpret_cast<const float2 *>(&Bs[kk][32 + tx * 2]);
            const float ap[4] = {av.x, av.y, av.z, av.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                accf[i][0] = fmaf(ap[i], bf.x, accf[i][0]);
                accf[i][1] = fmaf(ap[i], bf.y, accf[i][1]);
                accm[i][0] = fmaf(ap[i], bm.x, accm[i][0]);
                accm[i][1] = fmaf(ap[i], bm.y, accm[i][1]);
            }
        }
        __syncthreads();
    }

    // epilogue
    const int co0 = ngrp * 32 + tx * 2;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int pi = ty * 4 + i;
        const int oy = ty_tile * 8 + (pi >> 3), ox = tx_tile * 8 + (pi & 7);
        if (oy >= a.Hout || ox >= a.Wout) continue;
        const long long pix = ((long long)b * a.Hout + oy) * a.Wout + ox;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            const int co = co0 + j;
            if (co >= a.Cout) continue;
            float y = gated_epilogue(accf[i][j] + a.bias_f[co], accm[i][j] + a.bias_m[co], a.elu, a.bn_scale[co], a.bn_shift[co]);
            if (a.residual) y += to_f32<T>(static_cast<const T *>(a.residual)[pix * a.Cout + co]);
            if (a.out_mode == READ_OUT_NCHW_F32) {
                static_cast<float *>(a.out)[(((long long)b * a.Cout + co) * a.Hout + oy) * a.Wout + ox] = y;
            } else {
                static_cast<T *>(a.out)[pix * a.Cout + co] = from_f32<T>(y);
            }
            if (a.out2) {
                const float m = to_f32<T>(static_cast<const T *>(a.out2_mul)[pix * a.Cout + co]);
                // FAM consumes the STORED (rounded) activation: multiply what a reader of `out` would see
                const float ys = to_f32<T>(from_f32<T>(y));
                static_cast<T *>(a.out2)[pix * a.Cout + co] = from_f32<T>(ys * m);
            }
        }
    }
}

// ---- weight packing: torch [Cout,Cin,kh,kw] x2  ->  [Kpad][Npad] f32, k = (ky*kw+kx)*Cin + c,
//      column n = 64*(co/32) + (co%32) for f, +32 for m.
__global__ void pack_generic_kernel(const float *__restrict__ wf, const float *__restrict__ wm, int Cout, int Cin, int k,
                                    int Npad, int Kpad, float *__restrict__ out)
{
    const long long total = (long long)Kpad * Npad;
    const int K = k * k * Cin;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i % Npad);
        const int kk = (int)(i / Npad);
        const int grp = n / 64, r = n % 64;
        const int co = grp * 32 + (r & 31);
        const bool is_m = r >= 32;
        float v = 0.f;
        if (kk < K && co < Cout) {
            const int tap = kk / Cin, c = kk % Cin;
            const int ky = tap / k, kx = tap % k;
            const float *w = is_m ? wm : wf;
            v = w[(((long long)co * Cin + c) * k + ky) * k + kx];
        }
        out[i] = v;
    }
}

template <typename TI, typename TO>
__global__ void nchw_to_nhwc_kernel(const TI *__restrict__ in, int B, int C, int H, int W, TO *__restrict__ out)
{
    const long long total = (long long)B * C * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        long long r = i / C;
        const int x = (int)(r % W);
        r /= W;
        const int y = (int)(r % H);
        const int b = (int)(r / H);
        out[i] = from_f32<TO>(to_f32<TI>(in[(((long long)b * C + c) * H + y) * W + x]));
    }
}
template <typename TI>
__global__ void nhwc_to_nchw_kernel(const TI *__restrict__ in, int B, int C, int H, int W, float *__restrict__ out)
{
    const long long total = (long long)B * C * H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(i % W);
        long long r = i / W;
        const int y = (int)(r % H);
        r /= H;
        const int c = (int)(r % C);
        const int b = (int)(r / C);
        out[i] = to_f32<TI>(in[(((long long)b * H + y) * W + x) * C + c]);
    }
}

// Bilinear x4 upsample, align_corners=False (nn.Upsample(scale_factor=4, mode='bilinear'), unet.py:200), NHWC.  Used by the bf16
// engine so the decoder's 1x1 merge convs read plain (identity) sources.
// One thread per LOW-resolution pixel and 8 channels: the 4x4 output block of a source pixel (X, Y) depends on
// the 3x3 neighbourhood only, with constant weights (output column 4X + j samples X - 0.375 + j / 4: {3/8 L + 5/8 C,
// 1/8 L + 7/8 C, 7/8 C + 1/8 R, 5/8 C + 3/8 R}; borders clamp L / R onto C exactly as torch's max(src, 0) / min(i0 + 1, n - 1)).
// 9 loads, vertical then horizontal lerp in registers, 16 stores: ~35 instructions per output vector instead of ~250 (a
// per-output kernel spends its time in three 64-bit divisions per 16 bytes written).
template <typename T>
__global__ void __launch_bounds__(128) upsample_bilinear4_block_kernel(const T *__restrict__ in, int B, int h, int w, int C, T *__restrict__ out)
{
    const int cg = C >> 3;
    const int total = B * h * w * cg;                       // < 2^31 (host check)
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (idx % cg) * 8;
    int t = idx / cg;
    const int X = t % w;
    t /= w;
    const int Y = t % h;
    const int b = t / h;
    const int xs[3] = {X > 0 ? X - 1 : 0, X, X < w - 1 ? X + 1 : w - 1};
    const int ys[3] = {Y > 0 ? Y - 1 : 0, Y, Y < h - 1 ? Y + 1 : h - 1};
    float v[3][3][8];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Vec8<T>::load(in + (((long long)b * h + ys[i]) * w + xs[j]) * C + c, v[i][j]);
    // weights of (first tap, second tap) and which source rows / columns they are, for the 4 output phases
    const float w0[4] = {0.375f, 0.125f, 0.875f, 0.625f}, w1[4] = {0.625f, 0.875f, 0.125f, 0.375f};
    const int W4 = w * 4;
    T *obase = out + (((long long)b * h * 4 + Y * 4) * W4 + X * 4) * C + c;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int ia = i < 2 ? 0 : 1;                       // rows (Y-1, Y) for phases 0, 1; (Y, Y+1) for phases 2, 3
        float r[3][8];
#pragma unroll
        for (int j = 0; j < 3; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) r[j][k] = w0[i] * v[ia][j][k] + w1[i] * v[ia + 1][j][k];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int ja = j < 2 ? 0 : 1;
            float o[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) o[k] = w0[j] * r[ja][k] + w1[j] * r[ja + 1][k];
            Vec8<T>::store(obase + ((long long)i * W4 + j) * C, o);
        }
    }
}

int generic_npad(int Cout) { return ((Cout + 31) / 32) * 64; }
int generic_kpad(int K) { return ((K + GC_BK - 1) / GC_BK) * GC_BK; }

int launch_generic(const read_conv_desc &d, cudaStream_t st)
{
    GenericArgs a{};
    int cb = 0;
    for (int i = 0; i < d.n_src; ++i) {
        a.src[i] = SrcView{d.src[i].ptr, d.src[i].C, d.src[i].H, d.src[i].W, d.src[i].mode, d.src[i].factor, cb};
        cb += d.src[i].C;
    }
    a.n_src = d.n_src;
    a.mul = d.mul;
    a.B = d.B; a.Hin = d.Hin; a.Win = d.Win; a.Cin = d.Cin;
    a.Hout = d.Hout; a.Wout = d.Wout; a.Cout = d.Cout;
    a.k = d.k; a.stride = d.stride; a.pad = d.pad; a.elu = d.elu;
    a.w = d.w_generic;
    a.Npad = generic_npad(d.Cout);
    a.K = d.k * d.k * d.Cin;
    a.Kpad = generic_kpad(a.K);
    a.bias_f = d.bias_f; a.bias_m = d.bias_m; a.bn_scale = d.bn_scale; a.bn_shift = d.bn_shift;
    a.residual = d.residual;
    a.out = d.out; a.out_mode = d.out_mode; a.out2 = d.out2; a.out2_mul = d.out2_mul;
    a.tiles_x = (d.Wout + 7) / 8;
    a.tiles_y = (d.Hout + 7) / 8;
    const long long tiles = (long long)a.tiles_x * a.tiles_y * d.B;
    if (tiles == 0) return READ_OK;
    if (tiles > 0x7FFFFFFFll) { set_error("conv: too many tiles"); return READ_ERR_INVALID; }
    dim3 grid((unsigned)tiles, (unsigned)((d.Cout + 31) / 32));
    if (d.act_dtype == READ_ACT_F32) gated_conv_generic_kernel<float><<<grid, GC_THREADS, 0, st>>>(a);
    else gated_conv_generic_kernel<__nv_bfloat16><<<grid, GC_THREADS, 0, st>>>(a);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb

using namespace rb;

// Viewer output path (READ/gl/nn.py:123-124, viewer.py:267): RGB planes [3,H,W] f32 -> [H,W,4] f32 with alpha, optionally
// flipped vertically.  One float4 store per pixel, three coalesced plane reads.
__global__ void frame_to_rgba_kernel(const float *__restrict__ in, int H, int W, int flip, float alpha, float4 *__restrict__ out)
{
    const long long n = (long long)H * W;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int y = (int)(i / W), x = (int)(i - (long long)y * W);
        const int ys = flip ? (H - 1 - y) : y;
        const long long o = (long long)ys * W + x;
        out[i] = make_float4(in[o], in[n + o], in[2 * n + o], alpha);
    }
}

extern "C" {

int read_generic_npad(int Cout) { return generic_npad(Cout); }

int read_pack_weights_generic(const float *wf, const float *wm, int Cout, int Cin, int k, float *out, void *stream)
{
    RB_CHECK_ARG(wf && wm && out && Cout >= 1 && Cin >= 1 && k >= 1, "pack_generic: bad arguments");
    const int Npad = generic_npad(Cout), Kpad = generic_kpad(k * k * Cin);
    const long long total = (long long)Npad * Kpad;
    long long blocks = (total + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    pack_generic_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(wf, wm, Cout, Cin, k, Npad, Kpad, out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_upsample_bilinear4(const void *in, int act_dtype, int B, int h, int w, int C, void *out, void *stream)
{
    RB_CHECK_ARG(in && out && B >= 1 && h >= 1 && w >= 1 && C >= 8 && C % 8 == 0, "upsample: bad arguments");
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, "upsample: 16B alignment");
    const long long total = (long long)B * h * w * (C / 8);
    RB_CHECK_ARG(total < (1ll << 31), "upsample: tensor too large");
    if (total == 0) return READ_OK;
    const unsigned blocks = (unsigned)((total + 127) / 128);
    if (act_dtype == READ_ACT_F32)
        upsample_bilinear4_block_kernel<float><<<blocks, 128, 0, (cudaStream_t)stream>>>((const float *)in, B, h, w, C, (float *)out);
    else
        upsample_bilinear4_block_kernel<__nv_bfloat16><<<blocks, 128, 0, (cudaStream_t)stream>>>(
            (const __nv_bfloat16 *)in, B, h, w, C, (__nv_bfloat16 *)out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_frame_to_rgba(const float *rgb_planes, int H, int W, int flip_vertical, float alpha, float *out_hwc4, void *stream)
{
    RB_CHECK_ARG(rgb_planes && out_hwc4 && H >= 0 && W >= 0, "frame_to_rgba: bad arguments");
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(out_hwc4) & 15) == 0, "frame_to_rgba: output must be 16-byte aligned");
    const long long n = (long long)H * W;
    if (n == 0) return READ_OK;
    frame_to_rgba_kernel<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(rgb_planes, H, W, flip_vertical, alpha,
                                                                        reinterpret_cast<float4 *>(out_hwc4));
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_nchw_f32_to_nhwc(const float *in, int B, int C, int H, int W, int act_dtype, void *out, void *stream)
{
    RB_CHECK_ARG(in && out && B >= 0 && C >= 1 && H >= 0 && W >= 0, "nchw->nhwc: bad arguments");
    const long long total = (long long)B * C * H * W;
    if (total == 0) return READ_OK;
    long long blocks = (total + 255) / 256;
    if (blocks > (long long)num_sms() * 32) blocks = (long long)num_sms() * 32;
    if (act_dtype == READ_ACT_F32)
        nchw_to_nhwc_kernel<float, float><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(in, B, C, H, W, (float *)out);
    else
        nchw_to_nhwc_kernel<float, __nv_bfloat16><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(in, B, C, H, W, (__nv_bfloat16 *)out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_nhwc_to_nchw_f32(const void *in, int act_dtype, int B, int C, int H, int W, float *out, void *stream)
{
    RB_CHECK_ARG(in && out && B >= 0 && C >= 1 && H >= 0 && W >= 0, "nhwc->nchw: bad arguments");
    const long long total = (long long)B * C * H * W;
    if (total == 0) return READ_OK;
    long long blocks = (total + 255) / 256;
    if (blocks > (long long)num_sms() * 32) blocks = (long long)num_sms() * 32;
    if (act_dtype == READ_ACT_F32)
        nhwc_to_nchw_kernel<float><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const float *)in, B, C, H, W, out);
    else
        nhwc_to_nchw_kernel<__nv_bfloat16><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16 *)in, B, C, H, W, out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"
