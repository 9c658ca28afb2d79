// Shared pieces of the gated-conv kernels.
#pragma once
#include "common.cuh"

namespace rb {

// BasicConv tail (READ/models/unet.py:44-51): BN( A(f) * sigmoid(m) ), eval-mode BN folded to scale/shift.
// f, m already include their biases.
__device__ __forceinline__ float gated_epilogue(float f, float m, int elu, float scale, float shift)
{
    const float a = (elu && f <= 0.f) ? expm1f(f) : f;   // nn.ELU(alpha=1)
    const float s = 1.f / (1.f + expf(-m));              // nn.Sigmoid
    return fmaf(a * s, scale, shift);
}

// Fast variant for the bf16 tensor-core path, activation chosen at compile time: 1 MUFU for ELU (ex2), 1 MUFU for the
// gate (tanh); the no-activation layers never touch the ex2 pipe.
template <bool ELU>
__device__ __forceinline__ float gate_fast(float f, float m, float scale, float shift)
{
    float a = f;
    if (ELU) {
        float e;
        asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(f * 1.4426950408889634f));
        a = f <= 0.f ? (e - 1.f) : f;
    }
    float th;
    asm("tanh.approx.f32 %0, %1;" : "=f"(th) : "f"(0.5f * m));
    return fmaf(a * fmaf(0.5f, th, 0.5f), scale, shift);
}

// floor(x / d) without integer division (a runtime IDIV costs ~20 instructions and every warp of every role decodes
// every tile).  floor((x + 0.5) * (1/d)) is exact for the x < 2^22 we ever see: the fractional part of (x+0.5)/d is at
// least 0.5/d away from an integer, far more than the fp32 rounding error.
__device__ __forceinline__ int fdiv_small(int x, float inv_d) { return (int)(((float)x + 0.5f) * inv_d); }

// Epilogue parameters of the wgmma kernels and the register epilogue of the gather kernel and of the TMA kernel's final NCHW
// layer (the TMA kernel's NHWC layers go through shared memory, conv_tc.cu: epilogue_smem).  Accumulator layout of wgmma m64nN (fp32): register
// 4*j + 2*i + c of lane l holds row (l >> 2) + 8*i of the warp's 16 rows, column 8*j + 2*(l & 3) + c.  Columns [0, N/2) are
// conv_f, [N/2, N) conv_m of the same output channels; a thread therefore owns both gates of two adjacent channels.
struct EpiArgs {
    int H, W, Cout;
    int elu, raw, nchw;                   // raw: store the accumulators themselves ([.., N] channels); nchw: final layer, fp32 NCHW
    const float4 *par;                    // shared memory, per channel {bias_f, bias_m, bn_scale, bn_shift}
    const __nv_bfloat16 *residual, *out2_mul, *addin;
    void *out;
    __nv_bfloat16 *out2;
    int addin_H, addin_W;                 // addin: [B, addin_H, addin_W, N] added (nearest x2) to the accumulators
};

__device__ __forceinline__ uint32_t bf16x2_bits(float lo, float hi)
{
    uint32_t d;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(d) : "f"(hi), "f"(lo));
    return d;
}
__device__ __forceinline__ float2 bf16x2_val(uint32_t u) { return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xFFFF0000u)); }
template <int N>
constexpr int e_nj() { return N / 16; }   // 8-column groups per gate

// Both rows of the thread: pixels (b, y[i], x[i]), output channels nt * N/2 + ...  (no RAW output, no add-in: those layers run
// on the TMA kernel).  Every global load of a column chunk (residual, FAM multiplier) is issued before its first store: the
// stores may alias them as far as the compiler knows, so loads interleaved with stores would each pay a full memory latency.
template <int N>
__device__ __forceinline__ void epilogue_tile(const float (&d)[N / 2], int lane, int b, const int (&y)[2], const int (&x)[2],
                                              const bool (&inside)[2], int nt, const EpiArgs &e)
{
    constexpr int HALF = N / 2;
    constexpr int NJ = e_nj<N>();
    const int q2 = 2 * (lane & 3);
    long long pix[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) pix[i] = ((long long)b * e.H + y[i]) * e.W + x[i];
#pragma unroll
    for (int j0 = 0; j0 < NJ; j0 += (N <= 64 ? 1 : 4)) {
        constexpr int JC = N <= 64 ? 1 : 4;    // the N <= 64 instances run two CTAs per SM (register bound): one column group per chunk
        uint32_t rv[2][JC], mv[2][JC];
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int jj = 0; jj < JC; ++jj) {
                const int col = 8 * (j0 + jj) + q2;
                const int co = nt * HALF + col;
                const bool ok = inside[i] && j0 + jj < NJ && co < e.Cout && !e.nchw;
                const long long o = pix[i] * e.Cout + co;
                rv[i][jj] = (ok && e.residual) ? __ldg(reinterpret_cast<const unsigned int *>(e.residual + o)) : 0u;
                mv[i][jj] = (ok && e.out2) ? __ldg(reinterpret_cast<const unsigned int *>(e.out2_mul + o)) : 0u;
            }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!inside[i]) continue;
#pragma unroll
            for (int jj = 0; jj < JC; ++jj) {
                const int j = j0 + jj;
                if (j >= NJ) break;
                const int col = 8 * j + q2;
                const int co = nt * HALF + col;
                if (co >= e.Cout) continue;
                const float f0 = d[4 * j + 2 * i], f1 = d[4 * j + 2 * i + 1];
                const float m0 = d[4 * (j + NJ) + 2 * i], m1 = d[4 * (j + NJ) + 2 * i + 1];
                const float4 p0 = e.par[co], p1 = e.par[co + 1];
                float y0, y1;
                if (e.elu) {
                    y0 = gate_fast<true>(f0 + p0.x, m0 + p0.y, p0.z, p0.w);
                    y1 = gate_fast<true>(f1 + p1.x, m1 + p1.y, p1.z, p1.w);
                } else {
                    y0 = gate_fast<false>(f0 + p0.x, m0 + p0.y, p0.z, p0.w);
                    y1 = gate_fast<false>(f1 + p1.x, m1 + p1.y, p1.z, p1.w);
                }
                if (e.nchw) {
                    float *op = static_cast<float *>(e.out);
                    op[(((long long)b * e.Cout + co) * e.H + y[i]) * e.W + x[i]] = y0;
                    if (co + 1 < e.Cout) op[(((long long)b * e.Cout + co + 1) * e.H + y[i]) * e.W + x[i]] = y1;
                    continue;
                }
                const long long o = pix[i] * e.Cout + co;
                const float2 r = bf16x2_val(rv[i][jj]);            // zero without a residual
                const uint32_t pk = bf16x2_bits(y0 + r.x, y1 + r.y);
                *reinterpret_cast<uint32_t *>(static_cast<__nv_bfloat16 *>(e.out) + o) = pk;
                if (e.out2) {
                    const float2 ys = bf16x2_val(pk);            // the stored (rounded) activation
                    const float2 mm = bf16x2_val(mv[i][jj]);
                    *reinterpret_cast<uint32_t *>(e.out2 + o) = bf16x2_bits(ys.x * mm.x, ys.y * mm.y);
                }
            }
        }
    }
}

int generic_npad(int Cout);
int generic_kpad(int K);
int launch_generic(const read_conv_desc &d, cudaStream_t st);

// wgmma path, TMA-loaded halo tiles (conv_tc.cu)
struct TcPlan;
bool tc_supported(const read_conv_desc &d);
int tc_plan_create(const read_conv_desc &d, TcPlan **out);
int tc_plan_launch(const TcPlan *p, cudaStream_t st, int max_ctas = 0);     // max_ctas > 0: persistent grid of at most that many CTAs
void tc_plan_destroy(TcPlan *p);
void tc_plan_set_reverse(TcPlan *p, int reverse);      // walk the tiles bottom-up (same result; L2 reuse between consecutive layers)

// wgmma path with gathered A operand (conv_tc_gather.cu)
struct TcgPlan;
bool tcg_supported(const read_conv_desc &d);
int tcg_plan_create(const read_conv_desc &d, TcgPlan **out);
int tcg_plan_launch(const TcgPlan *p, cudaStream_t st, int max_ctas = 0);
void tcg_plan_destroy(TcgPlan *p);
int64_t tcg_weight_elems(int Cout, int Cin, int k);
int tcg_pack(const float *wf, const float *wm, int Cout, int Cin, int k, void *out, cudaStream_t st);

}  // namespace rb
