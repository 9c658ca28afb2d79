// General gated convolution on the Hopper tensor cores (wgmma): implicit GEMM whose A operand is GATHERED by four
// producer warps (cp.async 16-byte chunks, zero-fill for padding) into 128B-swizzled rows of shared memory.  Covers every
// BasicConv shape of READ/models/unet.py that the TMA kernel (conv_tc.cu) cannot express as shifted tile loads:
//   * stride-2 3x3 and 4x4 convolutions with channel counts the TMA kernel does not take (feat_extract[1,2,6], [3,4,7])
//   * virtual concat of up to 4 sources (SCM / AFF / decoder merges: unet.py:88,105,263,271,279)
//   * nearest up/down resampling of a source (F.interpolate, unet.py:239-250) and bilinear x4 (nn.Upsample, :200)
//   * channel counts that are only multiples of 8 (8->32 first conv, 32->3 last conv, SCM 16/56/120/248)
//   * NCHW fp32 output for the final layer
//
// GEMM view: M = 128 output pixels (8 rows x 16 cols), K = (tap, cin) flattened in 8-channel chunks and padded to
// 64-element blocks, N = conv_f | conv_m channels (<= 128 per tile).  Weights arrive by TMA and are read by wgmma through
// shared-memory descriptors; the A rows are read with ldmatrix into wgmma's register operand; accumulators live in the
// registers of two consumer warpgroups (64 pixels each), whose epilogue is the fused bias/ELU/sigmoid/BN/residual tail of
// conv_common.cuh.
//
// Warp roles (384 threads, 1 CTA/SM, persistent): warps 0-3 = producers, one warp per ring stage: lane 0 loads the stage's
// weights by TMA and every lane gathers a fixed 16-byte K chunk of 4 tile columns x 8 rows of A; warps 4-11 = consumers.
#include "common.cuh"
#include "conv_common.cuh"
#include "ptx.cuh"
#include <cuda.h>
#include <mutex>
#include <new>

namespace rb {

constexpr int G_THREADS = 384;
constexpr int G_CONS_WARP0 = 4;              // warps 0..3 produce, warps 4..11 are two consumer warpgroups
constexpr int G_TW = 16, G_TH = 8;
constexpr int G_MAX_STAGES = 4;              // one gather warp per ring stage
constexpr uint32_t G_SMEM_BUDGET = 200 * 1024;
constexpr int G_KBLK = 64;                     // elements per K block (128-byte rows, SWIZZLE_128B)

struct GSrc {
    const __nv_bfloat16 *ptr;
    int C, H, W, mode, shift, c_begin;   // shift = log2(resample factor)
};

// Per-source parameters the producers read from shared memory (dynamic indexing of the kernel-parameter constant bank
// is slow).  Nearest resampling is one formula for identity / down / up: src = (dst << shl) >> shr; a coordinate that
// is inside the (virtual) conv input is always inside the source, so no clamp is needed.
struct __align__(16) SrcS {
    const __nv_bfloat16 *ptr;
    int plane;                 // H*W*C elements per image (< 2^31)
    int C;
    int rs;                    // W*C (row stride in elements)
    int shl, shr, bil;
    int W, H, pad0_, pad1_;    // bilinear path only
};

struct GArgs {
    GSrc src[READ_MAX_SRC];
    int n_src;
    int B, Hin, Win, Cin, Hout, Wout, Cout, Cout_pad;
    int ksize, stride, pad;
    int K, kblocks;
    int n_tile, n_tiles;
    int tiles_x, tiles_y;
    float inv_tx, inv_ty, inv_nt;   // reciprocals for the division-free tile decode
    int stages;
    int pdl;                   // launched with programmatic stream serialization
    uint32_t a_bytes, b_bytes;
    const float *bias_f, *bias_m, *scale, *shift;
    EpiArgs epi;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// the mbarrier receives one (pre-counted) arrival from this thread once all its prior cp.async have completed
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar)
{
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}

__device__ __forceinline__ uint32_t g_pack2(float a, float b)
{
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&v);
}
__device__ __forceinline__ float2 g_unpack2(uint32_t u) { return __bfloat1622float2(*reinterpret_cast<__nv_bfloat162 *>(&u)); }

// bilinear x4, align_corners=False (torch upsample_bilinear2d): src = max(0.25*(dst+0.5)-0.5, 0).  Only the fp32-parity
// engine and the unit tests route a bilinear source through this kernel (the bf16 engine upsamples with its own kernel).
__device__ __noinline__ void gather_bilinear_row(const SrcS &sv, const __nv_bfloat16 *sbase, int ix, int iy, bool valid,
                                                 uint32_t dst)
{
    uint4 o = make_uint4(0, 0, 0, 0);
    if (valid) {
        float fx = 0.25f * ((float)ix + 0.5f) - 0.5f;
        fx = fx < 0.f ? 0.f : fx;
        const int x0 = (int)fx;
        const int xp = (x0 < sv.W - 1) ? 1 : 0;
        const float lx = fx - (float)x0, hx = 1.f - lx;
        float fy = 0.25f * ((float)iy + 0.5f) - 0.5f;
        fy = fy < 0.f ? 0.f : fy;
        const int y0 = (int)fy;
        const int yp = (y0 < sv.H - 1) ? 1 : 0;
        const float ly = fy - (float)y0, hy = 1.f - ly;
        const __nv_bfloat16 *p = sbase + ((long long)y0 * sv.W + x0) * sv.C;
        const uint4 v00 = __ldg(reinterpret_cast<const uint4 *>(p));
        const uint4 v01 = __ldg(reinterpret_cast<const uint4 *>(p + (long long)xp * sv.C));
        const uint4 v10 = __ldg(reinterpret_cast<const uint4 *>(p + (long long)yp * sv.W * sv.C));
        const uint4 v11 = __ldg(reinterpret_cast<const uint4 *>(p + ((long long)yp * sv.W + xp) * sv.C));
        const uint32_t *a00 = &v00.x, *a01 = &v01.x, *a10 = &v10.x, *a11 = &v11.x;
        uint32_t r[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float2 f00 = g_unpack2(a00[q]), f01 = g_unpack2(a01[q]), f10 = g_unpack2(a10[q]), f11 = g_unpack2(a11[q]);
            r[q] = g_pack2(hy * (hx * f00.x + lx * f01.x) + ly * (hx * f10.x + lx * f11.x),
                           hy * (hx * f00.y + lx * f01.y) + ly * (hx * f10.y + lx * f11.y));
        }
        o = make_uint4(r[0], r[1], r[2], r[3]);
    }
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(o.x), "r"(o.y), "r"(o.z), "r"(o.w) : "memory");
}

template <int STRIDE, int N>
__global__ void __launch_bounds__(G_THREADS, 1)
gated_conv_tc_gather_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ GArgs a)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (s_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *smem_al = smem_raw + (smem_base - s_u32(smem_raw));

    const uint32_t stage_bytes = a.a_bytes + a.b_bytes;
    const uint32_t ring_bytes = stage_bytes * (uint32_t)a.stages;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_al + ring_bytes);
    const uint32_t full0 = s_u32(bars);
    const uint32_t empty0 = full0 + 8 * G_MAX_STAGES;
    float4 *s_par4 = reinterpret_cast<float4 *>(bars + 2 * G_MAX_STAGES);   // Cout_pad x {bias_f, bias_m, scale, shift}

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int CP = a.Cout_pad;
    if (a.pdl) pdl_launch_dependents();
    // per-(K block, 16-byte chunk) decode table, built once per CTA so the producers' hot loop has no division:
    // {source index (-1 = zero padding of K), ky, kx, channel offset inside the source}
    int4 *s_tab = reinterpret_cast<int4 *>(s_par4 + CP);
    SrcS *s_src = reinterpret_cast<SrcS *>(s_tab + a.kblocks * 8);
    if (threadIdx.x < READ_MAX_SRC) {
        const GSrc &g = a.src[threadIdx.x < a.n_src ? threadIdx.x : 0];
        SrcS v;
        v.ptr = g.ptr;
        v.plane = g.H * g.W * g.C;
        v.C = g.C;
        v.rs = g.W * g.C;
        v.shl = g.mode == READ_SRC_NEAREST_DOWN ? g.shift : 0;
        v.shr = g.mode == READ_SRC_NEAREST_UP ? g.shift : 0;
        v.bil = g.mode == READ_SRC_BILINEAR_UP4 ? 1 : 0;
        v.W = g.W; v.H = g.H; v.pad0_ = 0; v.pad1_ = 0;
        s_src[threadIdx.x] = v;
    }
    for (int i = threadIdx.x; i < a.kblocks * 8; i += G_THREADS) {
        const int kel = i * 8;
        int4 e = make_int4(-1, 0, 0, 0);
        if (kel < a.K) {
            const int tap = kel / a.Cin;
            const int c = kel - tap * a.Cin;
            int si = 0;
            for (int q = 1; q < READ_MAX_SRC; ++q)
                if (q < a.n_src && c >= a.src[q].c_begin) si = q;
            e = make_int4(si, tap / a.ksize, tap % a.ksize, c - a.src[si].c_begin);
        }
        s_tab[i] = e;
    }
    for (int i = threadIdx.x; i < CP; i += G_THREADS)
        s_par4[i] = i < a.Cout ? make_float4(a.bias_f[i], a.bias_m[i], a.scale[i], a.shift[i]) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < a.stages; ++s) {
            mbar_init(full0 + 8 * s, 32 + 1);   // the 32 lanes of the stage's gather warp + its lane 0's weight TMA
            mbar_init(empty0 + 8 * s, 8);       // the 8 consumer warps
        }
        mbar_fence_init();
    }
    __syncthreads();
    // everything above touched only static data (weights' descriptors, folded constants): with programmatic dependent launch
    // it overlapped the previous kernel's tail; activations / residuals below need that kernel to have completed
    if (a.pdl) pdl_wait();

    const int m_tiles = a.tiles_x * a.tiles_y * a.B;
    const long long total_tiles = (long long)m_tiles * a.n_tiles;
    const int n_total = a.n_tile * a.n_tiles;

    if (warp < G_CONS_WARP0) {
        // ===================== producers: 4 warps, ONE WARP PER RING STAGE =====================
        // Warp w owns ring slot w (a slot must have ONE producer that sees every one of its phases, or the parity wait on its
        // empty barrier could alias two phases) and fills it on its own: lane 0 starts the TMA of the stage's weight block,
        // then lane -> (16-byte K chunk j = lane & 7, tile column px = 4*g + (lane >> 3), g = 0..3), 8 tile rows each, 32
        // copies per lane and stage.  The stages are gathered concurrently by the 4 warps.
        const uint32_t w = (uint32_t)warp;
        if (w >= (uint32_t)a.stages) return;
        const uint32_t my_empty = empty0 + 8 * w;
        const int j = lane & 7;
        const int pq = lane >> 3;
        uint32_t s = 0, ph = 0;           // ring slot of the current iteration and its phase (tracked for EVERY iteration)
        const int4 *tab = s_tab + j;
        for (long long tl = blockIdx.x; tl < total_tiles; tl += gridDim.x) {
            const int mt = fdiv_small((int)tl, a.inv_nt);
            const int nt = (int)tl - mt * a.n_tiles;
            const int q_ = fdiv_small(mt, a.inv_tx);
            const int tx = mt - q_ * a.tiles_x;
            const int b = fdiv_small(q_, a.inv_ty);
            const int ty = q_ - b * a.tiles_y;
            const int oy0 = ty * G_TH;
            const int iyb = oy0 * STRIDE - a.pad;
            const int rows_ok = a.Hout - oy0;          // tile rows i < rows_ok produce output
            for (int kb = 0; kb < a.kblocks; ++kb) {
                if (s == w) {
                    mbar_wait(my_empty, ph ^ 1u);
                    const uint32_t dst0 = smem_base + s * stage_bytes;
                    if (lane == 0) {
                        mbar_arrive_expect_tx(full0 + 8 * s, a.b_bytes);
                        tma_load_2d(&tmB, full0 + 8 * s, dst0 + a.a_bytes, 0, nt * a.n_tile + kb * n_total);
                    }
                    const int4 e = tab[kb * 8];
                    const SrcS &sv = s_src[e.x < 0 ? 0 : e.x];
                    const __nv_bfloat16 *sbase = sv.ptr + (long long)b * sv.plane;
                    const int iy0 = iyb + e.y;
                    if (!sv.bil) {
                        const int shl = sv.shl, shr = sv.shr, rs = sv.rs, C = sv.C;
                        // per-row source offsets (elements), -1 = row outside the image / the output
                        int roff[G_TH];
#pragma unroll
                        for (int i = 0; i < G_TH; ++i) {
                            const int iy = iy0 + i * STRIDE;
                            const bool rv = (e.x >= 0) && (i < rows_ok) && ((unsigned)iy < (unsigned)a.Hin);
                            roff[i] = rv ? ((iy << shl) >> shr) * rs + e.w : -1;
                        }
#pragma unroll
                        for (int g = 0; g < 4; ++g) {
                            const int px = g * 4 + pq;
                            const int ox = tx * G_TW + px;
                            const int ix = ox * STRIDE - a.pad + e.z;
                            const bool xv = (ox < a.Wout) && ((unsigned)ix < (unsigned)a.Win);
                            const int xoff = ((ix << shl) >> shr) * C;
                            const uint32_t dcol = dst0 + (uint32_t)px * 128u + (uint32_t)((j ^ (px & 7)) << 4);
#pragma unroll
                            for (int i = 0; i < G_TH; ++i) {
                                const bool valid = xv && roff[i] >= 0;
                                cp_async16(dcol + (uint32_t)i * 2048u, sbase + (valid ? roff[i] + xoff : 0), valid ? 16u : 0u);
                            }
                        }
                        // asynchronous arrival: the barrier counts this lane in when its copies above have landed
                        cp_async_arrive_noinc(full0 + 8 * s);
                    } else {
                        for (int g = 0; g < 4; ++g) {
                            const int px = g * 4 + pq;
                            const int ox = tx * G_TW + px;
                            const int ix = ox * STRIDE - a.pad + e.z;
                            const bool xv = (e.x >= 0) && (ox < a.Wout) && ((unsigned)ix < (unsigned)a.Win);
                            const uint32_t dcol = dst0 + (uint32_t)px * 128u + (uint32_t)((j ^ (px & 7)) << 4);
                            for (int i = 0; i < G_TH; ++i) {
                                const int iy = iy0 + i * STRIDE;
                                const bool valid = xv && (i < rows_ok) && (iy >= 0) && (iy < a.Hin);
                                gather_bilinear_row(sv, sbase + e.w, ix, iy, valid, dcol + (uint32_t)i * 2048u);
                            }
                        }
                        mbar_arrive(full0 + 8 * s);
                    }
                }
                if (++s == (uint32_t)a.stages) { s = 0; ph ^= 1u; }
            }
        }
    } else {
        // ===================== consumers: two warpgroups, 64 pixels (4 tile rows) each =====================
        const int wg = (warp - G_CONS_WARP0) >> 2, wiw = warp & 3;
        const uint32_t lrow = (uint32_t)(64 * wg + 16 * wiw + (lane & 7) + 8 * ((lane >> 3) & 1));   // this lane's ldmatrix row
        const uint32_t khalf = (uint32_t)(lane >> 4) * 16u;
        uint32_t s = 0, ph = 0;
        EpiArgs e = a.epi;
        e.par = s_par4;
        for (long long t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const int mt = fdiv_small((int)t, a.inv_nt);
            const int nt = (int)t - mt * a.n_tiles;
            const int q_ = fdiv_small(mt, a.inv_tx);
            const int tx = mt - q_ * a.tiles_x;
            const int b = fdiv_small(q_, a.inv_ty);
            const int ty = q_ - b * a.tiles_y;
            float acc[N / 2];
#pragma unroll
            for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
            for (int kb = 0; kb < a.kblocks; ++kb) {
                mbar_wait(full0 + 8 * s, ph);
                const uint32_t stage = smem_base + s * stage_bytes;
                uint32_t fr[G_KBLK / 16][4];
#pragma unroll
                for (int kk = 0; kk < G_KBLK / 16; ++kk) ldmatrix_x4(stage + swz(lrow * 128u + 32u * kk + khalf, 128u), fr[kk]);
                wgmma_fence();
                wgmma_fence_acc(acc);
#pragma unroll
                for (int kk = 0; kk < G_KBLK / 16; ++kk) Wgmma<N>::mma(acc, fr[kk], wgmma_desc(stage + a.a_bytes + 32u * kk, 128u), 1u);
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_acc(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty0 + 8 * s);
                if (++s == (uint32_t)a.stages) { s = 0; ph ^= 1u; }
            }
            const int y0 = ty * G_TH + 4 * wg + wiw, x0 = tx * G_TW + (lane >> 2);
            const int xs[2] = {x0, x0 + 8}, ys[2] = {y0, y0};
            const bool in[2] = {x0 < a.Wout && y0 < a.Hout, x0 + 8 < a.Wout && y0 < a.Hout};
            epilogue_tile<N>(acc, lane, b, ys, xs, in, nt, e);
        }
    }
}

// ------------------------------------------------------------------ weight packing
// out[((kb * n_total + n) * 64 + kk)],  k = kb*64 + kk = (tap*Cin + c) ; n -> (tile, f|m half, channel); zero padded
__global__ void pack_tcg_kernel(const float *__restrict__ wf, const float *__restrict__ wm, int Cout, int Cin, int k,
                                int kblocks, int n_tile, int n_tiles, __nv_bfloat16 *__restrict__ out)
{
    const int K = k * k * Cin;
    const int n_total = n_tile * n_tiles;
    const int half = n_tile / 2;
    const long long total = (long long)kblocks * n_total * G_KBLK;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int kk = (int)(i % G_KBLK);
        long long r = i / G_KBLK;
        const int n = (int)(r % n_total);
        const int kb = (int)(r / n_total);
        const int kel = kb * G_KBLK + kk;
        const int nt = n / n_tile, rr = n % n_tile;
        const bool is_m = rr >= half;
        const int co = nt * half + (rr % half);
        float v = 0.f;
        if (kel < K && co < Cout) {
            const int tap = kel / Cin, c = kel % Cin;
            const int ky = tap / k, kx = tap % k;
            const float *w = is_m ? wm : wf;
            v = w[(((long long)co * Cin + c) * k + ky) * k + kx];
        }
        out[i] = __float2bfloat16_rn(v);
    }
}

// ------------------------------------------------------------------ host side
struct GGeom {
    int cout_pad, n_tile, n_tiles, kblocks;
};
static bool g_geom(int Cin, int Cout, int k, GGeom *g)
{
    if (Cin % 8 != 0 || Cout < 1) return false;
    int cp, n_tile, n_tiles;
    if (Cout <= 64) {
        cp = ((Cout + 7) / 8) * 8;
        n_tile = 2 * cp;
        n_tiles = 1;
    } else {                                   // accumulators in registers: at most 128 columns (64 fp32 per thread)
        cp = ((Cout + 63) / 64) * 64;
        n_tile = 128;
        n_tiles = cp / 64;
    }
    if (n_tile % 16 != 0 || n_tile > 128) return false;
    if (g) *g = GGeom{cp, n_tile, n_tiles, (k * k * Cin + G_KBLK - 1) / G_KBLK};
    return true;
}

bool tcg_supported(const read_conv_desc &d)
{
    if (d.act_dtype != READ_ACT_BF16 || d.mul != nullptr) return false;
    if (d.out_mode == READ_OUT_RAW_NHWC || d.addin != nullptr) return false;      // TMA kernel only
    if (d.out_mode == READ_OUT_NHWC && d.Cout % 8 != 0) return false;
    for (int i = 0; i < d.n_src; ++i) {
        if (d.src[i].C % 8 != 0) return false;
        const int f = d.src[i].factor;
        const bool resampled = d.src[i].mode == READ_SRC_NEAREST_DOWN || d.src[i].mode == READ_SRC_NEAREST_UP;
        if (resampled && (f < 2 || (f & (f - 1)) != 0)) return false;      // power-of-two factors only (shifts)
    }
    return g_geom(d.Cin, d.Cout, d.k, nullptr);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_tiled();

struct TcgPlan {
    CUtensorMap tmB;
    GArgs args;
    size_t smem_bytes;
};

int tcg_plan_create(const read_conv_desc &d, TcgPlan **out)
{
    GGeom g;
    if (!tcg_supported(d) || !g_geom(d.Cin, d.Cout, d.k, &g)) {
        set_error("wgmma gather conv: unsupported layer");
        return READ_ERR_UNSUPPORTED;
    }
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) {
        set_error("wgmma gather conv: cuTensorMapEncodeTiled not available from the driver");
        return READ_ERR_CUDA;
    }
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(d.w_tc) & 127) == 0, "wgmma gather conv: packed weights must be 128B aligned");
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "wgmma gather conv: output must be 16B aligned");
    TcgPlan *p = new (std::nothrow) TcgPlan{};
    RB_CHECK_ARG(p != nullptr, "wgmma gather conv: out of host memory");
    {
        const cuuint64_t rows = (cuuint64_t)g.kblocks * g.n_tile * g.n_tiles;
        cuuint64_t dims[2] = {(cuuint64_t)G_KBLK, rows};
        cuuint64_t strides[1] = {(cuuint64_t)G_KBLK * 2};
        cuuint32_t box[2] = {(cuuint32_t)G_KBLK, (cuuint32_t)g.n_tile};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&p->tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(d.w_tc), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            set_error("wgmma gather conv: cuTensorMapEncodeTiled(weights) failed with %d", (int)r);
            delete p;
            return READ_ERR_CUDA;
        }
    }
    GArgs &a = p->args;
    int cb = 0;
    for (int i = 0; i < d.n_src; ++i) {
        int sh = 0;
        while ((1 << sh) < d.src[i].factor) ++sh;
        a.src[i] = GSrc{static_cast<const __nv_bfloat16 *>(d.src[i].ptr), d.src[i].C, d.src[i].H, d.src[i].W, d.src[i].mode,
                        sh, cb};
        cb += d.src[i].C;
    }
    for (int i = d.n_src; i < READ_MAX_SRC; ++i) a.src[i] = a.src[0];
    a.n_src = d.n_src;
    a.B = d.B; a.Hin = d.Hin; a.Win = d.Win; a.Cin = d.Cin;
    a.Hout = d.Hout; a.Wout = d.Wout; a.Cout = d.Cout; a.Cout_pad = g.cout_pad;
    a.ksize = d.k; a.stride = d.stride; a.pad = d.pad;
    a.K = d.k * d.k * d.Cin; a.kblocks = g.kblocks;
    a.n_tile = g.n_tile; a.n_tiles = g.n_tiles;
    a.tiles_x = (d.Wout + G_TW - 1) / G_TW;
    a.tiles_y = (d.Hout + G_TH - 1) / G_TH;
    a.inv_tx = 1.0f / (float)a.tiles_x;
    a.inv_ty = 1.0f / (float)a.tiles_y;
    a.inv_nt = 1.0f / (float)a.n_tiles;
    if ((long long)d.B * d.Hout * d.Wout * d.Cout >= (1ll << 31)) {
        set_error("wgmma gather conv: output too large for 32-bit offsets");
        delete p;
        return READ_ERR_UNSUPPORTED;
    }
    if ((long long)a.tiles_x * a.tiles_y * d.B * a.n_tiles >= (1ll << 22)) {
        set_error("wgmma gather conv: too many tiles for the division-free decode");
        delete p;
        return READ_ERR_UNSUPPORTED;
    }
    a.a_bytes = 128u * G_KBLK * 2u;
    a.b_bytes = (uint32_t)g.n_tile * G_KBLK * 2u;
    int stages = (int)(G_SMEM_BUDGET / (a.a_bytes + a.b_bytes));
    if (stages > G_MAX_STAGES) stages = G_MAX_STAGES;
    a.stages = stages;
    if (stages < 3 || (d.stride != 1 && d.stride != 2)) {
        set_error("wgmma gather conv: unsupported geometry (stages %d, stride %d)", stages, d.stride);
        delete p;
        return READ_ERR_UNSUPPORTED;
    }
    a.bias_f = d.bias_f; a.bias_m = d.bias_m; a.scale = d.bn_scale; a.shift = d.bn_shift;
    EpiArgs &e = a.epi;
    e.H = d.Hout; e.W = d.Wout; e.Cout = d.Cout;
    e.elu = d.elu;
    e.raw = 0;
    e.nchw = d.out_mode == READ_OUT_NCHW_F32 ? 1 : 0;
    e.par = nullptr;
    e.residual = static_cast<const __nv_bfloat16 *>(d.residual);
    e.out2_mul = static_cast<const __nv_bfloat16 *>(d.out2_mul);
    e.addin = nullptr;
    e.out = d.out;
    e.out2 = static_cast<__nv_bfloat16 *>(d.out2);
    e.addin_H = e.addin_W = 0;
    p->smem_bytes = 1024 + (size_t)stages * (a.a_bytes + a.b_bytes) + 8 * (2 * G_MAX_STAGES) + 16 * (size_t)g.cout_pad + 16 * (size_t)g.kblocks * 8 + sizeof(SrcS) * READ_MAX_SRC + 64;
    *out = p;
    return READ_OK;
}

extern int g_tc_pdl;

template <int STRIDE, int N>
static int launch_tcg(const TcgPlan *p, const GArgs &a, cudaLaunchConfig_t &lcfg)
{
    RB_CUDA(cudaFuncSetAttribute(gated_conv_tc_gather_kernel<STRIDE, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_bytes));
    RB_CUDA(cudaLaunchKernelEx(&lcfg, gated_conv_tc_gather_kernel<STRIDE, N>, p->tmB, a));
    return READ_OK;
}

template <int STRIDE>
static int launch_tcg_n(const TcgPlan *p, const GArgs &a, cudaLaunchConfig_t &lcfg)
{
    switch (a.n_tile) {
    case 16: return launch_tcg<STRIDE, 16>(p, a, lcfg);
    case 32: return launch_tcg<STRIDE, 32>(p, a, lcfg);
    case 48: return launch_tcg<STRIDE, 48>(p, a, lcfg);
    case 64: return launch_tcg<STRIDE, 64>(p, a, lcfg);
    case 80: return launch_tcg<STRIDE, 80>(p, a, lcfg);
    case 96: return launch_tcg<STRIDE, 96>(p, a, lcfg);
    case 112: return launch_tcg<STRIDE, 112>(p, a, lcfg);
    case 128: return launch_tcg<STRIDE, 128>(p, a, lcfg);
    default: set_error("wgmma gather conv: no kernel instance for n_tile=%d", a.n_tile); return READ_ERR_UNSUPPORTED;
    }
}

int tcg_plan_launch(const TcgPlan *p, cudaStream_t st, int max_ctas)
{
    GArgs a = p->args;
    const long long total_tiles = (long long)a.tiles_x * a.tiles_y * a.B * a.n_tiles;
    if (total_tiles == 0) return READ_OK;
    long long grid = num_sms();
    if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
    if (grid > total_tiles) grid = total_tiles;
    a.pdl = g_tc_pdl ? 1 : 0;
    cudaLaunchAttribute lattr[1];
    lattr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    lattr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t lcfg{};
    lcfg.gridDim = dim3((unsigned)grid);
    lcfg.blockDim = dim3(G_THREADS);
    lcfg.dynamicSmemBytes = p->smem_bytes;
    lcfg.stream = st;
    lcfg.attrs = lattr;
    lcfg.numAttrs = a.pdl ? 1 : 0;
    const int rc = a.stride == 1 ? launch_tcg_n<1>(p, a, lcfg) : launch_tcg_n<2>(p, a, lcfg);
    if (rc != READ_OK) return rc;
    RB_LAUNCH_CHECK();
    return READ_OK;
}

void tcg_plan_destroy(TcgPlan *p) { delete p; }

int64_t tcg_weight_elems(int Cout, int Cin, int k)
{
    GGeom g;
    if (!g_geom(Cin, Cout, k, &g)) return -1;
    return (int64_t)g.kblocks * g.n_tile * g.n_tiles * G_KBLK;
}

int tcg_pack(const float *wf, const float *wm, int Cout, int Cin, int k, void *out, cudaStream_t st)
{
    GGeom g;
    if (!g_geom(Cin, Cout, k, &g)) {
        set_error("pack_tc_gather: unsupported channel counts %d -> %d", Cin, Cout);
        return READ_ERR_INVALID;
    }
    const long long total = (long long)g.kblocks * g.n_tile * g.n_tiles * G_KBLK;
    long long blocks = (total + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    pack_tcg_kernel<<<(unsigned)blocks, 256, 0, st>>>(wf, wm, Cout, Cin, k, g.kblocks, g.n_tile, g.n_tiles, (__nv_bfloat16 *)out);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb
