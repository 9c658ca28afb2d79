// Gated convolution as an implicit GEMM on the Hopper tensor cores (wgmma + TMA + mbarrier), sm_90a.
//
// One kernel computes  y = BN( A(conv_f(x)+b_f) * sigmoid(conv_m(x)+b_m) ) [+ residual]  (BasicConv,
// READ/models/unet.py:22-53) for stride-1 k x k and stride-2 3x3 / 4x4 convolutions over NHWC bf16 activations:
//
//   GEMM view   D[M = 128 output pixels (16 rows x 8 cols of one image), N = f|m channels] +=
//               A[M, K = one filter tap x CIN_BLK input channels] * B[N, K]
//   A operand   ONE TMA 4-D tile load {c, x, y, b} per tile and K chunk: the (16+k-1)-row x (8+k-1)-column halo tile, rows of
//               CIN_BLK bf16 with the matching 32/64/128-byte swizzle.  Every filter tap (ky, kx) reads its 128 pixel rows out of
//               that tile with ldmatrix (pixel (py + ky, px + kx) of the halo) into wgmma's register A operand, so the input is
//               fetched once per tile (x1.41 halo) and no im2col is ever materialised.  Pixels outside the image are ZERO-FILLED by
//               the TMA unit == the conv's zero padding (unet.py:29,36).
//   B operand   packed weights [tap][kchunk][n][CIN_BLK] bf16, conv_f and conv_m side by side in N so ONE accumulator tile
//               holds both gates of the same output channels; read by wgmma through K-major shared-memory descriptors.
//               When the whole layer fits (<= 144 KB: the C=32 and C=64 layers) the weights are loaded ONCE per CTA and stay
//               resident in shared memory; otherwise they stream through their own mbarrier ring.
//   D           fp32 in registers: two consumer warpgroups, each owning 64 pixels (8 rows) of the tile.
//   epilogue    bias, ELU, sigmoid gate, BN affine, residual add, bf16 pack (optionally a second output y*z for the following
//               FAM, unet.py:115) through an epilogue stage in shared memory: the producer TMA-loads the tile's residual / FAM
//               multiplier / add-in into the stage, each consumer warpgroup overwrites them in place with its 64 output pixels
//               and TMA-stores the result (clipped at the image edge).  Only the final NCHW fp32 layer stores from registers.
//
// Warp roles (288 threads, persistent over tiles): warps 0..7 = two consumer warpgroups (wgmma + epilogue), warp 8 = TMA
// producer, which runs ahead through the A (and streamed B) rings and the epilogue ring while the consumers compute.  Layers
// with N <= 64 whose weights, three A stages and two epilogue stages fit half the shared-memory budget run two CTAs per SM:
// one CTA's epilogue overlaps the other's MMAs.
//
// Stride 2 (3x3 / 4x4, pad 1): input column 2x + kx - 1 is an EVEN column for kx odd and an ODD one for kx even, so a stage
// holds four phase tiles E/O x E/O, each loaded by one TMA with traversal stride 2 in x and y (tile[j][i] = in(sx + 2i, sy + 2j),
// sx = 2*X0 for E, 2*X0 - 1 for O); tap (ky, kx) reads phase tile ((ky+1)&1, (kx+1)&1) at pixel offset (ky>>1, kx>>1).
#include "common.cuh"
#include "conv_common.cuh"
#include "ptx.cuh"
#include <cuda.h>
#include <mutex>
#include <new>

namespace rb {

constexpr int TC_TW = 8, TC_TH = 16;          // 128-pixel M tile: 16 rows of 8 pixels
constexpr int TC_THREADS = 288;               // two consumer warpgroups + one producer warp
constexpr int TC_PRODUCER_WARP = 8;
constexpr int TC_MAX_STAGES = 16;
// H100 shared memory: at most 227 KB per CTA, 228 KB per SM of which the hardware reserves 1 KB per resident CTA
constexpr uint32_t TC_SMEM_PER_CTA = 227 * 1024, TC_SMEM_PER_SM = 228 * 1024;
__host__ __device__ constexpr int tc_ctas_per_sm(int n_tile) { return n_tile <= 64 ? 2 : 1; }
constexpr uint32_t TC_RESIDENT_MAX = 144 * 1024;
constexpr int TC_E_STAGES = 2;                 // epilogue stages
// barrier slots (uint64 each): the A and B rings and the resident weights, then the full and empty barriers of a body's
// e_stages epilogue stages; the per-channel parameters follow the barriers
constexpr int BAR_AFULL = 0, BAR_AEMPTY = 16, BAR_BFULL = 32, BAR_BEMPTY = 48, BAR_BRES = 64;
struct TcBarSlots { int efull, eempty, params; };
__host__ __device__ constexpr TcBarSlots tc_bar_slots(int e_stages) { return {BAR_BRES + 2, BAR_BRES + 2 + e_stages, BAR_BRES + 2 + 2 * e_stages}; }
constexpr uint32_t TC_CONSUMER_WARPS = 8;

// activation tensor maps: one per source of a virtual concat (1x1 convs: torch.cat along channels, unet.py:88,105,263;
// a nearest-DOWN resampled source is a traversal-stride load of the full-resolution tensor)
// The epilogue's maps (NHWC outputs only): residual and out2_mul are loaded as the tile's 16 rows x 8 pixels, the add-in as the
// nearest-x2 source region of 8 rows x 4 pixels; out and out2 are stored per warpgroup, 8 rows x 8 pixels.  Channels come in
// blocks of at most 64 (128-byte rows, the widest swizzle).
struct TcMaps {
    CUtensorMap a[READ_MAX_SRC];
    CUtensorMap res, mul, add, out, out2;
};

struct TcArgs {
    int B, H, W, Cin, Cout, cout_pad;     // cout_pad > Cout only for the final (Cout <= 8, NCHW f32) layer
    int ksize, pad;
    int cin_blk, kchunks;
    int n_tile, n_tiles;
    int tiles_x, tiles_y;
    int a_stages, b_stages, b_resident;
    int halo_w;                            // smem tile width in pixels: TC_TW + ksize - 1 (stride 1) or TC_TW + 1 (stride 2)
    uint32_t a_tx_bytes;                   // bytes one tile load delivers
    uint32_t tile_bytes;                   // that rounded up to 1 KB; a_bytes = tile_bytes (stride 1) or 4 x tile_bytes (stride 2)
    int stride;                            // 1, or 2: four phase tiles (even / odd input columns x rows) per stage
    int n_src;                             // sources of the virtual concat (> 1 only for 1x1 convs)
    int src_kc_end[READ_MAX_SRC];          // K chunks [src_kc_end[s-1], src_kc_end[s]) come from source s
    int src_shift[READ_MAX_SRC];           // log2 of the source's nearest-down factor (coordinate multiplier)
    uint32_t a_bytes, b_bytes, b_region_off;   // halo stage bytes, one weight tile bytes, byte offset of the B region
    int pdl;                               // launched with programmatic stream serialization (griddepcontrol in the kernel)
    int ctas_per_sm;                       // 2: the layer fits half the shared-memory budget and its kernel instance two CTAs' registers
    int rev_total;                         // 0, or the number of work units: unit t is mapped to rev_total - 1 - t (read_conv_plan_set_tile_order)
    uint32_t e_bytes, e_region_off;        // one epilogue stage (out | out2 | add-in regions), byte offset of the epilogue ring
    uint32_t e_out2_off, e_add_off, e_tx_bytes;   // region offsets inside a stage, bytes the producer loads into one stage
    const float *bias_f, *bias_m, *scale, *shift;
    EpiArgs epi;
};

struct TileCoord {
    int nt, tx, ty, b;
};
__device__ __forceinline__ TileCoord decode_tile(int t, const TcArgs &a)
{
    if (a.rev_total) t = a.rev_total - 1 - t;
    TileCoord c;
    c.nt = t % a.n_tiles;
    int m = t / a.n_tiles;
    c.tx = m % a.tiles_x;
    m /= a.tiles_x;
    c.ty = m % a.tiles_y;
    c.b = m / a.tiles_y;
    return c;
}

// The issuer releases the epilogue stage e_pend once its previous TMA store has read it: the producer may refill it
__device__ __forceinline__ void release_epilogue_stage(bool issuer, int e_pend, uint32_t eempty0)
{
    if (issuer && e_pend >= 0) {
        bulk_wait_group_read<0>();
        mbar_arrive(eempty0 + 8 * e_pend);
    }
}

// Byte offset of channel c of pixel p in an epilogue region of P pixels: blocks of CB channels, each P rows of 2*CB bytes with
// the TMA swizzle of that row length.  Reads and writes in the accumulator layout (8 pixels x 4 channel pairs per warp access)
// touch 32 distinct banks.
template <int CB, int P>
__device__ __forceinline__ uint32_t epi_off(int p, int c)
{
    return (uint32_t)(c / CB) * (P * 2u * CB) + swz((uint32_t)p * (2u * CB) + (uint32_t)(c % CB) * 2u, 2u * CB);
}

// Epilogue of one warp's 16 pixels (tile rows r0, r0 + 1) from the accumulators (layout: conv_common.cuh, epilogue_tile) into
// the epilogue stage st: the out region [128 px][N/2 channels] (RAW: [128 px][N]) holds the residual when there is one and
// receives the output in place, the out2 region likewise holds out2_mul and receives out2, the add-in region [32 px][N] holds
// the nearest-x2 source of the tile.  The arithmetic is epilogue_tile's.
template <int N>
__device__ __forceinline__ void epilogue_smem(const float (&d)[N / 2], uint8_t *st, int lane, int r0, int nt, const float4 *par,
                                              const TcArgs &a)
{
    constexpr int HALF = N / 2, NJ = e_nj<N>();
    constexpr int CBA = N < 64 ? N : 64;                    // add-in channel block
    const EpiArgs &e = a.epi;
    const int q2 = 2 * (lane & 3), px = lane >> 2;
    auto ld = [&](uint32_t off) { return bf16x2_val(*reinterpret_cast<const uint32_t *>(st + off)); };
    auto stw = [&](uint32_t off, uint32_t v) { *reinterpret_cast<uint32_t *>(st + off) = v; };
    const float2 zero = make_float2(0.f, 0.f);
    if (e.raw) {
        // the out region holds the tile's residual when there is one (RAW 3x3: input gradient of a ResBlock, conv_bwd.cu)
        constexpr int CB = N < 64 ? N : 64;
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = r0 + i, c = 8 * j + q2;
                const float2 a2 = e.addin ? ld(a.e_add_off + epi_off<CBA, 32>((r >> 1) * (TC_TW / 2) + (px >> 1), c)) : zero;
                const uint32_t o = epi_off<CB, 128>(r * TC_TW + px, c);
                const float2 rs = e.residual ? ld(o) : zero;
                stw(o, bf16x2_bits(d[4 * j + 2 * i] + a2.x + rs.x, d[4 * j + 2 * i + 1] + a2.y + rs.y));
            }
        return;
    }
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = r0 + i, col = 8 * j + q2, co = nt * HALF + col;
            float2 fa = zero, ma = zero;
            if (e.addin) {
                const int pa = (r >> 1) * (TC_TW / 2) + (px >> 1);
                fa = ld(a.e_add_off + epi_off<CBA, 32>(pa, col));
                ma = ld(a.e_add_off + epi_off<CBA, 32>(pa, HALF + col));
            }
            const float f0 = d[4 * j + 2 * i] + fa.x, f1 = d[4 * j + 2 * i + 1] + fa.y;
            const float m0 = d[4 * (j + NJ) + 2 * i] + ma.x, m1 = d[4 * (j + NJ) + 2 * i + 1] + ma.y;
            const float4 p0 = par[co], p1 = par[co + 1];
            float y0, y1;
            if (e.elu) {
                y0 = gate_fast<true>(f0 + p0.x, m0 + p0.y, p0.z, p0.w);
                y1 = gate_fast<true>(f1 + p1.x, m1 + p1.y, p1.z, p1.w);
            } else {
                y0 = gate_fast<false>(f0 + p0.x, m0 + p0.y, p0.z, p0.w);
                y1 = gate_fast<false>(f1 + p1.x, m1 + p1.y, p1.z, p1.w);
            }
            const uint32_t o = epi_off<HALF, 128>(r * TC_TW + px, col);
            const float2 rs = e.residual ? ld(o) : zero;
            const uint32_t pk = bf16x2_bits(y0 + rs.x, y1 + rs.y);
            stw(o, pk);
            if (e.out2) {
                const float2 ys = bf16x2_val(pk);                // the stored (rounded) activation
                const float2 mm = ld(a.e_out2_off + o);
                stw(a.e_out2_off + o, bf16x2_bits(ys.x * mm.x, ys.y * mm.y));
            }
        }
}

// ------------------------------------------------------------------ the kernel
// KS = filter size, STR = stride, KKN = 16-element K steps per K chunk (cin_blk / 16), N = n_tile (wgmma N).  Filter size and
// stride are compile-time so that the tap loop unrolls into constant shared-memory offsets.
template <int KS, int STR, int KKN, int N>
__global__ void __launch_bounds__(TC_THREADS, tc_ctas_per_sm(N))
gated_conv_tc_kernel(const __grid_constant__ TcMaps tm, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ TcArgs a)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t smem_base = (s_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *smem_al = smem_raw + (smem_base - s_u32(smem_raw));

    constexpr int ntaps = KS * KS;
    constexpr TcBarSlots e_bars = tc_bar_slots(TC_E_STAGES);
    const uint32_t b_region = smem_base + a.b_region_off;
    const uint32_t e_region = smem_base + a.e_region_off;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_al + a.e_region_off + TC_E_STAGES * a.e_bytes);
    const uint32_t bar0 = s_u32(bars);
    const uint32_t afull0 = bar0 + 8 * BAR_AFULL, aempty0 = bar0 + 8 * BAR_AEMPTY;
    const uint32_t bfull0 = bar0 + 8 * BAR_BFULL, bempty0 = bar0 + 8 * BAR_BEMPTY, bres = bar0 + 8 * BAR_BRES;
    const uint32_t efull0 = bar0 + 8 * e_bars.efull, eempty0 = bar0 + 8 * e_bars.eempty;
    float4 *s_par = reinterpret_cast<float4 *>(bars + e_bars.params);

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    if (a.pdl) pdl_launch_dependents();
    for (int i = threadIdx.x; i < a.cout_pad; i += TC_THREADS)
        s_par[i] = i < a.Cout ? make_float4(a.bias_f[i], a.bias_m[i], a.scale[i], a.shift[i]) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (warp == TC_PRODUCER_WARP && lane == 0) {
        for (int i = 0; i < a.n_src; ++i) tma_prefetch_desc(&tm.a[i]);
        tma_prefetch_desc(&tmB);
        if (N > 16) {
            if (a.epi.residual) tma_prefetch_desc(&tm.res);
            if (a.epi.out2) tma_prefetch_desc(&tm.mul);
            if (a.epi.addin) tma_prefetch_desc(&tm.add);
        }
        for (int s = 0; s < TC_MAX_STAGES; ++s) {
            mbar_init(afull0 + 8 * s, 1);
            mbar_init(aempty0 + 8 * s, TC_CONSUMER_WARPS);
            mbar_init(bfull0 + 8 * s, 1);
            mbar_init(bempty0 + 8 * s, TC_CONSUMER_WARPS);
        }
        for (int s = 0; s < TC_E_STAGES; ++s) {
            mbar_init(efull0 + 8 * s, 1);
            mbar_init(eempty0 + 8 * s, 2);          // one arrival per consumer warpgroup
        }
        mbar_init(bres, 1);
        mbar_fence_init();
    }
    __syncthreads();

    const int total_tiles = a.tiles_x * a.tiles_y * a.B * a.n_tiles;   // < 2^31 (checked by the host)
    const int n_total = a.n_tile * a.n_tiles;

    if (warp == TC_PRODUCER_WARP) {
        // ===================== TMA producer (whole warp loops, one elected lane issues) =====================
        if (a.b_resident && elect_one()) {
            const int nb = ntaps * a.kchunks;
            mbar_arrive_expect_tx(bres, (uint32_t)nb * a.b_bytes);
            for (int i = 0; i < nb; ++i) tma_load_2d(&tmB, bres, b_region + (uint32_t)i * a.b_bytes, 0, i * n_total);
        }
        __syncwarp();
        if (a.pdl) pdl_wait();        // activations come from the previous kernel; the (static) weights above do not
        uint32_t as = 0, aph = 0, bs = 0, bph = 0, es = 0, eph = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const TileCoord tc_ = decode_tile(t, a);
            const int x0 = tc_.tx * TC_TW - a.pad, y0 = tc_.ty * TC_TH - a.pad;
            for (int kc = 0; kc < a.kchunks; ++kc) {
                mbar_wait(aempty0 + 8 * as, aph ^ 1u);
                if (elect_one()) {
                    const uint32_t full = afull0 + 8 * as, dst = smem_base + as * a.a_bytes;
                    if (STR == 1) {
                        mbar_arrive_expect_tx(full, a.a_tx_bytes);
                        // virtual concat (1x1, pad 0): chunk kc belongs to source si; a down-sampled source is read with
                        // traversal stride 2^shift from coordinate (x0, y0) << shift
                        int si = 0, kc0 = 0;
                        for (int q = 0; q < READ_MAX_SRC - 1; ++q)
                            if (q + 1 < a.n_src && kc >= a.src_kc_end[q]) { si = q + 1; kc0 = a.src_kc_end[q]; }
                        const int sh = a.src_shift[si];
                        tma_load_4d(&tm.a[si], full, dst, (kc - kc0) * a.cin_blk, x0 << sh, y0 << sh, tc_.b);
                    } else {
                        mbar_arrive_expect_tx(full, 4u * a.a_tx_bytes);
                        const int ex = 2 * tc_.tx * TC_TW, ey = 2 * tc_.ty * TC_TH;        // even-phase origin in the input
#pragma unroll
                        for (int ph4 = 0; ph4 < 4; ++ph4)
                            tma_load_4d(&tm.a[0], full, dst + (uint32_t)ph4 * a.tile_bytes, kc * a.cin_blk, ex - (ph4 & 1), ey - (ph4 >> 1), tc_.b);
                    }
                }
                __syncwarp();
                if (++as == (uint32_t)a.a_stages) { as = 0; aph ^= 1u; }
                if (!a.b_resident) {
                    for (int tap = 0; tap < ntaps; ++tap) {
                        mbar_wait(bempty0 + 8 * bs, bph ^ 1u);
                        if (elect_one()) {
                            mbar_arrive_expect_tx(bfull0 + 8 * bs, a.b_bytes);
                            tma_load_2d(&tmB, bfull0 + 8 * bs, b_region + bs * a.b_bytes, 0, (tap * a.kchunks + kc) * n_total + tc_.nt * a.n_tile);
                        }
                        __syncwarp();
                        if (++bs == (uint32_t)a.b_stages) { bs = 0; bph ^= 1u; }
                    }
                }
            }
            if (N > 16) {
                // the tile's epilogue operands, after its A chunks: a stage is freed only when the epilogue of the tile
                // after its own starts, and the next tile's A loads must not wait for that
                mbar_wait(eempty0 + 8 * es, eph ^ 1u);
                if (elect_one()) {
                    const uint32_t full = efull0 + 8 * es, dst = e_region + es * a.e_bytes;
                    mbar_arrive_expect_tx(full, a.e_tx_bytes);       // 0 bytes (a plain arrival) when the epilogue loads nothing
                    const int ex = tc_.tx * TC_TW, ey = tc_.ty * TC_TH, c0 = tc_.nt * (N / 2);
                    if (a.epi.residual) {
                        if (a.epi.raw) {             // RAW rows of N channels, in blocks of at most 64 like the stores
                            constexpr int CB = N < 64 ? N : 64;
                            for (int c = 0; c < N; c += CB) tma_load_4d(&tm.res, full, dst + 256u * c, tc_.nt * N + c, ex, ey, tc_.b);
                        } else {
                            tma_load_4d(&tm.res, full, dst, c0, ex, ey, tc_.b);
                        }
                    }
                    if (a.epi.out2) tma_load_4d(&tm.mul, full, dst + a.e_out2_off, c0, ex, ey, tc_.b);
                    if (a.epi.addin)
                        for (int c = 0; c < N; c += 64) tma_load_4d(&tm.add, full, dst + a.e_add_off + 64u * c, c, ex >> 1, ey >> 1, tc_.b);
                }
                __syncwarp();
                if (++es == (uint32_t)TC_E_STAGES) { es = 0; eph ^= 1u; }
            }
        }
        return;
    }

    // ===================== consumers: two warpgroups, 64 pixels (8 tile rows) each =====================
    const int wg = warp >> 2, wiw = warp & 3;
    constexpr uint32_t row_bytes = KKN * 32u;                  // cin_blk bf16
    // this lane's ldmatrix row (pixel of the tile) and 8-element half of the K step
    constexpr int HALO_W = STR == 1 ? TC_TW + KS - 1 : TC_TW + 1;     // halo tile width in pixels (== a.halo_w)
    const int lr = 64 * wg + 16 * wiw + (lane & 7) + 8 * ((lane >> 3) & 1);
    const uint32_t a_base = (uint32_t)((lr >> 3) * HALO_W + (lr & 7)) * row_bytes;   // tap (0, 0) of this lane's pixel
    const uint32_t khalf = (uint32_t)(lane >> 4) * 16u;
    if (a.pdl) pdl_wait();        // the outputs may still be read by earlier kernels
    if (a.b_resident) mbar_wait(bres, 0);
    uint32_t as = 0, aph = 0, bs = 0, bph = 0, es = 0, eph = 0;
    const bool issuer = wiw == 0 && lane == 0;      // issues the warpgroup's TMA stores and releases its epilogue stages
    int e_pend = -1;                               // stage whose stores the issuer has not yet seen read
    for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const TileCoord tc_ = decode_tile(t, a);
        float acc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        for (int kc = 0; kc < a.kchunks; ++kc) {
            mbar_wait(afull0 + 8 * as, aph);
            const uint32_t stage = smem_base + as * a.a_bytes;
            // A fragments of tap t+1 are loaded while the MMAs of tap t run: two register buffers, the tap loop fully unrolled
            uint32_t fr[2][KKN][4];
            auto load_a = [&](int tap, uint32_t (&f)[KKN][4]) {
                const int ky = tap / KS, kx = tap % KS;
                const uint32_t off = STR == 1
                    ? a_base + (uint32_t)(ky * HALO_W + kx) * row_bytes
                    : a_base + (uint32_t)((((ky + 1) & 1) << 1) | ((kx + 1) & 1)) * a.tile_bytes + (uint32_t)((ky >> 1) * HALO_W + (kx >> 1)) * row_bytes;
#pragma unroll
                for (int kk = 0; kk < KKN; ++kk) ldmatrix_x4(stage + swz(off + 32u * kk + khalf, row_bytes), f[kk]);
            };
            uint32_t prev_bs = 0;
            load_a(0, fr[0]);
#pragma unroll
            for (int tap = 0; tap < ntaps; ++tap) {
                uint32_t b_addr;
                if (a.b_resident) {
                    b_addr = b_region + (uint32_t)(tap * a.kchunks + kc) * a.b_bytes;
                } else {
                    mbar_wait(bfull0 + 8 * bs, bph);
                    b_addr = b_region + bs * a.b_bytes;
                }
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < KKN; ++kk) Wgmma<N>::mma(acc, fr[tap & 1][kk], wgmma_desc(b_addr + 32u * kk, row_bytes), 1u);
                wgmma_commit();
                wgmma_wait<1>();          // tap t-1 retired: its A buffer and (streamed) B stage are free
                if (!a.b_resident) {
                    if (tap > 0) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bempty0 + 8 * prev_bs);
                    }
                    prev_bs = bs;
                    if (++bs == (uint32_t)a.b_stages) { bs = 0; bph ^= 1u; }
                }
                if (tap + 1 < ntaps) load_a(tap + 1, fr[(tap + 1) & 1]);
            }
            wgmma_wait<0>();
            wgmma_fence_acc(acc);
            __syncwarp();
            if (lane == 0) {
                if (!a.b_resident) mbar_arrive(bempty0 + 8 * prev_bs);
                mbar_arrive(aempty0 + 8 * as);
            }
            if (++as == (uint32_t)a.a_stages) { as = 0; aph ^= 1u; }
        }
        if constexpr (N == 16) {     // the final layer (Cout <= 8): fp32 NCHW, stored from the registers
            EpiArgs e = a.epi;
            e.par = s_par;
            const int x0 = tc_.tx * TC_TW + (lane >> 2), y0 = tc_.ty * TC_TH + 8 * wg + 2 * wiw;
            const int xs[2] = {x0, x0}, ys[2] = {y0, y0 + 1};
            const bool in[2] = {x0 < a.W && y0 < a.H, x0 < a.W && y0 + 1 < a.H};
            epilogue_tile<N>(acc, lane, tc_.b, ys, xs, in, tc_.nt, e);
        } else {
            release_epilogue_stage(issuer, e_pend, eempty0);
            mbar_wait(efull0 + 8 * es, eph);
            epilogue_smem<N>(acc, smem_al + a.e_region_off + es * a.e_bytes, lane, 8 * wg + 2 * wiw, tc_.nt, s_par, a);
            fence_proxy_async_smem();
            named_bar_sync(1 + wg, 128);
            if (issuer) {
                const uint32_t st = e_region + es * a.e_bytes;
                const int ex = tc_.tx * TC_TW, ey = tc_.ty * TC_TH + 8 * wg;
                if (ey < a.H) {          // the TMA unit clips the rest of the box at the image edge
                    if (a.epi.raw) {
                        constexpr int CB = N < 64 ? N : 64;
#pragma unroll
                        for (int c = 0; c < N; c += CB) tma_store_4d(&tm.out, st + 256u * c + 128u * CB * wg, tc_.nt * N + c, ex, ey, tc_.b);
                    } else {
                        tma_store_4d(&tm.out, st + 64u * N * wg, tc_.nt * (N / 2), ex, ey, tc_.b);
                        if (a.epi.out2) tma_store_4d(&tm.out2, st + a.e_out2_off + 64u * N * wg, tc_.nt * (N / 2), ex, ey, tc_.b);
                    }
                }
                bulk_commit_group();
            }
            e_pend = (int)es;
            if (++es == (uint32_t)TC_E_STAGES) { es = 0; eph ^= 1u; }
        }
    }
    if (issuer) bulk_wait_group<0>();     // the stores have read shared memory and written the outputs before the CTA retires
}

// ------------------------------------------------------------------ weight-stationary body: 3x3 stride-1, 32 -> 32 channels
// At 32 channels the kernel above spends more shared-memory time moving the 128 x 288 activation operand through ldmatrix than
// its MMAs take.  Here the roles swap: the weights (64 rows = 32 conv_f + 32 conv_m channels, K = 9 taps x 32 channels) are
// wgmma's register A operand, loaded ONCE per CTA (72 registers per thread), and the 128 pixels of a tile are N, read by the
// tensor core straight out of the halo tile: 18 m64n128k16 per tile and no A loads.
//   halo tile   no swizzle, [8-channel chunk][18 rows][10 px][16 B], one 4-D TMA per chunk (box {8, 10, 18, 1}, chunk stride
//               padded to 128 B).  Every core matrix (8 px x 16 B) is 128 contiguous bytes, and tap (ky, kx) is the start
//               address + ky * row + kx * 16 B: LBO = the chunk stride, SBO = the row stride.
//   A rows      the ldmatrix row addresses pick the packed weight rows so that warp w's rows 0..7 are conv_f and rows 8..15
//               conv_m of the SAME channels 8w .. 8w+7: each thread then holds both gates of one channel for 32 pixels (tile
//               row j = accumulator group j, pixels 2 (l & 3), + 1), and the weight packing is the other body's.
//   epilogue    ws_epilogue_rows: epilogue_smem's arithmetic per element; the residual comes in with ldmatrix.trans and the
//               output goes back with stmatrix.trans (8 channels x 8 pixels per block) into the 64-byte-swizzled NHWC stage,
//               stored by one TMA (ws_store_block).
// Warp roles: the producer warp as above; each consumer warpgroup takes whole tiles (the CTA's even / odd ones), so one
// warpgroup's epilogue runs under the other's MMAs.  One CTA per SM (72 + 64 registers per thread are live across the MMAs).
constexpr int WS_E_STAGES = 4;                 // two per consumer warpgroup: tile k uses stage k % 4
// one halo row of one 8-channel chunk, and the chunk, of a TW x TH-pixel tile (TMA destinations are 128 B aligned)
__host__ __device__ constexpr uint32_t ws_row_bytes(int tw) { return (uint32_t)(tw + 2) * 16u; }
__host__ __device__ constexpr uint32_t ws_chunk_bytes(int tw, int th) { return ((uint32_t)(th + 2) * ws_row_bytes(tw) + 127u) & ~127u; }
constexpr uint32_t WS_ROW_BYTES = ws_row_bytes(TC_TW);
constexpr uint32_t WS_CHUNK_BYTES = ws_chunk_bytes(TC_TW, TC_TH);
constexpr uint32_t WS_BLOCK_BYTES = 128u * 32u * 2u;   // one 32-channel block of an epilogue stage

// The shared memory of a weight-stationary body with E epilogue stages, from its 1 KB aligned base (offsets and sizes:
// tc_plan_create): halo ring | resident weights | epilogue ring | barriers | per-channel parameters
template <int E>
struct WsSmem {
    uint32_t base, b_region, e_region;
    uint32_t afull0, aempty0, bfull0, bempty0, bres, efull0, eempty0;
    float4 *par;
    __device__ __forceinline__ explicit WsSmem(const TcArgs &a)
    {
        extern __shared__ uint8_t smem_raw[];
        base = (s_u32(smem_raw) + 1023u) & ~1023u;
        b_region = base + a.b_region_off;
        e_region = base + a.e_region_off;
        uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + (base - s_u32(smem_raw)) + a.e_region_off + E * a.e_bytes);
        const uint32_t bar0 = s_u32(bars);
        afull0 = bar0 + 8 * BAR_AFULL, aempty0 = bar0 + 8 * BAR_AEMPTY, bres = bar0 + 8 * BAR_BRES;
        bfull0 = bar0 + 8 * BAR_BFULL, bempty0 = bar0 + 8 * BAR_BEMPTY;
        efull0 = bar0 + 8 * tc_bar_slots(E).efull, eempty0 = bar0 + 8 * tc_bar_slots(E).eempty;
        par = reinterpret_cast<float4 *>(bars + tc_bar_slots(E).params);
    }
};

// Prologue of the role-swapped bodies: per-channel parameters, descriptor prefetch, and the barriers, with a_arrivals per
// halo stage (the warps that read it; with STREAMED weights also per weight stage) and e_arrivals per epilogue stage (the
// warpgroups that store from it).
template <int E, bool STREAMED = false>
__device__ __forceinline__ void ws_prologue(const WsSmem<E> &sm, const TcMaps &tm, const CUtensorMap &tmB, const TcArgs &a,
                                            uint32_t a_arrivals, uint32_t e_arrivals)
{
    if (a.pdl) pdl_launch_dependents();
    for (int i = threadIdx.x; i < a.Cout; i += TC_THREADS) sm.par[i] = make_float4(a.bias_f[i], a.bias_m[i], a.scale[i], a.shift[i]);
    if (threadIdx.x == 32 * TC_PRODUCER_WARP) {
        tma_prefetch_desc(&tm.a[0]);
        tma_prefetch_desc(&tmB);
        if (a.epi.residual) tma_prefetch_desc(&tm.res);
        for (int s = 0; s < a.a_stages; ++s) {
            mbar_init(sm.afull0 + 8 * s, 1);
            mbar_init(sm.aempty0 + 8 * s, a_arrivals);
        }
        if (STREAMED)
            for (int s = 0; s < a.b_stages; ++s) {
                mbar_init(sm.bfull0 + 8 * s, 1);
                mbar_init(sm.bempty0 + 8 * s, a_arrivals);
            }
        for (int s = 0; s < E; ++s) {
            mbar_init(sm.efull0 + 8 * s, 1);
            mbar_init(sm.eempty0 + 8 * s, e_arrivals);
        }
        mbar_init(sm.bres, 1);
        mbar_fence_init();
    }
    __syncthreads();
}

// Producer: the halo of tile tc (TW x TH pixels from (x0, y0)) into the next stage (as, aph) of the halo ring, as C / 8
// unswizzled 8-channel chunks of input channels c0 .. c0 + C - 1 from pixel (x0 - 1, y0 - 1)
template <int C, int E, int TW = TC_TW, int TH = TC_TH>
__device__ __forceinline__ void ws_load_halo(const WsSmem<E> &sm, const TcMaps &tm, const TcArgs &a, const TileCoord &tc,
                                             uint32_t &as, uint32_t &aph, int c0 = 0)
{
    mbar_wait(sm.aempty0 + 8 * as, aph ^ 1u);
    if (elect_one()) {
        const uint32_t full = sm.afull0 + 8 * as, dst = sm.base + as * a.a_bytes;
        mbar_arrive_expect_tx(full, a.a_tx_bytes);
#pragma unroll
        for (int c = 0; c < C / 8; ++c)
            tma_load_4d(&tm.a[0], full, dst + (uint32_t)c * ws_chunk_bytes(TW, TH), c0 + 8 * c, tc.tx * TW - 1, tc.ty * TH - 1, tc.b);
    }
    __syncwarp();
    if (++as == (uint32_t)a.a_stages) { as = 0; aph ^= 1u; }
}

// Producer: the residual of tile tc (TW x TH pixels), output channels c0 .. c0 + C - 1, into the next epilogue stage (es, eph),
// as C / 32 boxes of 32 channels, block h at h * TW * TH * 64 bytes; a plain arrival without a residual
template <int C, int E, int TW = TC_TW, int TH = TC_TH>
__device__ __forceinline__ void ws_load_residual(const WsSmem<E> &sm, const TcMaps &tm, const TcArgs &a, const TileCoord &tc,
                                                 uint32_t &es, uint32_t &eph, int c0 = 0)
{
    mbar_wait(sm.eempty0 + 8 * es, eph ^ 1u);
    if (elect_one()) {
        const uint32_t full = sm.efull0 + 8 * es, dst = sm.e_region + es * a.e_bytes;
        mbar_arrive_expect_tx(full, a.e_tx_bytes);
        if (a.epi.residual)
#pragma unroll
            for (int h = 0; h < C / 32; ++h)
                tma_load_4d(&tm.res, full, dst + (uint32_t)h * (TW * TH * 64u), c0 + 32 * h, tc.tx * TW, tc.ty * TH, tc.b);
    }
    __syncwarp();
    if (++es == (uint32_t)E) { es = 0; eph ^= 1u; }
}

// Consumer: NR (4 or 1) tile rows j0 .. of the epilogue, pixels x0 .. x0 + 7 of each, in place in the warpgroup's
// 64-byte-swizzled [TH rows][TW px][32 ch] block st of an epilogue stage.  acc holds both gates of this thread's channel
// (parameters par) for two pixels of every 8-pixel row of the block: row j at acc[4 j ..].  The residual comes in with
// ldmatrix.trans, the arithmetic is epilogue_smem's per element, and the bf16 output goes back with stmatrix.trans.
template <int NA = 64, int TW = TC_TW, int NR = 4>
__device__ __forceinline__ void ws_epilogue_rows(const float (&acc)[NA], int j0, uint32_t st, float4 par, const EpiArgs &e, int x0 = 0)
{
    static_assert(NR == 4 || NR == 1, "ldmatrix / stmatrix of four or one 8x8 blocks");
    const int lane = threadIdx.x & 31, wiw = (threadIdx.x >> 5) & 3;
    // this lane's ldmatrix / stmatrix row: pixel x0 + (lane & 7) of tile row j0 + (lane >> 3), channels 8 wiw ..
    const uint32_t e_row = ((uint32_t)(lane >> 3) * TW + (lane & 7)) * 64u + 16u * wiw;
    const uint32_t addr = st + swz(e_row + ((uint32_t)j0 * TW + (uint32_t)x0) * 64u, 64u);
    uint32_t rv[NR] = {};
    if (e.residual) {
        if constexpr (NR == 4) ldmatrix_x4_trans(addr, rv);
        else ldmatrix_x1_trans(addr, rv);
    }
    uint32_t ov[NR];
#pragma unroll
    for (int i = 0; i < NR; ++i) {
        const int j = j0 + i;
        const float f0 = acc[4 * j] + par.x, f1 = acc[4 * j + 1] + par.x;
        const float m0 = acc[4 * j + 2] + par.y, m1 = acc[4 * j + 3] + par.y;
        float y0, y1;
        if (e.elu) {
            y0 = gate_fast<true>(f0, m0, par.z, par.w);
            y1 = gate_fast<true>(f1, m1, par.z, par.w);
        } else {
            y0 = gate_fast<false>(f0, m0, par.z, par.w);
            y1 = gate_fast<false>(f1, m1, par.z, par.w);
        }
        const float2 rs = bf16x2_val(rv[i]);             // zero without a residual
        ov[i] = bf16x2_bits(y0 + rs.x, y1 + rs.y);
    }
    if constexpr (NR == 4) stmatrix_x4_trans(addr, ov);
    else stmatrix_x1_trans(addr, ov);
}

// Consumer: the warpgroup's finished block st, output channels c0 .. c0 + 31 of the TW x TH-pixel tile t, made visible to the
// TMA unit and stored by the issuer (the TMA unit clips the box at the image edge)
template <int TW = TC_TW, int TH = TC_TH>
__device__ __forceinline__ void ws_store_block(const TcMaps &tm, const TcArgs &a, uint32_t st, int c0, int t, int wg, bool issuer)
{
    fence_proxy_async_smem();
    named_bar_sync(1 + wg, 128);
    if (issuer) {
        const TileCoord tc = decode_tile(t, a);
        tma_store_4d(&tm.out, st, c0, tc.tx * TW, tc.ty * TH, tc.b);
        bulk_commit_group();
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1)
gated_conv_tc_ws_kernel(const __grid_constant__ TcMaps tm, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ TcArgs a)
{
    const WsSmem<WS_E_STAGES> sm(a);
    ws_prologue(sm, tm, tmB, a, 4, 1);      // a tile's halo and epilogue stages belong to the one warpgroup that takes it
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int total_tiles = a.tiles_x * a.tiles_y * a.B;   // one n-tile

    if (warp == TC_PRODUCER_WARP) {
        if (elect_one()) {
            mbar_arrive_expect_tx(sm.bres, 9u * a.b_bytes);
            for (int i = 0; i < 9; ++i) tma_load_2d(&tmB, sm.bres, sm.b_region + (uint32_t)i * a.b_bytes, 0, i * a.n_tile);
        }
        __syncwarp();
        if (a.pdl) pdl_wait();
        uint32_t as = 0, aph = 0, es = 0, eph = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const TileCoord tc_ = decode_tile(t, a);
            ws_load_halo<32>(sm, tm, a, tc_, as, aph);
            ws_load_residual<32>(sm, tm, a, tc_, es, eph);
        }
        return;
    }

    const int wg = warp >> 2, wiw = warp & 3;
    if (a.pdl) pdl_wait();        // the outputs may still be read by earlier kernels
    mbar_wait(sm.bres, 0);
    uint32_t wa[9][2][4];
    {
        // packed row n: conv_f channel n (n < 32), conv_m channel n - 32; 64-byte swizzled rows of 32 channels
        const uint32_t n = 8u * wiw + (lane & 7) + 32u * ((lane >> 3) & 1);
#pragma unroll
        for (int tap = 0; tap < 9; ++tap)
#pragma unroll
            for (int kk = 0; kk < 2; ++kk)
                ldmatrix_x4(sm.b_region + (uint32_t)tap * a.b_bytes + swz(n * 64u + 32u * kk + 16u * (lane >> 4), 64u), wa[tap][kk]);
    }
    const float4 par = sm.par[8 * wiw + (lane >> 2)];
    const bool issuer = wiw == 0 && lane == 0;      // issues the warpgroup's TMA stores and releases its epilogue stages
    int e_pend = -1;
    uint32_t as = (uint32_t)wg, aph = 0;            // a_stages >= 2
    for (int k = wg, t = blockIdx.x + wg * gridDim.x; t < total_tiles; k += 2, t += 2 * gridDim.x) {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        mbar_wait(sm.afull0 + 8 * as, aph);
        const uint32_t stage = sm.base + as * a.a_bytes;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap)
#pragma unroll
            for (int kk = 0; kk < 2; ++kk)
                Wgmma<128>::mma(acc, wa[tap][kk],
                                wgmma_desc_noswz(stage + (uint32_t)(tap / 3) * WS_ROW_BYTES + (uint32_t)(tap % 3) * 16u + 2u * kk * WS_CHUNK_BYTES,
                                                 WS_CHUNK_BYTES, WS_ROW_BYTES),
                                1u);
        wgmma_commit();
        release_epilogue_stage(issuer, e_pend, sm.eempty0);
        wgmma_wait<0>();
        wgmma_fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(sm.aempty0 + 8 * as);
        as += 2;
        if (as >= (uint32_t)a.a_stages) { as -= (uint32_t)a.a_stages; aph ^= 1u; }

        const int es = k % WS_E_STAGES;
        mbar_wait(sm.efull0 + 8 * es, (uint32_t)(k / WS_E_STAGES) & 1u);
        const uint32_t st = sm.e_region + es * a.e_bytes;
#pragma unroll
        for (int j0 = 0; j0 < TC_TH; j0 += 4) ws_epilogue_rows(acc, j0, st, par, a.epi);
        ws_store_block(tm, a, st, 0, t, wg, issuer);
        e_pend = es;
    }
    if (issuer) bulk_wait_group<0>();
}

// ------------------------------------------------------------------ weight-stationary body: 3x3 stride-1, 64 -> 64 channels
// The same role swap at 64 channels: D[128 weight rows = 64 conv_f + 64 conv_m][128 pixels] += W[128, K = 9 taps x 64] X[128, K].
// The weights (144 KB) no longer fit in registers, so they are wgmma's SHARED-MEMORY A operand, resident for the CTA's life.
//   A rows      the producer loads each tap's packed [128 rows: f0..63, m0..63][64 K] tile as sixteen 8-row boxes (one 1 KB
//               128-byte-swizzle atom each) and lays them out f-group g, m-group g, f-group g + 1, ...: warpgroup h's 64 rows of a
//               tap are the 8 KB at h * 8 KB, and warp w's 16 rows are conv_f then conv_m of channels 32h + 8w .. + 7, so each
//               thread holds both gates of one channel for 32 pixels as in the 32-channel body.  The packing is unchanged.
//   B (pixels)  the 32-channel body's unswizzled halo tile with eight 8-channel chunks (23 KB per stage); K step kk starts at
//               chunk 2 kk, tap (ky, kx) adds ky * row + kx * 16 B.
//   overlap     both warpgroups work on the same tile (warpgroup h: output channels 32h .. 32h + 31, 36 m64n128k16 per tile)
//               and each keeps TWO accumulator sets: tile t's epilogue runs under tile t + 1's MMAs.  Those are issued in four
//               groups between the epilogue's four 4-row blocks: issued as one batch of 36, they held the warps back until
//               most of them had run (0.143 ms per layer against 0.113 ms interleaved, H100 80GB HBM3 at 700 W).  The tile
//               loop is unrolled by two so the set of each tile is known at compile time.
//   epilogue    as in the 32-channel body; warpgroup h owns the [128 px][32 ch] 64-byte-swizzled block h of the epilogue stage
//               and stores it with its own TMA store.
// Shared memory: 144 KB weights + 2 halo stages + 2 epilogue stages of 16 KB + barriers and parameters, one CTA per SM.
constexpr uint32_t WS64_TAP_BYTES = 128u * 64u * 2u;     // one tap's packed weight tile

__global__ void __launch_bounds__(TC_THREADS, 1)
gated_conv_tc_ws64_kernel(const __grid_constant__ TcMaps tm, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ TcArgs a)
{
    const WsSmem<TC_E_STAGES> sm(a);
    ws_prologue(sm, tm, tmB, a, TC_CONSUMER_WARPS, 2);      // both warpgroups read every halo stage and store from every epilogue stage
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int total_tiles = a.tiles_x * a.tiles_y * a.B;   // one n-tile

    if (warp == TC_PRODUCER_WARP) {
        if (elect_one()) {
            mbar_arrive_expect_tx(sm.bres, 9u * WS64_TAP_BYTES);
            for (int tap = 0; tap < 9; ++tap)
                for (int g = 0; g < 8; ++g) {
                    const uint32_t dst = sm.b_region + (uint32_t)tap * WS64_TAP_BYTES + (uint32_t)g * 2048u;
                    tma_load_2d(&tmB, sm.bres, dst, 0, tap * 128 + 8 * g);                // conv_f channels 8g .. 8g + 7
                    tma_load_2d(&tmB, sm.bres, dst + 1024u, 0, tap * 128 + 64 + 8 * g);   // conv_m, the same channels
                }
        }
        __syncwarp();
        if (a.pdl) pdl_wait();
        uint32_t as = 0, aph = 0, es = 0, eph = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const TileCoord tc_ = decode_tile(t, a);
            ws_load_halo<64>(sm, tm, a, tc_, as, aph);
            ws_load_residual<64>(sm, tm, a, tc_, es, eph);
        }
        return;
    }

    const int wg = warp >> 2, wiw = warp & 3;
    if (a.pdl) pdl_wait();        // the outputs may still be read by earlier kernels
    mbar_wait(sm.bres, 0);
    const float4 par = sm.par[32 * wg + 8 * wiw + (lane >> 2)];
    const bool issuer = wiw == 0 && lane == 0;      // issues the warpgroup's TMA stores and releases its epilogue stages
    int e_pend = -1;
    uint32_t as = 0, aph = 0, es = 0, eph = 0;       // halo and epilogue stages of tile t

    // The MMAs of taps [tap0, tap1) of one tile, committed as one group.  The weight rows' base (this warpgroup's 64 rows of tap
    // 0) comes through a shuffle of wg: warp-uniform to the compiler, so the descriptors live in uniform registers (otherwise
    // ptxas serialises every wgmma), and computed per call, so the compiler does not hoist 36 loop-invariant descriptors out of
    // the tile loop and spill them.
    auto mma_taps = [&](float (&acc)[64], uint32_t stage, int tap0, int tap1) {
        const uint32_t w_base = sm.b_region + (uint32_t)__shfl_sync(0xffffffffu, wg, 0) * 8192u;
        wgmma_fence();
#pragma unroll
        for (int tap = tap0; tap < tap1; ++tap)
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
                wgmma_ss_m64n128k16(acc, wgmma_desc(w_base + (uint32_t)tap * WS64_TAP_BYTES + 32u * kk, 128u),
                                    wgmma_desc_noswz(stage + (uint32_t)(tap / 3) * WS_ROW_BYTES + (uint32_t)(tap % 3) * 16u +
                                                         2u * kk * WS_CHUNK_BYTES,
                                                     WS_CHUNK_BYTES, WS_ROW_BYTES),
                                    1u);
        wgmma_commit();
    };
    auto zero = [](float (&acc)[64]) {
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    };
    // tile t's MMAs (into cur) are in flight: issue tile t + gridDim.x's into nxt and run tile t's epilogue under them.  The
    // next tile's MMAs go out in four groups (taps 0-2, 3-4, 5-6, 7-8) between the epilogue's four 4-row blocks, so the epilogue
    // does not wait behind the issue of all 36.
    int t = blockIdx.x;
    auto step = [&](float (&cur)[64], float (&nxt)[64]) {
        const int tn = t + (int)gridDim.x;
        uint32_t as_n = as + 1u, aph_n = aph;
        if (as_n == (uint32_t)a.a_stages) { as_n = 0; aph_n ^= 1u; }
        const uint32_t stage_n = sm.base + as_n * a.a_bytes;
        if (tn < total_tiles) {
            mbar_wait(sm.afull0 + 8 * as_n, aph_n);
            zero(nxt);
            mma_taps(nxt, stage_n, 0, 3);
        }
        release_epilogue_stage(issuer, e_pend, sm.eempty0);
        if (tn < total_tiles) wgmma_wait<1>();      // tile t's MMAs have retired
        else wgmma_wait<0>();
        wgmma_fence_acc(cur);
        __syncwarp();
        if (lane == 0) mbar_arrive(sm.aempty0 + 8 * as);
        as = as_n;
        aph = aph_n;

        mbar_wait(sm.efull0 + 8 * es, eph);
        const uint32_t st = sm.e_region + es * a.e_bytes + (uint32_t)wg * WS_BLOCK_BYTES;
#pragma unroll
        for (int j0 = 0; j0 < TC_TH; j0 += 4) {
            ws_epilogue_rows(cur, j0, st, par, a.epi);
            if (j0 < TC_TH - 4 && tn < total_tiles) mma_taps(nxt, stage_n, 3 + j0 / 2, 5 + j0 / 2);
        }
        ws_store_block(tm, a, st, 32 * wg, t, wg, issuer);
        e_pend = (int)es;
        if (++es == (uint32_t)TC_E_STAGES) { es = 0; eph ^= 1u; }
        t = tn;
        return t < total_tiles;
    };

    float acc0[64], acc1[64];
    if (t < total_tiles) {
        mbar_wait(sm.afull0, 0);
        zero(acc0);
        mma_taps(acc0, sm.base, 0, 9);
        while (step(acc0, acc1) && step(acc1, acc0)) {
        }
        wgmma_wait<0>();
    }
    if (issuer) bulk_wait_group<0>();
}

// ------------------------------------------------------------------ role-swapped body with streamed weights: 3x3 stride-1, C -> C, C = 128 / 256
// The 64-channel body's role swap for the layers whose weights (576 KB / 2.25 MB) do not fit shared memory.  The general body
// streams an n-tile's whole weight set out of L2 for every 128-pixel tile, so each weight byte feeds 128 pixels; here a work
// unit is (16 x R-pixel tile, n-tile of 64 output channels), and each weight byte feeds 16 R = 256 or 272 pixels:
//   D[128 weight rows = 64 conv_f + 64 conv_m][16 R pixels] += W[128, K = 9 taps x C] X[16 R, K]
//   A (weights)  streamed through the weight ring, one stage per (K chunk of 64 channels, tap): the n-tile's packed 128 x 64 tile
//                loaded as sixteen 8-row boxes in the 64-channel body's order (f-group g, m-group g, f-group g + 1, ...), so
//                warpgroup h reads its 64 rows (conv_f and conv_m of channels 32h .. 32h + 31) at h * 8 KB.  The packing is
//                the general body's.
//   B (pixels)   one halo stage per K chunk: [8-channel chunk][R + 2 rows][18 px][16 B], unswizzled.  Each K step is two
//                m64n(8R)k16 with the same A descriptor, for pixel columns 0..7 and 8..15 of the tile (128 B apart): SBO = the
//                halo row (288 B), LBO = the chunk stride, tap (ky, kx) at + ky * 288 + kx * 16 B.
//   K order      K chunk, tap, 16-wide step: the general body's, so each output sums its products in the same order.
//   accumulators one set of 2 x 4R per thread (both gates of one channel, two pixels of every 8-pixel row of the tile).
//   epilogue     ws_epilogue_rows / ws_store_block over [R rows][16 px][32 ch] blocks; it does not overlap the MMAs (the
//                producer keeps loading the next unit's halo and weights meanwhile).
// R = 16 or 17 is chosen per layer by tc_wss_rows.  One CTA per SM, at most 168 registers per thread: nine warps spread over
// the SM's four register-file quarters put three warps in one of them.  The ring sizes are compile-time so that every stage
// index and phase is a bit field of one running count.
constexpr int WSS_TW = 16;                                 // tile width in pixels
constexpr int WSS_A_STAGES = 2, WSS_B_STAGES = 4;          // halo stages, weight stages
constexpr uint32_t WSS_STAGE_BYTES = 128u * 64u * 2u;     // one weight stage: 128 packed rows of one tap and K chunk

template <int R>
__global__ void __launch_bounds__(TC_THREADS, 1)
gated_conv_tc_wss_kernel(const __grid_constant__ TcMaps tm, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ TcArgs a)
{
    constexpr uint32_t ROW = ws_row_bytes(WSS_TW), CHUNK = ws_chunk_bytes(WSS_TW, R);
    constexpr uint32_t BLOCK = WSS_TW * R * 64u;        // one warpgroup's [R][16 px][32 ch] block of an epilogue stage
    const WsSmem<TC_E_STAGES> sm(a);
    ws_prologue<TC_E_STAGES, true>(sm, tm, tmB, a, TC_CONSUMER_WARPS, 2);   // both warpgroups read every stage
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int total = a.tiles_x * a.tiles_y * a.B * a.n_tiles;
    const int n_total = a.n_tile * a.n_tiles;

    if (warp == TC_PRODUCER_WARP) {
        if (a.pdl) pdl_wait();
        uint32_t as = 0, aph = 0, es = 0, eph = 0, nb = 0;
        for (int t = blockIdx.x; t < total; t += gridDim.x) {
            const TileCoord tc_ = decode_tile(t, a);
            for (int kc = 0; kc < a.kchunks; ++kc) {
                ws_load_halo<64, TC_E_STAGES, WSS_TW, R>(sm, tm, a, tc_, as, aph, 64 * kc);
                for (int tap = 0; tap < 9; ++tap, ++nb) {
                    const uint32_t bs = nb % WSS_B_STAGES;
                    mbar_wait(sm.bempty0 + 8 * bs, ((nb / WSS_B_STAGES) & 1u) ^ 1u);
                    if (elect_one()) {
                        const uint32_t full = sm.bfull0 + 8 * bs, dst = sm.b_region + bs * WSS_STAGE_BYTES;
                        const int row0 = (tap * a.kchunks + kc) * n_total + tc_.nt * a.n_tile;
                        mbar_arrive_expect_tx(full, WSS_STAGE_BYTES);
                        for (int g = 0; g < 8; ++g) {
                            tma_load_2d(&tmB, full, dst + (uint32_t)g * 2048u, 0, row0 + 8 * g);                // conv_f channels 8g ..
                            tma_load_2d(&tmB, full, dst + (uint32_t)g * 2048u + 1024u, 0, row0 + 64 + 8 * g);   // conv_m, the same
                        }
                    }
                    __syncwarp();
                }
            }
            ws_load_residual<64, TC_E_STAGES, WSS_TW, R>(sm, tm, a, tc_, es, eph, tc_.nt * 64);
        }
        return;
    }

    const int wg = warp >> 2, wiw = warp & 3;
    if (a.pdl) pdl_wait();        // the outputs may still be read by earlier kernels
    const bool issuer = wiw == 0 && lane == 0;      // issues the warpgroup's TMA stores and releases its epilogue stages
    // halo and weight stages consumed so far: stage = count % stages, phase = (count / stages) & 1
    uint32_t na = 0, nb = 0;
    auto release = [&](uint32_t bar) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar);
    };
    for (int k = 0, t = blockIdx.x; t < total; ++k, t += gridDim.x) {
        const TileCoord tc_ = decode_tile(t, a);
        float acc[2][4 * R];
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int i = 0; i < 4 * R; ++i) acc[c][i] = 0.f;
        // a weight stage is released once the MMA group after the one that read it has been issued and the one that read it
        // has retired (wgmma_wait<1>); a halo stage likewise after its last tap's group
        for (int kc = 0; kc < a.kchunks; ++kc, ++na) {
            mbar_wait(sm.afull0 + 8 * (na % WSS_A_STAGES), (na / WSS_A_STAGES) & 1u);
            const uint32_t halo = sm.base + (na % WSS_A_STAGES) * a.a_bytes;
#pragma unroll
            for (int tap = 0; tap < 9; ++tap, ++nb) {
                const uint32_t bs = nb % WSS_B_STAGES;
                mbar_wait(sm.bfull0 + 8 * bs, (nb / WSS_B_STAGES) & 1u);
                // warpgroup-uniform weight base through a shuffle, recomputed per group (see gated_conv_tc_ws64_kernel)
                const uint32_t w_base = sm.b_region + bs * WSS_STAGE_BYTES + (uint32_t)__shfl_sync(0xffffffffu, wg, 0) * 8192u;
                const uint32_t x_base = halo + (uint32_t)(tap / 3) * ROW + (uint32_t)(tap % 3) * 16u;
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        const uint64_t wd = wgmma_desc(w_base + 32u * kk, 128u);
                        const uint64_t xd = wgmma_desc_noswz(x_base + 2u * kk * CHUNK + 128u * c, CHUNK, ROW);
                        if constexpr (R == 16) wgmma_ss_m64n128k16(acc[c], wd, xd, 1u);
                        else wgmma_ss_m64n136k16(acc[c], wd, xd, 1u);
                    }
                wgmma_commit();
                wgmma_wait<1>();
                if (tap > 0 || kc > 0) release(sm.bempty0 + 8 * ((nb - 1u) % WSS_B_STAGES));
                if (tap == 0 && kc > 0) release(sm.aempty0 + 8 * ((na - 1u) % WSS_A_STAGES));
            }
        }
        const uint32_t es = (uint32_t)k % TC_E_STAGES;
        release_epilogue_stage(issuer, k > 0 ? (int)((uint32_t)(k - 1) % TC_E_STAGES) : -1, sm.eempty0);
        wgmma_wait<0>();
#pragma unroll
        for (int c = 0; c < 2; ++c) wgmma_fence_acc(acc[c]);
        release(sm.bempty0 + 8 * ((nb - 1u) % WSS_B_STAGES));
        release(sm.aempty0 + 8 * ((na - 1u) % WSS_A_STAGES));

        const float4 par = sm.par[tc_.nt * 64 + 32 * wg + 8 * wiw + (lane >> 2)];
        mbar_wait(sm.efull0 + 8 * es, ((uint32_t)k / TC_E_STAGES) & 1u);
        const uint32_t st = sm.e_region + es * a.e_bytes + (uint32_t)wg * BLOCK;
#pragma unroll
        for (int c = 0; c < 2; ++c) {
#pragma unroll
            for (int j0 = 0; j0 + 4 <= R; j0 += 4) ws_epilogue_rows<4 * R, WSS_TW, 4>(acc[c], j0, st, par, a.epi, 8 * c);
#pragma unroll
            for (int j = R / 4 * 4; j < R; ++j) ws_epilogue_rows<4 * R, WSS_TW, 1>(acc[c], j, st, par, a.epi, 8 * c);
        }
        ws_store_block<WSS_TW, R>(tm, a, st, tc_.nt * 64 + 32 * wg, t, wg, issuer);
    }
    if (issuer) bulk_wait_group<0>();
}

// ------------------------------------------------------------------ weight packing
// out[((tap*kchunks + kc) * n_total + n) * cin_blk + kk],  n -> (tile nt, f|m half, channel)
__global__ void pack_tc_kernel(const float *__restrict__ wf, const float *__restrict__ wm, int Cout, int cout_pad, int Cin,
                               int k, int cin_blk, int n_tile, __nv_bfloat16 *__restrict__ out)
{
    const int kchunks = (Cin + cin_blk - 1) / cin_blk;       // Cin 8 with 16-channel K steps: the upper half of every row is zero
    const int n_total = 2 * cout_pad;
    const int half = n_tile / 2;
    const long long total = (long long)k * k * kchunks * n_total * cin_blk;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int kk = (int)(i % cin_blk);
        long long r = i / cin_blk;
        const int n = (int)(r % n_total);
        r /= n_total;
        const int kc = (int)(r % kchunks);
        const int tap = (int)(r / kchunks);
        const int nt = n / n_tile, rr = n % n_tile;
        const bool is_m = rr >= half;
        const int co = nt * half + (rr % half);
        const int c = kc * cin_blk + kk;
        const int ky = tap / k, kx = tap % k;
        const float *w = is_m ? wm : wf;
        out[i] = __float2bfloat16_rn((co < Cout && c < Cin) ? w[(((long long)co * Cin + c) * k + ky) * k + kx] : 0.f);
    }
}

// Input gradient of a stride-1 3x3 conv pair (conv_f, conv_m: [Cout][Cin][3][3]) as a RAW plan of the same kernel: a 3x3 conv of
// [df | dm] (2*Cout channels, in the column order of the forward RAW output: blocks of n_tile_f columns, conv_f half then conv_m
// half) with the filters flipped in space and transposed, dX[n] = sum_{tap, c} dfm[c] * w[o(c)][n][2-ky][2-kx].  The plan's N
// columns are the Cin input channels in order, so its RAW output is dX itself.  k = 1 packs the input gradient of the input
// channels c0 .. c0 + cn - 1 of a 1x1 conv (one source of a concat) as a RAW 1x1 plan with n_out >= cn columns, the columns
// beyond cn zero filters.
__global__ void pack_tc_dgrad_kernel(const float *__restrict__ wf, const float *__restrict__ wm, int Cout, int Cin, int k, int half_f,
                                     int cin_blk, int kchunks, int c0, int cn, int n_out, __nv_bfloat16 *__restrict__ out)
{
    const long long total = (long long)k * k * kchunks * n_out * cin_blk;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int kk = (int)(i % cin_blk);
        long long r = i / cin_blk;
        const int n = (int)(r % n_out);
        r /= n_out;
        const int kc = (int)(r % kchunks);
        const int tap = (int)(r / kchunks);
        const int c = kc * cin_blk + kk;                         // column of [df | dm]
        const int rr = c % (2 * half_f);
        const int o = (c / (2 * half_f)) * half_f + rr % half_f;
        const float *w = rr >= half_f ? wm : wf;
        const int ky = k - 1 - tap / k, kx = k - 1 - tap % k;
        out[i] = __float2bfloat16_rn(c < 2 * Cout && n < cn ? w[(((long long)o * Cin + c0 + n) * k + ky) * k + kx] : 0.f);
    }
}

// ------------------------------------------------------------------ host side
struct TcGeom {
    int cin_blk, kchunks, n_tile, n_tiles, cout_pad;
};
// K-chunk granularity of a layer: the widest block (64 or 32 channels) that divides EVERY source of a virtual concat
static int desc_chan_gran(const read_conv_desc &d)
{
    int gsrc = d.Cin;
    for (int i = 0; i < d.n_src && d.n_src > 1; ++i)
        if (d.src[i].C % 64 != 0) gsrc = 32;
    return gsrc;
}

static bool tc_geom(int Cin, int Cout, int stride, TcGeom *g, int chan_gran = 64)
{
    int cin_blk;
    // stride 2 keeps four phase tiles per stage: 32-channel K chunks keep a 3-stage ring within shared memory
    if (Cin % 64 == 0 && stride == 1 && chan_gran % 64 == 0) cin_blk = 64;
    else if (Cin % 32 == 0) cin_blk = 32;
    // 8- and 16-channel inputs (the descriptor pyramid itself: feat_extract.0, SCM*.main.0; SCM2.main.1): ONE 16-channel K step,
    // 32-byte rows with SWIZZLE_32B.  An 8-channel tensor is loaded with a 16-channel box: the TMA unit zero-fills the
    // out-of-range half of every row, the packed weights carry zeros there - no padded copy of the input exists anywhere.
    else if ((Cin == 8 || Cin == 16) && stride == 1) cin_blk = 16;
    else return false;
    int cout_pad = Cout;
    if (Cout <= 8) cout_pad = 8;                 // final layer: N = 16 (f|m of 8 padded channels)
    else if (Cout % 16 != 0) return false;
    const int n_total = 2 * cout_pad;
    const int n_tile = n_total <= 128 ? n_total : 128;   // accumulators in registers: 64 fp32 per thread
    if (n_total % n_tile != 0) return false;
    if (cout_pad > 8 && (n_tile / 2) % 16 != 0) return false;
    if (cin_blk == 16 && (n_total / n_tile != 1 || cout_pad <= 8 || !(cout_pad == 16 || cout_pad == 32 || cout_pad == 64))) return false;
    if (g) *g = TcGeom{cin_blk, (Cin + cin_blk - 1) / cin_blk, n_tile, n_total / n_tile, cout_pad};
    return true;
}

bool tc_supported(const read_conv_desc &d)
{
    if (d.act_dtype != READ_ACT_BF16) return false;
    if (d.mul != nullptr || d.n_src < 1 || d.n_src > READ_MAX_SRC) return false;
    if (d.n_src == 1) {
        if (d.src[0].mode != READ_SRC_IDENTITY) return false;
    } else {
        // virtual concat: 1x1 convs whose sources are identity or nearest-DOWN by a power of two, 32-channel granular
        if (d.k != 1 || d.stride != 1) return false;
        int csum = 0;
        for (int i = 0; i < d.n_src; ++i) {
            const read_src &sv = d.src[i];
            if (sv.mode == READ_SRC_NEAREST_DOWN) {
                if (sv.factor < 2 || (sv.factor & (sv.factor - 1)) != 0) return false;
            } else if (sv.mode != READ_SRC_IDENTITY) {
                return false;
            }
            if (sv.C % 32 != 0) return false;
            csum += sv.C;
        }
        if (csum != d.Cin) return false;
    }
    if (d.stride == 1) {
        if (!(d.k == 3 || d.k == 1) || d.pad != (d.k - 1) / 2) return false;
        if (d.Hin != d.Hout || d.Win != d.Wout) return false;
    } else if (d.stride == 2) {            // 3x3 / 4x4, pad 1, even input: four phase tiles (see the kernel)
        if (!(d.k == 3 || d.k == 4) || d.pad != 1) return false;
        if (d.Hin != 2 * d.Hout || d.Win != 2 * d.Wout) return false;
    } else {
        return false;
    }
    if (d.Cout <= 8) {
        if (d.out_mode != READ_OUT_NCHW_F32 || d.residual || d.out2) return false;   // final layer only
    } else if (d.out_mode != READ_OUT_NHWC && d.out_mode != READ_OUT_RAW_NHWC) {
        return false;
    }
    if (d.out_mode == READ_OUT_RAW_NHWC && d.k == 3 && d.stride == 1) {
        // accumulators of a 3x3 stride-1 conv over one tensor, optionally plus a residual of the output's [B, H, W, 2*Cout]
        // shape: the training path's recomputed [f | m] and ResBlock input gradients (read_b200/blocks.py)
        if (d.n_src != 1 || d.addin != nullptr || d.out2 != nullptr) return false;
        if ((long long)d.B * d.Hout * d.Wout * 2 * d.Cout >= (1ll << 31)) return false;
    } else if (d.out_mode == READ_OUT_RAW_NHWC && d.stride == 2) {
        // the recomputed [f | m] of a stride-2 3x3 / 4x4 conv (bf16 training): no epilogue operands
        if (d.residual != nullptr || d.addin != nullptr || d.out2 != nullptr) return false;
        if ((long long)d.B * d.Hout * d.Wout * 2 * d.Cout >= (1ll << 31)) return false;
    } else if (d.out_mode == READ_OUT_RAW_NHWC || d.addin != nullptr) {
        // terms of a 1x1 conv over a multi-resolution concat: served by the lean epilogue (Cout 16 / 32 / 64)
        if (d.k != 1 || d.stride != 1) return false;
        if (!(d.Cout == 16 || d.Cout == 32 || d.Cout == 64)) return false;
        if (d.out_mode == READ_OUT_RAW_NHWC && (d.residual || d.out2)) return false;
        if ((long long)d.B * d.Hout * d.Wout * 2 * d.Cout >= (1ll << 31)) return false;
    }
    TcGeom g;
    if (!tc_geom(d.Cin, d.Cout, d.stride, &g, desc_chan_gran(d))) return false;
    for (int i = 0; i < d.n_src && d.n_src > 1; ++i)
        if (d.src[i].C % g.cin_blk != 0) return false;       // K chunks may not straddle two sources
    return true;
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_tiled()
{
    static PFN_encodeTiled fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    });
    return fn;
}

struct TcPlan {
    TcMaps tmA;
    CUtensorMap tmB;
    TcArgs args;
    size_t smem_bytes;
    int reverse;
    int ws;                                // 0, or the channel count of a role-swapped layer (tc_ws_layer): 32 runs
                                           // gated_conv_tc_ws_kernel, 64 gated_conv_tc_ws64_kernel, 128 and 256
                                           // gated_conv_tc_wss_kernel<tile_h>
    int tile_h;                            // output tile rows: TC_TH, or R of gated_conv_tc_wss_kernel<R>
};

// The layers of the role-swapped bodies: 3x3 stride-1 C -> C gated convs, C = 32 or 64 (weight-stationary) or 128 or 256
// (streamed weights), with an NHWC output and at most a residual
static bool tc_ws_layer(const read_conv_desc &d)
{
    return d.k == 3 && d.stride == 1 && (d.Cin == 32 || d.Cin == 64 || d.Cin == 128 || d.Cin == 256) && d.Cout == d.Cin &&
           d.n_src == 1 && d.out_mode == READ_OUT_NHWC && d.out2 == nullptr && d.addin == nullptr;
}

// Tile rows R of a streamed-weight role-swapped layer (gated_conv_tc_wss_kernel<R>, R = 16 or 17): the fewest pixel slots on
// the busiest CTA, ceil(units / SMs) x 16 R, and on a tie the fewer halo rows loaded
static int tc_wss_rows(const read_conv_desc &d, int n_tiles)
{
    const long long ctas = num_sms(), tiles_x = (d.Wout + WSS_TW - 1) / WSS_TW;
    int best = 0;
    long long best_slots = 0, best_halo = 0;
    for (int r = 16; r <= 17; ++r) {
        const long long tiles_y = (d.Hout + r - 1) / r, units = tiles_x * tiles_y * d.B * n_tiles;
        const long long slots = (units + ctas - 1) / ctas * WSS_TW * r, halo = tiles_y * (r + 2);
        if (!best || slots < best_slots || (slots == best_slots && halo < best_halo)) {
            best = r;
            best_slots = slots;
            best_halo = halo;
        }
    }
    return best;
}

// The plan values that depend on the kernel body, for a layer whose weights, like its activations, have the swizzle sw of
// their K chunk.  The role-swapped bodies read the halo as unswizzled 8-channel chunks and load the residual and store the
// output as 32-channel blocks of whole tiles; from 64 channels they load their weights as 8-row boxes, one swizzle atom each,
// to interleave conv_f and conv_m, and from 128 channels their tiles are 16 pixels wide and tc_wss_rows high.
struct TcBodyLayout {
    int ws;                                // TcPlan::ws
    int tile_w, tile_h;                    // pixels of the output tile
    int halo_c;                            // channels of one halo box
    CUtensorMapSwizzle halo_sw;
    int w_rows;                            // rows of one weight box
    int epi_c, out_rows;                   // channels of the output and residual boxes, rows of the output box
    uint32_t tile_bytes;                   // TcArgs::tile_bytes, 0: the halo tile's bytes
    int e_stages;                          // epilogue stages
};
static TcBodyLayout tc_body_layout(const read_conv_desc &d, const TcGeom &g, CUtensorMapSwizzle sw)
{
    const int oc = d.out_mode == READ_OUT_RAW_NHWC ? g.n_tile : g.n_tile / 2;     // channels of one output pixel in the tile
    TcBodyLayout L{0, TC_TW, TC_TH, g.cin_blk, sw, g.n_tile, oc < 64 ? oc : 64, TC_TH / 2, 0, TC_E_STAGES};
    if (tc_ws_layer(d)) {
        L.ws = d.Cin;
        if (d.Cin >= 128) {
            L.tile_w = WSS_TW;
            L.tile_h = tc_wss_rows(d, g.n_tiles);
        }
        L.halo_c = 8;
        L.halo_sw = CU_TENSOR_MAP_SWIZZLE_NONE;
        if (d.Cin >= 64) L.w_rows = 8;
        L.epi_c = 32;
        L.out_rows = L.tile_h;
        L.tile_bytes = (uint32_t)(g.cin_blk / 8) * ws_chunk_bytes(L.tile_w, L.tile_h);
        if (d.Cin == 32) L.e_stages = WS_E_STAGES;
    }
    return L;
}

int tc_plan_create(const read_conv_desc &d, TcPlan **out)
{
    TcGeom g;
    if (!tc_supported(d) || !tc_geom(d.Cin, d.Cout, d.stride, &g, desc_chan_gran(d))) {
        set_error("wgmma conv: unsupported layer");
        return READ_ERR_UNSUPPORTED;
    }
    PFN_encodeTiled enc = get_encode_tiled();
    if (!enc) {
        set_error("wgmma conv: cuTensorMapEncodeTiled not available from the driver");
        return READ_ERR_CUDA;
    }
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(d.w_tc) & 127) == 0, "wgmma conv: packed weights must be 128B aligned");
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(d.out) & 15) == 0, "wgmma conv: output must be 16B aligned");
    RB_CHECK_ARG(d.residual == nullptr || (reinterpret_cast<uintptr_t>(d.residual) & 15) == 0, "wgmma conv: residual must be 16B aligned");
    RB_CHECK_ARG(d.addin == nullptr || (reinterpret_cast<uintptr_t>(d.addin) & 15) == 0, "wgmma conv: addin must be 16B aligned");
    RB_CHECK_ARG(d.out2 == nullptr || ((reinterpret_cast<uintptr_t>(d.out2) | reinterpret_cast<uintptr_t>(d.out2_mul)) & 15) == 0,
                 "wgmma conv: out2 and out2_mul must be 16B aligned");
    const CUtensorMapSwizzle sw = g.cin_blk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : (g.cin_blk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    const TcBodyLayout L = tc_body_layout(d, g, sw);
    const long long tiles = (long long)((d.Wout + L.tile_w - 1) / L.tile_w) * ((d.Hout + L.tile_h - 1) / L.tile_h) * d.B * g.n_tiles;
    RB_CHECK_ARG(tiles < (1ll << 31), "wgmma conv: too many tiles");
    TcPlan *p = new (std::nothrow) TcPlan{};
    RB_CHECK_ARG(p != nullptr, "wgmma conv: out of host memory");

    const bool s2 = d.stride == 2;
    const int halo_rows = s2 ? L.tile_h + 1 : L.tile_h + d.k - 1;
    const int halo_w = s2 ? L.tile_w + 1 : L.tile_w + d.k - 1;
    const uint32_t a_tx_bytes = (uint32_t)halo_rows * halo_w * g.cin_blk * 2u;
    p->ws = L.ws;
    for (int si = 0; si < d.n_src; ++si) {   // activations: dims {C, W, H, B}; box = one halo tile (all filter taps)
        const read_src &sv = d.src[si];
        const unsigned f = (d.n_src > 1 && sv.mode == READ_SRC_NEAREST_DOWN) ? (unsigned)sv.factor : (s2 ? 2u : 1u);
        cuuint64_t dims[4] = {(cuuint64_t)sv.C, (cuuint64_t)sv.W, (cuuint64_t)sv.H, (cuuint64_t)d.B};
        cuuint64_t strides[3] = {(cuuint64_t)sv.C * 2, (cuuint64_t)sv.W * sv.C * 2, (cuuint64_t)sv.H * sv.W * sv.C * 2};
        // traversal stride f in x and y (conv stride 2, or a nearest-down source): the box spans (n-1)*f+1 input
        // elements and delivers n of them
        cuuint32_t box[4] = {(cuuint32_t)L.halo_c, (cuuint32_t)((halo_w - 1) * f + 1), (cuuint32_t)((halo_rows - 1) * f + 1), 1};
        cuuint32_t estr[4] = {1, f, f, 1};
        CUresult r = enc(&p->tmA.a[si], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(sv.ptr), dims, strides, box,
                         estr, CU_TENSOR_MAP_INTERLEAVE_NONE, L.halo_sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            set_error("wgmma conv: cuTensorMapEncodeTiled(activations, source %d) failed with %d", si, (int)r);
            delete p;
            return READ_ERR_CUDA;
        }
    }
    for (int si = d.n_src; si < READ_MAX_SRC; ++si) p->tmA.a[si] = p->tmA.a[0];
    {   // weights: dims {cin_blk, taps * kchunks * n_total}
        const cuuint64_t rows = (cuuint64_t)d.k * d.k * g.kchunks * 2 * g.cout_pad;
        cuuint64_t dims[2] = {(cuuint64_t)g.cin_blk, rows};
        cuuint64_t strides[1] = {(cuuint64_t)g.cin_blk * 2};
        cuuint32_t box[2] = {(cuuint32_t)g.cin_blk, (cuuint32_t)L.w_rows};
        cuuint32_t estr[2] = {1, 1};
        CUresult r = enc(&p->tmB, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(d.w_tc), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            set_error("wgmma conv: cuTensorMapEncodeTiled(weights) failed with %d", (int)r);
            delete p;
            return READ_ERR_CUDA;
        }
    }
    // epilogue maps, NHWC bf16 {C, W, H, B}; boxes of at most 64 channels with the swizzle of their row length
    const bool nchw = d.out_mode == READ_OUT_NCHW_F32, raw = d.out_mode == READ_OUT_RAW_NHWC;
    auto enc_epi = [&](CUtensorMap *m, const void *ptr, int C, int W, int H, int bc, int bw, int bh, const char *what) {
        cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)d.B};
        cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
        cuuint32_t box[4] = {(cuuint32_t)bc, (cuuint32_t)bw, (cuuint32_t)bh, 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        const CUtensorMapSwizzle esw = bc == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (bc == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
        CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(ptr), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, esw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) set_error("wgmma conv: cuTensorMapEncodeTiled(%s) failed with %d", what, (int)r);
        return r == CUDA_SUCCESS;
    };
    const int half = g.n_tile / 2;
    if (!nchw) {
        const int out_c = raw ? 2 * d.Cout : d.Cout, acb = g.n_tile < 64 ? g.n_tile : 64;     // out_c: also the residual's
        bool ok = enc_epi(&p->tmA.out, d.out, out_c, d.Wout, d.Hout, L.epi_c, L.tile_w, L.out_rows, "out");
        if (ok && d.out2) ok = enc_epi(&p->tmA.out2, d.out2, d.Cout, d.Wout, d.Hout, half, TC_TW, TC_TH / 2, "out2");
        if (ok && d.out2) ok = enc_epi(&p->tmA.mul, d.out2_mul, d.Cout, d.Wout, d.Hout, half, TC_TW, TC_TH, "out2_mul");
        if (ok && d.residual) ok = enc_epi(&p->tmA.res, d.residual, out_c, d.Wout, d.Hout, L.epi_c, L.tile_w, L.tile_h, "residual");
        if (ok && d.addin) ok = enc_epi(&p->tmA.add, d.addin, g.n_tile, d.addin_W, d.addin_H, acb, TC_TW / 2, TC_TH / 2, "addin");
        if (!ok) {
            delete p;
            return READ_ERR_CUDA;
        }
    }
    TcArgs &a = p->args;
    a.B = d.B; a.H = d.Hout; a.W = d.Wout; a.Cin = d.Cin; a.Cout = d.Cout; a.cout_pad = g.cout_pad;
    a.ksize = d.k; a.pad = d.pad;
    a.cin_blk = g.cin_blk; a.kchunks = g.kchunks; a.n_tile = g.n_tile; a.n_tiles = g.n_tiles;
    a.tiles_x = (d.Wout + L.tile_w - 1) / L.tile_w;
    a.tiles_y = (d.Hout + L.tile_h - 1) / L.tile_h;
    p->tile_h = L.tile_h;
    a.halo_w = halo_w;
    a.stride = d.stride;
    a.n_src = d.n_src;
    {
        int kc = 0;
        for (int si = 0; si < READ_MAX_SRC; ++si) {
            int sh = 0;
            if (si < d.n_src) {
                kc += d.src[si].C / g.cin_blk;
                if (d.n_src > 1 && d.src[si].mode == READ_SRC_NEAREST_DOWN)
                    while ((1 << sh) < d.src[si].factor) ++sh;
            } else {
                kc = 1 << 30;
            }
            a.src_kc_end[si] = kc;
            a.src_shift[si] = sh;
        }
    }
    a.a_tx_bytes = a_tx_bytes;
    a.tile_bytes = ((L.tile_bytes ? L.tile_bytes : a_tx_bytes) + 1023u) & ~1023u;   // 1 KB aligned (swizzle patterns are address based)
    a.a_bytes = s2 ? 4u * a.tile_bytes : a.tile_bytes;
    a.b_bytes = (uint32_t)g.n_tile * g.cin_blk * 2u;
    const uint32_t total_b = (uint32_t)(d.k * d.k * g.kchunks) * a.b_bytes;
    // epilogue stage: out region (the tile's pixels x its output channels), out2 region, add-in region (32 pixels x N);
    // every region is a multiple of 1 KB, so each keeps the 1 KB alignment of the swizzle patterns
    if (!nchw) {
        const uint32_t out_b = (uint32_t)(L.tile_w * L.tile_h) * (raw ? 2u : 1u) * (uint32_t)g.n_tile;
        const uint32_t out2_b = d.out2 ? 128u * (uint32_t)g.n_tile : 0u, add_b = d.addin ? 64u * (uint32_t)g.n_tile : 0u;
        a.e_out2_off = out_b;
        a.e_add_off = out_b + out2_b;
        a.e_bytes = out_b + out2_b + add_b;
        a.e_tx_bytes = (d.residual ? out_b : 0u) + out2_b + add_b;
    }
    const uint32_t e_ring = (uint32_t)L.e_stages * a.e_bytes;
    // the rings get what a CTA may have minus the alignment pad, barriers and per-channel parameters (smem_bytes below)
    const uint32_t fixed = 1024 + 8 * tc_bar_slots(L.e_stages).params + 16 * (uint32_t)g.cout_pad + 64;
    const uint32_t budget_2 = TC_SMEM_PER_SM / 2 - 1024 - fixed, budget_1 = TC_SMEM_PER_CTA - fixed;
    // two CTAs per SM when the kernel instance allows it and the layer keeps resident weights, the epilogue ring and >= 3 A
    // stages in half of the SM
    a.ctas_per_sm = (!p->ws && tc_ctas_per_sm(g.n_tile) > 1 && g.n_tiles == 1 && total_b <= TC_RESIDENT_MAX &&
                     total_b + e_ring + 3 * a.a_bytes <= budget_2) ? 2 : 1;
    const uint32_t budget = a.ctas_per_sm > 1 ? budget_2 : budget_1;
    a.b_resident = (g.n_tiles == 1 && total_b <= TC_RESIDENT_MAX && total_b + e_ring + 2 * a.a_bytes <= budget) ? 1 : 0;
    uint32_t b_region_bytes;
    if (p->ws >= 128) {
        // streamed-weight role swap: two halo stages, four 16 KB weight stages and the epilogue ring; at 256 channels and
        // R = 17 two 44 KB halo stages, two 34 KB epilogue stages and 5.6 KB of alignment pad, barriers and parameters,
        // 225.6 KB of the 227 KB a CTA may have
        a.a_stages = WSS_A_STAGES;
        a.b_stages = WSS_B_STAGES;
        b_region_bytes = (uint32_t)a.b_stages * a.b_bytes;
        if (a.a_stages * a.a_bytes + b_region_bytes + e_ring > budget) {
            set_error("wgmma conv: streamed-weight role-swapped layer does not fit shared memory (%u B needed)",
                      a.a_stages * a.a_bytes + b_region_bytes + e_ring + fixed);
            delete p;
            return READ_ERR_UNSUPPORTED;
        }
    } else if (a.b_resident) {
        int st = (int)((budget - total_b - e_ring) / a.a_bytes);
        a.a_stages = st > TC_MAX_STAGES ? TC_MAX_STAGES : st;
        a.b_stages = 0;
        b_region_bytes = total_b;
    } else {
        a.a_stages = 3;
        if (3 * a.a_bytes + e_ring + 2 * a.b_bytes > budget) {
            set_error("wgmma conv: layer does not fit shared memory (A stage %u B, B tile %u B, epilogue stage %u B)", a.a_bytes,
                      a.b_bytes, a.e_bytes);
            delete p;
            return READ_ERR_UNSUPPORTED;
        }
        int st = (int)((budget - 3 * a.a_bytes - e_ring) / a.b_bytes);
        a.b_stages = st > TC_MAX_STAGES ? TC_MAX_STAGES : st;
        b_region_bytes = (uint32_t)a.b_stages * a.b_bytes;
    }
    // the weight-stationary bodies rely on both.  At 64 channels: 144 KB of weights, two 23 KB halo stages, two 16 KB epilogue
    // stages and about 2.7 KB of alignment pad, barriers and parameters, 224.7 KB of the 227 KB a CTA may have
    if (p->ws && p->ws < 128 && (!a.b_resident || a.a_stages < 2)) {
        set_error("wgmma conv: weight-stationary layer without resident weights or two A stages (%u B of shared memory needed)",
                  total_b + e_ring + 2 * a.a_bytes + fixed);
        delete p;
        return READ_ERR_UNSUPPORTED;
    }
    a.b_region_off = (uint32_t)a.a_stages * a.a_bytes;
    a.e_region_off = a.b_region_off + b_region_bytes;
    a.bias_f = d.bias_f; a.bias_m = d.bias_m; a.scale = d.bn_scale; a.shift = d.bn_shift;
    EpiArgs &e = a.epi;
    e.H = d.Hout; e.W = d.Wout; e.Cout = d.Cout;
    e.elu = d.elu;
    e.raw = d.out_mode == READ_OUT_RAW_NHWC ? 1 : 0;
    e.nchw = d.out_mode == READ_OUT_NCHW_F32 ? 1 : 0;
    e.par = nullptr;
    e.residual = static_cast<const __nv_bfloat16 *>(d.residual);
    e.out2_mul = static_cast<const __nv_bfloat16 *>(d.out2_mul);
    e.addin = static_cast<const __nv_bfloat16 *>(d.addin);
    e.out = d.out;
    e.out2 = static_cast<__nv_bfloat16 *>(d.out2);
    e.addin_H = d.addin_H; e.addin_W = d.addin_W;
    p->smem_bytes = (size_t)a.e_region_off + e_ring + fixed;
    *out = p;
    return READ_OK;
}

int g_tc_pdl = 1;         // programmatic dependent launch between consecutive conv kernels (read_set_option "tc_pdl")

typedef void (*TcKernel)(TcMaps, CUtensorMap, TcArgs);

static int launch_tc(TcKernel kernel, const TcPlan *p, const TcArgs &a, cudaLaunchConfig_t &lcfg)
{
    RB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_bytes));
    RB_CUDA(cudaLaunchKernelEx(&lcfg, kernel, p->tmA, p->tmB, a));
    return READ_OK;
}

template <int KS, int STR>
static int launch_tc_kn(const TcPlan *p, const TcArgs &a, cudaLaunchConfig_t &lcfg)
{
    const int kkn = a.cin_blk / 16;
#define RB_TC_N(KKN_)                                                                       \
    switch (a.n_tile) {                                                                     \
    case 16: return launch_tc(gated_conv_tc_kernel<KS, STR, KKN_, 16>, p, a, lcfg);         \
    case 32: return launch_tc(gated_conv_tc_kernel<KS, STR, KKN_, 32>, p, a, lcfg);         \
    case 64: return launch_tc(gated_conv_tc_kernel<KS, STR, KKN_, 64>, p, a, lcfg);         \
    case 128: return launch_tc(gated_conv_tc_kernel<KS, STR, KKN_, 128>, p, a, lcfg);       \
    default: break;                                                                         \
    }
    if (kkn == 1) { RB_TC_N(1) }
    else if (kkn == 2) { RB_TC_N(2) }
    else if (kkn == 4) { RB_TC_N(4) }
#undef RB_TC_N
    set_error("wgmma conv: no kernel instance for cin_blk=%d n_tile=%d", a.cin_blk, a.n_tile);
    return READ_ERR_UNSUPPORTED;
}

int tc_plan_launch(const TcPlan *p, cudaStream_t st, int max_ctas)
{
    TcArgs a = p->args;
    a.pdl = g_tc_pdl ? 1 : 0;
    const long long total_tiles = (long long)a.tiles_x * a.tiles_y * a.B * a.n_tiles;
    if (total_tiles == 0) return READ_OK;
    a.rev_total = p->reverse ? (int)total_tiles : 0;
    long long grid = (long long)num_sms() * a.ctas_per_sm;
    if (max_ctas > 0 && grid > max_ctas) grid = max_ctas;
    if (grid > total_tiles) grid = total_tiles;
    // cudaLaunchKernelEx with programmatic stream serialization: the kernel may be scheduled while its predecessor in the
    // stream drains; it calls griddepcontrol.wait before touching anything an earlier kernel produced (ptx.cuh: pdl_wait)
    cudaLaunchAttribute lattr[1];
    lattr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    lattr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t lcfg{};
    lcfg.gridDim = dim3((unsigned)grid);
    lcfg.blockDim = dim3(TC_THREADS);
    lcfg.dynamicSmemBytes = p->smem_bytes;
    lcfg.stream = st;
    lcfg.attrs = lattr;
    lcfg.numAttrs = a.pdl ? 1 : 0;
    int rc;
    if (p->ws == 32) rc = launch_tc(gated_conv_tc_ws_kernel, p, a, lcfg);
    else if (p->ws == 64) rc = launch_tc(gated_conv_tc_ws64_kernel, p, a, lcfg);
    else if (p->ws >= 128 && p->tile_h == 16) rc = launch_tc(gated_conv_tc_wss_kernel<16>, p, a, lcfg);
    else if (p->ws >= 128 && p->tile_h == 17) rc = launch_tc(gated_conv_tc_wss_kernel<17>, p, a, lcfg);
    else if (a.stride == 1 && a.ksize == 1) rc = launch_tc_kn<1, 1>(p, a, lcfg);
    else if (a.stride == 1 && a.ksize == 3) rc = launch_tc_kn<3, 1>(p, a, lcfg);
    else if (a.stride == 2 && a.ksize == 3) rc = launch_tc_kn<3, 2>(p, a, lcfg);
    else if (a.stride == 2 && a.ksize == 4) rc = launch_tc_kn<4, 2>(p, a, lcfg);
    else {
        set_error("wgmma conv: no kernel instance for k=%d stride=%d", a.ksize, a.stride);
        return READ_ERR_UNSUPPORTED;
    }
    if (rc != READ_OK) return rc;
    RB_LAUNCH_CHECK();
    return READ_OK;
}

void tc_plan_set_reverse(TcPlan *p, int reverse) { p->reverse = reverse ? 1 : 0; }

void tc_plan_destroy(TcPlan *p) { delete p; }

}  // namespace rb

using namespace rb;

static int pack_tc_impl(const float *wf, const float *wm, int Cout, int Cin, int k, int stride, int chan_gran, void *out_bf16,
                        void *stream);

extern "C" {

int64_t read_tc_weight_elems(int Cout, int Cin, int k)
{
    TcGeom g;
    if (!tc_geom(Cin, Cout, 1, &g)) return -1;
    return (int64_t)k * k * g.kchunks * g.cin_blk * 2 * g.cout_pad;
}

int read_pack_weights_tc(const float *wf, const float *wm, int Cout, int Cin, int k, void *out_bf16, void *stream)
{
    return read_pack_weights_tc_strided(wf, wm, Cout, Cin, k, 1, out_bf16, stream);
}

int read_pack_weights_tc_for(const read_conv_desc *d, const float *wf, const float *wm, void *out_bf16, void *stream)
{
    RB_CHECK_ARG(d != nullptr, "pack_tc: null descriptor");
    return pack_tc_impl(wf, wm, d->Cout, d->Cin, d->k, d->stride, desc_chan_gran(*d), out_bf16, stream);
}

int read_pack_weights_tc_strided(const float *wf, const float *wm, int Cout, int Cin, int k, int stride, void *out_bf16,
                                 void *stream)
{
    return pack_tc_impl(wf, wm, Cout, Cin, k, stride, 64, out_bf16, stream);
}

int read_pack_weights_tc_dgrad(const float *wf, const float *wm, int Cout, int Cin, void *out_bf16, void *stream)
{
    TcGeom gf, gd;
    RB_CHECK_ARG(wf && wm && out_bf16, "pack_tc_dgrad: null pointer");
    RB_CHECK_ARG(Cin % 32 == 0 && tc_geom(Cin, Cout, 1, &gf) && tc_geom(2 * Cout, Cin / 2, 1, &gd) && gd.cout_pad == Cin / 2,
                 "pack_tc_dgrad: unsupported channel counts %d -> %d", Cin, Cout);
    const long long total = 9ll * gd.kchunks * gd.cin_blk * Cin;
    long long blocks = (total + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    pack_tc_dgrad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(wf, wm, Cout, Cin, 3, gf.n_tile / 2, gd.cin_blk,
                                                                             gd.kchunks, 0, Cin, Cin, (__nv_bfloat16 *)out_bf16);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_pack_weights_tc_dgrad1x1(const float *wf, const float *wm, int Cout, int Cin, int c0, int cn, void *out_bf16, void *stream)
{
    TcGeom gd;
    RB_CHECK_ARG(wf && wm && out_bf16, "pack_tc_dgrad1x1: null pointer");
    RB_CHECK_ARG(Cout % 16 == 0 && Cout > 0 && (Cout <= 64 || Cout % 64 == 0),
                 "pack_tc_dgrad1x1: Cout must be 16, 32, 48, 64 or a multiple of 64 (got %d)", Cout);
    RB_CHECK_ARG((cn == 16 || cn == 32 || cn == 64 || cn == 128) && c0 >= 0 && c0 + cn <= Cin,
                 "pack_tc_dgrad1x1: input channels %d..%d of %d: the slice must lie in the input and hold 16, 32, 64 or 128 channels",
                 c0, c0 + cn - 1, Cin);
    const int n_out = cn < 32 ? 32 : cn;                  // N = 16 is below the RAW plans' smallest N tile: zero filters pad it
    RB_CHECK_ARG(tc_geom(2 * Cout, n_out / 2, 1, &gd) && gd.n_tiles == 1, "pack_tc_dgrad1x1: unsupported channel counts %d -> %d",
                 Cin, Cout);
    const long long total = (long long)gd.kchunks * gd.cin_blk * n_out;
    long long blocks = (total + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    pack_tc_dgrad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(wf, wm, Cout, Cin, 1, Cout < 64 ? Cout : 64, gd.cin_blk,
                                                                             gd.kchunks, c0, cn, n_out, (__nv_bfloat16 *)out_bf16);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"

static int pack_tc_impl(const float *wf, const float *wm, int Cout, int Cin, int k, int stride, int chan_gran, void *out_bf16,
                        void *stream)
{
    TcGeom g;
    RB_CHECK_ARG(wf && wm && out_bf16, "pack_tc: null pointer");
    RB_CHECK_ARG(stride == 1 || stride == 2, "pack_tc: stride must be 1 or 2");
    RB_CHECK_ARG(tc_geom(Cin, Cout, stride, &g, chan_gran), "pack_tc: unsupported channel counts %d -> %d", Cin, Cout);
    const long long total = (long long)k * k * g.kchunks * g.cin_blk * 2 * g.cout_pad;
    long long blocks = (total + 255) / 256;
    if (blocks > 65535) blocks = 65535;
    pack_tc_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(wf, wm, Cout, g.cout_pad, Cin, k, g.cin_blk, g.n_tile,
                                                                      (__nv_bfloat16 *)out_bf16);
    RB_LAUNCH_CHECK();
    return READ_OK;
}
