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
//   epilogue    bias, ELU, sigmoid gate, BN affine, residual add, bf16 pack -> global, straight from the accumulators
//               (optionally a second output y*z for the following FAM, unet.py:115).
//
// Warp roles (288 threads, persistent over tiles): warps 0..7 = two consumer warpgroups (wgmma + epilogue), warp 8 = TMA
// producer, which runs ahead through the A (and streamed B) rings while the consumers compute.  Layers with N <= 64 whose
// weights and four A stages fit half the shared-memory budget run two CTAs per SM: one CTA's epilogue overlaps the other's MMAs.
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
constexpr uint32_t TC_SMEM_BUDGET = 200 * 1024;
constexpr uint32_t TC_SMEM_BUDGET_SMALL_N = 100 * 1024;   // N <= 64: two CTAs per SM
__host__ __device__ constexpr int tc_ctas_per_sm(int n_tile) { return n_tile <= 64 ? 2 : 1; }
constexpr uint32_t TC_RESIDENT_MAX = 144 * 1024;
// barrier slots (uint64 each)
constexpr int BAR_AFULL = 0, BAR_AEMPTY = 16, BAR_BFULL = 32, BAR_BEMPTY = 48, BAR_BRES = 64, BAR_PARAMS = 66;
constexpr uint32_t TC_CONSUMER_WARPS = 8;

// activation tensor maps: one per source of a virtual concat (1x1 convs: torch.cat along channels, unet.py:88,105,263;
// a nearest-DOWN resampled source is a traversal-stride load of the full-resolution tensor)
struct TcMaps {
    CUtensorMap a[READ_MAX_SRC];
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
    const uint32_t b_region = smem_base + a.b_region_off;
    const uint32_t b_region_bytes = a.b_resident ? (uint32_t)(ntaps * a.kchunks) * a.b_bytes : (uint32_t)a.b_stages * a.b_bytes;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_al + a.b_region_off + b_region_bytes);
    const uint32_t bar0 = s_u32(bars);
    const uint32_t afull0 = bar0 + 8 * BAR_AFULL, aempty0 = bar0 + 8 * BAR_AEMPTY;
    const uint32_t bfull0 = bar0 + 8 * BAR_BFULL, bempty0 = bar0 + 8 * BAR_BEMPTY, bres = bar0 + 8 * BAR_BRES;
    float4 *s_par = reinterpret_cast<float4 *>(bars + BAR_PARAMS);

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    if (a.pdl) pdl_launch_dependents();
    for (int i = threadIdx.x; i < a.cout_pad; i += TC_THREADS)
        s_par[i] = i < a.Cout ? make_float4(a.bias_f[i], a.bias_m[i], a.scale[i], a.shift[i]) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (warp == TC_PRODUCER_WARP && lane == 0) {
        for (int i = 0; i < a.n_src; ++i) tma_prefetch_desc(&tm.a[i]);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < TC_MAX_STAGES; ++s) {
            mbar_init(afull0 + 8 * s, 1);
            mbar_init(aempty0 + 8 * s, TC_CONSUMER_WARPS);
            mbar_init(bfull0 + 8 * s, 1);
            mbar_init(bempty0 + 8 * s, TC_CONSUMER_WARPS);
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
        uint32_t as = 0, aph = 0, bs = 0, bph = 0;
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
    if (a.pdl) pdl_wait();        // residual / add-in / FAM-multiplier tensors come from earlier kernels
    if (a.b_resident) mbar_wait(bres, 0);
    uint32_t as = 0, aph = 0, bs = 0, bph = 0;
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
        EpiArgs e = a.epi;
        e.par = s_par;
        const int x0 = tc_.tx * TC_TW + (lane >> 2), y0 = tc_.ty * TC_TH + 8 * wg + 2 * wiw;
        const int xs[2] = {x0, x0}, ys[2] = {y0, y0 + 1};
        const bool in[2] = {x0 < a.W && y0 < a.H, x0 < a.W && y0 + 1 < a.H};
        epilogue_tile<N>(acc, lane, tc_.b, ys, xs, in, tc_.nt, e);
    }
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
    if (d.out_mode == READ_OUT_RAW_NHWC || d.addin != nullptr) {
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
};

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
    const long long tiles = (long long)((d.Wout + TC_TW - 1) / TC_TW) * ((d.Hout + TC_TH - 1) / TC_TH) * d.B * g.n_tiles;
    RB_CHECK_ARG(tiles < (1ll << 31), "wgmma conv: too many tiles");
    TcPlan *p = new (std::nothrow) TcPlan{};
    RB_CHECK_ARG(p != nullptr, "wgmma conv: out of host memory");

    const bool s2 = d.stride == 2;
    const int halo_rows = s2 ? TC_TH + 1 : TC_TH + d.k - 1;
    const int halo_w = s2 ? TC_TW + 1 : TC_TW + d.k - 1;
    const CUtensorMapSwizzle sw = g.cin_blk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B
                                  : (g.cin_blk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    for (int si = 0; si < d.n_src; ++si) {   // activations: dims {C, W, H, B}; box = one halo tile (all filter taps)
        const read_src &sv = d.src[si];
        const unsigned f = (d.n_src > 1 && sv.mode == READ_SRC_NEAREST_DOWN) ? (unsigned)sv.factor : (s2 ? 2u : 1u);
        cuuint64_t dims[4] = {(cuuint64_t)sv.C, (cuuint64_t)sv.W, (cuuint64_t)sv.H, (cuuint64_t)d.B};
        cuuint64_t strides[3] = {(cuuint64_t)sv.C * 2, (cuuint64_t)sv.W * sv.C * 2, (cuuint64_t)sv.H * sv.W * sv.C * 2};
        // traversal stride f in x and y (conv stride 2, or a nearest-down source): the box spans (n-1)*f+1 input
        // elements and delivers n of them
        cuuint32_t box[4] = {(cuuint32_t)g.cin_blk, (cuuint32_t)((halo_w - 1) * f + 1), (cuuint32_t)((halo_rows - 1) * f + 1), 1};
        cuuint32_t estr[4] = {1, f, f, 1};
        CUresult r = enc(&p->tmA.a[si], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void *>(sv.ptr), dims, strides, box,
                         estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
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
        cuuint32_t box[2] = {(cuuint32_t)g.cin_blk, (cuuint32_t)g.n_tile};
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
    TcArgs &a = p->args;
    a.B = d.B; a.H = d.Hout; a.W = d.Wout; a.Cin = d.Cin; a.Cout = d.Cout; a.cout_pad = g.cout_pad;
    a.ksize = d.k; a.pad = d.pad;
    a.cin_blk = g.cin_blk; a.kchunks = g.kchunks; a.n_tile = g.n_tile; a.n_tiles = g.n_tiles;
    a.tiles_x = (d.Wout + TC_TW - 1) / TC_TW;
    a.tiles_y = (d.Hout + TC_TH - 1) / TC_TH;
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
    a.a_tx_bytes = (uint32_t)halo_rows * halo_w * g.cin_blk * 2u;
    a.tile_bytes = (a.a_tx_bytes + 1023u) & ~1023u;    // tiles stay 1 KB aligned (swizzle patterns are address based)
    a.a_bytes = s2 ? 4u * a.tile_bytes : a.tile_bytes;
    a.b_bytes = (uint32_t)g.n_tile * g.cin_blk * 2u;
    const uint32_t total_b = (uint32_t)(d.k * d.k * g.kchunks) * a.b_bytes;
    // two CTAs per SM when the kernel instance allows it and the layer keeps resident weights + >= 4 A stages in half the budget
    a.ctas_per_sm = (tc_ctas_per_sm(g.n_tile) > 1 && g.n_tiles == 1 && total_b <= TC_RESIDENT_MAX &&
                     total_b + 4 * a.a_bytes <= TC_SMEM_BUDGET_SMALL_N) ? 2 : 1;
    const uint32_t budget = a.ctas_per_sm > 1 ? TC_SMEM_BUDGET_SMALL_N : TC_SMEM_BUDGET;
    a.b_resident = (g.n_tiles == 1 && total_b <= TC_RESIDENT_MAX && total_b + 2 * a.a_bytes <= budget) ? 1 : 0;
    uint32_t b_region_bytes;
    if (a.b_resident) {
        int st = (int)((budget - total_b) / a.a_bytes);
        a.a_stages = st > TC_MAX_STAGES ? TC_MAX_STAGES : st;
        a.b_stages = 0;
        b_region_bytes = total_b;
    } else {
        a.a_stages = 3;
        if (3 * a.a_bytes + 2 * a.b_bytes > budget) {
            set_error("wgmma conv: layer does not fit shared memory (A stage %u B, B tile %u B)", a.a_bytes, a.b_bytes);
            delete p;
            return READ_ERR_UNSUPPORTED;
        }
        int st = (int)((budget - 3 * a.a_bytes) / a.b_bytes);
        a.b_stages = st > TC_MAX_STAGES ? TC_MAX_STAGES : st;
        b_region_bytes = (uint32_t)a.b_stages * a.b_bytes;
    }
    a.b_region_off = (uint32_t)a.a_stages * a.a_bytes;
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
    p->smem_bytes = 1024 + (size_t)a.b_region_off + b_region_bytes + 8 * BAR_PARAMS + 16 * (size_t)g.cout_pad + 64;
    *out = p;
    return READ_OK;
}

int g_tc_pdl = 1;         // programmatic dependent launch between consecutive conv kernels (read_set_option "tc_pdl")

template <int KS, int STR, int KKN, int N>
static int launch_tc(const TcPlan *p, const TcArgs &a, cudaLaunchConfig_t &lcfg)
{
    RB_CUDA(cudaFuncSetAttribute(gated_conv_tc_kernel<KS, STR, KKN, N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p->smem_bytes));
    RB_CUDA(cudaLaunchKernelEx(&lcfg, gated_conv_tc_kernel<KS, STR, KKN, N>, p->tmA, p->tmB, a));
    return READ_OK;
}

template <int KS, int STR>
static int launch_tc_kn(const TcPlan *p, const TcArgs &a, cudaLaunchConfig_t &lcfg)
{
    const int kkn = a.cin_blk / 16;
#define RB_TC_N(KKN_)                                                                       \
    switch (a.n_tile) {                                                                     \
    case 16: return launch_tc<KS, STR, KKN_, 16>(p, a, lcfg);                               \
    case 32: return launch_tc<KS, STR, KKN_, 32>(p, a, lcfg);                               \
    case 64: return launch_tc<KS, STR, KKN_, 64>(p, a, lcfg);                               \
    case 128: return launch_tc<KS, STR, KKN_, 128>(p, a, lcfg);                             \
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
    if (a.stride == 1 && a.ksize == 1) rc = launch_tc_kn<1, 1>(p, a, lcfg);
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
