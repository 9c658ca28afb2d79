// Descriptor gather for sm_90a.
// Replaces PointTexture.forward (READ/models/texture.py:42-70; its autograd backward, the scatter-add, is in train.cu):
//   feat[b,c,y,x] = texture_[0,c,(int64)idx[b,0,y,x]]      (empty pixel carries idx 0 -> point 0)
// Descriptors are read from a point-major [N,D] shadow so a pixel touches one 32-byte sector.
// gather_items_kernel: the same for a batch whose items sample different textures (a texture table in the kernel parameters).
#include "common.cuh"

namespace rb {

__global__ void tex_to_point_major_kernel(const float *__restrict__ cn, int D, long long N, float *__restrict__ nd)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < N;
         i += (long long)gridDim.x * blockDim.x) {
        if (D == 8) {
            float v[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) v[c] = __ldg(cn + (long long)c * N + i);
            float4 *o = reinterpret_cast<float4 *>(nd + i * 8);
            o[0] = make_float4(v[0], v[1], v[2], v[3]);
            o[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
            for (int c = 0; c < D; ++c) nd[i * D + c] = __ldg(cn + (long long)c * N + i);
        }
    }
}

__global__ void tex_to_channel_major_kernel(const float *__restrict__ nd, int D, long long N, float *__restrict__ cn)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < N;
         i += (long long)gridDim.x * blockDim.x) {
        for (int c = 0; c < D; ++c) cn[(long long)c * N + i] = nd[i * D + c];
    }
}

__device__ __forceinline__ float tex_act(float v, int act)
{
    if (act == READ_TEXACT_SIGMOID) return 1.f / (1.f + expf(-v));
    if (act == READ_TEXACT_TANH) return tanhf(v);
    return v;
}

// SRC: 0 = float index map, 1 = packed zbuf, 2 = int32 index map (clouds of more than 2^24 + 1 points)
template <int SRC, int LAYOUT>
__global__ void gather_kernel(const float *__restrict__ tex, int D, long long N, const void *__restrict__ src, int B,
                              int h, int w, int act, void *__restrict__ out)
{
    const long long hw = (long long)h * w;
    const long long total = (long long)B * hw;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total;
         p += (long long)gridDim.x * blockDim.x) {
        long long id;
        if (SRC == 0) {
            id = (long long)static_cast<const float *>(src)[p];           // texture.py:52 .long()
        } else if (SRC == 2) {
            id = static_cast<const int32_t *>(src)[p];
        } else {
            const unsigned long long k = static_cast<const unsigned long long *>(src)[p];
            id = (k == ZBUF_EMPTY) ? 0ll : (long long)(k & 0xFFFFFFFFull);
        }
        // the reference does not bounds-check (index_select would raise); clamp to stay memory-safe
        if (id < 0) id = 0;
        if (id >= N) id = N - 1;
        const long long b = p / hw, q = p - b * hw;
        if (D == 8) {
            const float4 *t = reinterpret_cast<const float4 *>(tex + id * 8);
            const float4 a = __ldg(t), c = __ldg(t + 1);
            float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
            if (act != READ_TEXACT_NONE) {
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = tex_act(v[i], act);
            }
            if (LAYOUT == READ_FEAT_NCHW_F32) {
                float *o = static_cast<float *>(out) + b * 8 * hw + q;
#pragma unroll
                for (int i = 0; i < 8; ++i) o[i * hw] = v[i];
            } else if (LAYOUT == READ_FEAT_NHWC_F32) {
                float4 *o = reinterpret_cast<float4 *>(static_cast<float *>(out) + p * 8);
                o[0] = make_float4(v[0], v[1], v[2], v[3]);
                o[1] = make_float4(v[4], v[5], v[6], v[7]);
            } else {
                __nv_bfloat162 r[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) r[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
                *reinterpret_cast<uint4 *>(static_cast<__nv_bfloat16 *>(out) + p * 8) = *reinterpret_cast<uint4 *>(r);
            }
        } else {
            for (int c = 0; c < D; ++c) {
                const float v = tex_act(__ldg(tex + id * D + c), act);
                if (LAYOUT == READ_FEAT_NCHW_F32) static_cast<float *>(out)[(b * D + c) * hw + q] = v;
                else if (LAYOUT == READ_FEAT_NHWC_F32) static_cast<float *>(out)[p * D + c] = v;
                else static_cast<__nv_bfloat16 *>(out)[p * D + c] = __float2bfloat16_rn(v);
            }
        }
    }
}

// gather_kernel<0, LAYOUT> at D == 8 for a batch whose items sample different textures: item b reads slot t.slot[b] of the table
// (kernel parameter space), with its ids clamped to that texture's N.  IdT: float or int32_t index map
template <typename IdT, int LAYOUT>
__global__ void gather_items_kernel(const __grid_constant__ read_tex_table t, const IdT *__restrict__ ids, int h, int w, int act,
                                    void *__restrict__ out)
{
    const long long hw = (long long)h * w;
    const long long total = (long long)t.n_items * hw;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total;
         p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / hw, q = p - b * hw;
        const int s = t.slot[b];
        const long long N = t.N[s];
        long long id = (long long)ids[p];
        if (id < 0) id = 0;
        if (id >= N) id = N - 1;
        const float4 *tp = reinterpret_cast<const float4 *>(t.tex_nd[s] + id * 8);
        const float4 a = __ldg(tp), c = __ldg(tp + 1);
        float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
        if (act != READ_TEXACT_NONE) {
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = tex_act(v[i], act);
        }
        if (LAYOUT == READ_FEAT_NCHW_F32) {
            float *o = static_cast<float *>(out) + b * 8 * hw + q;
#pragma unroll
            for (int i = 0; i < 8; ++i) o[i * hw] = v[i];
        } else if (LAYOUT == READ_FEAT_NHWC_F32) {
            float4 *o = reinterpret_cast<float4 *>(static_cast<float *>(out) + p * 8);
            o[0] = make_float4(v[0], v[1], v[2], v[3]);
            o[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
            __nv_bfloat162 r[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) r[i] = __floats2bfloat162_rn(v[2 * i], v[2 * i + 1]);
            *reinterpret_cast<uint4 *>(static_cast<__nv_bfloat16 *>(out) + p * 8) = *reinterpret_cast<uint4 *>(r);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Fused pyramid resolve for the per-frame fast path (4 nested levels, D = 8): ONE pass over the level-0 packed
// z-buffer derives levels 1..3 (2x2 min, see raster.cu: zbuf_derive_kernel), stores them, gathers the descriptors of
// all four levels into the net's NHWC input buffers, and optionally resets level 0 to "empty" for the next frame
// (replaces 3 derive + 4 gather + 1 clear launches).  One warp = one 8x8 block of level-0 pixels; lane = (row, 2 cols).
__device__ __forceinline__ void load_desc8(const float *tex, long long N, unsigned long long key, float4 (&d)[2])
{
    long long id = (key == ZBUF_EMPTY) ? 0ll : (long long)(key & 0xFFFFFFFFull);
    if (id >= N) id = N - 1;
    const float4 *t = reinterpret_cast<const float4 *>(tex + id * 8);
    d[0] = __ldg(t);
    d[1] = __ldg(t + 1);
}
template <typename TO> __device__ __forceinline__ void write_desc8(TO *out, long long pix, const float4 (&d)[2]);
template <> __device__ __forceinline__ void write_desc8<__nv_bfloat16>(__nv_bfloat16 *out, long long pix, const float4 (&d)[2])
{
    __nv_bfloat162 r[4] = {__floats2bfloat162_rn(d[0].x, d[0].y), __floats2bfloat162_rn(d[0].z, d[0].w),
                           __floats2bfloat162_rn(d[1].x, d[1].y), __floats2bfloat162_rn(d[1].z, d[1].w)};
    *reinterpret_cast<uint4 *>(out + pix * 8) = *reinterpret_cast<uint4 *>(r);
}
template <> __device__ __forceinline__ void write_desc8<float>(float *out, long long pix, const float4 (&d)[2])
{
    float4 *o = reinterpret_cast<float4 *>(out + pix * 8);
    o[0] = d[0];
    o[1] = d[1];
}

int g_gather_variant = 3;     // read_set_option("gather_variant"): 3 = the production kernel (default); 0 / 1 / 2 = restructured variants
                              // (gathers hoisted above the stores; measured slower, not re-measured on H100) kept for A/B only

struct FusedArgs {
    const float *tex;
    long long N;
    unsigned long long *z[4];     // level base pointers (all B views)
    void *out[4];
    int B, W, H;                  // level-0 size; level l is (W>>l, H>>l)
    int reset0;
};

__device__ __forceinline__ unsigned long long umin64(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
__device__ __forceinline__ unsigned long long shfl_xor64(unsigned long long v, int m)
{
    return (unsigned long long)__shfl_xor_sync(0xffffffffu, (long long)v, m);
}

template <typename TO, int V>
__global__ void __launch_bounds__(256, V == 1 ? 4 : 1) pyramid_resolve_gather_kernel(const __grid_constant__ FusedArgs a)
{
    const int lane = threadIdx.x & 31;
    const int bw = a.W >> 3, bh = a.H >> 3;
    const long long nblocks = (long long)a.B * bw * bh;
    const int row = lane >> 2, col = (lane & 3) * 2;
    for (long long blk = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; blk < nblocks;
         blk += ((long long)gridDim.x * blockDim.x) >> 5) {
        const int bx = (int)(blk % bw);
        long long t = blk / bw;
        const int by = (int)(t % bh);
        const int b = (int)(t / bh);
        const int x = bx * 8 + col, y = by * 8 + row;
        const long long p0 = ((long long)b * a.H + y) * a.W + x;
        unsigned long long *zp = a.z[0] + p0;
        const ulonglong2 k = *reinterpret_cast<const ulonglong2 *>(zp);            // x is even, level base is 16B aligned
        if (a.reset0) *reinterpret_cast<ulonglong2 *>(zp) = make_ulonglong2(ZBUF_EMPTY, ZBUF_EMPTY);
        // level 1: 2x2 min = horizontal pair (in-lane) + vertical pair (lane ^ 4)
        unsigned long long m1 = umin64(k.x, k.y);
        m1 = umin64(m1, shfl_xor64(m1, 4));
        // level 2: level-1 neighbours: horizontal lane ^ 1, vertical lane ^ 8
        unsigned long long m2 = umin64(m1, shfl_xor64(m1, 1));
        m2 = umin64(m2, shfl_xor64(m2, 8));
        // level 3: horizontal lane ^ 2, vertical lane ^ 16
        unsigned long long m3 = umin64(m2, shfl_xor64(m2, 2));
        m3 = umin64(m3, shfl_xor64(m3, 16));
        // ALL descriptor reads of the block are issued before the first store (the level-1..3 gathers would otherwise wait
        // behind the level-0 stores: up to five serial DRAM round trips per block; this way it is two: keys, then descriptors)
        const bool p1 = (row & 1) == 0, p2 = p1 && (row & 2) == 0 && (lane & 1) == 0, p3 = lane == 0;
        if (V == 0) {           // round-1 order: every gather next to its store
            TO *o0 = static_cast<TO *>(a.out[0]);
            float4 d[2];
            load_desc8(a.tex, a.N, k.x, d); write_desc8<TO>(o0, p0, d);
            load_desc8(a.tex, a.N, k.y, d); write_desc8<TO>(o0, p0 + 1, d);
            if (p1) {
                const long long p1i = ((long long)b * (a.H >> 1) + (y >> 1)) * (a.W >> 1) + (x >> 1);
                a.z[1][p1i] = m1;
                load_desc8(a.tex, a.N, m1, d); write_desc8<TO>(static_cast<TO *>(a.out[1]), p1i, d);
            }
            if (p2) {
                const long long p2i = ((long long)b * (a.H >> 2) + (y >> 2)) * (a.W >> 2) + (x >> 2);
                a.z[2][p2i] = m2;
                load_desc8(a.tex, a.N, m2, d); write_desc8<TO>(static_cast<TO *>(a.out[2]), p2i, d);
            }
            if (p3) {
                const long long p3i = ((long long)b * (a.H >> 3) + (y >> 3)) * (a.W >> 3) + (x >> 3);
                a.z[3][p3i] = m3;
                load_desc8(a.tex, a.N, m3, d); write_desc8<TO>(static_cast<TO *>(a.out[3]), p3i, d);
            }
            continue;
        }
        float4 d0[2], d1[2], d2[2], d3[2], d4[2];
        load_desc8(a.tex, a.N, k.x, d0);
        load_desc8(a.tex, a.N, k.y, d1);
        if (p1) load_desc8(a.tex, a.N, m1, d2);
        if (p2) load_desc8(a.tex, a.N, m2, d3);
        if (p3) load_desc8(a.tex, a.N, m3, d4);
        TO *o0 = static_cast<TO *>(a.out[0]);
        write_desc8<TO>(o0, p0, d0);
        write_desc8<TO>(o0, p0 + 1, d1);
        if (p1) {
            const int W1 = a.W >> 1, H1 = a.H >> 1;
            const long long p1i = ((long long)b * H1 + (y >> 1)) * W1 + (x >> 1);
            a.z[1][p1i] = m1;
            write_desc8<TO>(static_cast<TO *>(a.out[1]), p1i, d2);
        }
        if (p2) {
            const int W2 = a.W >> 2, H2 = a.H >> 2;
            const long long p2i = ((long long)b * H2 + (y >> 2)) * W2 + (x >> 2);
            a.z[2][p2i] = m2;
            write_desc8<TO>(static_cast<TO *>(a.out[2]), p2i, d3);
        }
        if (p3) {
            const int W3 = a.W >> 3, H3 = a.H >> 3;
            const long long p3i = ((long long)b * H3 + (y >> 3)) * W3 + (x >> 3);
            a.z[3][p3i] = m3;
            write_desc8<TO>(static_cast<TO *>(a.out[3]), p3i, d4);
        }
    }
}

// the production kernel (gather_variant 3, unchanged since round 1)
template <typename TO>
__device__ __forceinline__ void store_desc8(TO *out, long long pix, const float *tex, long long N, unsigned long long key);

template <>
__device__ __forceinline__ void store_desc8<__nv_bfloat16>(__nv_bfloat16 *out, long long pix, const float *tex, long long N,
                                                           unsigned long long key)
{
    long long id = (key == ZBUF_EMPTY) ? 0ll : (long long)(key & 0xFFFFFFFFull);
    if (id >= N) id = N - 1;
    const float4 *t = reinterpret_cast<const float4 *>(tex + id * 8);
    const float4 a = __ldg(t), c = __ldg(t + 1);
    __nv_bfloat162 r[4] = {__floats2bfloat162_rn(a.x, a.y), __floats2bfloat162_rn(a.z, a.w), __floats2bfloat162_rn(c.x, c.y),
                           __floats2bfloat162_rn(c.z, c.w)};
    *reinterpret_cast<uint4 *>(out + pix * 8) = *reinterpret_cast<uint4 *>(r);
}
template <>
__device__ __forceinline__ void store_desc8<float>(float *out, long long pix, const float *tex, long long N,
                                                   unsigned long long key)
{
    long long id = (key == ZBUF_EMPTY) ? 0ll : (long long)(key & 0xFFFFFFFFull);
    if (id >= N) id = N - 1;
    const float4 *t = reinterpret_cast<const float4 *>(tex + id * 8);
    float4 *o = reinterpret_cast<float4 *>(out + pix * 8);
    o[0] = __ldg(t);
    o[1] = __ldg(t + 1);
}

template <typename TO>
__global__ void __launch_bounds__(256) pyramid_resolve_gather_r1_kernel(const __grid_constant__ FusedArgs a)
{
    const int lane = threadIdx.x & 31;
    const int bw = a.W >> 3, bh = a.H >> 3;
    const long long nblocks = (long long)a.B * bw * bh;
    const int row = lane >> 2, col = (lane & 3) * 2;
    for (long long blk = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; blk < nblocks;
         blk += ((long long)gridDim.x * blockDim.x) >> 5) {
        const int bx = (int)(blk % bw);
        long long t = blk / bw;
        const int by = (int)(t % bh);
        const int b = (int)(t / bh);
        const int x = bx * 8 + col, y = by * 8 + row;
        const long long p0 = ((long long)b * a.H + y) * a.W + x;
        unsigned long long *zp = a.z[0] + p0;
        const ulonglong2 k = *reinterpret_cast<const ulonglong2 *>(zp);            // x is even, level base is 16B aligned
        if (a.reset0) *reinterpret_cast<ulonglong2 *>(zp) = make_ulonglong2(ZBUF_EMPTY, ZBUF_EMPTY);
        TO *o0 = static_cast<TO *>(a.out[0]);
        store_desc8<TO>(o0, p0, a.tex, a.N, k.x);
        store_desc8<TO>(o0, p0 + 1, a.tex, a.N, k.y);
        // level 1: 2x2 min = horizontal pair (in-lane) + vertical pair (lane ^ 4)
        unsigned long long m1 = umin64(k.x, k.y);
        m1 = umin64(m1, shfl_xor64(m1, 4));
        // level 2: level-1 neighbours: horizontal lane ^ 1, vertical lane ^ 8
        unsigned long long m2 = umin64(m1, shfl_xor64(m1, 1));
        m2 = umin64(m2, shfl_xor64(m2, 8));
        // level 3: horizontal lane ^ 2, vertical lane ^ 16
        unsigned long long m3 = umin64(m2, shfl_xor64(m2, 2));
        m3 = umin64(m3, shfl_xor64(m3, 16));
        if ((row & 1) == 0) {
            const int W1 = a.W >> 1, H1 = a.H >> 1;
            const long long p1 = ((long long)b * H1 + (y >> 1)) * W1 + (x >> 1);
            a.z[1][p1] = m1;
            store_desc8<TO>(static_cast<TO *>(a.out[1]), p1, a.tex, a.N, m1);
            if ((row & 2) == 0 && (lane & 1) == 0) {
                const int W2 = a.W >> 2, H2 = a.H >> 2;
                const long long p2 = ((long long)b * H2 + (y >> 2)) * W2 + (x >> 2);
                a.z[2][p2] = m2;
                store_desc8<TO>(static_cast<TO *>(a.out[2]), p2, a.tex, a.N, m2);
                if (lane == 0) {
                    const int W3 = a.W >> 3, H3 = a.H >> 3;
                    const long long p3 = ((long long)b * H3 + (y >> 3)) * W3 + (x >> 3);
                    a.z[3][p3] = m3;
                    store_desc8<TO>(static_cast<TO *>(a.out[3]), p3, a.tex, a.N, m3);
                }
            }
        }
    }
}

template <int SRC>
static int launch_gather(const float *tex, int D, long long N, const void *src, int B, int h, int w, int layout,
                         int act, void *out, cudaStream_t st)
{
    const long long total = (long long)B * h * w;
    if (total == 0) return READ_OK;
    const unsigned g = grid_for(total);
    switch (layout) {
    case READ_FEAT_NCHW_F32:
        gather_kernel<SRC, READ_FEAT_NCHW_F32><<<g, 256, 0, st>>>(tex, D, N, src, B, h, w, act, out);
        break;
    case READ_FEAT_NHWC_F32:
        gather_kernel<SRC, READ_FEAT_NHWC_F32><<<g, 256, 0, st>>>(tex, D, N, src, B, h, w, act, out);
        break;
    case READ_FEAT_NHWC_BF16:
        gather_kernel<SRC, READ_FEAT_NHWC_BF16><<<g, 256, 0, st>>>(tex, D, N, src, B, h, w, act, out);
        break;
    default:
        set_error("gather: unknown layout %d", layout);
        return READ_ERR_INVALID;
    }
    RB_LAUNCH_CHECK();
    return READ_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Net-input staging for the two viewer options of NetAndTexture (READ/models/compose.py:162-171) on the fused path:
//   supersampling ss > 1: the pyramid is rendered at ss x the net resolution and every level's feature map is reduced with
//     F.interpolate(scale_factor=1/ss, mode='bilinear') (align_corners=False): src = (dst + 0.5) * ss - 0.5, taps i0 = floor(src),
//     i1 = min(i0 + 1, n - 1), weight src - i0 (even ss: the two central pixels, equal weights; odd ss: the central pixel);
//   temporal_average: input = (input + last_input) / 2, and the AVERAGED input becomes last_input (compose.py:167-171).
// One pass: f32 NHWC features at render resolution -> [bilinear reduce] -> [average with / update `last`] -> NHWC act dtype.
template <typename T>
__global__ void stage_inputs_kernel(const float *__restrict__ src, int B, int hs, int ws, int C, int factor, float *last,
                                    int have_last, T *__restrict__ dst)
{
    const int hd = hs / factor, wd = ws / factor;
    const long long total = (long long)B * hd * wd * C;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        long long t = i / C;
        const int x = (int)(t % wd);
        t /= wd;
        const int y = (int)(t % hd);
        const int b = (int)(t / hd);
        float v;
        if (factor == 1) {
            v = src[i];
        } else {
            const float fx = ((float)x + 0.5f) * (float)factor - 0.5f, fy = ((float)y + 0.5f) * (float)factor - 0.5f;
            const int x0 = (int)fx, y0 = (int)fy;                    // fx, fy >= 0 for factor >= 1
            const int x1 = x0 + 1 < ws ? x0 + 1 : ws - 1, y1 = y0 + 1 < hs ? y0 + 1 : hs - 1;
            const float lx = fx - (float)x0, ly = fy - (float)y0;
            const float *p = src + (long long)b * hs * ws * C + c;
            const float v00 = p[((long long)y0 * ws + x0) * C], v01 = p[((long long)y0 * ws + x1) * C];
            const float v10 = p[((long long)y1 * ws + x0) * C], v11 = p[((long long)y1 * ws + x1) * C];
            // torch's upsample_bilinear2d: w-lerp inside h-lerp, weights (1 - l), l
            v = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
        }
        if (last != nullptr) {
            if (have_last) v = (v + last[i]) / 2.f;
            last[i] = v;
        }
        dst[i] = from_f32<T>(v);
    }
}

template <typename IdT>
static int gather_items(const read_tex_table *table, const IdT *ids, int h, int w, int layout, int activation, void *out, cudaStream_t st)
{
    int rc = check_tex_table(table, h, w, true, false, "gather (items)");
    if (rc) return rc;
    RB_CHECK_ARG(ids && out && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "gather (items): null or unaligned ids / output");
    const long long total = (long long)table->n_items * h * w;
    if (total == 0) return READ_OK;
    const unsigned g = grid_for(total);
    switch (layout) {
    case READ_FEAT_NCHW_F32: gather_items_kernel<IdT, READ_FEAT_NCHW_F32><<<g, 256, 0, st>>>(*table, ids, h, w, activation, out); break;
    case READ_FEAT_NHWC_F32: gather_items_kernel<IdT, READ_FEAT_NHWC_F32><<<g, 256, 0, st>>>(*table, ids, h, w, activation, out); break;
    case READ_FEAT_NHWC_BF16: gather_items_kernel<IdT, READ_FEAT_NHWC_BF16><<<g, 256, 0, st>>>(*table, ids, h, w, activation, out); break;
    default:
        set_error("gather (items): unknown layout %d", layout);
        return READ_ERR_INVALID;
    }
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb

using namespace rb;

extern "C" {

int read_texture_to_point_major(const float *tex_cn, int D, int64_t N, float *tex_nd, void *stream)
{
    RB_CHECK_ARG(tex_cn && tex_nd && D >= 1 && N >= 1, "texture transpose: bad arguments");
    RB_CHECK_ARG(D != 8 || (reinterpret_cast<uintptr_t>(tex_nd) & 15) == 0, "texture transpose: output must be 16B aligned");
    tex_to_point_major_kernel<<<grid_for(N), 256, 0, (cudaStream_t)stream>>>(tex_cn, D, N, tex_nd);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_texture_to_channel_major(const float *tex_nd, int D, int64_t N, float *tex_cn, void *stream)
{
    RB_CHECK_ARG(tex_cn && tex_nd && D >= 1 && N >= 1, "texture transpose: bad arguments");
    tex_to_channel_major_kernel<<<grid_for(N), 256, 0, (cudaStream_t)stream>>>(tex_nd, D, N, tex_cn);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

static int check_gather(const float *tex, int D, int64_t N, const void *src, int B, int h, int w, const void *out)
{
    RB_CHECK_ARG(tex && src && out, "gather: null pointer");
    RB_CHECK_ARG(D >= 1 && N >= 1 && B >= 0 && h >= 0 && w >= 0, "gather: bad shape");
    RB_CHECK_ARG(D != 8 || (reinterpret_cast<uintptr_t>(tex) & 15) == 0, "gather: descriptors must be 16B aligned");
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(out) & 15) == 0, "gather: output must be 16B aligned");
    return READ_OK;
}

int read_gather_from_index(const float *tex_nd, int D, int64_t N, const float *ids, int B, int h, int w, int layout,
                           int activation, void *out, void *stream)
{
    int rc = check_gather(tex_nd, D, N, ids, B, h, w, out);
    if (rc) return rc;
    return launch_gather<0>(tex_nd, D, N, ids, B, h, w, layout, activation, out, (cudaStream_t)stream);
}

int read_gather_from_index_i32(const float *tex_nd, int D, int64_t N, const int32_t *ids, int B, int h, int w, int layout,
                               int activation, void *out, void *stream)
{
    int rc = check_gather(tex_nd, D, N, ids, B, h, w, out);
    if (rc) return rc;
    return launch_gather<2>(tex_nd, D, N, ids, B, h, w, layout, activation, out, (cudaStream_t)stream);
}

int read_gather_from_index_items(const read_tex_table *table, const float *ids, int h, int w, int layout, int activation, void *out,
                                 void *stream)
{
    return gather_items<float>(table, ids, h, w, layout, activation, out, (cudaStream_t)stream);
}

int read_gather_from_index_items_i32(const read_tex_table *table, const int32_t *ids, int h, int w, int layout, int activation,
                                     void *out, void *stream)
{
    return gather_items<int32_t>(table, ids, h, w, layout, activation, out, (cudaStream_t)stream);
}

int read_gather_from_zbuf(const float *tex_nd, int D, int64_t N, const uint64_t *zbuf_level, int B, int h, int w,
                          int layout, int activation, void *out, void *stream)
{
    int rc = check_gather(tex_nd, D, N, zbuf_level, B, h, w, out);
    if (rc) return rc;
    return launch_gather<1>(tex_nd, D, N, zbuf_level, B, h, w, layout, activation, out, (cudaStream_t)stream);
}

int read_pyramid_resolve_gather(const float *tex_nd, int D, int64_t N, uint64_t *zbuf, int B, int view0, int nviews,
                                int W, int H, int L, int layout, void *const *outs, int reset_level0, void *stream)
{
    RB_CHECK_ARG(view0 >= 0 && nviews >= 1 && view0 + nviews <= B, "pyramid resolve: bad view range");
    RB_CHECK_ARG(tex_nd && zbuf && outs, "pyramid resolve: null pointer");
    RB_CHECK_ARG(D == 8 && L == 4, "pyramid resolve: fused path needs D == 8 and L == 4");
    RB_CHECK_ARG(B >= 1 && W >= 8 && H >= 8 && W % 8 == 0 && H % 8 == 0, "pyramid resolve: W and H must be multiples of 8");
    RB_CHECK_ARG(layout == READ_FEAT_NHWC_BF16 || layout == READ_FEAT_NHWC_F32, "pyramid resolve: NHWC layouts only");
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(tex_nd) & 15) == 0 && (reinterpret_cast<uintptr_t>(zbuf) & 15) == 0,
                 "pyramid resolve: descriptors / z-buffer must be 16B aligned");
    const LevelGeom g = level_geom(B, W, H, L);
    FusedArgs a{};
    a.tex = tex_nd; a.N = N; a.B = nviews; a.W = W; a.H = H; a.reset0 = reset_level0;
    for (int l = 0; l < 4; ++l) {
        RB_CHECK_ARG(outs[l] != nullptr && (reinterpret_cast<uintptr_t>(outs[l]) & 15) == 0, "pyramid resolve: bad output %d", l);
        a.z[l] = reinterpret_cast<unsigned long long *>(zbuf) + g.off[l] + (long long)view0 * g.w[l] * g.h[l];
        a.out[l] = outs[l];
    }
    const long long nblocks = (long long)nviews * (W >> 3) * (H >> 3);
    long long ctas = (nblocks + 7) / 8;
    const long long cap = (long long)num_sms() * 16;
    if (ctas > cap) ctas = cap;
    const int v = g_gather_variant;
#define RB_PRG(T_) do { if (v == 3) pyramid_resolve_gather_r1_kernel<T_><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(a); \
                        else if (v == 1) pyramid_resolve_gather_kernel<T_, 1><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(a); \
                        else if (v == 2) pyramid_resolve_gather_kernel<T_, 2><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(a); \
                        else pyramid_resolve_gather_kernel<T_, 0><<<(unsigned)ctas, 256, 0, (cudaStream_t)stream>>>(a); } while (0)
    if (layout == READ_FEAT_NHWC_BF16) RB_PRG(__nv_bfloat16);
    else RB_PRG(float);
#undef RB_PRG
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_stage_net_inputs(const float *src, int B, int hs, int ws, int C, int factor, float *last, int have_last, int act_dtype,
                          void *dst, void *stream)
{
    RB_CHECK_ARG(src && dst, "stage_net_inputs: null pointer");
    RB_CHECK_ARG(B >= 1 && C >= 1 && factor >= 1 && hs >= factor && ws >= factor, "stage_net_inputs: bad shape");
    RB_CHECK_ARG(hs % factor == 0 && ws % factor == 0, "stage_net_inputs: the render size must be a multiple of the supersampling factor");
    RB_CHECK_ARG(act_dtype == READ_ACT_F32 || act_dtype == READ_ACT_BF16, "stage_net_inputs: bad act_dtype");
    const long long total = (long long)B * (hs / factor) * (ws / factor) * C;
    long long blocks = (total + 255) / 256;
    if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
    if (act_dtype == READ_ACT_BF16)
        stage_inputs_kernel<__nv_bfloat16><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, B, hs, ws, C, factor, last, have_last,
                                                                                              (__nv_bfloat16 *)dst);
    else
        stage_inputs_kernel<float><<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, B, hs, ws, C, factor, last, have_last, (float *)dst);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"
