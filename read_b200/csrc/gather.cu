// Descriptor gather for sm_90a.
// Replaces PointTexture.forward (READ/models/texture.py:42-70; its autograd backward, the scatter-add, is in train.cu):
//   feat[b,c,y,x] = texture_[0,c,(int64)idx[b,0,y,x]]      (empty pixel carries idx 0 -> point 0)
// Descriptors are read from a point-major [N,D] shadow so a pixel touches one 32-byte sector.
// One kernel body (gather_kernel) serves both jobs: one texture (GatherOne), and a batch whose items sample different textures
// (GatherItems: a texture table in the kernel parameters).
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

// the raw id of an index-map entry (texture.py:52 .long() of a float map, or an int32 map) or of a packed z-buffer key
__device__ __forceinline__ long long raw_id(float v) { return (long long)v; }
__device__ __forceinline__ long long raw_id(int32_t v) { return v; }
__device__ __forceinline__ long long raw_id(unsigned long long key) { return zbuf_point_id(key); }

// the 8 features of flat pixel p = b * hw + q in each output layout: 8 planes of hw floats (the only use of hw), or 32 (f32) /
// 16 (bf16) bytes at p
template <int LAYOUT>
__device__ __forceinline__ void store_feat8(void *out, long long p, long long hw, const float (&v)[8])
{
    if (LAYOUT == READ_FEAT_NCHW_F32) {
        const long long b = p / hw;
        float *o = static_cast<float *>(out) + b * 8 * hw + (p - b * hw);
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

// The jobs of gather_kernel: rows(b, N) the point-major descriptors item b reads and their count N, d() the channel count (a
// compile-time 8 for a table) and items() the batch size.
// One texture of N points and D channels for every item.
struct GatherOne {
    const float *tex;
    long long N;
    int D, B;
    __device__ __forceinline__ const float *rows(long long, long long &n) const { n = N; return tex; }
    __device__ __forceinline__ int d() const { return D; }
    __host__ __device__ __forceinline__ int items() const { return B; }
};

// A texture table (kernel parameter space): item b reads slot t.slot[b].
struct GatherItems {
    read_tex_table t;
    __device__ __forceinline__ const float *rows(long long b, long long &n) const
    {
        const int s = t.slot[b];
        n = t.N[s];
        return t.tex_nd[s];
    }
    __device__ __forceinline__ int d() const { return 8; }
    __host__ __device__ __forceinline__ int items() const { return t.n_items; }
};

// feat[b, :, q] = act(rows[clamp(id)]) for every pixel; SrcT: float or int32_t index map, or packed z-buffer keys
template <class Job, typename SrcT, int LAYOUT>
__global__ void gather_kernel(const __grid_constant__ Job j, const SrcT *__restrict__ src, int h, int w, int act,
                              void *__restrict__ out)
{
    const long long hw = (long long)h * w;
    const long long total = (long long)j.items() * hw;
    const int D = j.d();
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total;
         p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / hw;
        long long N;
        const float *tex = j.rows(b, N);
        long long id = raw_id(src[p]);
        // the reference does not bounds-check (index_select would raise); clamp to stay memory-safe
        if (id < 0) id = 0;
        if (id >= N) id = N - 1;
        if (D == 8) {
            const float4 *t = reinterpret_cast<const float4 *>(tex + id * 8);
            const float4 a = __ldg(t), c = __ldg(t + 1);
            float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
            if (act != READ_TEXACT_NONE) {
#pragma unroll
                for (int i = 0; i < 8; ++i) v[i] = tex_act(v[i], act);
            }
            store_feat8<LAYOUT>(out, p, hw, v);
        } else {
            const long long q = p - b * hw;
            for (int c = 0; c < D; ++c) {
                const float v = tex_act(__ldg(tex + id * D + c), act);
                if (LAYOUT == READ_FEAT_NCHW_F32) static_cast<float *>(out)[(b * D + c) * hw + q] = v;
                else if (LAYOUT == READ_FEAT_NHWC_F32) static_cast<float *>(out)[p * D + c] = v;
                else static_cast<__nv_bfloat16 *>(out)[p * D + c] = __float2bfloat16_rn(v);
            }
        }
    }
}

// what: the caller's name in the unknown-layout message
template <class Job, typename SrcT>
static int launch_gather(const Job &j, const SrcT *src, int h, int w, int layout, int act, void *out, cudaStream_t st,
                         const char *what)
{
    const long long total = (long long)j.items() * h * w;
    if (total == 0) return READ_OK;
    const unsigned g = grid_for(total);
    switch (layout) {
    case READ_FEAT_NCHW_F32: gather_kernel<Job, SrcT, READ_FEAT_NCHW_F32><<<g, 256, 0, st>>>(j, src, h, w, act, out); break;
    case READ_FEAT_NHWC_F32: gather_kernel<Job, SrcT, READ_FEAT_NHWC_F32><<<g, 256, 0, st>>>(j, src, h, w, act, out); break;
    case READ_FEAT_NHWC_BF16: gather_kernel<Job, SrcT, READ_FEAT_NHWC_BF16><<<g, 256, 0, st>>>(j, src, h, w, act, out); break;
    default:
        set_error("%s: unknown layout %d", what, layout);
        return READ_ERR_INVALID;
    }
    RB_LAUNCH_CHECK();
    return READ_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Fused pyramid resolve for the per-frame fast path (4 nested levels, D = 8): ONE pass over the level-0 packed
// z-buffer derives levels 1..3 (2x2 min, see raster.cu: zbuf_derive_kernel), stores them, gathers the descriptors of
// all four levels into the net's NHWC input buffers, and optionally resets level 0 to "empty" for the next frame
// (replaces 3 derive + 4 gather + 1 clear launches).  One warp = one 8x8 block of level-0 pixels; lane = (row, 2 cols).
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

// the descriptor of a key's point into pixel pix of an NHWC level (a key's id is never negative).  f32 stores each half as it is
// loaded: loading both halves first, as store_feat8's callers do, makes the compiler schedule this kernel differently
template <int LAYOUT>
__device__ __forceinline__ void gather_key8(void *out, long long pix, const float *tex, long long N, unsigned long long key)
{
    long long id = zbuf_point_id(key);
    if (id >= N) id = N - 1;
    const float4 *t = reinterpret_cast<const float4 *>(tex + id * 8);
    if (LAYOUT == READ_FEAT_NHWC_F32) {
        float4 *o = reinterpret_cast<float4 *>(static_cast<float *>(out) + pix * 8);
        o[0] = __ldg(t);
        o[1] = __ldg(t + 1);
    } else {
        const float4 a = __ldg(t), c = __ldg(t + 1);
        const float v[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
        store_feat8<LAYOUT>(out, pix, 0, v);
    }
}

template <int LAYOUT>
__global__ void __launch_bounds__(256) pyramid_resolve_gather_kernel(const __grid_constant__ FusedArgs a)
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
        gather_key8<LAYOUT>(a.out[0], p0, a.tex, a.N, k.x);
        gather_key8<LAYOUT>(a.out[0], p0 + 1, a.tex, a.N, k.y);
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
            gather_key8<LAYOUT>(a.out[1], p1, a.tex, a.N, m1);
            if ((row & 2) == 0 && (lane & 1) == 0) {
                const int W2 = a.W >> 2, H2 = a.H >> 2;
                const long long p2 = ((long long)b * H2 + (y >> 2)) * W2 + (x >> 2);
                a.z[2][p2] = m2;
                gather_key8<LAYOUT>(a.out[2], p2, a.tex, a.N, m2);
                if (lane == 0) {
                    const int W3 = a.W >> 3, H3 = a.H >> 3;
                    const long long p3 = ((long long)b * H3 + (y >> 3)) * W3 + (x >> 3);
                    a.z[3][p3] = m3;
                    gather_key8<LAYOUT>(a.out[3], p3, a.tex, a.N, m3);
                }
            }
        }
    }
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
    return launch_gather(GatherItems{*table}, ids, h, w, layout, activation, out, st, "gather (items)");
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
    return launch_gather(GatherOne{tex_nd, N, D, B}, ids, h, w, layout, activation, out, (cudaStream_t)stream, "gather");
}

int read_gather_from_index_i32(const float *tex_nd, int D, int64_t N, const int32_t *ids, int B, int h, int w, int layout,
                               int activation, void *out, void *stream)
{
    int rc = check_gather(tex_nd, D, N, ids, B, h, w, out);
    if (rc) return rc;
    return launch_gather(GatherOne{tex_nd, N, D, B}, ids, h, w, layout, activation, out, (cudaStream_t)stream, "gather");
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
    return launch_gather(GatherOne{tex_nd, N, D, B}, reinterpret_cast<const unsigned long long *>(zbuf_level), h, w, layout, activation,
                         out, (cudaStream_t)stream, "gather");
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
    const unsigned ctas = grid_for(32ll * nviews * (W >> 3) * (H >> 3));      // one warp per 8x8 block
    if (layout == READ_FEAT_NHWC_BF16) pyramid_resolve_gather_kernel<READ_FEAT_NHWC_BF16><<<ctas, 256, 0, (cudaStream_t)stream>>>(a);
    else pyramid_resolve_gather_kernel<READ_FEAT_NHWC_F32><<<ctas, 256, 0, (cudaStream_t)stream>>>(a);
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
    const unsigned g = grid_for(total);
    if (act_dtype == READ_ACT_BF16)
        stage_inputs_kernel<__nv_bfloat16><<<g, 256, 0, (cudaStream_t)stream>>>(src, B, hs, ws, C, factor, last, have_last, (__nv_bfloat16 *)dst);
    else
        stage_inputs_kernel<float><<<g, 256, 0, (cudaStream_t)stream>>>(src, B, hs, ws, C, factor, last, have_last, (float *)dst);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"
