// Point-cloud views (include/read_b200.h, read_point_view; DESIGN.md §4.3): the colour of each pixel's winning point from its own
// attributes, as the reference viewer's non-neural path draws it.  One thread per output pixel: an 8-byte key load, the rows of
// the winning point the mode reads, one 16-byte store.
#include "common.cuh"

namespace rb {
namespace {

__device__ __forceinline__ float half_of(float v) { return __fadd_rn(__fmul_rn(v, 0.5f), 0.5f); }

__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2)
{
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

__device__ __forceinline__ float3 normalize3(float v0, float v1, float v2)
{
    const float s = __fsqrt_rn(dot3(v0, v1, v2, v0, v1, v2));
    return make_float3(__fdiv_rn(v0, s), __fdiv_rn(v1, s), __fdiv_rn(v2, s));
}

__device__ __forceinline__ float4 half_rgb(float3 v) { return make_float4(half_of(v.x), half_of(v.y), half_of(v.z), 1.f); }

__device__ __forceinline__ float3 position(const float *__restrict__ xyz, long long id)
{
    return make_float3(__ldg(xyz + 3 * id), __ldg(xyz + 3 * id + 1), __ldg(xyz + 3 * id + 2));
}

// the colour of point `id` (key id `raw`, unclamped) under MODE
template <int MODE>
__device__ __forceinline__ float4 shade(const read_point_view_desc &d, long long id, unsigned raw)
{
    if constexpr (MODE == READ_VIEW_COLOR) {
        const float4 c = __ldg(reinterpret_cast<const float4 *>(d.colors) + id);
        return make_float4(c.x, c.y, c.z, 1.f);
    } else if constexpr (MODE == READ_VIEW_NORMALS) {
        const float4 n = __ldg(reinterpret_cast<const float4 *>(d.normals) + id);
        switch (d.submode) {
        case 0:
            return half_rgb(make_float3(n.x, n.y, n.z));
        case 1: {
            const float3 p = position(d.xyz, id);
            const float3 v = normalize3(__fsub_rn(d.cam[0], p.x), __fsub_rn(d.cam[1], p.y), __fsub_rn(d.cam[2], p.z));
            const float k = __fmul_rn(2.f, dot3(n.x, n.y, n.z, v.x, v.y, v.z));
            return half_rgb(normalize3(__fsub_rn(v.x, __fmul_rn(k, n.x)), __fsub_rn(v.y, __fmul_rn(k, n.y)),
                                       __fsub_rn(v.z, __fmul_rn(k, n.z))));
        }
        case 2: {
            const float w0 = __fadd_rn(d.cam[0], n.x), w1 = __fadd_rn(d.cam[1], n.y), w2 = __fadd_rn(d.cam[2], n.z);
            const float *m = d.m_view;
            return half_rgb(normalize3(__fadd_rn(dot3(m[0], m[1], m[2], w0, w1, w2), m[3]),
                                       __fadd_rn(dot3(m[4], m[5], m[6], w0, w1, w2), m[7]),
                                       __fadd_rn(dot3(m[8], m[9], m[10], w0, w1, w2), m[11])));
        }
        case 3: {
            const float3 p = position(d.xyz, id);
            return half_rgb(normalize3(__fsub_rn(d.cam[0], p.x), __fsub_rn(d.cam[1], p.y), __fsub_rn(d.cam[2], p.z)));
        }
        default:
            return make_float4(n.x, n.y, n.z, 1.f);
        }
    } else if constexpr (MODE == READ_VIEW_DEPTH) {
        const float3 p = position(d.xyz, id);
        const float *m = d.total_m;
        const float c2 = __fadd_rn(__fmaf_rn(p.z, m[10], __fmaf_rn(p.y, m[9], __fmul_rn(p.x, m[8]))), m[11]);
        return make_float4(c2, c2, c2, 1.f);
    } else if constexpr (MODE == READ_VIEW_UV) {
        return make_float4(d.submode == 0 ? __uint2float_rn(raw) : 0.f, 0.f, 0.f, 1.f);
    } else if constexpr (MODE == READ_VIEW_XYZ) {
        const float3 p = position(d.xyz, id);
        return make_float4(__fdiv_rn(__fsub_rn(p.x, d.lo[0]), __fadd_rn(__fsub_rn(d.hi[0], d.lo[0]), 1e-9f)),
                           __fdiv_rn(__fsub_rn(p.y, d.lo[1]), __fadd_rn(__fsub_rn(d.hi[1], d.lo[1]), 1e-9f)),
                           __fdiv_rn(__fsub_rn(p.z, d.lo[2]), __fadd_rn(__fsub_rn(d.hi[2], d.lo[2]), 1e-9f)), 1.f);
    } else {
        static_assert(MODE == READ_VIEW_LABEL, "unknown view mode");
        return make_float4(__fdiv_rn(__ldg(d.normals + 4 * id), 255.f), 0.f, 0.f, 1.f);
    }
}

}  // namespace

template <int MODE>
__global__ void __launch_bounds__(256) point_view_kernel(const unsigned long long *__restrict__ zbuf, int H, int W,
                                                         const read_point_view_desc d, float4 *__restrict__ out)
{
    const long long i = blockIdx.x * 256ll + threadIdx.x;
    if (i >= (long long)H * W) return;
    const int y = (int)(i / W), x = (int)(i - (long long)y * W);
    const int ys = d.flip_vertical ? H - 1 - y : y;
    const unsigned long long key = __ldg(zbuf + (long long)ys * W + x);
    float4 c;
    if (key == ZBUF_EMPTY) {
        c = make_float4(d.clear[0], d.clear[1], d.clear[2], d.clear[3]);
    } else {
        const unsigned raw = (unsigned)key;
        const long long id = raw < d.n ? (long long)raw : d.n - 1;
        c = shade<MODE>(d, id, raw);
    }
    out[i] = c;
}

template <int MODE>
static void launch(const uint64_t *zbuf, int H, int W, const read_point_view_desc &d, float *out, cudaStream_t s)
{
    const long long n = (long long)H * W;
    point_view_kernel<MODE><<<(unsigned)((n + 255) / 256), 256, 0, s>>>(
        reinterpret_cast<const unsigned long long *>(zbuf), H, W, d, reinterpret_cast<float4 *>(out));
}

}  // namespace rb

using namespace rb;

extern "C" int read_point_view(const uint64_t *zbuf_level0, int H, int W, const read_point_view_desc *desc, float *out_hwc4,
                               void *stream)
{
    RB_CHECK_ARG(zbuf_level0 && desc && out_hwc4 && H >= 0 && W >= 0, "point_view: bad arguments");
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(out_hwc4) & 15) == 0, "point_view: output must be 16-byte aligned");
    const read_point_view_desc &d = *desc;
    RB_CHECK_ARG(d.mode >= READ_VIEW_COLOR && d.mode <= READ_VIEW_LABEL, "point_view: unknown mode %d", d.mode);
    RB_CHECK_ARG(d.submode >= 0 && d.submode <= 4, "point_view: submode %d not in 0..4", d.submode);
    const bool colors = d.mode == READ_VIEW_COLOR;
    const bool normals = d.mode == READ_VIEW_NORMALS || d.mode == READ_VIEW_LABEL;
    const bool xyz = d.mode == READ_VIEW_DEPTH || d.mode == READ_VIEW_XYZ ||
                     (d.mode == READ_VIEW_NORMALS && (d.submode == 1 || d.submode == 3));
    RB_CHECK_ARG(!(colors || normals || xyz) || d.n >= 1, "point_view: the mode reads a table of n >= 1 rows");
    RB_CHECK_ARG(!colors || (d.colors && (reinterpret_cast<uintptr_t>(d.colors) & 15) == 0),
                 "point_view: colors must be non-null and 16-byte aligned");
    RB_CHECK_ARG(!normals || (d.normals && (reinterpret_cast<uintptr_t>(d.normals) & 15) == 0),
                 "point_view: normals must be non-null and 16-byte aligned");
    RB_CHECK_ARG(!xyz || d.xyz, "point_view: xyz must be non-null");
    RB_CHECK_ARG((long long)H * W < (1ll << 31) * 256, "point_view: view too large");
    if ((long long)H * W == 0) return READ_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    switch (d.mode) {
    case READ_VIEW_COLOR: launch<READ_VIEW_COLOR>(zbuf_level0, H, W, d, out_hwc4, s); break;
    case READ_VIEW_NORMALS: launch<READ_VIEW_NORMALS>(zbuf_level0, H, W, d, out_hwc4, s); break;
    case READ_VIEW_DEPTH: launch<READ_VIEW_DEPTH>(zbuf_level0, H, W, d, out_hwc4, s); break;
    case READ_VIEW_UV: launch<READ_VIEW_UV>(zbuf_level0, H, W, d, out_hwc4, s); break;
    case READ_VIEW_XYZ: launch<READ_VIEW_XYZ>(zbuf_level0, H, W, d, out_hwc4, s); break;
    default: launch<READ_VIEW_LABEL>(zbuf_level0, H, W, d, out_hwc4, s); break;
    }
    RB_LAUNCH_CHECK();
    return READ_OK;
}
