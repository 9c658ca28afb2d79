/*
 * ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product path.
 *
 * CPU restatement of the reference rasterizer (the only CUDA kernel in
 * JOP-Lee/READ), evaluated SEQUENTIALLY in ascending point id, which is the
 * deterministic z-buffer the reference intends (and which its OpenGL variant
 * implements: GL_LESS depth test, points drawn in id order,
 * READ/gl/render.py:55-70).
 *
 * Follows, line for line in meaning:
 *   MyRender/CloudProjection/point_render.cu:107-122  math::MatrixMul (M*p, divide by w)
 *   MyRender/CloudProjection/point_render.cu:125-167  DepthProject (cull, pixel map, z rule)
 *   MyRender/CloudProjection/point_render.cu:169-200  GPU_PCPR (zeroed [B,h,w] float outputs)
 *
 * Arithmetic order is the one nvcc emits for the reference kernel
 * (SURVEY.md §8 a3'):  dot(row,(x,y,z,1)) = fadd(fma(z,m2,fma(y,m1,x*m0)),m3);
 * correctly-rounded fp32 division; u = fl(fl(W*fl(x+1))*0.5); int() truncates.
 * Build with -ffp-contract=off so the compiler adds no contraction of its own;
 * every fused op below is an explicit fmaf().
 *
 * Parity status: the reference ships no golden vectors for this path
 * (SURVEY.md §4) — "parity unpinned" by reference tests; this restatement is
 * pinned by hand-derived known-answer tests (tests/test_oracle_kat.py) and
 * against the recorded outputs of the reference extension built from source
 * (tests/golden/ref_pcpr_*.npz) on collision-free scenes.
 *
 * Documented deviations from a literal execution of the racy reference kernel:
 *   - NaN clip coordinates (w == 0 and numerator 0) are culled; the reference
 *     would pass the cull (all comparisons false) and F2I(NaN)=0 lands them in
 *     pixel (0,0).  Callers/tests avoid this measure-zero case.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* One view, one level.  index/depth: [h*w] float, caller-zeroed or not (we zero). */
void oracle_depth_project(const float *xyz, int64_t n, const float *M /*16, row-major*/,
                          int w, int h, float *index, float *depth)
{
    memset(index, 0, sizeof(float) * (size_t)w * h);
    memset(depth, 0, sizeof(float) * (size_t)w * h);
    for (int64_t id = 0; id < n; ++id) {
        const float x = xyz[3 * id + 0], y = xyz[3 * id + 1], z = xyz[3 * id + 2];
        float c[4];
        for (int r = 0; r < 4; ++r) {
            const float *m = M + 4 * r;
            float t = x * m[0];
            t = fmaf(y, m[1], t);
            t = fmaf(z, m[2], t);
            c[r] = t + m[3];
        }
        const float cx = c[0] / c[3], cy = c[1] / c[3], cz = c[2] / c[3];
        if (isnan(cx) || isnan(cy) || isnan(cz)) continue;            /* documented deviation */
        if (cx < -1 || cx > 1 || cy < -1 || cy > 1 || cz < -1 || cz > 1) continue; /* :139 */
        const float u = ((float)w * (cx + 1.0f)) * 0.5f;               /* :141 */
        const float v = ((float)h * (1.0f - cy)) * 0.5f;               /* :142 */
        const float d = (cz + 1.0f) * 0.5f;                            /* :143 */
        const int xx = (int)u, yy = (int)v;                            /* :145-146 trunc */
        if (xx < 0 || xx >= w || yy < 0 || yy >= h) continue;          /* :147 */
        const size_t ind = (size_t)yy * w + xx;
        if (depth[ind] > d || depth[ind] == 0.0f) {                    /* :155 */
            depth[ind] = d;
            index[ind] = (float)id;                                    /* :158, 0 denotes empty */
        }
    }
}

/* B views: index/depth [B,h,w]; M [B,16].  point_render.cu:186-192 (serial loop over b). */
void oracle_pcpr_forward(const float *xyz, int64_t n, const float *M, int B,
                         int w, int h, float *index, float *depth)
{
    for (int b = 0; b < B; ++b)
        oracle_depth_project(xyz, n, M + 16 * b, w, h,
                             index + (size_t)b * w * h, depth + (size_t)b * w * h);
}

/* Count of points that are exactly on the near plane after projection (d == 0) or NaN:
 * the cases where sequential reference semantics are degenerate; tests assert 0. */
int64_t oracle_count_degenerate(const float *xyz, int64_t n, const float *M)
{
    int64_t cnt = 0;
    for (int64_t id = 0; id < n; ++id) {
        const float x = xyz[3 * id + 0], y = xyz[3 * id + 1], z = xyz[3 * id + 2];
        float c[4];
        for (int r = 0; r < 4; ++r) {
            const float *m = M + 4 * r;
            float t = x * m[0];
            t = fmaf(y, m[1], t);
            t = fmaf(z, m[2], t);
            c[r] = t + m[3];
        }
        const float cx = c[0] / c[3], cy = c[1] / c[3], cz = c[2] / c[3];
        if (isnan(cx) || isnan(cy) || isnan(cz)) { ++cnt; continue; }
        if (cx < -1 || cx > 1 || cy < -1 || cy > 1 || cz < -1 || cz > 1) continue;
        if ((cz + 1.0f) * 0.5f == 0.0f) ++cnt;
    }
    return cnt;
}
