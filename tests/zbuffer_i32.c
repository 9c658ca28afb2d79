/*
 * TEST INFRASTRUCTURE ONLY (tests/oracle_i32.py compiles it).
 *
 * oracle/zbuffer.c's oracle_pcpr_forward with int32 ids, for clouds of more than 2^24 + 1 points, whose ids a float32 index map
 * cannot all hold: the same sequential z-buffer (ascending id, per pixel the minimum depth, tie -> lowest id, empty -> index 0 /
 * depth 0) with the same arithmetic (SURVEY.md §8 a3': dot = fadd(fma(z,m2,fma(y,m1,x*m0)),m3), correctly-rounded fp32 division,
 * u = fl(fl(W*fl(x+1))*0.5), int() truncates; built with -ffp-contract=off so only the explicit fmaf() fuse), the same culling of
 * NaN clip coordinates, and the index written as int32.  tests/test_large_scene_host.py pins it to the float oracle wherever
 * float32 holds the ids.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* B views: index [B,h,w] int32, depth [B,h,w] f32; M [B,16] row-major. */
void oracle_pcpr_forward_i32(const float *xyz, int64_t n, const float *Ms, int B, int w, int h, int32_t *index_all,
                             float *depth_all)
{
    for (int b = 0; b < B; ++b) {
        const float *M = Ms + 16 * b;
        int32_t *index = index_all + (size_t)b * w * h;
        float *depth = depth_all + (size_t)b * w * h;
        memset(index, 0, sizeof(int32_t) * (size_t)w * h);
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
            if (isnan(cx) || isnan(cy) || isnan(cz)) continue;
            if (cx < -1 || cx > 1 || cy < -1 || cy > 1 || cz < -1 || cz > 1) continue;
            const float u = ((float)w * (cx + 1.0f)) * 0.5f;
            const float v = ((float)h * (1.0f - cy)) * 0.5f;
            const float d = (cz + 1.0f) * 0.5f;
            const int xx = (int)u, yy = (int)v;
            if (xx < 0 || xx >= w || yy < 0 || yy >= h) continue;
            const size_t ind = (size_t)yy * w + xx;
            if (depth[ind] > d || depth[ind] == 0.0f) {
                depth[ind] = d;
                index[ind] = (int32_t)id;
            }
        }
    }
}
