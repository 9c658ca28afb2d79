/*
 * TEST INFRASTRUCTURE ONLY (tests/oracle_sprite.py compiles it).
 *
 * Point sprites restated on oracle/zbuffer.c's sequential z-buffer (DESIGN.md §4.2).  Per point, in ascending id: the same clip
 * coordinates (dot = fadd(fma(z,m2,fma(y,m1,x*m0)),m3), correctly-rounded fp32 division, NaN culled), the same frustum test, depth
 * d = (cz+1)/2 (a point with d == 0 draws nothing) and centre pixel u = fl(fl(w*fl(cx+1))*0.5), v = fl(fl(h*fl(1-cy))*0.5),
 * xx = (int)u, yy = (int)v; a centre outside the level draws nothing.  Then, per level l:
 *   size = s_i if s_i > 0 else N_l;  relative levels: size = fmaxf(1, size / c2), c2 the clip-space z (fp32 division);
 *   wd = (int)fminf(fmaxf(floorf(size + 0.5), 1), 64);  k = wd / 2;
 *   columns: odd wd: xx-k .. xx+k; even wd: xr-k .. xr+k-1, xr = xx + (u - xx >= 0.5); rows likewise with v / yy;
 *   every covered pixel inside the level keeps the smaller of its key and (depth bits << 32 | id): per pixel the nearest point,
 *   equal depths to the lower id.
 * Built with -ffp-contract=off so only the explicit fmaf() fuse.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define MAX_POINT_SIZE 64

/* z: the L levels one after another, level l as [B, h[l], w[l]] uint64 keys, ~0 = empty (the function fills it). */
void oracle_sprite_project(const float *xyz, int64_t n, const float *Ms, int B, int L, const int *w, const int *h,
                           const float *N, const int *rel, const float *psize, uint64_t *z)
{
    size_t total = 0;
    for (int l = 0; l < L; ++l) total += (size_t)B * w[l] * h[l];
    memset(z, 0xFF, sizeof(uint64_t) * total);
    for (int b = 0; b < B; ++b) {
        const float *M = Ms + 16 * b;
        for (int64_t id = 0; id < n; ++id) {
            const float x = xyz[3 * id + 0], y = xyz[3 * id + 1], zz = xyz[3 * id + 2];
            float c[4];
            for (int r = 0; r < 4; ++r) {
                const float *m = M + 4 * r;
                float t = x * m[0];
                t = fmaf(y, m[1], t);
                t = fmaf(zz, m[2], t);
                c[r] = t + m[3];
            }
            const float cx = c[0] / c[3], cy = c[1] / c[3], cz = c[2] / c[3];
            if (isnan(cx) || isnan(cy) || isnan(cz)) continue;
            if (cx < -1 || cx > 1 || cy < -1 || cy > 1 || cz < -1 || cz > 1) continue;
            const float d = (cz + 1.0f) * 0.5f;
            if (d == 0.0f) continue;
            uint32_t dbits;
            memcpy(&dbits, &d, 4);
            const uint64_t key = ((uint64_t)dbits << 32) | (uint32_t)id;
            size_t off = 0;
            for (int l = 0; l < L; ++l) {
                uint64_t *zl = z + off + (size_t)b * w[l] * h[l];
                off += (size_t)B * w[l] * h[l];
                const float u = ((float)w[l] * (cx + 1.0f)) * 0.5f;
                const float v = ((float)h[l] * (1.0f - cy)) * 0.5f;
                const int xx = (int)u, yy = (int)v;
                if (xx < 0 || xx >= w[l] || yy < 0 || yy >= h[l]) continue;
                float size = (psize && psize[id] > 0.0f) ? psize[id] : N[l];
                if (rel[l]) size = fmaxf(1.0f, size / c[2]);
                const int wd = (int)fminf(fmaxf(floorf(size + 0.5f), 1.0f), (float)MAX_POINT_SIZE);
                const int k = wd / 2;
                const int x0 = (wd & 1) ? xx - k : xx + (u - (float)xx >= 0.5f) - k;
                const int y0 = (wd & 1) ? yy - k : yy + (v - (float)yy >= 0.5f) - k;
                for (int py = y0; py < y0 + wd; ++py) {
                    if (py < 0 || py >= h[l]) continue;
                    for (int px = x0; px < x0 + wd; ++px) {
                        if (px < 0 || px >= w[l]) continue;
                        uint64_t *p = zl + (size_t)py * w[l] + px;
                        if (key < *p) *p = key;
                    }
                }
            }
        }
    }
}
