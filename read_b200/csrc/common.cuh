// Shared helpers for the read_b200 CUDA library (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/read_b200.h"

namespace rb {

void set_error(const char *fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int num_sms();
// grid of a grid-stride kernel over n items in blocks of 256 threads: one item per thread, at most 16 blocks per SM
inline unsigned grid_for(long long n)
{
    const long long blocks = (n + 255) / 256, cap = 16ll * num_sms();
    return (unsigned)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}
// channel counts of the train-mode BatchNorm entry points (bn_train.cu, conv_bwd.cu): the gate backward's, without 48
inline bool bn_channels_ok(int C) { return C == 16 || C == 32 || C == 64 || (C % 64 == 0 && C > 0 && C <= 256); }

#define RB_CHECK_ARG(cond, ...)                        \
    do {                                               \
        if (!(cond)) {                                 \
            rb::set_error(__VA_ARGS__);                \
            return READ_ERR_INVALID;                   \
        }                                              \
    } while (0)

#define RB_CUDA(call)                                                                          \
    do {                                                                                       \
        cudaError_t e__ = (call);                                                              \
        if (e__ != cudaSuccess) {                                                              \
            rb::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,                 \
                          cudaGetErrorString(e__));                                            \
            return READ_ERR_CUDA;                                                              \
        }                                                                                      \
    } while (0)

#define RB_LAUNCH_CHECK()                                                                      \
    do {                                                                                       \
        cudaError_t e__ = cudaPeekAtLastError();                                               \
        if (e__ != cudaSuccess) {                                                              \
            rb::set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,             \
                          cudaGetErrorString(e__));                                            \
            (void)cudaGetLastError();                                                          \
            return READ_ERR_CUDA;                                                              \
        }                                                                                      \
        rb::count_launch();                                                                    \
    } while (0)

// shared argument checks of the multi-texture gather entry points (read_tex_table, include/read_b200.h)
inline int check_tex_table(const read_tex_table *t, int h, int w, bool forward, bool sparse, const char *what)
{
    RB_CHECK_ARG(t != nullptr, "%s: null table", what);
    RB_CHECK_ARG(t->n_slots >= 1 && t->n_slots <= READ_MAX_TEX_SLOTS, "%s: n_slots %d not in 1..%d", what, t->n_slots,
                 READ_MAX_TEX_SLOTS);
    RB_CHECK_ARG(t->n_items >= 1 && t->n_items <= READ_MAX_TEX_ITEMS, "%s: n_items %d not in 1..%d", what, t->n_items,
                 READ_MAX_TEX_ITEMS);
    RB_CHECK_ARG(h >= 0 && w >= 0, "%s: bad shape", what);
    for (int b = 0; b < t->n_items; ++b) RB_CHECK_ARG(t->slot[b] < t->n_slots, "%s: item %d maps to slot %d", what, b, t->slot[b]);
    for (int s = 0; s < t->n_slots; ++s) {
        RB_CHECK_ARG(t->N[s] >= 1, "%s: slot %d has no points", what, s);
        if (forward)
            RB_CHECK_ARG(t->tex_nd[s] && (reinterpret_cast<uintptr_t>(t->tex_nd[s]) & 15) == 0,
                         "%s: slot %d: descriptors must be non-null and 16B aligned", what, s);
        else if (sparse)
            RB_CHECK_ARG(!t->grad_nd[s] || t->touched[s], "%s: slot %d: an accumulator without touched flags", what, s);
    }
    return READ_OK;
}

// max positive int64: larger than any real key (depth bits <= 0x3F800000) under BOTH signed and unsigned
// comparison, so a min-reduction may be typed int64 (torch.distributed / ncclInt64) or uint64.
static constexpr unsigned long long ZBUF_EMPTY = 0x7FFFFFFFFFFFFFFFull;
// the point a key names: its low 32 bits, and point 0 for an empty pixel (the reference's index maps hold 0 there)
__device__ __forceinline__ unsigned zbuf_point_id(unsigned long long key) { return key == ZBUF_EMPTY ? 0u : (unsigned)key; }

struct LevelGeom {
    int w[READ_MAX_LEVELS], h[READ_MAX_LEVELS];
    long long off[READ_MAX_LEVELS];   // entry offset of level l (all B views)
    long long total;
};
inline LevelGeom level_geom(int B, int W, int H, int L)
{
    LevelGeom g{};
    long long o = 0;
    double s = 1.0;
    for (int l = 0; l < L; ++l) {
        g.w[l] = (int)(W * s);   // int(W*0.5**l), myrender.py:33
        g.h[l] = (int)(H * s);
        g.off[l] = o;
        o += (long long)B * g.w[l] * g.h[l];
        s *= 0.5;
    }
    g.total = o;
    return g;
}

// activation storage helpers
template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

}  // namespace rb
