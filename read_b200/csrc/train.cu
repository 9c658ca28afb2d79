// Descriptor side of the training step (SURVEY.md §8f rank 2, §8e "Training"): the reference back-propagates into PointTexture
// through a dense [D, B*N] index_add_ per pyramid level (READ/models/texture.py:55-63 under autograd) and steps a dense
// torch.optim.RMSprop over all N points (READ/pipelines/ogl.py:16,97-102) - 160-320 MB of gradient and 3 x 320 MB of optimizer
// traffic per step for a few 10^4 visible points.  Here everything past the net's input gradient touches only visible points:
//   gather_backward_sparse   grad[id,:] += dL/dfeat[:, pixel]  (point-major accumulator) and touched[id] = 1
//   gather_backward_items    the same (sparse or dense) for a batch whose items sample different textures: each item's pixels go
//                            to its own texture's accumulator (a batch that mixes scenes in one net call)
//   sparse_rmsprop           for touched points only: lazily decayed square_avg, parameter update written to BOTH the
//                            checkpoint-layout parameter [1,D,N] and its point-major shadow [N,D], gradient row and flag cleared
//   compact / scatter pairs  (id, grad[D]) lists for the data-parallel exchange: ranks all-gather their touched rows instead of
//                            all-reducing dense [N,D] gradients (train.py:138-139 nn.DataParallel broadcasts the whole texture).
// Equivalence with the dense optimizer: RMSprop without momentum moves a parameter only when its gradient is non-zero; a point
// that is not touched only has its square_avg multiplied by alpha each step.  Storing the step of the last update and applying
// alpha^(t - t_last) on the next touch reproduces the dense state exactly (up to the rounding of powf vs repeated products).
#include "common.cuh"

namespace rb {

// IdT: float or int32_t index map (every kernel of this file that reads ids)
template <typename IdT>
__global__ void gather_backward_sparse_kernel(const float *__restrict__ go, const IdT *__restrict__ ids, int B, int D, int h,
                                              int w, long long N, float *__restrict__ gt, unsigned char *__restrict__ touched)
{
    extern __shared__ float zero_acc[];   // [D]: pixels that show point 0 (and every empty pixel) are pre-reduced per block
    for (int c = threadIdx.x; c < D; c += blockDim.x) zero_acc[c] = 0.f;
    __syncthreads();
    const long long hw = (long long)h * w;
    const long long total = (long long)B * hw;
    bool any_zero = false;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        long long id = (long long)ids[p];
        if (id < 0) id = 0;
        if (id >= N) id = N - 1;
        const long long b = p / hw, q = p - b * hw;
        const float *g = go + b * D * hw + q;
        if (id == 0) {
            any_zero = true;
            for (int c = 0; c < D; ++c) atomicAdd(&zero_acc[c], g[c * hw]);
        } else {
            for (int c = 0; c < D; ++c) atomicAdd(gt + id * D + c, g[c * hw]);
            touched[id] = 1;
        }
    }
    const int zero_any = __syncthreads_or(any_zero ? 1 : 0);
    if (zero_any) {
        for (int c = threadIdx.x; c < D; c += blockDim.x) atomicAdd(gt + c, zero_acc[c]);
        if (threadIdx.x == 0) touched[0] = 1;
    }
}

// gather_backward_kernel (SPARSE = false) / gather_backward_sparse_kernel (true) at D == 8 for a batch whose items sample different
// textures: item b's pixels go to slot t.slot[b]'s accumulator.  Point 0 is pre-reduced per block AND per slot (a shared [slot][8]
// accumulator): with one shared row, every empty pixel of one slot's sparse crop would serialise on another's point 0.
template <typename IdT, bool SPARSE>
__global__ void gather_backward_items_kernel(const float *__restrict__ go, const IdT *__restrict__ ids,
                                             const __grid_constant__ read_tex_table t, int h, int w)
{
    __shared__ float zero_acc[READ_MAX_TEX_SLOTS][8];
    __shared__ int zero_any[READ_MAX_TEX_SLOTS];
    for (int i = threadIdx.x; i < READ_MAX_TEX_SLOTS * 8; i += blockDim.x) zero_acc[i >> 3][i & 7] = 0.f;
    for (int i = threadIdx.x; i < READ_MAX_TEX_SLOTS; i += blockDim.x) zero_any[i] = 0;
    __syncthreads();
    const long long hw = (long long)h * w;
    const long long total = (long long)t.n_items * hw;
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        const long long b = p / hw, q = p - b * hw;
        const int s = t.slot[b];
        float *gt = t.grad_nd[s];
        if (gt == nullptr) continue;
        const long long N = t.N[s];
        long long id = (long long)ids[p];
        if (id < 0) id = 0;
        if (id >= N) id = N - 1;
        const float *g = go + b * 8 * hw + q;
        if (id == 0) {
            zero_any[s] = 1;
#pragma unroll
            for (int c = 0; c < 8; ++c) atomicAdd(&zero_acc[s][c], g[c * hw]);
        } else {
#pragma unroll
            for (int c = 0; c < 8; ++c) atomicAdd(gt + id * 8 + c, g[c * hw]);
            if (SPARSE) t.touched[s][id] = 1;
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < t.n_slots * 8; i += blockDim.x) {
        const int s = i >> 3, c = i & 7;
        if (!zero_any[s]) continue;
        atomicAdd(t.grad_nd[s] + c, zero_acc[s][c]);
        if (SPARSE && c == 0) t.touched[s][0] = 1;
    }
}

// L2 regulariser of PointTexture (reg_weight * mean(texture^2)): *out = w * sum(param^2) / numel over the whole [1,D,N] parameter.
// Each thread squares and adds 4 consecutive words in fp32 (one float4) and accumulates those partials in fp64; the CTA's threads
// are combined by a fixed tree in shared memory, the CTAs' sums by the last CTA to finish (counter + fence, as bn_stats_kernel), in
// CTA order.  The grid depends on the device alone, so two calls on the same parameter give the same bits.
constexpr int RL_THREADS = 256;
constexpr int RL_MAX_CTAS = 4096;

__device__ __forceinline__ double rl_block_sum(double v, double *red)
{
    red[threadIdx.x] = v;
    __syncthreads();
#pragma unroll
    for (int s = RL_THREADS / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    return red[0];
}

__global__ void __launch_bounds__(RL_THREADS)
reg_loss_kernel(const float *__restrict__ param, long long numel, double w, float *__restrict__ out, double *__restrict__ part,
                unsigned int *__restrict__ counter)
{
    __shared__ double red[RL_THREADS];
    __shared__ bool last;
    const long long n4 = numel >> 2, stride = (long long)gridDim.x * RL_THREADS;
    const long long tid = blockIdx.x * (long long)RL_THREADS + threadIdx.x;
    const float4 *p4 = reinterpret_cast<const float4 *>(param);
    double acc = 0.0;
#pragma unroll 4
    for (long long v = tid; v < n4; v += stride) {
        const float4 a = __ldcs(p4 + v);
        acc += (double)fmaf(a.w, a.w, fmaf(a.z, a.z, fmaf(a.y, a.y, a.x * a.x)));
    }
    if (tid < (numel & 3)) {                                     // the last numel % 4 words: threads 0.. of CTA 0
        const float x = param[n4 * 4 + tid];
        acc += (double)(x * x);
    }
    const double cta = rl_block_sum(acc, red);
    if (threadIdx.x == 0) part[blockIdx.x] = cta;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    double s = 0.0;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += RL_THREADS) s += __ldcg(part + b);
    const double total = rl_block_sum(s, red);
    if (threadIdx.x == 0) {
        *out = (float)(w * total / (double)numel);
        *counter = 0u;
    }
}

// one thread per point; D <= 16.  D == 8 (the reference's descriptor size) takes a fully unrolled path: the point's 2 + 2 + 8 loads
// (gradient row, square_avg row, 8 channel-major parameter words) are all in flight before the first use - the generic loop below
// made 16 dependent DRAM round trips per touched point and ran slower than the DENSE torch optimizer.
// REG: the step of a texture whose L2 regulariser was back-propagated (read_sparse_rmsprop_step_reg).  Its gradient k * param
// reaches every point, so every point is updated with g = (touched ? acc : 0) + fl(k * param), k read from *reg_coef; the decay
// of the points that were not updated since last_step still applies lazily.
template <bool REG>
__global__ void sparse_rmsprop_kernel(float *__restrict__ param_cn, float *__restrict__ shadow_nd, float *__restrict__ grad_nd,
                                      unsigned char *__restrict__ touched, float *__restrict__ square_avg, int *__restrict__ last_step,
                                      long long N, int D, int step, float lr, float alpha, float eps, float weight_decay,
                                      const float *__restrict__ reg_coef)
{
    const float k = REG ? *reg_coef : 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < N; i += (long long)gridDim.x * blockDim.x) {
        bool t = true;
        if constexpr (REG) {
            t = touched[i] != 0;
            if (t) touched[i] = 0;
        } else {
            if (!touched[i]) continue;
            touched[i] = 0;
        }
        const int dt = step - last_step[i];
        last_step[i] = step;
        const float decay = dt == 1 ? alpha : powf(alpha, (float)dt);
        if (D == 8) {
            float4 *gp = reinterpret_cast<float4 *>(grad_nd + i * 8), *qp = reinterpret_cast<float4 *>(square_avg + i * 8);
            const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
            const float4 g0 = t ? gp[0] : zero, g1 = t ? gp[1] : zero, q0 = qp[0], q1 = qp[1];
            float p[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) p[c] = param_cn[(long long)c * N + i];
            if (t) {
                gp[0] = make_float4(0.f, 0.f, 0.f, 0.f);
                gp[1] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
            float q[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                if (REG) g[c] = __fadd_rn(g[c], __fmul_rn(k, p[c]));          // two roundings, as autograd's sum of the two terms
                if (weight_decay != 0.f) g[c] = fmaf(weight_decay, p[c], g[c]);
                q[c] = fmaf(decay, q[c], (1.f - alpha) * g[c] * g[c]);
                p[c] -= lr * g[c] / (sqrtf(q[c]) + eps);
                param_cn[(long long)c * N + i] = p[c];
            }
            qp[0] = make_float4(q[0], q[1], q[2], q[3]);
            qp[1] = make_float4(q[4], q[5], q[6], q[7]);
            if (shadow_nd) {
                float4 *sp = reinterpret_cast<float4 *>(shadow_nd + i * 8);
                sp[0] = make_float4(p[0], p[1], p[2], p[3]);
                sp[1] = make_float4(p[4], p[5], p[6], p[7]);
            }
            continue;
        }
        for (int c = 0; c < D; ++c) {
            float g = t ? grad_nd[i * D + c] : 0.f;
            if (t) grad_nd[i * D + c] = 0.f;
            float p = param_cn[(long long)c * N + i];
            if (REG) g = __fadd_rn(g, __fmul_rn(k, p));
            if (weight_decay != 0.f) g = fmaf(weight_decay, p, g);
            // torch.optim.RMSprop (momentum 0, not centered): sq = alpha sq + (1 - alpha) g^2; p -= lr g / (sqrt(sq) + eps)
            const float sq = fmaf(decay, square_avg[i * D + c], (1.f - alpha) * g * g);
            square_avg[i * D + c] = sq;
            p -= lr * g / (sqrtf(sq) + eps);
            param_cn[(long long)c * N + i] = p;
            if (shadow_nd) shadow_nd[i * D + c] = p;
        }
    }
}

// square_avg as the dense optimizer would hold it after `step` steps (checkpoints / state_dict)
__global__ void square_avg_materialize_kernel(const float *__restrict__ square_avg, const int *__restrict__ last_step, long long N,
                                              int D, int step, float alpha, float *__restrict__ out_cn)
{
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < N; i += (long long)gridDim.x * blockDim.x) {
        const int dt = step - last_step[i];
        const float decay = dt <= 0 ? 1.f : powf(alpha, (float)dt);
        for (int c = 0; c < D; ++c) out_cn[(long long)c * N + i] = decay * square_avg[i * D + c];
    }
}

// touched rows -> (id, grad[D]) pairs, order unspecified; *count receives the number of pairs (must be zeroed by the caller)
__global__ void compact_touched_kernel(const float *__restrict__ grad_nd, const unsigned char *__restrict__ touched, long long N, int D,
                                       int *__restrict__ count, int capacity, int *__restrict__ out_ids, float *__restrict__ out_grads)
{
    const int lane = threadIdx.x & 31;
    const long long stride = (long long)gridDim.x * blockDim.x;
    const long long n_round = ((N + stride - 1) / stride) * stride;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_round; i += stride) {
        const bool t = i < N && touched[i];
        const unsigned m = __ballot_sync(0xFFFFFFFFu, t);
        if (m == 0) continue;
        int base = 0;
        if (lane == 0) base = atomicAdd(count, __popc(m));
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (t) {
            const int k = base + __popc(m & ((1u << lane) - 1u));
            if (k < capacity) {
                out_ids[k] = (int)i;
                for (int c = 0; c < D; ++c) out_grads[(long long)k * D + c] = grad_nd[i * D + c];
            }
        }
    }
}

__global__ void scatter_pairs_kernel(const int *__restrict__ ids, const float *__restrict__ grads, int n, int D, long long N,
                                     float *__restrict__ grad_nd, unsigned char *__restrict__ touched)
{
    for (long long j = blockIdx.x * (long long)blockDim.x + threadIdx.x; j < (long long)n * D; j += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(j / D), c = (int)(j - (long long)k * D);
        const int id = ids[k];
        if (id < 0 || id >= N) continue;
        atomicAdd(grad_nd + (long long)id * D + c, grads[j]);
        if (c == 0) touched[id] = 1;
    }
}

static unsigned tgrid(long long total)
{
    long long blocks = (total + 255) / 256;
    const long long cap = (long long)num_sms() * 16;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return (unsigned)blocks;
}

template <typename IdT, bool SPARSE>
static int gather_backward_items(const float *grad_out, const IdT *ids, const read_tex_table *table, int h, int w, void *stream,
                                 const char *what)
{
    int rc = check_tex_table(table, h, w, false, SPARSE, what);
    if (rc) return rc;
    RB_CHECK_ARG(grad_out && ids, "%s: null pointer", what);
    const long long total = (long long)table->n_items * h * w;
    if (total == 0) return READ_OK;
    gather_backward_items_kernel<IdT, SPARSE><<<tgrid(total), 256, 0, (cudaStream_t)stream>>>(grad_out, ids, *table, h, w);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

template <typename IdT>
static int gather_backward_sparse(const float *grad_out, const IdT *ids, int B, int D, int h, int w, int64_t N, float *grad_nd,
                                  unsigned char *touched, cudaStream_t st)
{
    RB_CHECK_ARG(grad_out && ids && grad_nd && touched, "gather backward (sparse): null pointer");
    RB_CHECK_ARG(D >= 1 && D <= 1024 && N >= 1 && B >= 0 && h >= 0 && w >= 0, "gather backward (sparse): bad shape");
    const long long total = (long long)B * h * w;
    if (total == 0) return READ_OK;
    gather_backward_sparse_kernel<IdT><<<tgrid(total), 256, D * sizeof(float), st>>>(grad_out, ids, B, D, h, w, N, grad_nd, touched);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb

using namespace rb;

extern "C" {

int read_gather_backward_sparse(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N,
                                float *grad_nd, unsigned char *touched, void *stream)
{
    return gather_backward_sparse<float>(grad_out, ids, B, D, h, w, N, grad_nd, touched, (cudaStream_t)stream);
}

int read_gather_backward_sparse_i32(const float *grad_out, const int32_t *ids, int B, int D, int h, int w, int64_t N, float *grad_nd,
                                    unsigned char *touched, void *stream)
{
    return gather_backward_sparse<int32_t>(grad_out, ids, B, D, h, w, N, grad_nd, touched, (cudaStream_t)stream);
}

int read_gather_backward_items(const float *grad_out, const float *ids, const read_tex_table *table, int h, int w, void *stream)
{
    return gather_backward_items<float, false>(grad_out, ids, table, h, w, stream, "gather backward (items)");
}

int read_gather_backward_items_i32(const float *grad_out, const int32_t *ids, const read_tex_table *table, int h, int w, void *stream)
{
    return gather_backward_items<int32_t, false>(grad_out, ids, table, h, w, stream, "gather backward (items)");
}

int read_gather_backward_sparse_items(const float *grad_out, const float *ids, const read_tex_table *table, int h, int w,
                                      void *stream)
{
    return gather_backward_items<float, true>(grad_out, ids, table, h, w, stream, "gather backward (sparse, items)");
}

int read_gather_backward_sparse_items_i32(const float *grad_out, const int32_t *ids, const read_tex_table *table, int h, int w,
                                          void *stream)
{
    return gather_backward_items<int32_t, true>(grad_out, ids, table, h, w, stream, "gather backward (sparse, items)");
}

int read_sparse_rmsprop_step(float *param_cn, float *shadow_nd, float *grad_nd, unsigned char *touched, float *square_avg,
                             int32_t *last_step, int64_t N, int D, int step, float lr, float alpha, float eps, float weight_decay,
                             void *stream)
{
    RB_CHECK_ARG(param_cn && grad_nd && touched && square_avg && last_step, "sparse rmsprop: null pointer");
    RB_CHECK_ARG(N >= 1 && D >= 1 && D <= 16 && step >= 1, "sparse rmsprop: bad shape / step");
    sparse_rmsprop_kernel<false><<<tgrid(N), 256, 0, (cudaStream_t)stream>>>(param_cn, shadow_nd, grad_nd, touched, square_avg, last_step,
                                                                             N, D, step, lr, alpha, eps, weight_decay, nullptr);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_sparse_rmsprop_step_reg(float *param_cn, float *shadow_nd, float *grad_nd, unsigned char *touched, float *square_avg,
                                 int32_t *last_step, int64_t N, int D, int step, float lr, float alpha, float eps, float weight_decay,
                                 const float *reg_coef, void *stream)
{
    RB_CHECK_ARG(param_cn && grad_nd && touched && square_avg && last_step && reg_coef, "sparse rmsprop (reg): null pointer");
    RB_CHECK_ARG(N >= 1 && D >= 1 && D <= 16 && step >= 1, "sparse rmsprop (reg): bad shape / step");
    sparse_rmsprop_kernel<true><<<tgrid(N), 256, 0, (cudaStream_t)stream>>>(param_cn, shadow_nd, grad_nd, touched, square_avg, last_step,
                                                                            N, D, step, lr, alpha, eps, weight_decay, reg_coef);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int64_t read_reg_loss_workspace_bytes(int D, int64_t N)
{
    if (D < 1 || D > 16 || N < 1) return -1;
    return 256 + (int64_t)RL_MAX_CTAS * (int64_t)sizeof(double);
}

int read_reg_loss(const float *param_cn, int D, int64_t N, double reg_weight, float *out, void *workspace, void *stream)
{
    RB_CHECK_ARG(param_cn && out && workspace, "reg_loss: null pointer");
    RB_CHECK_ARG(N >= 1 && D >= 1 && D <= 16, "reg_loss: bad shape (D %d, N %lld)", D, (long long)N);
    RB_CHECK_ARG(((reinterpret_cast<uintptr_t>(param_cn) | reinterpret_cast<uintptr_t>(workspace)) & 15) == 0,
                 "reg_loss: param and workspace must be 16B aligned");
    const long long numel = (long long)D * N;
    long long blocks = ((numel >> 2) + RL_THREADS - 1) / RL_THREADS;
    const long long cap = 8ll * num_sms() < RL_MAX_CTAS ? 8ll * num_sms() : RL_MAX_CTAS;
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    const cudaStream_t st = (cudaStream_t)stream;
    unsigned int *counter = (unsigned int *)workspace;
    RB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned int), st));
    reg_loss_kernel<<<(unsigned)blocks, RL_THREADS, 0, st>>>(param_cn, numel, reg_weight, out, (double *)((char *)workspace + 256),
                                                            counter);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_square_avg_dense(const float *square_avg, const int32_t *last_step, int64_t N, int D, int step, float alpha, float *out_cn,
                          void *stream)
{
    RB_CHECK_ARG(square_avg && last_step && out_cn && N >= 1 && D >= 1, "square_avg_dense: bad arguments");
    square_avg_materialize_kernel<<<tgrid(N), 256, 0, (cudaStream_t)stream>>>(square_avg, last_step, N, D, step, alpha, out_cn);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_compact_touched(const float *grad_nd, const unsigned char *touched, int64_t N, int D, int32_t *count, int capacity,
                         int32_t *out_ids, float *out_grads, void *stream)
{
    RB_CHECK_ARG(grad_nd && touched && count && out_ids && out_grads && N >= 1 && D >= 1 && capacity >= 0, "compact_touched: bad arguments");
    compact_touched_kernel<<<tgrid(N), 256, 0, (cudaStream_t)stream>>>(grad_nd, touched, N, D, count, capacity, out_ids, out_grads);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

int read_scatter_pairs(const int32_t *ids, const float *grads, int n, int D, int64_t N, float *grad_nd, unsigned char *touched,
                       void *stream)
{
    RB_CHECK_ARG(n >= 0 && D >= 1 && N >= 1, "scatter_pairs: bad arguments");
    if (n == 0) return READ_OK;
    RB_CHECK_ARG(ids && grads && grad_nd && touched, "scatter_pairs: null pointer");
    scatter_pairs_kernel<<<tgrid((long long)n * D), 256, 0, (cudaStream_t)stream>>>(ids, grads, n, D, N, grad_nd, touched);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // extern "C"
