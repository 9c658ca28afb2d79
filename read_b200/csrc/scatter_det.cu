// Deterministic descriptor-gradient scatter, the backward of the gather under torch.use_deterministic_algorithms(True)
// (read_b200/texture.py: _Gather, read_b200/train.py: _GatherSparse).  The default kernels (gather.cu: gather_backward_kernel,
// train.cu: gather_backward_sparse_kernel) add every pixel's gradient into its point's row with fp32 atomics, so the order of the
// additions changes from run to run.  Here it is fixed (include/read_b200.h states it for a restatement):
//   keys     key[p] = clamp(id[p], 0, N - 1), value p, for every flat pixel p = (b * h + y) * w + x
//   sort     cub::DeviceRadixSort::SortPairs on the key: a stable sort, so each id's pixels stay in ascending p
//   chunks   the sorted sequence is cut into chunks of SD_CHUNK positions; one thread per (chunk, channel) sums each run of equal
//            ids inside its chunk in sorted order, from 0.  A run that is a whole segment (the id's pixels all lie in this chunk)
//            is added to its row directly; the first and last runs of a chunk, when they belong to a longer segment, are stored
//   combine  the thread of a segment's first chunk adds the segment's chunk sums in chunk order, starting from its own, and adds
//            the result to the row once
// So each row has exactly one writer per call, and the dense (grad_tex_nd) and sparse (grad_nd + touched) forms share the code.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace rb {

constexpr int SD_CHUNK = 128, SD_THREADS = 256;

__global__ void sd_keys_kernel(const float *__restrict__ ids, long long total, long long N, unsigned *__restrict__ key,
                               int *__restrict__ pix)
{
    for (long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
        long long id = (long long)ids[p];
        if (id < 0) id = 0;
        if (id >= N) id = N - 1;
        key[p] = (unsigned)id;
        pix[p] = (int)p;
    }
}

template <bool SPARSE>
__device__ __forceinline__ void sd_add_row(float *out, unsigned char *touched, unsigned id, int D, int c, float s)
{
    out[(long long)id * D + c] += s;
    if (SPARSE && c == 0) touched[id] = 1;
}

// thread (chunk k, channel c): the runs of equal ids in sorted positions [k * SD_CHUNK, (k + 1) * SD_CHUNK)
template <bool SPARSE>
__global__ void __launch_bounds__(SD_THREADS)
sd_chunk_kernel(const float *__restrict__ go, const unsigned *__restrict__ key, const int *__restrict__ pix, long long total,
                int D, long long hw, long long nchunks, float *__restrict__ out, unsigned char *__restrict__ touched,
                float *__restrict__ first, float *__restrict__ last)
{
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nchunks * D; t += (long long)gridDim.x * blockDim.x) {
        const long long k = t / D, i0 = k * SD_CHUNK, i1 = i0 + SD_CHUNK < total ? i0 + SD_CHUNK : total;
        const int c = (int)(t - k * D);
        long long head = i0;
        float s = 0.f;
        unsigned id = key[i0];
        for (long long i = i0; i < i1; ++i) {
            const long long p = pix[i], b = p / hw;
            s += go[(b * D + c) * hw + (p - b * hw)];
            const unsigned nx = i + 1 < total ? key[i + 1] : ~0u;
            if (i + 1 < i1 && nx == id) continue;
            // the run [head, i] ends here: a whole segment, or a piece of one that crosses a chunk boundary
            const bool starts = head > 0 ? key[head - 1] != id : true, ends = nx != id;
            if (starts && ends) {
                sd_add_row<SPARSE>(out, touched, id, D, c, s);
            } else {
                if (head == i0) first[t] = s;
                if (i + 1 == i1) last[t] = s;
            }
            s = 0.f;
            head = i + 1;
            id = nx;
        }
    }
}

// thread (chunk k, channel c): if chunk k holds the first piece of a segment that continues into chunk k + 1, it adds the segment's
// pieces in chunk order and writes the row
template <bool SPARSE>
__global__ void __launch_bounds__(SD_THREADS)
sd_combine_kernel(const unsigned *__restrict__ key, long long total, int D, long long nchunks, const float *__restrict__ first,
                  const float *__restrict__ last, float *__restrict__ out, unsigned char *__restrict__ touched)
{
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < nchunks * D; t += (long long)gridDim.x * blockDim.x) {
        const long long k = t / D, i0 = k * SD_CHUNK, i1 = i0 + SD_CHUNK;
        const int c = (int)(t - k * D);
        if (i1 >= total) continue;
        const unsigned id = key[i1 - 1];
        if (key[i1] != id) continue;                                   // chunk k's last run ends with the chunk
        if (i0 > 0 && key[i0] == id && key[i0 - 1] == id) continue;    // the segment began in an earlier chunk
        long long lo = i1, hi = total;                                 // the segment's end: the first position with a larger key
        while (lo < hi) {
            const long long mid = (lo + hi) / 2;
            if (key[mid] == id) lo = mid + 1;
            else hi = mid;
        }
        const long long kend = (lo - 1) / SD_CHUNK;                    // the segment's last chunk
        float s = last[t];
        for (long long k2 = k + 1; k2 <= kend; ++k2) s += first[k2 * D + c];
        sd_add_row<SPARSE>(out, touched, id, D, c, s);
    }
}

struct SdLayout {
    long long total, nchunks;
    int end_bit;
    size_t key_in, key_out, pix_in, pix_out, first, last, temp, temp_bytes, bytes;
};

static size_t sd_round(size_t n) { return (n + 255) / 256 * 256; }

static bool sd_layout(int B, int D, int h, int w, long long N, SdLayout &L)
{
    if (B < 0 || h < 0 || w < 0 || D < 1 || D > 1024 || N < 1 || N > 0x7FFFFFFFll) return false;
    L.total = (long long)B * h * w;
    if (L.total > 0x7FFFFFFFll) return false;
    L.nchunks = (L.total + SD_CHUNK - 1) / SD_CHUNK;
    L.end_bit = 1;
    while ((1ll << L.end_bit) < N) ++L.end_bit;
    L.temp_bytes = 0;
    if (L.total > 0 && cub::DeviceRadixSort::SortPairs(nullptr, L.temp_bytes, (const unsigned *)nullptr, (unsigned *)nullptr,
                                                       (const int *)nullptr, (int *)nullptr, (int)L.total, 0, L.end_bit) !=
                           cudaSuccess)
        return false;
    const size_t n4 = sd_round((size_t)L.total * 4), c4 = sd_round((size_t)L.nchunks * D * 4);
    L.key_in = 0;
    L.key_out = L.key_in + n4;
    L.pix_in = L.key_out + n4;
    L.pix_out = L.pix_in + n4;
    L.first = L.pix_out + n4;
    L.last = L.first + c4;
    L.temp = L.last + c4;
    L.bytes = L.temp + sd_round(L.temp_bytes);
    return true;
}

static unsigned sd_grid(long long n)
{
    long long blocks = (n + SD_THREADS - 1) / SD_THREADS;
    const long long cap = 16ll * num_sms();
    return (unsigned)(blocks < 1 ? 1 : blocks > cap ? cap : blocks);
}

template <bool SPARSE>
static int sd_run(const float *go, const float *ids, int B, int D, int h, int w, long long N, float *out, unsigned char *touched,
                  void *workspace, cudaStream_t st)
{
    SdLayout L;
    RB_CHECK_ARG(sd_layout(B, D, h, w, N, L), "gather backward (deterministic): bad shape");
    if (L.total == 0) return READ_OK;
    RB_CHECK_ARG((reinterpret_cast<uintptr_t>(workspace) & 15) == 0, "gather backward (deterministic): workspace must be 16B aligned");
    char *ws = (char *)workspace;
    unsigned *key_in = (unsigned *)(ws + L.key_in), *key = (unsigned *)(ws + L.key_out);
    int *pix_in = (int *)(ws + L.pix_in), *pix = (int *)(ws + L.pix_out);
    float *first = (float *)(ws + L.first), *last = (float *)(ws + L.last);
    sd_keys_kernel<<<sd_grid(L.total), SD_THREADS, 0, st>>>(ids, L.total, N, key_in, pix_in);
    RB_LAUNCH_CHECK();
    size_t temp_bytes = L.temp_bytes;
    RB_CUDA(cub::DeviceRadixSort::SortPairs(ws + L.temp, temp_bytes, key_in, key, pix_in, pix, (int)L.total, 0, L.end_bit, st));
    count_launch();
    sd_chunk_kernel<SPARSE><<<sd_grid(L.nchunks * D), SD_THREADS, 0, st>>>(go, key, pix, L.total, D, (long long)h * w, L.nchunks,
                                                                           out, touched, first, last);
    RB_LAUNCH_CHECK();
    sd_combine_kernel<SPARSE><<<sd_grid(L.nchunks * D), SD_THREADS, 0, st>>>(key, L.total, D, L.nchunks, first, last, out, touched);
    RB_LAUNCH_CHECK();
    return READ_OK;
}

}  // namespace rb

using namespace rb;

extern "C" {

int64_t read_gather_backward_det_workspace_bytes(int B, int D, int h, int w, int64_t N)
{
    SdLayout L;
    if (!sd_layout(B, D, h, w, N, L)) return -1;
    return (int64_t)L.bytes;
}

int read_gather_backward_det(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N, float *grad_tex_nd,
                             void *workspace, void *stream)
{
    RB_CHECK_ARG(grad_out && ids && grad_tex_nd && workspace, "gather backward (deterministic): null pointer");
    return sd_run<false>(grad_out, ids, B, D, h, w, N, grad_tex_nd, nullptr, workspace, (cudaStream_t)stream);
}

int read_gather_backward_sparse_det(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N, float *grad_nd,
                                    unsigned char *touched, void *workspace, void *stream)
{
    RB_CHECK_ARG(grad_out && ids && grad_nd && touched && workspace, "gather backward (sparse, deterministic): null pointer");
    return sd_run<true>(grad_out, ids, B, D, h, w, N, grad_nd, touched, workspace, (cudaStream_t)stream);
}

}  // extern "C"
