/*
 * read_b200 — C ABI of the H100-native (sm_90a) READ render hot path.
 *
 * Plain C: pointers, sizes, ints.  No torch / C++ types cross this boundary.
 * All data pointers are CALLER-OWNED DEVICE memory unless a parameter is named
 * `*_host`.  Every launch is asynchronous on the caller's stream (`stream` is a
 * cudaStream_t passed as void*); no entry point synchronises the device,
 * allocates per call, or touches the host copy of the data.
 *
 * Return value: 0 on success, negative error code otherwise;
 * read_last_error() returns a thread-local message (the Python host raises
 * RuntimeError with it, matching the reference's AT_ASSERTM -> RuntimeError
 * behaviour, pcpr_cuda.cpp:17-21).
 *
 * Which reference interface each entry point replaces is cited per function
 * (paths relative to the JOP-Lee/READ tree).
 */
#ifndef READ_B200_H
#define READ_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define READ_MAX_LEVELS 8
#define READ_MAX_SRC 4

enum {
    READ_OK = 0,
    READ_ERR_INVALID = -1,   /* bad argument (shape, alignment, null)            */
    READ_ERR_CUDA = -2,      /* CUDA runtime / driver error, see read_last_error */
    READ_ERR_UNSUPPORTED = -3
};

int read_version(void);
const char *read_last_error(void);
/* Tuning options.  Results are bit-identical for every accepted setting; unknown names and out-of-range values are rejected.
 *   rasterizer: "raster_pipelined" (1), "raster_bulk_tma" (1), "raster_mode" (0..3, default 2), "raster_occupancy" (0 = auto), "raster_stream" (1),
 *               "raster_dedup" (0), "raster_run" (0 = auto), "raster_nbr_filter" (0), "raster_stages" (2; 3 = deeper point ring),
 *               "raster_carveout" (45: preferred shared-memory carveout in percent for the streaming kernel, -1 = driver default)
 *   convs:      read at launch: "tc_pdl" (1: programmatic dependent launch between consecutive conv kernels)
 *   The Python host applies READ_B200_OPTIONS="name=value,..." from the environment when it loads the library.
 * The options are process-wide tuning state (plain ints): set them before creating plans / launching, not concurrently with
 * launches from other threads.  Diagnostic knobs that skip work and therefore corrupt the output (raster_mode 4 / 5) exist only in builds compiled with -DREAD_DIAG and are absent from the shipped library. */
int read_set_option(const char *name, int value);
/* 1 if the current device is sm_90 (H100); the library refuses to launch elsewhere. */
int read_device_ok(void);

/* ------------------------------------------------------------------------------------------
 * Rasterizer.  Packed z-buffer entry: (uint64)float_bits(depth) << 32 | point_id ;
 * empty = 0x7FFFFFFFFFFFFFFF (max int64, so signed and unsigned min agree).  atomicMin on it == "min depth, ties -> lowest id", the
 * sequential semantics of DepthProject (MyRender/CloudProjection/point_render.cu:125-167).
 * Pyramid layout: level-major; level l holds [B, h_l, w_l] entries, w_l = int(W*0.5^l),
 * h_l = int(H*0.5^l) (src/READ/gl/myrender.py:33-34).
 * ---------------------------------------------------------------------------------------- */

/* Number of uint64 entries of a B-view, L-level pyramid (size your zbuf with this). */
int64_t read_pyramid_entries(int B, int W, int H, int L);
/* Entry offset of level l inside the pyramid, and its (w,h). */
int64_t read_pyramid_level_offset(int B, int W, int H, int l);
void read_level_size(int W, int H, int l, int *w, int *h);

/* Reset a pyramid (or any zbuf) to "empty". */
int read_zbuf_clear(uint64_t *zbuf, int64_t entries, void *stream);

/*
 * Replaces: the L calls of pcpr.forward made by MyRender.render
 * (src/READ/gl/myrender.py:32-40 -> pcpr_cuda.cpp:23-37 -> point_render.cu:169-200),
 * fused: every point is read, culled and projected ONCE for all B views and all L levels.
 *   xyz      [n,3] f32 device            total_m [B,16] f32 device, row-major 4x4 (proj @ inv(view))
 *   zbuf     pyramid of read_pyramid_entries(B,W,H,L) uint64, already cleared
 *   id_base  added to the local point index to form the global id written in the z-buffer
 *            (point-sharded multi-GPU rendering: each rank passes its shard's first global id)
 * Levels whose size is exactly half of the previous one are derived from it by a 2x2 min
 * (bit-identical to rasterising them directly, see DESIGN.md); the others get direct atomics.
 */
int read_raster_project(const float *xyz, int64_t n, int64_t id_base, const float *total_m, int B,
                        int W, int H, int L, uint64_t *zbuf, void *stream);
/* Second half of the above when a collective sits in between (multi-GPU): project only the levels
 * that need direct atomics (read_raster_project_direct), all-reduce(min) them, then derive the rest. */
int read_raster_project_direct(const float *xyz, int64_t n, int64_t id_base, const float *total_m, int B,
                               int W, int H, int L, uint64_t *zbuf, void *stream);
int read_raster_derive_levels(int B, int W, int H, int L, uint64_t *zbuf, void *stream);
/* Single-view frame path over a spatially sorted point store: pts4 is [n,4] f32 = (x, y, z, bit pattern of the ORIGINAL
 * point id), ordered so that neighbouring points are neighbours in space (read_b200.ops.SortedPoints sorts by the Morton
 * code of the 3-D grid cell when the scene is loaded, the equivalent of MyRender.update_ds).  Rasterises level 0 only
 * (nested levels; finish with read_raster_derive_levels or read_pyramid_resolve_gather).  The z-buffer is a min over
 * (depth | original id) keys, hence identical to read_raster_project_direct on the unsorted cloud. */
int read_raster_project_sorted(const float *pts4, int64_t n, const float *total_m, int W, int H, int L, uint64_t *zbuf,
                               void *stream);
/* Same for B <= 8 views in ONE pass over the store (total_m [B,16]; view b goes to level 0 of view b of a B-view pyramid,
 * i.e. zbuf + b*W*H): the multi-GPU frame path, where every rank rasterises its spatial tile for all views of the step. */
int read_raster_project_sorted_views(const float *pts4, int64_t n, const float *total_m, int B, int W, int H, int L,
                                     uint64_t *zbuf, void *stream);
/* Segmented store (scene editing and stitching, read_b200.ops.SegmentedPoints): pts4 is [n,4] f32 = (x, y, z, bit pattern of
 * the GLOBAL point id), n a multiple of 1024.  Segment i covers chunks [seg_first_chunk[i], + seg_chunks[i]) of 1024 rows
 * (segments may share rows: instances), is drawn with its matrices seg_m[i] ([nseg, B, 16] f32 on the device) and is skipped
 * entirely when seg_visible[i] is 0.  The table (host arrays) travels as kernel parameters.  Padding rows carry NaN
 * coordinates and an id word other than 0xFFFFFFFF.  Like read_raster_project_sorted_views: B <= 8 views in ONE pass,
 * level 0 of nested levels only. */
#define READ_MAX_SEGMENTS 128
int read_raster_project_segments(const float *pts4, int64_t n, const int64_t *seg_first_chunk, const int64_t *seg_chunks,
                                 const uint8_t *seg_visible, int nseg, const float *seg_m, int B, int W, int H, int L,
                                 uint64_t *zbuf, void *stream);
/* Segmented store with view-frustum culling of its chunks, up to READ_MAX_SEGMENTS_CULLED segments; the table lives on the
 * device, so a frame needs no host-side table walk and no synchronisation.
 *   seg_table   [nseg, 3] int32 on the device: (first chunk, chunk count, matrix slot) of segment s; matrices at
 *               seg_m[slot] ([nseg, B, 16] f32).  A segment whose range lies outside the store's n / 1024 chunks, or whose
 *               slot is not below nseg, draws nothing.
 *   nunits      the number of (segment, chunk) units = the sum of the table's chunk counts (units past it are not drawn).
 *   chunk_boxes [n / 1024, 6] f32: (min x, y, z, max x, y, z) of the non-NaN rows of each chunk; an all-padding chunk has
 *               min > max (an empty box).
 *   seg_visible [nseg] uint8 on the device (0 = hidden).
 * One launch culls every unit whose segment is hidden or whose box lies outside the clip volume in all B views (DESIGN.md
 * §4.1: the float64 test is conservative with respect to the per-point float32 test, so the frame is bit-identical to
 * read_raster_project_segments), compacts the survivors in segment-then-chunk order into the workspace, and a persistent
 * rasterizer draws them.  workspace: read_raster_cull_workspace_bytes(nunits) bytes of device memory, 16-byte aligned; its
 * first 4 bytes hold the surviving-unit count (uint32) once the launch has run.  B <= 8, level 0 of nested levels only. */
#define READ_MAX_SEGMENTS_CULLED 4096
int64_t read_raster_cull_workspace_bytes(int64_t nunits);
int read_raster_project_segments_culled(const float *pts4, int64_t n, const int32_t *seg_table, int nseg, int64_t nunits,
                                        const float *chunk_boxes, const uint8_t *seg_visible, const float *seg_m,
                                        void *workspace, int64_t workspace_bytes, int B, int W, int H, int L, uint64_t *zbuf,
                                        void *stream);
/* Point sprites (the reference's _pN / _psN input formats and per-point sizes; DESIGN.md §4.2).  A point is clipped, keyed and
 * given its centre pixel (xx, yy) exactly as at 1 pixel; it then covers a wd x wd square of pixels of each level:
 *   size  = N of the level's key (_pN), or max(1, N / c2) with c2 the point's clip-space z and an IEEE fp32 division (_psN);
 *           a per-point size s > 0 replaces N in either form, s == 0 keeps N;
 *   wd    = min(READ_MAX_POINT_SIZE, max(1, floor(size + 0.5)));
 *   odd wd = 2k+1: columns xx-k .. xx+k; even wd = 2k: columns xr-k .. xr+k-1 with xr = xx + (u - xx >= 0.5), rows likewise;
 *   pixels outside the level are dropped, and every covered pixel takes the (depth | id) key through the 64-bit min.
 * A level with N = 1 in the _pN form and no per-point sizes is a 1-pixel level: it is derived by the 2x2 min from the level
 * before it when that is a 1-pixel level of exactly twice its size, as today.  Every other level, sprite or not, is drawn
 * directly in the same pass over the store, so the levels need not nest.  The three entry points take the stores of
 * read_raster_project_sorted_views, read_raster_project_segments and read_raster_project_segments_culled with the same
 * arguments, write EVERY level of the (cleared) B-view pyramid (no derive step follows), and take B > 8 views for the sorted
 * store (one pass per 8 views).
 *   size[l], relative[l]  level l's N (finite, > 0) and form (0: _pN, 1: _psN), for l < L;
 *   point_sizes           NULL, or one float per store row (>= 0, finite), 16-byte aligned and padded with zeros to whole
 *                         1024-row chunks (the segmented stores already are); sorted and segmented stores permute it with
 *                         their rows. */
#define READ_MAX_POINT_SIZE 64
typedef struct {
    float size[READ_MAX_LEVELS];
    int32_t relative[READ_MAX_LEVELS];
    const float *point_sizes;
} read_sprite_desc;
int read_raster_sprites_sorted(const float *pts4, int64_t n, const float *total_m, int B, int W, int H, int L,
                               const read_sprite_desc *desc, uint64_t *zbuf, void *stream);
int read_raster_sprites_segments(const float *pts4, int64_t n, const int64_t *seg_first_chunk, const int64_t *seg_chunks,
                                 const uint8_t *seg_visible, int nseg, const float *seg_m, int B, int W, int H, int L,
                                 const read_sprite_desc *desc, uint64_t *zbuf, void *stream);
int read_raster_sprites_segments_culled(const float *pts4, int64_t n, const int32_t *seg_table, int nseg, int64_t nunits,
                                        const float *chunk_boxes, const uint8_t *seg_visible, const float *seg_m,
                                        void *workspace, int64_t workspace_bytes, int B, int W, int H, int L,
                                        const read_sprite_desc *desc, uint64_t *zbuf, void *stream);
/* Cylindrical panoramas (DESIGN.md §4.4).  view_m / seg_m hold WORLD -> CAMERA matrices (the inverse of a GL camera-to-world
 * view matrix: x right, y up, looking down -z), [B,16] or [nseg, B, 16].  Per point, in IEEE float32 with no contraction:
 *   (x, y, z) = rows 0-2 of m (p, 1), in the order of the pinhole path's dot products; f = -z; r = sqrt(x*x + f*f);
 *   visible only if znear <= r <= zfar;  v = (t_hi - y / r) * k_h, visible only if 0 <= v < H, row = (int)v;
 *   theta = atan2(x, f) from +, -, *, / (octant reduction and a degree-6 minimax polynomial; |theta| <= float32 pi);
 *   u = (theta + theta_half) * k_w, col = (int)u; full: col == width wraps to 0, otherwise visible only if 0 <= u < width;
 *   key = (bits(r) << 32) | id;  pixel (row, col + margin) of the level-0 plane, W = width + 2 margin columns wide;
 *   full: a point with col < margin also goes to col + margin + width, one with col >= width - margin to col + margin - width.
 * The constants come from read_b200/panorama.py (Panorama.desc), each computed in float64 and rounded once:
 *   theta_half = hfov / 2 (float32 pi at 360 degrees), k_w = width / hfov, t_hi = tan(elevation hi), k_h = H / (t_hi - t_lo).
 * width, margin and H are multiples of 16, 2 margin <= width <= READ_PANORAMA_MAX_WIDTH, margin = 0 unless full.  Level 0 only,
 * into a cleared pyramid whose levels nest (finish with read_raster_derive_levels or read_pyramid_resolve_gather).  The two
 * entry points take the stores and arguments of read_raster_project_sorted_views (B <= 8) and
 * read_raster_project_segments_culled; the culled one drops a unit when, in every view, its box lies entirely beyond zfar. */
#define READ_PANORAMA_MAX_WIDTH 65536
typedef struct {
    float theta_half, k_w, t_hi, k_h, znear, zfar;
    int32_t width;                               /* W: columns of the panorama, margins excluded */
    int32_t margin;                              /* M: wrapped columns drawn on each side (full circle only) */
    int32_t full;                                /* 1: 360 degrees */
} read_panorama_desc;
int read_raster_panorama_sorted(const float *pts4, int64_t n, const float *view_m, int B, int W, int H, int L,
                                const read_panorama_desc *desc, uint64_t *zbuf, void *stream);
int read_raster_panorama_segments_culled(const float *pts4, int64_t n, const int32_t *seg_table, int nseg, int64_t nunits,
                                         const float *chunk_boxes, const uint8_t *seg_visible, const float *seg_m,
                                         void *workspace, int64_t workspace_bytes, int B, int W, int H, int L,
                                         const read_panorama_desc *desc, uint64_t *zbuf, void *stream);
/* Bitmask of levels rasterised with direct atomics (bit l set) for this geometry. */
unsigned read_raster_direct_mask(int W, int H, int L);

/*
 * Replaces: the float outputs of GPU_PCPR (point_render.cu:176-177,196-199): for one level,
 * index [B,h,w] f32 (0 = empty) and depth [B,h,w] f32 (0 = empty) from the packed z-buffer.
 * Either output may be NULL.
 */
int read_zbuf_resolve(const uint64_t *zbuf_level, int64_t pixels, float *index_out, float *depth_out,
                      void *stream);
/* read_zbuf_resolve with an int32 index: the key's low 32 bits (the point id), 0 = empty.  For clouds of more than 2^24 + 1
 * points, whose ids a float32 map cannot all hold; the caller keeps N < 2^31. */
int read_zbuf_resolve_i32(const uint64_t *zbuf_level, int64_t pixels, int32_t *index_out, float *depth_out, void *stream);

/*
 * Replaces: pcpr.forward itself (pcpr_cuda.cpp:23-37): one level, B views.
 * zbuf_ws: workspace of B*h*w uint64 (cleared inside).  Outputs as GPU_PCPR.
 */
int read_pcpr_forward(const float *xyz, int64_t n, const float *total_m, int B, int w, int h,
                      uint64_t *zbuf_ws, float *index_out, float *depth_out, void *stream);

/* ------------------------------------------------------------------------------------------
 * Descriptor gather (PointTexture, READ/models/texture.py:42-70).
 * Descriptors live point-major [N, D] ("shadow" of the checkpoint's [1, D, N] parameter) so that
 * one pixel touches one 32-byte sector (D = 8 f32) instead of 8.
 * ---------------------------------------------------------------------------------------- */

/* [1,D,N] f32 channel-major  <->  [N,D] f32 point-major. */
int read_texture_to_point_major(const float *tex_cn, int D, int64_t N, float *tex_nd, void *stream);
int read_texture_to_channel_major(const float *tex_nd, int D, int64_t N, float *tex_cn, void *stream);

enum { READ_FEAT_NCHW_F32 = 0, READ_FEAT_NHWC_F32 = 1, READ_FEAT_NHWC_BF16 = 2 };
enum { READ_TEXACT_NONE = 0, READ_TEXACT_SIGMOID = 1, READ_TEXACT_TANH = 2 };

/* From a float index map (API path: PointTexture.forward(ids), texture.py:52-63).
 * ids [pixels] f32 (channel 0 of the uv input, already contiguous); out [B, D, h, w] or NHWC. */
int read_gather_from_index(const float *tex_nd, int D, int64_t N, const float *ids, int B, int h, int w,
                           int layout, int activation, void *out, void *stream);
/* Fused path: straight from the packed z-buffer level (skips the float index map). */
int read_gather_from_zbuf(const float *tex_nd, int D, int64_t N, const uint64_t *zbuf_level, int B, int h,
                          int w, int layout, int activation, void *out, void *stream);
/* Per-frame fast path for a 4-level NESTED pyramid (every level an exact half of the previous one, W,H % 8 == 0)
 * and D == 8: one kernel derives levels 1..3 from level 0 (bit-identical 2x2 min), stores them, gathers all four
 * feature maps (NHWC bf16 or f32; outs = HOST array of 4 device pointers) and, if reset_level0, leaves level 0
 * cleared for the next frame.  Views [view0, view0+nviews) of the B-view pyramid are processed (outs hold nviews views).
 * Call after read_raster_project_direct (replaces derive + 4 gathers + next clear). */
int read_pyramid_resolve_gather(const float *tex_nd, int D, int64_t N, uint64_t *zbuf, int B, int view0, int nviews,
                                int W, int H, int L, int layout, void *const *outs, int reset_level0, void *stream);
/* Backward of the gather (autograd of index_select, texture.py:61): grad_tex_nd[ids[p], :] += grad_out[.., p]
 * grad_out is NCHW f32 [B,D,h,w]; grad_tex_nd [N,D] f32 accumulates (caller zeroes).  Empty pixels carry
 * id 0, so point 0 receives their gradient exactly like the reference. */
int read_gather_backward(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N,
                         float *grad_tex_nd, void *stream);
/* Int32 index maps (clouds of more than 2^24 + 1 points): every entry point that reads an index map has an _i32 twin taking
 * `const int32_t *ids`, with otherwise the same arguments, clamping (id < 0 -> 0, id >= N -> N - 1), semantics and, for the
 * deterministic forms, the same workspace query and order of additions.  The float forms are unchanged. */
int read_gather_from_index_i32(const float *tex_nd, int D, int64_t N, const int32_t *ids, int B, int h, int w, int layout,
                               int activation, void *out, void *stream);
int read_gather_backward_i32(const float *grad_out, const int32_t *ids, int B, int D, int h, int w, int64_t N, float *grad_tex_nd,
                             void *stream);

/* Batches whose items sample different textures (a training batch that mixes scenes), D == 8.  The table travels BY VALUE in the
 * kernel parameters (no device-side table, no host-to-device copy).  Item b of the call samples slot slot[b]; its ids are clamped
 * to [0, N[slot] - 1] of its OWN texture, and its empty pixels (id 0) go to point 0 of that texture.
 *   read_gather_from_index_items     : read_gather_from_index per item, one launch (ids [n_items, h, w] f32, out [n_items, 8, h, w]
 *                                      or NHWC); bit-identical to one read_gather_from_index call per item
 *   read_gather_backward_items       : read_gather_backward per item into its slot's grad_nd (dense [N, 8] accumulators)
 *   read_gather_backward_sparse_items: read_gather_backward_sparse per item into its slot's grad_nd, setting its slot's touched
 * A slot with grad_nd == NULL receives nothing (its texture needs no gradient); a slot no item uses is left unchanged.  Pixels of
 * id 0 are pre-reduced per block and per slot in shared memory.  grad_out is NCHW f32 [n_items, 8, h, w]. */
#define READ_MAX_TEX_SLOTS 16
#define READ_MAX_TEX_ITEMS 64
typedef struct read_tex_table {
    const float *tex_nd[READ_MAX_TEX_SLOTS];    /* slot s: point-major [N[s], 8] f32 descriptors, 16B aligned (forward) */
    int64_t N[READ_MAX_TEX_SLOTS];
    float *grad_nd[READ_MAX_TEX_SLOTS];         /* slot s: [N[s], 8] f32 accumulator (backward), or NULL */
    unsigned char *touched[READ_MAX_TEX_SLOTS]; /* slot s: [N[s]] u8 flags (sparse backward) */
    int32_t n_slots;                            /* 1 .. READ_MAX_TEX_SLOTS */
    int32_t n_items;                            /* 1 .. READ_MAX_TEX_ITEMS: the batch size of the call */
    uint8_t slot[READ_MAX_TEX_ITEMS];           /* item -> slot, < n_slots */
} read_tex_table;
int read_gather_from_index_items(const read_tex_table *table, const float *ids, int h, int w, int layout, int activation, void *out,
                                 void *stream);
int read_gather_backward_items(const float *grad_out, const float *ids, const read_tex_table *table, int h, int w, void *stream);
int read_gather_backward_sparse_items(const float *grad_out, const float *ids, const read_tex_table *table, int h, int w,
                                      void *stream);
int read_gather_from_index_items_i32(const read_tex_table *table, const int32_t *ids, int h, int w, int layout, int activation,
                                     void *out, void *stream);
int read_gather_backward_items_i32(const float *grad_out, const int32_t *ids, const read_tex_table *table, int h, int w, void *stream);
int read_gather_backward_sparse_items_i32(const float *grad_out, const int32_t *ids, const read_tex_table *table, int h, int w,
                                          void *stream);

/* ------------------------------------------------------------------------------------------
 * Gated convolution (BasicConv, READ/models/unet.py:22-53) with everything around it fused:
 *   y = bn_scale * ( A(conv_f(x)+b_f) * sigmoid(conv_m(x)+b_m) ) + bn_shift  [+ residual]
 * x is a VIRTUAL concat of up to 4 NHWC sources, each resampled on the fly (nearest up/down by an
 * integer factor = F.interpolate default mode, unet.py:239-250; bilinear x4 align_corners=False =
 * nn.Upsample, unet.py:200), optionally multiplied elementwise by `mul` (FAM, unet.py:114-117).
 * ---------------------------------------------------------------------------------------- */
enum { READ_ACT_F32 = 0, READ_ACT_BF16 = 1 };
enum { READ_SRC_IDENTITY = 0, READ_SRC_NEAREST_DOWN = 1, READ_SRC_NEAREST_UP = 2, READ_SRC_BILINEAR_UP4 = 3 };
enum { READ_OUT_NHWC = 0, READ_OUT_NCHW_F32 = 1,
       /* pre-activation accumulators [conv_f | conv_m] (no bias / activation / BN), NHWC with 2*Cout channels: one term of a
        * 1x1 conv over a concat whose other sources live at a finer resolution (see `addin`); for a 3x3 stride-1 conv, plus an
        * optional residual of the same [B,H,W,2*Cout] shape (training: recomputed [f | m], input gradients) */
       READ_OUT_RAW_NHWC = 2 };
enum { READ_CONV_AUTO = 0, READ_CONV_GENERIC = 1, READ_CONV_TCGEN05 = 2, READ_CONV_TCGEN05_GATHER = 3 };

typedef struct read_src {
    const void *ptr;   /* [B, H, W, C] NHWC, activation dtype */
    int32_t C, H, W;
    int32_t mode;      /* READ_SRC_* */
    int32_t factor;    /* resample factor for NEAREST_* (2,4,8); ignored otherwise */
} read_src;

typedef struct read_conv_desc {
    int32_t act_dtype;              /* READ_ACT_* : storage type of sources / residual / NHWC out */
    int32_t n_src;
    read_src src[READ_MAX_SRC];
    const void *mul;                /* optional [B,Hin,Win,Cin], only with n_src==1 identity */
    int32_t B, Hin, Win, Cin;       /* logical (post-resample, post-concat) input */
    int32_t Hout, Wout, Cout;
    int32_t k, stride, pad;
    int32_t elu;                    /* 1: A = ELU(alpha=1); 0: identity */
    const float *w_generic;         /* packed f32 [k*k*Cin][Npad] (read_pack_weights_generic) or NULL */
    const void *w_tc;               /* packed bf16 for the wgmma kernels (read_pack_weights_tc) or NULL */
    const float *bias_f, *bias_m;   /* [Cout] */
    const float *bn_scale, *bn_shift; /* [Cout] folded eval-mode BatchNorm */
    const void *residual;           /* optional [B,Hout,Wout,Cout] added after BN (ResBlock / FAM skip) */
    void *out;
    int32_t out_mode;               /* READ_OUT_* */
    void *out2;                     /* optional second NHWC output: out2 = y * out2_mul (feeds a FAM) */
    const void *out2_mul;
    int32_t impl;                   /* READ_CONV_* : which kernel (must match the packed weights) */
    /* optional RAW tensor [B, ceil(Hout/2), ceil(Wout/2), 2*Cout] (activation dtype) added, nearest-upsampled x2, to the
     * accumulators BEFORE bias / activation.  A 1x1 conv commutes with nearest upsampling, so
     *   conv1x1(cat[a, up2(b)]) == conv1x1_a(a) + up2(conv1x1_b(b)):
     * the coarse sources of the AFF heads (unet.py:79-89,252-254) are convolved at their own resolution into RAW tensors
     * and enter here, instead of being gathered 4..64 times each at the fine resolution.  TMA-fed wgmma kernel only. */
    const void *addin;
    int32_t addin_H, addin_W;
} read_conv_desc;

typedef struct read_conv_plan read_conv_plan;

/* Npad of the generic packing for a given Cout (multiple of 32, f|m halves per 32-channel group). */
int read_generic_npad(int Cout);
/* Pack torch-layout weights [Cout,Cin,k,k] f32 (device) into the kernel layouts (device). */
int read_pack_weights_generic(const float *wf, const float *wm, int Cout, int Cin, int k, float *out,
                              void *stream);
int64_t read_tc_weight_elems(int Cout, int Cin, int k);
/* K-chunking of the packed layout depends on the conv stride (32-channel chunks for stride 2): pack with the stride the
 * plan will be created with.  read_pack_weights_tc == stride 1. */
int read_pack_weights_tc_strided(const float *wf, const float *wm, int Cout, int Cin, int k, int stride, void *out_bf16,
                                 void *stream);
/* Same, geometry taken from the layer descriptor (stride AND the channel granularity of a virtual concat's sources):
 * the form a caller should use for any descriptor that read_conv_tc_supported accepts. */
int read_pack_weights_tc_for(const read_conv_desc *d, const float *wf, const float *wm, void *out_bf16, void *stream);
int read_pack_weights_tc(const float *wf, const float *wm, int Cout, int Cin, int k, void *out_bf16,
                         void *stream);
/* Filters of the input gradient of a stride-1 3x3 conv pair (wf, wm: [Cout][Cin][3][3] f32), packed for a RAW plan of the TMA-fed
 * kernel with Cin' = 2*Cout, Cout' = Cin/2, k = 3: its input is [df | dm] in the column order of the forward RAW output (blocks of
 * 2*min(Cout, 64) columns, the conv_f half of each block first), its RAW output [B,H,W,Cin] is dX (plus the plan's residual).
 * Size: read_tc_weight_elems(Cin/2, 2*Cout, 3).  Cin % 32 == 0. */
int read_pack_weights_tc_dgrad(const float *wf, const float *wm, int Cout, int Cin, void *out_bf16, void *stream);
/* Filters of the input gradient of input channels c0 .. c0 + cn - 1 of a 1x1 conv pair (wf, wm: [Cout][Cin] f32): one source of a
 * concat, or a 128-channel slice of a wider input.  Packed for a RAW 1x1 plan with Cin' = 2*Cout (its input is [df | dm] in the
 * RAW column order) and Cout' = max(cn, 32) / 2: its RAW output [B,H,W,max(cn, 32)] is dX of those channels, the columns beyond
 * cn zero (cn = 16 is padded to the plans' smallest N tile).  Size: read_tc_weight_elems(max(cn, 32) / 2, 2*Cout, 1).
 * cn = 16, 32, 64 or 128; Cout = 16, 32, 48, 64 or a multiple of 64. */
int read_pack_weights_tc_dgrad1x1(const float *wf, const float *wm, int Cout, int Cin, int c0, int cn, void *out_bf16, void *stream);
/* 1 if the TMA-fed wgmma kernel supports this layer (stride-1 k x k / stride-2 3x3, 4x4 single source; 1x1 virtual concat of
 * identity / nearest-down sources; RAW 3x3 stride 1 over one source, optionally with a [B,H,W,2*Cout] residual; RAW stride-2
 * 3x3 / 4x4 without a residual; RAW 1x1 at Cout 16 / 32 / 64), else 0. */
int read_conv_tc_supported(const read_conv_desc *d);
/* Same for the wgmma kernel with a gathered A operand (any stride / concat / resampling, bf16 activations);
 * it has its own weight packing. */
int read_conv_tcg_supported(const read_conv_desc *d);
int64_t read_tcg_weight_elems(int Cout, int Cin, int k);
int read_pack_weights_tcg(const float *wf, const float *wm, int Cout, int Cin, int k, void *out_bf16, void *stream);

/* Plan = validated descriptor + chosen kernel + TMA tensor maps.  Host-side only, no device work. */
int read_conv_plan_create(const read_conv_desc *d, read_conv_plan **out);
int read_conv_plan_launch(const read_conv_plan *p, void *stream);
int read_conv_plan_impl(const read_conv_plan *p);   /* READ_CONV_GENERIC / _TCGEN05 / _TCGEN05_GATHER */
/* Cap the persistent grid of a tensor-core plan at max_ctas CTAs (0 = one per SM, the default): a caller that runs two independent
 * layer chains on two streams gives each a share of the SMs so that both are resident at once (read_b200/engine.py). */
int read_conv_plan_set_max_ctas(read_conv_plan *p, int max_ctas);
/* Tile traversal order of a tcgen05 TMA plan: 0 = top-down (default), 1 = bottom-up.  Same result.  A layer that walks the image in the
 * opposite direction of its producer starts on the tiles the producer wrote LAST, i.e. the ones still in the 126 MB L2: consecutive
 * layers of a chain alternate (read_b200/engine.py). */
int read_conv_plan_set_tile_order(read_conv_plan *p, int reversed);
void read_conv_plan_destroy(read_conv_plan *p);

/* nn.Upsample(scale_factor=4, mode='bilinear') (unet.py:200), NHWC [B,h,w,C] -> [B,4h,4w,C], C % 8 == 0. */
int read_upsample_bilinear4(const void *in, int act_dtype, int B, int h, int w, int C, void *out, void *stream);

/* Layout converters at the net boundary. */
/* Viewer output path (replaces READ/gl/nn.py:123-124 `permute + cat alpha` and the flip of viewer.py:267):
 * RGB planes [3,H,W] f32 -> [H,W,4] f32 (alpha constant), optionally flipped vertically. */
int read_frame_to_rgba(const float *rgb_planes, int H, int W, int flip_vertical, float alpha, float *out_hwc4, void *stream);

/* Point-cloud views (the reference viewer's non-neural path: NNScene's GLSL program, READ/gl/programs.py:60-300; DESIGN.md §4.3).
 * Shades level 0 of a 1-view z-buffer [H,W] (rasterised by any of the entry points above) into [H,W,4] f32, one 16-byte store
 * per pixel; with flip_vertical, output row y is z-buffer row H-1-y (as read_frame_to_rgba).  An empty pixel gets clear[];
 * a drawn pixel gets (r, g, b, 1) from its point, id = the key's low 32 bits, clamped to n - 1 for the table reads.
 * Colour per mode (mode0 of the shader; sub = submode, the shader's mode1), every operation an IEEE round-to-nearest one in
 * the order written, no contraction; half(v) = v*0.5 + 0.5, normalize(v) = v_i / sqrt((v0*v0 + v1*v1) + v2*v2):
 *   COLOR   colors[id].rgb (the point colours, or the PCA colours the host computed)
 *   NORMALS sub 0: half(n);  1: half(normalize(d - (2*dot(n, d))*n)) with d = normalize(cam - p), dot(a, b) = (a0*b0 + a1*b1) + a2*b2;
 *           2: half(normalize(m_view rows 0..2 . (cam + n, 1))), row i . v = ((m[i0]*v0 + m[i1]*v1) + m[i2]*v2) + m[i3];
 *           3: half(normalize(cam - p));  4: n
 *   DEPTH   (c2, c2, c2), c2 = fadd(fma(z, m[10], fma(y, m[9], x*m[8])), m[11]) of total_m: the rasterizer's own clip z
 *   UV      sub 0: (float(id), 0, 0) of the unclamped id;  1..4: (0, 0, 0)
 *   XYZ     (p - lo) / ((hi - lo) + 1e-9f) per axis
 *   LABEL   (n.x / 255, 0, 0)
 * with p = xyz[id] ([n,3] f32), n = normals[id].xyz.  colors and normals are [n,4] f32 rows (16-byte aligned); a table the mode
 * does not read may be NULL.  A zero vector normalises to NaN. */
enum { READ_VIEW_COLOR = 0, READ_VIEW_NORMALS = 1, READ_VIEW_DEPTH = 2, READ_VIEW_UV = 3, READ_VIEW_XYZ = 4, READ_VIEW_LABEL = 5 };
typedef struct {
    int32_t mode;            /* READ_VIEW_* */
    int32_t submode;         /* 0..4 */
    const float *colors;     /* [n,4] f32 */
    const float *normals;    /* [n,4] f32 */
    const float *xyz;        /* [n,3] f32 */
    int64_t n;               /* rows of the tables (>= 1 when the mode reads one) */
    float total_m[16];       /* row-major proj @ inv(view), as the rasterizer took it */
    float m_view[16];        /* row-major inv(view) */
    float cam[3];            /* view[:3, 3] */
    float lo[3], hi[3];      /* the cloud's per-axis min and max */
    float clear[4];
    int32_t flip_vertical;
} read_point_view_desc;
int read_point_view(const uint64_t *zbuf_level0, int H, int W, const read_point_view_desc *desc, float *out_hwc4, void *stream);

/* Net-input staging for NetAndTexture's viewer options on the fused path (READ/models/compose.py:162-171): src = f32 NHWC
 * features [B,hs,ws,C] at render resolution; factor = supersampling (bilinear reduce exactly as F.interpolate(scale_factor=1/ss,
 * mode='bilinear')); last (nullable) = f32 [B,hs/factor,ws/factor,C] temporal-average state: out = (cur + last) / 2 when
 * have_last, and last := out; dst = NHWC in act_dtype (the engine's input buffer). */
int read_stage_net_inputs(const float *src, int B, int hs, int ws, int C, int factor, float *last, int have_last, int act_dtype,
                          void *dst, void *stream);

int read_nchw_f32_to_nhwc(const float *in, int B, int C, int H, int W, int act_dtype, void *out, void *stream);
int read_nhwc_to_nchw_f32(const void *in, int act_dtype, int B, int C, int H, int W, float *out, void *stream);

/* ------------------------------------------------------------------------------------------
 * Strip-parallel refinement net across GPUs (SURVEY.md §8f rank 1): halo rows travel between neighbouring ranks through
 * peer-mapped mailboxes (cudaMalloc + CUDA IPC), one kernel per exchange, no NCCL on the path (csrc/halo.cu).
 * read_ipc_alloc: cudaMalloc `bytes` (zero-filled) and export its 64-byte IPC handle; read_ipc_open maps a peer's handle
 * (another process on the same node) with lazy peer access.  read_epoch_bump increments the device-resident frame counter.
 * read_halo_exchange: push `bytes` from src_up / src_dn into the neighbours' mailbox slots (peer pointers) and publish the
 * current epoch in their flag words; then wait until both neighbours' epochs arrived in this rank's flags and copy this rank's
 * mailbox slots into dst_top / dst_bot.  Null pointers = no neighbour on that side.  Asynchronous on `stream`. */
typedef struct read_halo_desc {
    const void *src_up, *src_dn;               /* local rows to send to the strip above / below */
    void *peer_up_slot, *peer_dn_slot;         /* destination slots inside the neighbours' mailboxes */
    void *peer_up_flag, *peer_dn_flag;         /* uint32 flag words inside the neighbours' mailboxes */
    const void *slot_from_up, *slot_from_dn;   /* this rank's mailbox slots (written by the neighbours) */
    const void *flag_from_up, *flag_from_dn;   /* this rank's flag words */
    void *dst_top, *dst_bot;                   /* halo rows of the local tensor */
    int64_t bytes;                             /* per direction, multiple of 16 */
    const void *epoch;                         /* uint32 device word, see read_epoch_bump */
    void *cta_counter;                         /* uint32 device word private to this exchange, zero-initialised */
} read_halo_desc;
int read_ipc_alloc(int64_t bytes, void **dev_ptr, unsigned char *handle64);
int read_ipc_open(const unsigned char *handle64, void **peer_ptr);
int read_ipc_close(void *peer_ptr);
int read_ipc_free(void *dev_ptr);
int read_epoch_bump(uint32_t *epoch, void *stream);
int read_halo_exchange(const read_halo_desc *d, void *stream);

/* ------------------------------------------------------------------------------------------
 * Descriptor side of the training step (SURVEY.md §8f rank 2; replaces autograd's dense index_add_ of READ/models/texture.py:55-63
 * and the dense torch.optim.RMSprop of READ/pipelines/ogl.py:16,97-102).  grad_nd [N,D] f32 and touched [N] u8 are persistent,
 * zero-initialised accumulators owned by the caller.
 *   read_gather_backward_sparse : grad_nd[id,:] += grad_out[b,:,y,x] for every pixel (ids [B,h,w] f32, grad_out [B,D,h,w] f32);
 *                                 touched[id] = 1
 *   read_sparse_rmsprop_step    : for touched points only - square_avg (point-major [N,D]) decayed lazily by alpha^(step -
 *                                 last_step[i]), RMSprop update (momentum 0, not centered) applied to param_cn ([1,D,N], the
 *                                 checkpoint layout) AND to shadow_nd ([N,D], may be null); the point's grad row and flag are
 *                                 cleared.  step counts optimizer steps from 1.
 *   read_square_avg_dense       : the dense optimizer's square_avg [1,D,N] after `step` steps (state_dict export)
 *   read_compact_touched        : touched rows -> (id, grad[D]) pairs; *count (zeroed by the caller) receives their number
 *   read_scatter_pairs          : grad_nd[id,:] += grads[k,:], touched[id] = 1 (pairs received from other ranks)
 * The L2 regulariser of PointTexture (reg_weight * mean(param^2), READ/models/texture.py:40-41) without a dense gradient: its
 * gradient is k * param with one scalar k per texture, so the step takes k instead of a [1,D,N] gradient.  D in 1..16, N >= 1.
 *   read_reg_loss_workspace_bytes : size of the workspace of read_reg_loss (-1 for a bad shape)
 *   read_reg_loss               : *out (device f32 scalar) = reg_weight * sum(param_cn^2) / (D * N) over param_cn [1,D,N] f32.
 *                                 fp32 partials of 4 words accumulated in fp64 per thread, then a fixed-order fp64 combine (the
 *                                 grid depends only on the device): repeated calls give the same bits.  param_cn and workspace
 *                                 16-byte aligned; the workspace (caller-owned) must not be shared by concurrent calls.
 *   read_sparse_rmsprop_step_reg: read_sparse_rmsprop_step with the regulariser's gradient added for EVERY point: g = (touched[i] ?
 *                                 grad_nd[i,c] : 0) + fl(k * param[c,i]) (two roundings), k = *reg_coef (device f32, e.g. 2 *
 *                                 the upstream gradient * reg_weight / numel), then weight decay, the lazy decay by alpha^(step -
 *                                 last_step[i]) and the update, written to param_cn and shadow_nd; touched rows and flags are
 *                                 cleared and last_step[i] = step for all points. */
int read_gather_backward_sparse(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N,
                                float *grad_nd, unsigned char *touched, void *stream);
int read_gather_backward_sparse_i32(const float *grad_out, const int32_t *ids, int B, int D, int h, int w, int64_t N, float *grad_nd,
                                    unsigned char *touched, void *stream);
int read_sparse_rmsprop_step(float *param_cn, float *shadow_nd, float *grad_nd, unsigned char *touched, float *square_avg,
                             int32_t *last_step, int64_t N, int D, int step, float lr, float alpha, float eps, float weight_decay,
                             void *stream);
int read_square_avg_dense(const float *square_avg, const int32_t *last_step, int64_t N, int D, int step, float alpha, float *out_cn,
                          void *stream);
int read_compact_touched(const float *grad_nd, const unsigned char *touched, int64_t N, int D, int32_t *count, int capacity,
                         int32_t *out_ids, float *out_grads, void *stream);
int read_scatter_pairs(const int32_t *ids, const float *grads, int n, int D, int64_t N, float *grad_nd, unsigned char *touched,
                       void *stream);
int64_t read_reg_loss_workspace_bytes(int D, int64_t N);
int read_reg_loss(const float *param_cn, int D, int64_t N, double reg_weight, float *out, void *workspace, void *stream);
int read_sparse_rmsprop_step_reg(float *param_cn, float *shadow_nd, float *grad_nd, unsigned char *touched, float *square_avg,
                                 int32_t *last_step, int64_t N, int D, int step, float lr, float alpha, float eps, float weight_decay,
                                 const float *reg_coef, void *stream);

/* ------------------------------------------------------------------------------------------
 * Backward of the gated convs, bf16 training with eval-mode BatchNorm (read_b200/blocks.py): the 3x3 stride-1 convs (the residual
 * blocks EBlock / DBlock, READ/models/unet.py:56-76, and the single convs feat_extract.0 / .5, SCM*.main.0 / .2, AFFs.*.conv.1,
 * FAM*.merge) and, under train_precision 'bf16_all', the 1x1 convs (Convs.*, AFFs.*.conv.0, SCM*.main.1 / .3, SCM*.conv) and the
 * stride-2 3x3 / 4x4 convs (feat_extract.1 / .2 / .3 / .4 / .6 / .7).
 * Activations NHWC bf16; [f | m] rows are in the forward RAW output's column order (see read_pack_weights_tc_dgrad).  Reductions
 * ACCUMULATE (+=) into caller-zeroed fp32 buffers.
 *   read_gate_backward      : fm = pre-activation accumulators [P, 2C] (without bias), dy = gradient of the conv's output [P, C];
 *                             dfm [P, 2C] = [df | dm] with dg = dy*bn_scale, df = dg*sigmoid(m)*A'(f), dm = dg*A(f)*sigmoid'(m);
 *                             dbias_f/m = sum df / dm, dgamma = sum dy*(g - mean)*inv_std, dbeta = sum dy.  C = 16, 32, 48, 64,
 *                             128, 192 or 256 (C <= 64 or C % 64 == 0: the channel counts that have the RAW column order); the RGB
 *                             output conv (C = 3) is run padded to C = 16 by the caller
 *   read_conv3x3_wgrad      : dwf / dwm [Cout][Cin][3][3] += sum over pixels of [df | dm] x im2col(x), x [B,H,W,Cin] with zero
 *                             padding 1.  Cin = 8, 16 or a multiple of 32; Cout = 16, 32, 64 or a multiple of 64
 *   read_conv3x3_dgrad_cin8 : input gradient dx [B,H,W,8] (bf16, overwritten) of a conv with Cin = 8 (the descriptor pyramid), from
 *                             dfm [B,H,W,2*Cout] and the fp32 filters wf / wm [Cout][8][3][3].  Cout = 16, 32 or 64.  The input
 *                             gradient of wider inputs is a RAW plan with read_pack_weights_tc_dgrad filters
 *   read_conv_wgrad         : read_conv3x3_wgrad for k x k stride s: 1x1 and 3x3 stride 1, 3x3 and 4x4 stride 2 (pad 1, the input
 *                             exactly twice the output: Hin == 2*Hout, Win == 2*Wout).  dwf / dwm [Cout][Cin][k][k], x [B,Hin,Win,Cin],
 *                             dfm [B,Hout,Wout,2*Cout]; same channel rules
 *   read_pack_weights_dgrad_s2 : the filters of read_conv_dgrad_s2: [k*k][Cin][2*Cout] bf16, the 2*Cout columns in the RAW order
 *   read_conv_dgrad_s2      : input gradient dx [B,2*Hout,2*Wout,Cin] (bf16, overwritten) of a stride-2 pad-1 3x3 / 4x4 conv from
 *                             dfm [B,Hout,Wout,2*Cout].  Cin a multiple of 32; Cout 16, 32, 64 or a multiple of 64.  The input
 *                             gradient of a 1x1 conv is a RAW 1x1 plan with read_pack_weights_tc_dgrad1x1 filters
 * ---------------------------------------------------------------------------------------- */
int read_gate_backward(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f, const float *bias_m,
                       const float *bn_scale, const float *bn_mean, const float *bn_inv_std, void *dfm, float *dbias_f,
                       float *dbias_m, float *dgamma, float *dbeta, void *stream);
int read_conv3x3_wgrad(const void *dfm, const void *x, int B, int H, int W, int Cout, int Cin, float *dwf, float *dwm, void *stream);
int read_conv3x3_dgrad_cin8(const void *dfm, const float *wf, const float *wm, int B, int H, int W, int Cout, void *dx, void *stream);
int read_conv_wgrad(const void *dfm, const void *x, int B, int Hin, int Win, int Hout, int Wout, int Cout, int Cin, int k,
                    int stride, float *dwf, float *dwm, void *stream);
int read_pack_weights_dgrad_s2(const float *wf, const float *wm, int Cout, int Cin, int k, void *out_bf16, void *stream);
int read_conv_dgrad_s2(const void *dfm, const void *wt, int B, int Hout, int Wout, int Cout, int Cin, int k, void *dx, void *stream);

/* ------------------------------------------------------------------------------------------
 * Train-mode BatchNorm of the gated convs (read_b200/blocks.py, batch_stats=True), torch.nn.BatchNorm2d's semantics: the conv runs
 * with an identity epilogue (bn_scale 1, bn_shift 0, no residual) and writes g [P, C] (NHWC bf16); then
 *   read_bn_batch_stats     : per-channel mean and biased variance var of g over the P pixels; writes mean, inv_std = 1/sqrt(var+eps),
 *                             var (optional, may be NULL), scale = gamma*inv_std, shift = beta - mean*scale, and updates in place
 *                             running_mean = (1-momentum)*running_mean + momentum*mean and running_var likewise with the unbiased
 *                             var*P/(P-1).  Channels >= n_real are padding (g == 0): scale = shift = 0 and no running update; gamma,
 *                             beta, running_* have n_real entries.  workspace: read_bn_workspace_bytes(C) bytes, 16B aligned,
 *                             uninitialised, used by one call at a time.  Deterministic run to run
 *   read_bn_apply           : y = bf16(g*scale + shift [+ residual]); residual (optional) [P, C] bf16; y may be g
 *   read_bn_backward_reduce : sum_dy += sum dy, sum_dy_xhat += sum dy*(g - mean)*inv_std (= dbeta, dgamma) with g recomputed from the
 *                             RAW [f | m] and the biases (caller-zeroed fp32 [C])
 *   read_gate_backward_batch_stats : read_gate_backward with the batch-statistics terms: dg = scale*(dy - sum_dy/P
 *                             - xhat*sum_dy_xhat/P); writes dfm, accumulates dbias_f / dbias_m (dgamma / dbeta are the two sums)
 * C = 16, 32, 64 or a multiple of 64 up to 256; pixels >= 2; activations 16B aligned.
 * ---------------------------------------------------------------------------------------- */
int64_t read_bn_workspace_bytes(int C);
int read_bn_batch_stats(const void *g, int64_t pixels, int C, int n_real, const float *gamma, const float *beta, float eps,
                        float momentum, float *running_mean, float *running_var, float *mean, float *inv_std, float *var,
                        float *scale, float *shift, void *workspace, void *stream);
int read_bn_apply(const void *g, int64_t pixels, int C, const float *scale, const float *shift, const void *residual, void *y,
                  void *stream);
int read_bn_backward_reduce(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f, const float *bias_m,
                            const float *bn_mean, const float *bn_inv_std, float *sum_dy, float *sum_dy_xhat, void *stream);
int read_gate_backward_batch_stats(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f,
                                   const float *bias_m, const float *bn_scale, const float *bn_mean, const float *bn_inv_std,
                                   const float *sum_dy, const float *sum_dy_xhat, void *dfm, float *dbias_f, float *dbias_m,
                                   void *stream);

/* ------------------------------------------------------------------------------------------
 * Per-item train-mode BatchNorm (read_b200/blocks.py, UNet.train_batchnorm = 'per_item'): a call of `items` batch items, item i
 * being the `pixels` rows [i*pixels, (i+1)*pixels) of g / dy / fm, each normalised with its own statistics.  mean, inv_std, scale,
 * shift, sum_dy and sum_dy_xhat are fp32 [items, C]; the rest is as in the call-wide entry points above.
 *   read_bn_batch_stats_items : item i's mean / inv_std / scale / shift are bit-identical to read_bn_batch_stats on its rows alone;
 *                               the running statistics are updated once per item, in item order, bit-identical to `items` calls
 *                               of read_bn_batch_stats in a row.  workspace: read_bn_workspace_bytes_items(items, C) bytes
 *   read_bn_apply_items       : y = bf16(g*scale_i + shift_i [+ residual]) with the scale / shift of the pixel's item
 *   read_bn_backward_reduce_items : the two sums per (item, channel) into caller-zeroed [items, C]; dbeta / dgamma are their sums
 *                               over items
 *   read_gate_backward_batch_stats_items : the corrected gate backward with item i's sums and `pixels`; dbias_f / dbias_m
 *                               accumulate over all items
 * items in 1..65535, pixels (per item) >= 2.
 * ---------------------------------------------------------------------------------------- */
int64_t read_bn_workspace_bytes_items(int items, int C);
int read_bn_batch_stats_items(const void *g, int items, int64_t pixels, int C, int n_real, const float *gamma, const float *beta,
                              float eps, float momentum, float *running_mean, float *running_var, float *mean, float *inv_std,
                              float *scale, float *shift, void *workspace, void *stream);
int read_bn_apply_items(const void *g, int items, int64_t pixels, int C, const float *scale, const float *shift, const void *residual,
                        void *y, void *stream);
int read_bn_backward_reduce_items(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu, const float *bias_f,
                                  const float *bias_m, const float *bn_mean, const float *bn_inv_std, float *sum_dy,
                                  float *sum_dy_xhat, void *stream);
int read_gate_backward_batch_stats_items(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu,
                                         const float *bias_f, const float *bias_m, const float *bn_scale, const float *bn_mean,
                                         const float *bn_inv_std, const float *sum_dy, const float *sum_dy_xhat, void *dfm,
                                         float *dbias_f, float *dbias_m, void *stream);

/* ------------------------------------------------------------------------------------------
 * VGG19 perceptual loss (read_b200/vgg_loss.py, the reference's READ/criterions/vgg_loss.py).  The convs are RAW 3x3 plans of the
 * TMA-fed kernel (a plain conv of c filters = the gated pair of c/2 whose RAW column order is the natural channel order) and, for
 * the image's input gradient, read_conv3x3_dgrad_cin8; these entry points are the glue around them.  A call holds n output images
 * and n target images as ONE NHWC bf16 batch of 2n: images 0 .. n-1 the output, n .. 2n-1 the target.
 *   read_vgg_workspace_bytes : bytes of the workspace read_vgg_post needs on a loss layer (16B aligned, one call at a time)
 *   read_vgg_normalize   : input, target NCHW f32 [n,3,H,W] -> out [2n,H,W,8] bf16 = (x - mean[c]) / std[c] (channels 3..7 zero);
 *                          mean, std f32 [3] device
 *   read_vgg_post        : raw [2n,H,W,C] bf16 = a conv's RAW accumulators; y = ReLU(raw + bias[c]) for both halves.  term
 *                          (nullable: not a loss layer): *term (double, device) += scale * sum |y_out - y_tgt|, deterministic (fixed
 *                          combine order for a given shape).  code (nullable) int8 [n,H,W,C]: 0 where y_out = 0, else
 *                          2 + sign(y_out - y_tgt) (2 off the loss layers).  out (nullable): pool = 0: y [2n,H,W,C] (may be raw);
 *                          pool = 1: AvgPool2d(2, 2) of y, [2n,H/2,W/2,C] (floor).  C % 8 == 0
 *   read_vgg_dgrad_in    : dy [n,H,W,C] bf16 = [code != 0] * (U + (code - 2) * g[0] * coef), U = up [n,H,W,C] (pool = 0) or the
 *                          AvgPool2d(2, 2) backward of up [n,H/2,W/2,C] (pool = 1: up / 4, 0 on a dropped odd row / column), 0 when
 *                          up is NULL; g f32 [1] device
 *   read_vgg_image_grad  : dx [n,H,W,8] bf16 -> out [n,3,H,W] f32 = dx[c] / std[c] (channels 3..7 ignored)
 * partialconv=True: conv1_1 is a partial conv over the target's validity mask M [n,H,W] (1 where the target's channel sum
 * > 1e-9, else 0; the same M for output b and target b).  With cnt = valid pixels of M's 3x3 window at a pixel (zero padding),
 * upd = [cnt > 0] and ratio = upd * reciprocal(cnt) * 9 (fp32, torch's rounding of 9 / (cnt + 1e-8)):
 *   read_vgg_normalize_masked  : as read_vgg_normalize, both halves times M; mask (out) uint8 [n,H,W] = M
 *   read_vgg_post_partial      : as read_vgg_post with pool = 0 and y = ReLU((raw * ratio + bias[c]) * upd); mask uint8 [n,H,W]
 *   read_vgg_dgrad_in_partial  : as read_vgg_dgrad_in with pool = 0, times ratio
 *   read_vgg_image_grad_masked : as read_vgg_image_grad, times M
 * ---------------------------------------------------------------------------------------- */
int64_t read_vgg_workspace_bytes(void);
int read_vgg_normalize(const float *input, const float *target, int n, int H, int W, const float *mean, const float *std_, void *out,
                       void *stream);
int read_vgg_post(const void *raw, int n, int H, int W, int C, const float *bias, int pool, void *out, void *code, double *term,
                  double scale, void *workspace, void *stream);
int read_vgg_dgrad_in(const void *up, int pool, const void *code, int n, int H, int W, int C, const float *g, float coef, void *dy,
                      void *stream);
int read_vgg_image_grad(const void *dx, int n, int H, int W, const float *std_, float *out, void *stream);
int read_vgg_normalize_masked(const float *input, const float *target, int n, int H, int W, const float *mean, const float *std_,
                              void *out, void *mask, void *stream);
int read_vgg_post_partial(const void *raw, const void *mask, int n, int H, int W, int C, const float *bias, void *out, void *code,
                          double *term, double scale, void *workspace, void *stream);
int read_vgg_dgrad_in_partial(const void *up, const void *mask, const void *code, int n, int H, int W, int C, const float *g,
                              float coef, void *dy, void *stream);
int read_vgg_image_grad_masked(const void *dx, const void *mask, int n, int H, int W, const float *std_, float *out, void *stream);

/* ------------------------------------------------------------------------------------------
 * Deterministic training reductions (read_b200 picks them when torch.are_deterministic_algorithms_enabled()).  The entry points
 * above add partial sums with fp32 atomics, so their last bits vary from run to run; these compute the same quantities with a fixed
 * order of additions: the same inputs give the same bits on every call, on the same device and build.  Each takes a caller-owned
 * workspace (16B aligned, uninitialised, used by one call at a time) of the size its *_workspace_bytes query returns (-1: shape not
 * supported), and otherwise the arguments and accumulate (+=) semantics of its default form.
 *
 *   read_gather_backward_det / read_gather_backward_sparse_det : read_gather_backward / read_gather_backward_sparse.  Order: with
 *       key[p] = clamp(id[p], 0, N-1) for the flat pixel p = (b*h + y)*w + x, the pixels are sorted stably by key (so each id's
 *       pixels stay in ascending p).  The sorted sequence is cut into chunks of 128 positions.  Within a chunk, each run of equal
 *       keys is summed in sorted order in fp32, starting from 0.  An id whose pixels all lie in one chunk gets that run sum; an id
 *       whose pixels cross chunk boundaries gets its runs' sums added in chunk order (the first run's sum, + the next, ...).  That
 *       sum is added once to row id (grad_tex_nd, or grad_nd with touched[id] = 1), per channel independently.
 *       workspace: read_gather_backward_det_workspace_bytes(B, D, h, w, N); B*h*w < 2^31, N < 2^31
 *   read_gather_backward_items_det / read_gather_backward_sparse_items_det : read_gather_backward_items / _sparse_items.  Order:
 *       the same passes over ONE key space that stacks the slots' rows in slot order: with base[s] = N[0] + ... + N[s-1],
 *       key[p] = base[slot[b]] + clamp(id[p], 0, N[slot[b]] - 1) for the flat pixel p = (b*h + y)*w + x of item b.  So the pixels
 *       are sorted stably by (slot, clamped id), each (slot, id)'s pixels in ascending p (items in item order), and the same
 *       128-position chunks, run sums and chunk-order combination give each row's sum, added once to row id of its slot.  Runs
 *       never span two slots (their keys differ).  Slots with grad_nd == NULL take part in the sort but receive nothing.
 *       workspace: read_gather_backward_det_workspace_bytes(n_items, 8, h, w, base[n_slots]); base[n_slots] < 2^31
 *   read_gate_backward_det, read_bn_backward_reduce_det, read_gate_backward_batch_stats_det, read_bn_backward_reduce_items_det,
 *   read_gate_backward_batch_stats_items_det : the per-channel sums leave each CTA through the workspace (the CTA's threads added
 *       in thread order) and the last CTA to finish adds the CTAs' rows in a fixed order.  workspace: read_gate_det_workspace_bytes
 *       (items, C), items = 1 for the call-wide forms
 *   read_conv_wgrad_det : read_conv_wgrad (and read_conv3x3_wgrad as k = 3, stride = 1).  Each split-K part of the pixels writes its
 *       own copy of the gradients to the workspace; the copies are added in split order and then to dwf / dwm.  The number of
 *       splits depends on the device's SM count.  workspace: read_conv_wgrad_det_workspace_bytes(B, Hout, Wout, Cout, Cin, k,
 *       stride)
 * ---------------------------------------------------------------------------------------- */
int64_t read_gather_backward_det_workspace_bytes(int B, int D, int h, int w, int64_t N);
int read_gather_backward_det(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N, float *grad_tex_nd,
                             void *workspace, void *stream);
int read_gather_backward_sparse_det(const float *grad_out, const float *ids, int B, int D, int h, int w, int64_t N, float *grad_nd,
                                    unsigned char *touched, void *workspace, void *stream);
int read_gather_backward_items_det(const float *grad_out, const float *ids, const read_tex_table *table, int h, int w,
                                   void *workspace, void *stream);
int read_gather_backward_sparse_items_det(const float *grad_out, const float *ids, const read_tex_table *table, int h, int w,
                                          void *workspace, void *stream);
/* int32 index maps: the same workspace query and order; only the key build reads the other type */
int read_gather_backward_det_i32(const float *grad_out, const int32_t *ids, int B, int D, int h, int w, int64_t N, float *grad_tex_nd,
                                 void *workspace, void *stream);
int read_gather_backward_sparse_det_i32(const float *grad_out, const int32_t *ids, int B, int D, int h, int w, int64_t N,
                                        float *grad_nd, unsigned char *touched, void *workspace, void *stream);
int read_gather_backward_items_det_i32(const float *grad_out, const int32_t *ids, const read_tex_table *table, int h, int w,
                                       void *workspace, void *stream);
int read_gather_backward_sparse_items_det_i32(const float *grad_out, const int32_t *ids, const read_tex_table *table, int h, int w,
                                              void *workspace, void *stream);
int64_t read_gate_det_workspace_bytes(int items, int C);
int read_gate_backward_det(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f, const float *bias_m,
                           const float *bn_scale, const float *bn_mean, const float *bn_inv_std, void *dfm, float *dbias_f,
                           float *dbias_m, float *dgamma, float *dbeta, void *workspace, void *stream);
int read_bn_backward_reduce_det(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f,
                                const float *bias_m, const float *bn_mean, const float *bn_inv_std, float *sum_dy, float *sum_dy_xhat,
                                void *workspace, void *stream);
int read_gate_backward_batch_stats_det(const void *dy, const void *fm, int64_t pixels, int C, int elu, const float *bias_f,
                                       const float *bias_m, const float *bn_scale, const float *bn_mean, const float *bn_inv_std,
                                       const float *sum_dy, const float *sum_dy_xhat, void *dfm, float *dbias_f, float *dbias_m,
                                       void *workspace, void *stream);
int read_bn_backward_reduce_items_det(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu,
                                      const float *bias_f, const float *bias_m, const float *bn_mean, const float *bn_inv_std,
                                      float *sum_dy, float *sum_dy_xhat, void *workspace, void *stream);
int read_gate_backward_batch_stats_items_det(const void *dy, const void *fm, int items, int64_t pixels, int C, int elu,
                                             const float *bias_f, const float *bias_m, const float *bn_scale, const float *bn_mean,
                                             const float *bn_inv_std, const float *sum_dy, const float *sum_dy_xhat, void *dfm,
                                             float *dbias_f, float *dbias_m, void *workspace, void *stream);
int64_t read_conv_wgrad_det_workspace_bytes(int B, int Hout, int Wout, int Cout, int Cin, int k, int stride);
int read_conv_wgrad_det(const void *dfm, const void *x, int B, int Hin, int Win, int Hout, int Wout, int Cout, int Cin, int k,
                        int stride, float *dwf, float *dwm, void *workspace, void *stream);

/* Counts kernels launched by this library since load (bench.py's gpu_launches claim). */
int64_t read_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* READ_B200_H */
