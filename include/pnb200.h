/*
 * pnb200 -- C ABI of the GPU-native (Hopper, sm_90a) Point-NeRF per-ray hot path (libpnb200.so).
 *
 * Plain C: pointers, sizes, a CUDA stream handle.  No torch types, no hidden allocations: every
 * device buffer (inputs, outputs, workspaces) is owned by the caller; *_bytes() functions report the
 * workspace sizes.  Every entry point returns 0 on success or a negative pnb_status; the text of the
 * last error of the calling thread is available through pnb_last_error().  Nothing here synchronises
 * the stream unless its comment says so.
 *
 * Each entry point names the reference interface it replaces
 * (paths are into the reference tree, Xharlie/pointnerf):
 *   pnb_grid_build        models/neural_points/cuda/query_worldcoords.cu:18-162   (claim_occ, map_coor2occ,
 *                         fill_occ2pnts) + the allocations of :314-319 -- run ONCE per point-cloud version
 *                         instead of once per ray chunk.
 *   pnb_query             query_worldcoords.cu:165-302,381-391 (mask_raypos, first-SR selection,
 *                         get_shadingloc, query_neigh_along_ray_layered) and the ray generation of
 *                         models/rendering/diff_ray_marching.py:349-392 (positions are formed in-kernel from
 *                         campos + raydir * t[d], never materialised).
 *   pnb_query_export      query_worldcoords.cu:425-432 + models/neural_points/point_query.py:95-98: dense
 *                         [R',SR,K] / [R',SR,3] tensors in the reference layout for the drop-in
 *                         lighting_fast_querier.query_points().
 *   pnb_shade_forward     models/neural_points/neural_points.py:706-717 (gather),
 *                         models/aggregators/point_aggregators.py:727-814,488-644 (weights, PE, MLPs).
 *   pnb_composite_forward models/neural_points_volumetric_model.py:271-305, models/rendering/
 *                         diff_ray_marching.py:508-554 (ray distances, alpha compositing) and :87-123
 *                         (fill_invalid: results are written at full R).
 *   pnb_shade_backward / pnb_composite_backward: the autograd of the above (loss.backward() in
 *                         models/mvs_points_volumetric_model.py:98-118).
 */
#ifndef PNB200_H
#define PNB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* pnb_stream_t; /* cudaStream_t */

typedef enum {
    PNB_OK = 0,
    PNB_ERR_INVALID = -1,    /* bad argument (message in pnb_last_error) */
    PNB_ERR_CUDA = -2,       /* CUDA runtime error */
    PNB_ERR_WORKSPACE = -3,  /* workspace too small */
    PNB_ERR_UNSUPPORTED = -4 /* option value outside the implemented hot-path configuration */
} pnb_status;

#define PNB_MAX_K 8    /* query_worldcoords.cu:14 (#define KN 8) */
#define PNB_MAX_SR 128 /* sample slots per ray */
#define PNB_FEAT 32    /* point_features_dim of most shipped scripts (the default of pnb_points_t.feat_dim) */
#define PNB_FEAT_DTU 63 /* point_features_dim of the DTU scripts (point_{conf,dir,color}_mode "01": colour, dir, conf + 56 image features) */

/* counters written by pnb_grid_build (device int32[16], copied to host on request) */
enum {
    PNB_GC_N_OCC = 0,      /* occupied voxels */
    PNB_GC_MAX_PTS = 1,    /* max points in one voxel (before the P cap) */
    PNB_GC_OVERFLOW_O = 2, /* n_occ > max_o  (reference: random reservoir; here: all voxels kept, flagged) */
    PNB_GC_OVERFLOW_P = 3, /* some voxel > P (reference: random reservoir; here: first P by index, flagged) */
    PNB_GC_N_INRANGE = 4,  /* points inside the grid */
    PNB_GC_SLOT0_CELL = 5, /* linear index of the voxel that holds the lowest-index in-range point (Q1) */
    PNB_GC_FIRST_PT = 6    /* that point's index */
};

/* counters written by pnb_query (device int32[16]) */
enum {
    PNB_QC_N_CAND = 0,   /* candidate samples (occupied march steps kept, <= SR per ray) */
    PNB_QC_N_VALID = 1,  /* samples with >= 1 neighbour (S_v) */
    PNB_QC_N_PAIRS = 2,  /* valid (sample,k) pairs (P_v) */
    PNB_QC_R1 = 3,       /* rays with >= 1 candidate sample */
    PNB_QC_R2 = 4,       /* rays with >= 1 neighbour (R') */
    PNB_QC_OVERFLOW = 5  /* 1 if the candidate capacity was exceeded (results truncated) */
};

/* The voxel grid (device pointers into the caller's buffer) -- plain data, filled by pnb_grid_build. */
typedef struct {
    float lo[3];          /* grid origin = ranges[0:3] of point_query.py:64-66 */
    float svs[3];         /* scaled voxel size = vsize * vscale */
    int32_t dim[3];       /* scaled_vdim */
    int32_t P;            /* per-voxel point cap */
    int32_t parity_slot0; /* 1: replicate query_worldcoords.cu:147 (slot-0 voxel holds no points) */
    int32_t n_points;     /* N */
    uint32_t n_words;     /* ceil(dim0*dim1*dim2 / 32) */
    uint32_t* occ_bits;   /* dilated occupancy (coor_occ), 1 bit per voxel, z fastest */
    uint32_t* pt_bits;    /* voxels that hold >= 1 point */
    uint32_t* word_rank;  /* exclusive prefix of popc(pt_bits[w]): voxel -> dense slot */
    uint32_t* cell_start; /* [n_occ+1] CSR offsets into spts */
    float* spts;          /* [n_inrange] float4 (x, y, z, bitcast point index), voxel-major, ascending index */
    int32_t* counters;    /* device int32[16], see PNB_GC_* */
} pnb_grid_t;

/* Outputs of pnb_query (device pointers into the caller's workspace) -- sample-compacted layout. */
typedef struct {
    int32_t R, SR, K, D;
    int32_t cap_samples;     /* capacity of the per-candidate arrays */
    int32_t* nsamp;          /* [R]   candidate samples of ray r (0..SR) */
    uint32_t* samp_off;      /* [R+1] exclusive prefix of nsamp */
    uint16_t* steps;         /* [R*SR] march step index of candidate j of ray r */
    uint32_t* samp_ray;      /* [cap] ray of candidate s  (r*SR + j packed as r<<7 | j) */
    int32_t* cand_pidx;      /* [cap*K] neighbour point indices, -1 padded, canonical slot order */
    uint8_t* samp_nvalid;    /* [cap] number of neighbours (0..K) */
    uint32_t* valid_list;    /* [cap] candidate ids of valid samples, ascending */
    uint32_t* valid_rank;    /* [cap+1] exclusive prefix of (nvalid>0) */
    uint8_t* ray_hit;        /* [R] 1 if the ray has >= 1 neighbour (ray_mask of the reference) */
    uint32_t* ray_rank;      /* [R+1] scratch: exclusive prefix of ray_hit (filled by pnb_query_export) */
    uint32_t* scan_tmp;      /* scratch of the device-wide scans */
    int32_t* counters;       /* device int32[16], see PNB_QC_* */
    const float* raydir;     /* [R*3] as passed (borrowed) */
    const float* t;          /* borrowed */
    int32_t t_ray_stride;
    float campos[3];
    /* Explicit sample geometry of the perspective-frustum query (pnb_frustum_samples; all NULL for the world query, whose samples lie
     * at campos + raydir * t): the querier's [R',SR,3] tensors, borrowed.  Every slot of a hit ray is a candidate there, so candidate
     * s of ray r is row samp_off[r] / SR = ray_rank[r], slot s - samp_off[r], of these tensors. */
    const float* xs_loc_w;   /* world position of every slot (sample_loc_w) */
    const float* xs_loc;     /* perspective position x/z, y/z, z, jitter applied (sample_loc): dists[3..5] and the ray distances */
    const float* xs_dir;     /* view direction of every slot (sample_ray_dirs) */
} pnb_query_t;

/* Camera + scalar options of the shading / compositing stage. */
typedef struct {
    float campos[3];
    float camrotc2w[9]; /* row-major */
    float Rw2c[9];      /* row-major, points' world->canonical rotation (neural_points.Rw2c) */
    float vsize_z;      /* un-scaled opt.vsize[2]  (neural_points_volumetric_model.py:272) */
    float bg_color[3];
    int32_t raydist_mode_unit;
    int32_t agg_intrp_order; /* opt.agg_intrp_order (point_aggregators.py:573-633): 2 = density per neighbour, then the weighted sum
                              * (every shipped script; 0 is read as 2); 1 = alpha_branch on the K-aggregated feature */
} pnb_shade_opts_t;

/* MLP parameters, fp32, W^T layout [in][out] (transposed once per optimiser step by the host side), zero padded to K_pad rows.
 * block1.0 takes 7F + 60 inputs [f (F), PE3(f) (6F), PE5(dists) (60)] (point_aggregators.py:278-280): K_pad 288 for F = 32, 512 for
 * F = 63. */
typedef struct {
    const float* w[9]; /* block1.0 block1.2 block3.0 block3.2 alpha_branch.0 color_branch.0 .2 .4 .6 */
    const float* b[9];
    int32_t feat_dim;  /* F the block1.0 weights were built for (32 or 63; 0 is read as 32); must equal the points' */
} pnb_mlp_t;

/* Neural point attributes (the reference's parameter tensors, read in place). */
typedef struct {
    const float* xyz;   /* [N,3] */
    const float* emb;   /* [N,feat_dim] points_embeding */
    const float* color; /* [N,3] */
    const float* dir;   /* [N,3] */
    const float* conf;  /* [N]   */
    int32_t N;
    const float* rw2c;  /* [N][9] per-point Rw2c, row-major, or NULL (every point uses pnb_shade_opts_t.Rw2c).  Edited / composed
                         * scenes (run/editing.py) give each point its own frame: a pair's dists and dir use its point's frame, the
                         * view direction of a sample (PE(view) and every pair's extras) the frame of its slot-0 neighbour
                         * (point_aggregators.py:491-496, :506, :526, :566).  No gradient flows to it. */
    int32_t feat_dim;   /* point_features_dim F: 32 or 63 (0 is read as 32); any other width is PNB_ERR_UNSUPPORTED */
} pnb_points_t;

int pnb_version(void);
const char* pnb_last_error(void);
/* sizeof() of the POD structs as the library was compiled (0 grid, 1 query, 2 shade_opts, 3 mlp,
 * 4 points, 5 frustum, 6 vox) -- lets a foreign-language binding verify its mirror of the layout. */
size_t pnb_struct_size(int which);

/* ---- voxel grid ---- */
size_t pnb_grid_bytes(int N, const int32_t dim[3]);
/* Builds the grid into `buf` (>= pnb_grid_bytes).  h_counters (optional, int32[16]) receives the counters
 * AFTER a stream synchronise; pass NULL for a fully asynchronous build. */
int pnb_grid_build(pnb_grid_t* grid, void* buf, size_t buf_bytes, const float* d_xyz, int N,
                   const float lo[3], const float svs[3], const int32_t dim[3], const int32_t query_size[3],
                   int max_o, int P, int parity_slot0, pnb_stream_t stream, int32_t* h_counters);

/* ---- query ---- */
size_t pnb_query_bytes(int R, int SR, int K, int cap_samples);
/* cap_samples <= 0 -> R*SR (can never overflow).  t: [D] (t_ray_stride 0) or [R,D] (t_ray_stride D). */
int pnb_query(pnb_query_t* q, void* ws, size_t ws_bytes, const pnb_grid_t* grid, const float campos[3],
              const float* d_raydir, int R, const float* d_t, int t_ray_stride, int D, int SR, int K,
              float radius_limit, const int32_t kernel_size[3], int cap_samples, pnb_stream_t stream,
              int32_t* h_counters /* optional: synchronises */);
/* Dense reference layout.  d_ray_index [R] scratch (compacted row of each hit ray); outputs hold R rows of
 * capacity; rows >= R' are untouched.  ray_mask [R] int8.  sample_loc (perspective) may be NULL. */
int pnb_query_export(const pnb_query_t* q, const pnb_shade_opts_t* cam, int32_t* d_ray_row,
                     int8_t* d_ray_mask, int32_t* d_sample_pidx, float* d_sample_loc_w, float* d_sample_loc,
                     float* d_sample_ray_dirs, pnb_stream_t stream);

/* ---- shading + compositing, forward ---- */
size_t pnb_shade_bytes(int cap_samples);
/* sigma_rgb: [cap_samples] float4 per candidate sample (zeros for samples without neighbours). */
int pnb_shade_forward(const pnb_query_t* q, const pnb_points_t* pts, const pnb_mlp_t* mlp,
                      const pnb_shade_opts_t* opts, float* d_sigma_rgb, void* ws, size_t ws_bytes,
                      pnb_stream_t stream);
/* Full-R outputs (fill_invalid semantics): ray_color [R,3], opacity [R,SR], bg_T [R], ray_mask [R] int8. */
int pnb_composite_forward(const pnb_query_t* q, const pnb_shade_opts_t* opts, const float* d_sigma_rgb,
                          float* d_ray_color, float* d_opacity, float* d_bg_T, int8_t* d_ray_mask,
                          pnb_stream_t stream);
/* The same with a per-ray background bg_ray [R,3] (bgmodel plane: the reference composites without a background colour and
 * fill_invalid adds coarse_is_background * bg_ray, models/neural_points_volumetric_model.py:101-103, :294-295): ray_color is
 * bg_T * bg_ray + colour for a hit ray (product and sum rounded in that order) and bg_ray for a miss.  opts->bg_color is not read. */
int pnb_composite_forward_bg_ray(const pnb_query_t* q, const pnb_shade_opts_t* opts, const float* d_sigma_rgb, const float* d_bg_ray,
                                 float* d_ray_color, float* d_opacity, float* d_bg_T, int8_t* d_ray_mask, pnb_stream_t stream);

/* ---- auxiliary training outputs ----
 * `weight` [R',SR,K], `conf_coefficient` [R',SR,K] and `blend_weight` [R',SR] of the reference's output dict
 * (models/neural_points_volumetric_model.py:325-329; point_aggregators.py:421-429,727-732; neural_points.py:706-717;
 * diff_ray_marching.py:536-541) for the R' hit rays listed in d_rows (int64 ray ids, ascending), straight from the compacted query.
 * d_opacity: the [R,SR] opacity of pnb_composite_forward.  Empty slots follow the reference (weight 0, conf of point 0). */
int pnb_aux_outputs(const pnb_query_t* q, const pnb_points_t* pts, const long long* d_rows, int n_rows,
                    const float* d_opacity, float* d_weight, float* d_conf_coefficient, float* d_blend_weight,
                    pnb_stream_t stream);
/* d(loss)/d(points_conf) [N] (accumulated into) from d(loss)/d(conf_coefficient) [R',SR,K]: the clamp of neural_points.py:713 is a
 * straight-through estimator, every entry adds its gradient to the conf of its (clamped-to-0) point index. */
int pnb_aux_conf_backward(const pnb_query_t* q, const long long* d_rows, int n_rows,
                          const float* d_grad_conf_coefficient, float* d_grad_conf, pnb_stream_t stream);
/* Probe outputs of point growing (opt.prob == 1, models/neural_points_volumetric_model.py:331-351) from the compacted query and the
 * [R,SR] opacity of pnb_composite_forward: per ray the first slot of maximal opacity oi (torch.max's tie rule; slots past nsamp have
 * opacity 0), its opacity max_opacity [n], its position max_loc [n,3] (bit-identical to pnb_query_export's sample_loc_w; 0 past
 * nsamp), far_dist [n] = min over the K slots of |xyz[max(pidx,0)] - loc| (an empty slot measures point 0, as the reference's clamped
 * gather), and avg_{color [n,3], dir [n,3], conf [n], emb [n,F]} = sum_k w_k attr[max(pidx_k,0)] in k order with
 * w_k = weight * conf_coefficient at oi (bit-identical to the product of pnb_aux_outputs' two outputs; 0 for an empty slot).
 * d_rows: the R' hit rays (int64 ray ids, ascending; n = n_rows), or NULL for all rays (n_rows must be R; a ray that missed gets zeros
 * everywhere, as the reference's unmask fills it).  d_slot (int32 [n]) and d_weight ([n,K]) are optional copies of oi and w_k.
 * K > PNB_MAX_K, SR > PNB_MAX_SR or a width without an instantiation: PNB_ERR_UNSUPPORTED. */
int pnb_probe_outputs(const pnb_query_t* q, const pnb_points_t* pts, const long long* d_rows, int n_rows, const float* d_opacity,
                      float* d_max_opacity, float* d_max_loc, float* d_far_dist, float* d_avg_color, float* d_avg_dir,
                      float* d_avg_conf, float* d_avg_emb, int32_t* d_slot, float* d_weight, pnb_stream_t stream);

/* ---- shading forward on the tensor cores (wgmma, BF16x3 error-compensated split) ---- */
/* Packs block1 / block3 / colour-branch weights of a pnb_mlp_t (fp32 W^T buffers) into wgmma operand images (hi/lo bf16, one
 * [N x 16] image pair per K step in the shared-memory operand layout).  Call once per weight version.  d_out: >= pnb_mlp_pack_bytes(F)
 * bytes, F = mlp->feat_dim (block1.0: 18 K = 16 steps for F = 32, 32 for F = 63; 0 is read as 32). */
size_t pnb_mlp_pack_bytes(int feat_dim);
int pnb_mlp_pack(const pnb_mlp_t* mlp, void* d_out, size_t out_bytes, pnb_stream_t stream);
/* Frozen point cloud (rendering): the 7F point-only inputs [f, PE3(f)] of block1.0 (224 for F = 32, 441 for F = 63;
 * models/aggregators/point_aggregators.py:547-571) are hoisted out of the per-pair work into a per-point table
 * d_pre[N][256] = b1 + W1[:, :7F] . [f_n, PE3(f_n)] (fp32).  Call once per (points_embeding, block1.0) version. */
size_t pnb_point_pre_bytes(int N);
int pnb_point_pre(const pnb_points_t* pts, const pnb_mlp_t* mlp, float* d_pre, size_t pre_bytes, pnb_stream_t stream);
enum {
    PNB_TC_PAIRS = 1,           /* row packing + per-pair MLPs + K-reduction -> h-bar, sigma */
    PNB_TC_COLOR = 2,           /* colour branch -> sigma_rgb (both = a forward) */
    PNB_TC_FROZEN = 4,          /* pair kernel of a frozen cloud (k_shade_wg<FROZEN>): needs d_point_pre */
    PNB_TC_FEW_CTAS = 2048      /* test of the persistent tile loop: one CTA per 8 SMs instead of one per SM (same results) */
};
/* Same contract as pnb_shade_forward; the MLPs run as wgmma tiles.  mlp->w[5] must be zero padded to 288 rows; d_packed holds the images
 * of pnb_mlp_pack for the same F.
 * ws >= pnb_shade_tc_bytes(max_valid_samples).  d_err: device int32[>= 1], 0 on success, 9 if the query produced more valid
 * samples than max_valid_samples (the extra samples are dropped: their sigma_rgb is zeroed, every other result is exact),
 * any other non-zero value = an internal pipeline time-out (a bounded 2-s mbarrier wait expired; results invalid). */
size_t pnb_shade_tc_bytes(int max_valid_samples);
int pnb_shade_forward_tc(const pnb_query_t* q, const pnb_points_t* pts, const pnb_mlp_t* mlp, const void* d_packed,
                         const float* d_point_pre /* NULL unless PNB_TC_FROZEN */, const pnb_shade_opts_t* opts,
                         float* d_sigma_rgb, void* ws, size_t ws_bytes, int max_valid_samples, int flags, int* d_err,
                         pnb_stream_t stream);
/* Diagnostics / tests: device pointers of the row-packing tables inside a workspace laid out for max_valid_samples
 * (vorder uint32[n_valid], vcntp uint8[n_valid], quad_first uint32[n_quads + 1], pack_cnt int32[1] = n_quads). */
int pnb_shade_tc_tables(void* ws, size_t ws_bytes, int max_valid_samples, void** vorder, void** vcntp, void** quad_first,
                        void** pack_cnt);
/* Tests: device pointers of the pair kernel's products inside the same workspace.  hbar: the K-reduced feature of every valid
 * sample as k_color_wg's A operand, per 128 valid samples (vi >> 7) 8 blocks of 16 KB (bf16 hi 8 KB, then lo 8 KB, [128 x 32] in the
 * core-matrix layout of wgmma.cuh), one per 32 channels; sigma: float[n_valid], by valid-sample index. */
int pnb_shade_tc_buffers(void* ws, size_t ws_bytes, int max_valid_samples, void** hbar, void** sigma);

/* ---- backward (per-scene optimisation batches) ----
 * Replaces loss.backward() through the reference's eager autograd graph
 * (models/mvs_points_volumetric_model.py:98-118): given d(loss)/d(ray_color) [R,3], d(loss)/d(opacity) [R,SR] and
 * d(loss)/d(bg_T) [R] (the full-R layout of pnb_composite_forward; each may be NULL, at least one is given; NULL means that output
 * is not in the loss, and with d_ray_color alone the call is the colour-only backward) accumulates gradients of
 * points_embeding [N,F], points_color [N,3], points_dir [N,3],
 * points_conf [N] (any may be NULL) and of the 9 MLP layers in the layout of pnb_mlp_t (W^T [K_pad][N] and bias; the
 * caller zero-initialises all accumulators).  d_sigma_rgb_fwd: the forward's per-candidate (sigma, rgb) buffer.
 * n_valid / n_pairs: host copies of counters[PNB_QC_N_VALID] / [PNB_QC_N_PAIRS] (the pair-level buffers hold one row per valid pair).  ws >= pnb_backward_bytes.  The activations are recomputed and every layer
 * GEMM (recompute, dX, dW) runs on the tensor cores (wgmma, BF16x3 split, fp32 accumulate; dW by a deterministic split-K);
 * the recomputed pre-activations carry the BF16x3 error, so ~1e-6 of the LeakyReLU masks differ from an fp32 forward's (each changes
 * one pair's gradient by ~1/256; see the flags).  d_err: device int32,
 * set non-zero if a bounded pipeline wait of the tensor-core GEMMs expires (results invalid). */
enum {
    PNB_BWD_FP32_GEMM = 1,      /* every GEMM on the fp32 CUDA-core tiles (parity reference of the tensor-core engine) */
    PNB_BWD_FP32_RECOMPUTE = 4  /* forward recompute on the fp32 tiles (LeakyReLU masks of an fp32 forward), dX / dW on the tensor cores */
};
size_t pnb_backward_bytes(int n_valid, int cap_samples, int feat_dim /* F of the points; 0 is read as 32 */);
int pnb_shade_backward(const pnb_query_t* q, const pnb_points_t* pts, const pnb_mlp_t* mlp, const pnb_shade_opts_t* opts,
                       const float* d_sigma_rgb_fwd, const float* d_ray_color /* [R,3] or NULL */,
                       const float* d_opacity /* [R,SR] or NULL */, const float* d_bg_T /* [R] or NULL */, int n_valid, int n_pairs,
                       float* d_emb, float* d_color, float* d_dir, float* d_conf, float* const* d_mlp_w, float* const* d_mlp_b, void* ws,
                       size_t ws_bytes, int flags, int* d_err, pnb_stream_t stream);
/* Diagnostics / tests: device pointers of the forward recompute inside a workspace pnb_shade_backward ran in with the same n_valid,
 * cap_samples and feat_dim; the buffers keep their contents after it returns.  out[10] receives, in this order:
 *   H1, X3, H3, H4 (float, one row per valid pair: ld 256, 272 with H2 in columns 0..255, 256, 256), C1, C2, C3 (float [n_valid][128]):
 *     the post-activations of the 7 LeakyReLU layers (block1.0, block1.2, block3.0, block3.2, color_branch.0 .2 .4); the backward takes
 *     slope 1 where a value is > 0 and 0.01 elsewhere;
 *   pair_off (uint32 [n_valid + 1], the first pair row of each valid sample), row_samp (int32 [n_pairs], valid-sample index of each
 *     row), pidx (int32 [n_pairs], point index of each row). */
int pnb_backward_tables(void* ws, size_t ws_bytes, int n_valid, int cap_samples, int feat_dim, void** out);

/* ---- perspective-frustum neighbour query (wcoord_query 0, NN 2) ----
 * Replaces models/neural_points/query_point_indices.py:263-770 (get_occ_vox, near_vox_full, insert_vox_points,
 * query_neigh_along_ray_layered and their host glue) for the drop-in pointnerf_b200.query_point_indices.  Canonical serial semantics
 * and the reference's quirks: DESIGN.md §5 F1-F9.  The build depends on the points (in perspective coordinates x/z, y/z, z) and the
 * grid only, never on the rays, so one build serves every ray chunk of a view. */
enum {                             /* counters written by pnb_frustum_build (device int32[16]) */
    PNB_FB_N_VOX = 0,              /* voxels holding >= 1 point (truncated coordinates) */
    PNB_FB_MAX_PTS = 1,            /* max points in one voxel (before the P cap) */
    PNB_FB_OVERFLOW_P = 2,         /* voxels with > P points (reference: curand reservoir; here: first P by index) */
    PNB_FB_N_INSERT = 3,           /* points bucketed by truncated coordinates */
    PNB_FB_N_OCC = 4,              /* points inside the grid by floored coordinates */
    PNB_FB_MAX_COL_VOX = 5,        /* max occupied voxels in one column */
    PNB_FB_OVERFLOW_O = 6,         /* 1 if MAX_COL_VOX > max_o (or > 127, the int8 numbering): the reference wraps or overruns */
    PNB_FB_MAX_COL_SAMPLES = 7,    /* max dilated voxels in one column before the SR cap */
    PNB_FB_N_COL_CAPPED = 8        /* columns with more than SR dilated voxels (only the first SR are sampled) */
};
enum {                             /* counters written by pnb_frustum_query (device int32[16] in its workspace) */
    PNB_FQ_R2 = 0,                 /* rays with ray_mask 1 (R') */
    PNB_FQ_N_BAD_PIXEL = 1         /* pixels outside the grid (ray_mask 0; the reference reads out of bounds) */
};
typedef struct {
    float lo[3];            /* ranges[0:3] of get_hyperparameters: x/z, y/z of the image corner, near */
    float svs[3];           /* scaled voxel size (vsize * vscale) */
    float rvs[2];           /* pixel size: svs / vscale (x, y) */
    int32_t dim[3];         /* scaled_vdim */
    int32_t vscale[2];
    int32_t kernel_size[3];
    int32_t query_size[3];
    int32_t SR, K, P, n_points, max_o;
    uint32_t n_words;       /* words of one volume bitmask */
    uint32_t* pt_bits;      /* voxels holding a point by truncated coordinates (the CSR's voxels) */
    uint32_t* occ_bits;     /* voxels holding a point by floored coordinates (the voxels the query searches) */
    uint32_t* word_rank;    /* exclusive prefix of popc(pt_bits[w]) */
    uint32_t* vox_start;    /* CSR offsets into spts */
    float* spts;            /* float4 (x, y, z, bitcast point index), voxel-major, ascending index */
    int16_t* col_list;      /* [dim0*dim1, SR] first SR depth ids of each column's dilated occupancy, -1 padded */
    int32_t* col_far;       /* [dim0*dim1] last dilated depth id of each column (-1: none) */
    int32_t* counters;      /* device int32[16], see PNB_FB_* */
} pnb_frustum_t;

size_t pnb_frustum_bytes(int N, const int32_t dim[3], int SR);
/* NN != 2, inverse != 0, B != 1, K > PNB_MAX_K, SR > PNB_MAX_SR, or a query_size that does not cover the kernel_size search:
 * PNB_ERR_UNSUPPORTED.  max_o <= 0: derived (the reference's default).  h_counters (optional) synchronises. */
int pnb_frustum_build(pnb_frustum_t* fr, void* buf, size_t buf_bytes, const float* d_xyz_pers, int N, int B, const float lo[3],
                      const float svs[3], const int32_t dim[3], const int32_t vscale[3], const int32_t kernel_size[3],
                      const int32_t query_size[3], int SR, int K, int P, int max_o, int NN, int inverse, pnb_stream_t stream,
                      int32_t* h_counters);
/* Ray mask of R pixels (int32 [R,2], (x, y)) and the compaction scan; R' lands in counters[PNB_FQ_R2] of the workspace and, with
 * h_counters (which synchronises), on the host. */
size_t pnb_frustum_query_bytes(int R);
int pnb_frustum_query(const pnb_frustum_t* fr, const int32_t* d_pixel_idx, int R, void* ws, size_t ws_bytes, int8_t* d_ray_mask,
                      pnb_stream_t stream, int32_t* h_counters);
/* Dense reference layout for the R2 = R' rays of a pnb_frustum_query in the same workspace: pixel_idx_cur [R2,2],
 * sample_pidx [R2,SR,K] (-1 padded), sample_loc [R2,SR,3] (perspective; written for every slot).  radius_limit2 / depth_limit2: the
 * squared limits as the reference passes them (np.float32(limit ** 2)); 0 = no limit. */
int pnb_frustum_export(const pnb_frustum_t* fr, const int32_t* d_pixel_idx, int R, const void* ws, size_t ws_bytes,
                       const int8_t* d_ray_mask, int R2, float radius_limit2, float depth_limit2, int32_t* d_pixel_idx_cur,
                       int32_t* d_sample_pidx, float* d_sample_loc, pnb_stream_t stream);
/* Sample-compacted layout (pnb_query_t) of one frustum query for the shading, compositing, auxiliary, probe and backward entry points,
 * which then read the explicit geometry of the querier's tuple instead of forming positions from raydir and t.  d_ray_mask [R] int8
 * and R2 (its number of hit rays, on the host) come from pnb_frustum_query; d_sample_pidx [R2,SR,K] from pnb_frustum_export;
 * d_sample_loc_w, d_sample_loc (jitter applied) and d_sample_ray_dirs [R2,SR,3] from the querier's pers2w.  The four tensors are
 * borrowed and must outlive every call on q.  Every slot of a hit ray is a candidate sample (nsamp = SR): cand_pidx is
 * d_sample_pidx itself, samp_nvalid counts its non-negative entries (they come first, canonical order), ray_hit is the ray mask
 * (a hit ray may have no neighbour at all, as in the reference), and the counters are those of pnb_query.  Nothing synchronises. */
size_t pnb_frustum_samples_bytes(int R, int R2, int SR);
int pnb_frustum_samples(pnb_query_t* q, void* ws, size_t ws_bytes, const int8_t* d_ray_mask, int R, int R2, int SR, int K,
                        const int32_t* d_sample_pidx, const float* d_sample_loc_w, const float* d_sample_loc,
                        const float* d_sample_ray_dirs, pnb_stream_t stream);

/* ---- voxel down-sampling of a point cloud ----
 * Replaces models/mvs/mvs_utils.py:484-561 (construct_vox_points{,_closest,_ind,_xyz}: torch.unique(dim=0) of the floored voxel
 * indices, torch_scatter's scatter_mean and scatter_min) for pointnerf_b200.voxelize.  Results are canonical and identical from run to
 * run: voxels in torch.unique's lexicographic order, a fixed fp64 reduction tree for the centroid, the lowest point index among tied
 * residuals (DESIGN.md §5 "Voxel down-sampling"). */
enum {                             /* counters written by pnb_vox_build (device int32[16] in its workspace) */
    PNB_VC_N_VOX = 0,              /* M: occupied voxels */
    PNB_VC_MAX_PTS = 1,            /* max points in one voxel */
    PNB_VC_N_BIG = 2,              /* voxels of more than 256 points (reduced by a whole block) */
    PNB_VC_N_OUT_OF_KEY = 3        /* points whose voxel index does not fit the key (the call fails) */
};
typedef struct {
    int32_t n_points;              /* N */
    int32_t key_bits;              /* 32 (10 bits per axis, indices in [0, 1024)) or 64 (21 bits, indices in [-2^20, 2^20)) */
    int32_t n_vox;                 /* M */
    int32_t n_big;                 /* counters[PNB_VC_N_BIG] */
    const void* sorted_keys;       /* [N] uint32 | uint64, ascending */
    const uint32_t* sorted_idx;    /* [N] point indices, voxel-major, ascending inside a voxel */
    const uint32_t* seg_start;     /* [M+1] first sorted position of every voxel */
    const uint32_t* big_list;      /* [n_big] voxels of more than 256 points */
    int32_t* counters;             /* device int32[16], see PNB_VC_* */
} pnb_vox_t;

size_t pnb_vox_bytes(int N, int key_bits);
/* Voxel of every point of d_xyz [N,3] (fp32): floorf((p - space_min) / vox_sz) per axis, an IEEE fp32 subtract and a true fp32 divide;
 * d_space_min and d_vox_sz are device float[3].  Sorts, segments and, if d_inv_idx (int64 [N]) is given, writes every point's voxel.
 * Synchronises the stream once, to return M in v->n_vox and the counters in h_counters (int32[16], required).  A voxel index outside
 * the key's range: PNB_ERR_UNSUPPORTED.  v points into ws, which must outlive pnb_vox_outputs on it. */
int pnb_vox_build(pnb_vox_t* v, void* ws, size_t ws_bytes, const float* d_xyz, int N, const float* d_space_min, const float* d_vox_sz,
                  int key_bits, long long* d_inv_idx, pnb_stream_t stream, int32_t* h_counters);
/* Per-voxel outputs of a pnb_vox_build, each optional: d_grid_idx int32 [M,3]; d_centroid fp32 [M,3], the mean of d_val [N,3] (fp32)
 * over the voxel; d_min_idx int64 [M], the voxel's lowest point index, or with closest != 0 the point of d_val nearest its centroid.
 * Nothing synchronises. */
int pnb_vox_outputs(const pnb_vox_t* v, const float* d_val, int32_t* d_grid_idx, float* d_centroid, long long* d_min_idx, int closest,
                    pnb_stream_t stream);

/* ---- plane background of bgmodel plane ----
 * Replaces mvs_utils.get_rayplane_cross (models/mvs/mvs_utils.py:384-408) and the per-view work of MvsPointsVolumetricModel.set_bg
 * (models/mvs_points_volumetric_model.py:272-310: homo_warp_nongrid, homo_warp_fg_mask + id2mask, extract_from_2d_grid's bilinear
 * grid_sample, the +-0.03 plane-colour fit and the max over the views) for pointnerf_b200.plane_bg.  Every fp32 operation is rounded
 * explicitly in the order csrc/plane_bg.cu documents (DESIGN.md §5 "Plane background").  Views: d_w2c [G,4,4] (world -> camera, row 3
 * unread), d_K [G,3,3], d_hdwd int32 [G,2] (HD, WD: the bounds and the normalisation of the view), d_mask_off int64 [G] (offset of
 * view g's foreground mask, int8 [HD,WD] row-major, in d_masks).  Nothing synchronises. */
/* Ray / plane intersections d_xyz [R,3] of the rays d_raydir [R,3] from d_campos [3] with the plane through d_plane_pnt [3] of normal
 * d_plane_normal [3]; (0, 0, 0) where n . d < 0.001f. */
int pnb_plane_cross(const float* d_campos, const float* d_raydir, const float* d_plane_pnt, const float* d_plane_normal, int R,
                    float* d_xyz, pnb_stream_t stream);
/* Foreground masks of the points d_xyz [N,3]: zeroes d_masks (mask_bytes), then sets cell (ceil v, ceil u) of view g to 1 for every
 * point that projects in bounds, without a depth test.  1 <= G <= 65535. */
int pnb_plane_fg_masks(const float* d_xyz, int N, int G, const float* d_w2c, const float* d_K, const int32_t* d_hdwd,
                       const long long* d_mask_off, int8_t* d_masks, size_t mask_bytes, pnb_stream_t stream);
/* bg_ray d_bg [R,3] of the plane points d_xyz [R,3]: per view, the bilinear sample of d_img [G,3,H,W] (fp32) where the point projects
 * in bounds onto a cell whose mask is < 1 and all three channels fit d_plane_color [3] +- 0.03, else 0; the max over the G views. */
int pnb_plane_bg(const float* d_xyz, int R, int G, const float* d_w2c, const float* d_K, const int32_t* d_hdwd,
                 const long long* d_mask_off, const int8_t* d_masks, const float* d_img, int H, int W, const float* d_plane_color,
                 float* d_bg, pnb_stream_t stream);

/* ---- depth filter and visual hull of the initial point cloud ----
 * Replaces filter_utils.filter_by_masks_gpu (models/mvs/filter_utils.py:157-291, manual_depth_view 1) and mvs_utils.alpha_masking
 * (models/mvs/mvs_utils.py:573-607) for pointnerf_b200.depth_filter.  Every fp32 operation is rounded explicitly in the order
 * csrc/depth_filter.cu documents (DESIGN.md §5 "Depth filter and visual hull").
 * Views (V of them, all H x W): d_depth [V,H,W] fp32 (the depth maps), d_K [V,3,3], d_Kinv [V,3,3], d_c2w [V,3,4] (rows 0..2 of the
 * inverse extrinsics), d_pair [V,V,3,4] (pair (r, s): rows 0..2 of E_s inv(E_r)).  A call filters the nr ref views r0 .. r0+nr-1;
 * d_conf, d_mask and d_xyz are device arrays of nr device pointers, one per ref view: its confidence [H,W] fp32, points mask [H,W]
 * (nonzero bytes are true) and camera points [H,W,3] fp32 (raw x, y; the depth is read from d_depth). */
size_t pnb_depth_filter_bytes(int nr, int H, int W);
/* The geometric-consistency test of every pixel of the nr ref views against every other view, the averaged depth, the confidence /
 * mask / geo_cnsst_num decision and, with d_ranges (device float[6], lo then hi; NULL: none), the inclusive range test on the world
 * point.  Synchronises the stream once, to return the number of kept points of every ref view in h_counts (int64 [nr]).  ws must
 * outlive pnb_depth_filter_outputs on it. */
int pnb_depth_filter_build(void* ws, size_t ws_bytes, int V, int H, int W, int r0, int nr, const float* d_depth,
                           const float* const* d_conf, const uint8_t* const* d_mask, const float* const* d_xyz, const float* d_K,
                           const float* d_Kinv, const float* d_c2w, const float* d_pair, const float* d_ranges, float conf_thresh,
                           int geo_cnsst_num, pnb_stream_t stream, long long* h_counts);
/* The kept points of a pnb_depth_filter_build, ref view after ref view, each in row-major pixel order: d_xyz_cam [n,3] (raw x, y and
 * the averaged depth), d_xyz_world [n,3], d_conf_out [n] (n: the sum of h_counts).  Nothing synchronises. */
int pnb_depth_filter_outputs(const void* ws, size_t ws_bytes, int H, int W, int r0, int nr, const float* const* d_xyz,
                             const float* const* d_conf, const float* d_c2w, float* d_xyz_cam, float* d_xyz_world, float* d_conf_out,
                             pnb_stream_t stream);
/* Visual-hull mask d_mask [N] (bytes 0 / 1) of the points d_points [N,3] fp32 over V views: d_w2c [V,3,4] (rows 0..2), d_K [V,3,3],
 * d_alpha [V,H,W] fp32.  h_near_far (host float[2]: near - 1 and far, already rounded to fp32; NULL: no depth test); range_test != 0
 * adds 1 to the alpha of a point whose pixel is outside the image.  Nothing synchronises. */
int pnb_alpha_mask(const float* d_points, long long N, int V, const float* d_w2c, const float* d_K, const float* d_alpha, int H, int W,
                   const float* h_near_far, int range_test, uint8_t* d_mask, pnb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PNB200_H */
