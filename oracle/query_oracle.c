/*
 * TEST INFRASTRUCTURE ONLY -- not part of the shipped product path.
 *
 * Serial CPU restatement (plain C) of the reference's wcoord_query=-1 neighbour query:
 *   /root/reference/models/neural_points/cuda/query_worldcoords.cu
 *     claim_occ                       :18-78
 *     map_coor2occ                    :80-115
 *     fill_occ2pnts                   :117-162
 *     mask_raypos                     :165-189
 *     host glue (ray compaction, cumsum / first-SR rule)   :381-391
 *     get_shadingloc                  :192-214
 *     query_neigh_along_ray_layered   :217-302
 *     host glue (drop rays without neighbours)             :425-429
 * under the canonical serial semantics of SURVEY.md section 8(a) (Q1-Q7): the reference
 * kernels are racy (atomics) and use wall-clock-seeded curand on overflow; the canonical
 * form is "what a single thread visiting points/samples in ascending index order produces",
 * with overflow (more than max_o occupied voxels / more than P points per voxel) REPORTED
 * through counters instead of resolved randomly.
 *
 * Pinning: the reference ships no tests / golden vectors for this path (SURVEY 8c), and its
 * CUDA kernels cannot run in the build container (no GPU).  The restatement is therefore
 * pinned (i) structurally, line by line, against the cited source and (ii) by
 * tests/test_oracle_query.py against an independent brute-force numpy formulation.
 * Parity status: "pinned against own brute force + reference Python glue; reference CUDA
 * kernel itself not executed".
 *
 * Numerics that decide integers (must match the reference's SASS, SURVEY 8a):
 *   voxel coordinate  (int)floorf((p - lo) / svs)   IEEE fp32 sub then div  (.cu:40-42)
 *   sample position   campos + raydir * t           fp32 mul then add, NO fma (torch ops,
 *                                                   diff_ray_marching.py:386)
 *   distance          fmaf(dz,dz, fmaf(dx,dx, dy*dy))  (nvcc contraction of .cu:274)
 * Build with -ffp-contract=off so gcc never fuses what the reference does not.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define PNB_ORACLE_MAXK 8 /* query_worldcoords.cu:14  #define KN 8  (Q6) */

static inline int vox1(float p, float lo, float svs) {
    volatile float d = p - lo;     /* .cu:40 */
    volatile float q = d / svs;
    return (int)floorf(q);
}

/* counters[] layout (all int32):
 *  0 n_occ            number of occupied voxels (claim_occ's occ_idx, before the max_o cap)
 *  1 max_pts          max #points that fell in one voxel (before the P cap)
 *  2 overflow_o       1 if n_occ > max_o           (reference: random reservoir, Q3)
 *  3 overflow_p       1 if some voxel got > P pts  (reference: random reservoir, Q3)
 *  4 R1               rays surviving pass 1 (any occupied march step, .cu:381-382)
 *  5 R2               rays surviving pass 2 (any neighbour, .cu:425-426)
 *  6 n_valid_samples  samples with >= 1 neighbour  (S_v of SURVEY 8d)
 *  7 n_valid_pairs    (sample,k) slots with pidx>=0 (P_v of SURVEY 8d)
 *  8 n_cand           candidate points visited by the K-NN loop (for the bytes model)
 *  9 slot0_cell       linear cell index of the voxel that won slot 0 (Q1) or -1
 */
int pnb_oracle_query(
    const float* xyz, int N,
    const float* lo,          /* ranges[0:3]  = d_coord_shift */
    const float* svs,         /* scaled voxel size (vsize*vscale) */
    const int* dim,           /* scaled_vdim */
    const int* kernel_size, const int* query_size,
    int max_o, int P, float radius_limit,
    const float* campos,      /* 3 */
    const float* raydir, int R,
    const float* t, int t_ray_stride, int D, /* t[r*t_ray_stride + d]; stride 0 = shared table */
    const float* raypos,      /* optional R*D*3: if non-NULL these positions are used verbatim
                                 (the pybind op receives raypos, query_worldcoords.cpp:36) */
    int SR, int K,
    int parity_slot0,         /* 1: slot 0 holds no points (.cu:147, Q1); 0: every stored voxel keeps its points */
    int8_t* ray_mask,         /* R */
    int* sample_pidx,         /* R*SR*K, first R2 rows valid, -1 padded */
    float* sample_loc_w,      /* R*SR*3, first R2 rows valid, zeros where unfilled */
    int* counters)
{
    if (K > PNB_ORACLE_MAXK || K < 1) return -1;
    const long vol = (long)dim[0] * dim[1] * dim[2];
    int* coor_2_occ = (int*)malloc(sizeof(int) * (size_t)vol);      /* .cu:318 full(-1) */
    uint8_t* coor_occ = (uint8_t*)calloc((size_t)vol, 1);           /* .cu:314 zeros   */
    int* occ_2_coor = (int*)malloc(sizeof(int) * 3 * (size_t)(max_o > 0 ? max_o : 1));
    int* occ_numpnts = (int*)calloc((size_t)(max_o > 0 ? max_o : 1), sizeof(int));
    int* occ_2_pnts = (int*)malloc(sizeof(int) * (size_t)(max_o > 0 ? max_o : 1) * (size_t)P);
    if (!coor_2_occ || !coor_occ || !occ_2_coor || !occ_numpnts || !occ_2_pnts) return -2;
    for (long c = 0; c < vol; ++c) coor_2_occ[c] = -1;
    memset(occ_2_pnts, 0xff, sizeof(int) * (size_t)(max_o > 0 ? max_o : 1) * (size_t)P);
    memset(counters, 0, sizeof(int) * 10);
    counters[9] = -1;

    /* ---- claim_occ (.cu:18-78) + the coor_2_occ write of map_coor2occ (.cu:102), serial ---- */
    int n_occ = 0;
    for (int i = 0; i < N; ++i) {
        int c0 = vox1(xyz[3 * i + 0], lo[0], svs[0]);
        int c1 = vox1(xyz[3 * i + 1], lo[1], svs[1]);
        int c2 = vox1(xyz[3 * i + 2], lo[2], svs[2]);
        if (c0 < 0 || c0 >= dim[0] || c1 < 0 || c1 >= dim[1] || c2 < 0 || c2 >= dim[2]) continue; /* .cu:44 */
        long c = (long)c0 * dim[1] * dim[2] + (long)c1 * dim[2] + c2;
        if (coor_2_occ[c] == -1) {
            int slot = n_occ++;
            if (slot < max_o) {                     /* .cu:59-63 */
                occ_2_coor[3 * slot + 0] = c0; occ_2_coor[3 * slot + 1] = c1; occ_2_coor[3 * slot + 2] = c2;
                coor_2_occ[c] = slot;               /* .cu:102, after the full(-1) reset of .cu:337 */
                if (slot == 0) counters[9] = (int)c;
            } else {
                counters[2] = 1;                    /* Q3: reference resolves randomly; we flag */
                coor_2_occ[c] = -2;                 /* claimed but not stored: stays "no slot" below */
            }
        }
    }
    counters[0] = n_occ;
    const int n_slots = n_occ < max_o ? n_occ : max_o;
    for (long c = 0; c < vol; ++c) if (coor_2_occ[c] == -2) coor_2_occ[c] = -1;

    /* ---- map_coor2occ dilation (.cu:105-112) ---- */
    for (int s = 0; s < n_slots; ++s) {
        int c0 = occ_2_coor[3 * s], c1 = occ_2_coor[3 * s + 1], c2 = occ_2_coor[3 * s + 2];
        int x0 = c0 - query_size[0] / 2; if (x0 < 0) x0 = 0;
        int x1 = c0 + (query_size[0] + 1) / 2; if (x1 > dim[0]) x1 = dim[0];
        int y0 = c1 - query_size[1] / 2; if (y0 < 0) y0 = 0;
        int y1 = c1 + (query_size[1] + 1) / 2; if (y1 > dim[1]) y1 = dim[1];
        int z0 = c2 - query_size[2] / 2; if (z0 < 0) z0 = 0;
        int z1 = c2 + (query_size[2] + 1) / 2; if (z1 > dim[2]) z1 = dim[2];
        for (int x = x0; x < x1; ++x)
            for (int y = y0; y < y1; ++y)
                for (int z = z0; z < z1; ++z)
                    coor_occ[(long)x * dim[1] * dim[2] + (long)y * dim[2] + z] = 1;
    }

    /* ---- fill_occ2pnts (.cu:117-162), NOTE voxel_idx > 0 (.cu:147, Q1) unless parity_slot0 is 0 ---- */
    int* raw_cnt = (int*)calloc((size_t)(n_slots > 0 ? n_slots : 1), sizeof(int));
    for (int i = 0; i < N; ++i) {
        int c0 = vox1(xyz[3 * i + 0], lo[0], svs[0]);
        int c1 = vox1(xyz[3 * i + 1], lo[1], svs[1]);
        int c2 = vox1(xyz[3 * i + 2], lo[2], svs[2]);
        if (c0 < 0 || c0 >= dim[0] || c1 < 0 || c1 >= dim[1] || c2 < 0 || c2 >= dim[2]) continue;
        long c = (long)c0 * dim[1] * dim[2] + (long)c1 * dim[2] + c2;
        int s = coor_2_occ[c];
        if (s >= 0) { raw_cnt[s]++; if (raw_cnt[s] > counters[1]) counters[1] = raw_cnt[s]; }
        if (s > 0 || (s == 0 && !parity_slot0)) {
            int tmp = occ_numpnts[s]++;
            if (tmp < P) occ_2_pnts[(long)s * P + tmp] = i;
            else counters[3] = 1;                   /* Q3: reference reservoir-samples; we keep first P */
        }
    }
    free(raw_cnt);

    /* ---- mask_raypos + glue + get_shadingloc + query + glue, one ray at a time ---- */
    const float r2 = radius_limit * radius_limit;   /* .cu:410, fp32 product on host */
    const int nlayer = (kernel_size[0] + 1) / 2;    /* .cu:250 */
    int R1 = 0, R2 = 0;
    int* pidx_row = (int*)malloc(sizeof(int) * (size_t)SR * K);
    float* loc_row = (float*)malloc(sizeof(float) * (size_t)SR * 3);
    for (int r = 0; r < R; ++r) {
        ray_mask[r] = 0;
        const float* tr = raypos ? 0 : t + (long)r * t_ray_stride;
        const float dx = raypos ? 0.f : raydir[3 * r], dy = raypos ? 0.f : raydir[3 * r + 1], dz = raypos ? 0.f : raydir[3 * r + 2];
        int nsamp = 0, anyhit = 0;
        for (int j = 0; j < SR * 3; ++j) loc_row[j] = 0.f;          /* .cu:383 zeros */
        for (int j = 0; j < SR * K; ++j) pidx_row[j] = -1;          /* .cu:384 full(-1) */
        for (int d = 0; d < D; ++d) {
            volatile float px, py, pz;
            if (raypos) {
                px = raypos[((long)r * D + d) * 3]; py = raypos[((long)r * D + d) * 3 + 1]; pz = raypos[((long)r * D + d) * 3 + 2];
            } else {
                volatile float mx = dx * tr[d], my = dy * tr[d], mz = dz * tr[d];
                px = campos[0] + mx; py = campos[1] + my; pz = campos[2] + mz;
            }
            int c0 = vox1(px, lo[0], svs[0]), c1 = vox1(py, lo[1], svs[1]), c2 = vox1(pz, lo[2], svs[2]);
            if (c0 < 0 || c0 >= dim[0] || c1 < 0 || c1 >= dim[1] || c2 < 0 || c2 >= dim[2]) continue; /* .cu:185 */
            if (!coor_occ[(long)c0 * dim[1] * dim[2] + (long)c1 * dim[2] + c2]) continue;
            anyhit = 1;
            if (nsamp < SR) {                                        /* cumsum<=SR rule, .cu:390-391 */
                loc_row[3 * nsamp] = px; loc_row[3 * nsamp + 1] = py; loc_row[3 * nsamp + 2] = pz; /* .cu:207-211 */
                nsamp++;
            }
        }
        if (!anyhit) continue;                                       /* pass 1, .cu:381-388 */
        R1++;
        int any_nb = 0;
        for (int s = 0; s < nsamp; ++s) {                            /* query_neigh_along_ray_layered */
            const float cx = loc_row[3 * s], cy = loc_row[3 * s + 1], cz = loc_row[3 * s + 2];
            const int fx = vox1(cx, lo[0], svs[0]), fy = vox1(cy, lo[1], svs[1]), fz = vox1(cz, lo[2], svs[2]);
            int kid = 0, far_ind = 0;
            float far2 = 0.f;
            float buf[PNB_ORACLE_MAXK];
            int* out = pidx_row + (long)s * K;
            for (int layer = 0; layer < nlayer; ++layer) {
                int xa = -fx > -layer ? -fx : -layer, xb = dim[0] - fx < layer + 1 ? dim[0] - fx : layer + 1;
                int ya = -fy > -layer ? -fy : -layer, yb = dim[1] - fy < layer + 1 ? dim[1] - fy : layer + 1;
                int za = -fz > -layer ? -fz : -layer, zb = dim[2] - fz < layer + 1 ? dim[2] - fz : layer + 1;
                for (int x = xa; x < xb; ++x)
                    for (int y = ya; y < yb; ++y)
                        for (int z = za; z < zb; ++z) {
                            int ax = abs(x), ay = abs(y), az = abs(z);
                            int m = ax > ay ? ax : ay; m = m > az ? m : az;
                            if (m != layer) continue;                /* .cu:261 */
                            long c = (long)(fx + x) * dim[1] * dim[2] + (long)(fy + y) * dim[2] + (fz + z);
                            int occ = coor_2_occ[c];
                            if (occ < 0) continue;                   /* .cu:266 */
                            int cnt = occ_numpnts[occ] < P ? occ_numpnts[occ] : P;
                            for (int g = 0; g < cnt; ++g) {
                                int pi = occ_2_pnts[(long)occ * P + g];
                                float xv = xyz[3 * pi] - cx, yv = xyz[3 * pi + 1] - cy, zv = xyz[3 * pi + 2] - cz;
                                volatile float yy = yv * yv;
                                float d2 = fmaf(zv, zv, fmaf(xv, xv, yy)); /* SASS order, SURVEY 8a */
                                counters[8]++;
                                if (r2 == 0.f || d2 <= r2) {          /* .cu:275 */
                                    if (kid++ < K) {
                                        out[kid - 1] = pi; buf[kid - 1] = d2;
                                        if (d2 > far2) { far2 = d2; far_ind = kid - 1; }
                                    } else if (d2 < far2) {
                                        out[far_ind] = pi; buf[far_ind] = d2; far2 = d2;
                                        for (int i2 = 0; i2 < K; ++i2)
                                            if (buf[i2] > far2) { far2 = buf[i2]; far_ind = i2; }
                                    }
                                }
                            }
                        }
                if (kid >= K) break;                                 /* .cu:300 */
            }
            if (kid > 0) any_nb = 1;
        }
        if (!any_nb) continue;                                       /* pass 2, .cu:425-429 */
        ray_mask[r] = 1;
        memcpy(sample_pidx + (long)R2 * SR * K, pidx_row, sizeof(int) * (size_t)SR * K);
        memcpy(sample_loc_w + (long)R2 * SR * 3, loc_row, sizeof(float) * (size_t)SR * 3);
        for (int s = 0; s < SR; ++s) {
            int nv = 0;
            for (int k = 0; k < K; ++k) nv += pidx_row[s * K + k] >= 0;
            counters[7] += nv; counters[6] += nv > 0;
        }
        R2++;
    }
    counters[4] = R1; counters[5] = R2;
    free(pidx_row); free(loc_row);
    free(coor_2_occ); free(coor_occ); free(occ_2_coor); free(occ_numpnts); free(occ_2_pnts);
    return 0;
}
