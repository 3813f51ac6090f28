/* TEST INFRASTRUCTURE ONLY -- serial C restatement of the reference's perspective-frustum query
 * (the reference's models/neural_points/query_point_indices.py:263-770, NN 2, inverse 0, B 1) in the canonical order of DESIGN.md §5
 * (F1-F9).  It keeps the reference's own structure -- dense grids, the ray-driven marking of near_vox_full, the per-column numbering,
 * the per-voxel point table -- so that it checks libpnb200's CSR build and its ray independence (F7) rather than restating them.
 *
 * Compile with -ffp-contract=off: every fused multiply-add below is written as fmaf / fma, where the reference's SASS has one (F9).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { C_R2 = 0, C_OVERFLOW_P = 1, C_OVERFLOW_O = 2, C_MAX_O = 3, C_MAX_PTS = 4, C_N_BAD_PIXEL = 5, C_N_CAPPED = 6 };

static int imin(int a, int b) { return a < b ? a : b; }
static int imax(int a, int b) { return a > b ? a : b; }

int pnb_oracle_frustum(const float* pers, int N, const float lo[3], const float svs[3], const int dim[3], const int vscale[3],
                       const int ks[3], const int qs[3], int SR, int K, int P, int max_o_opt, float radius2, float depth2,
                       const int* pixel_idx, int R, int8_t* ray_mask, int* pixel_idx_cur, int* sample_pidx, float* sample_loc,
                       int* counters) {
    const int gx = dim[0], gy = dim[1], gz = dim[2];
    const size_t ncol = (size_t)gx * gy, vol = ncol * gz;
    const float rvs[2] = {(float)((double)svs[0] / vscale[0]), (float)((double)svs[1] / vscale[1])};
    uint8_t* occ = calloc(vol, 1);
    int8_t* loc = calloc(vol, 1);              /* get_occ_vox: -1 = holds a point; near_vox_full: 1 = marked */
    int* near_id = malloc(ncol * sizeof(int));
    int* far_id = malloc(ncol * sizeof(int));
    int16_t* list = malloc(ncol * (size_t)SR * sizeof(int16_t));
    uint8_t* pixel_map = calloc(ncol, 1);
    int* ordv = malloc(vol * sizeof(int));
    if (!occ || !loc || !near_id || !far_id || !list || !pixel_map || !ordv) return -1;
    for (size_t c = 0; c < ncol; ++c) { near_id[c] = gz; far_id[c] = -1; }
    for (size_t i = 0; i < ncol * (size_t)SR; ++i) list[i] = -1;
    memset(counters, 0, 16 * sizeof(int));

    /* get_occ_vox :280-311, points in ascending index (F1): the first point of a voxel dilates it, the rest return */
    for (int i = 0; i < N; ++i) {
        int c[3];
        int in = 1;
        for (int a = 0; a < 3; ++a) {
            float q = (pers[3 * i + a] - lo[a]) / svs[a];
            if (!(q >= 0.0f && q < (float)dim[a])) { in = 0; break; }
            c[a] = (int)floorf(q);
        }
        if (!in) continue;
        size_t v = ((size_t)c[0] * gy + c[1]) * gz + c[2];
        if (loc[v] < 0) continue;
        loc[v] = -1;
        for (int x = imax(0, c[0] - qs[0] / 2); x < imin(gx, c[0] + (qs[0] + 1) / 2); ++x)
            for (int y = imax(0, c[1] - qs[1] / 2); y < imin(gy, c[1] + (qs[1] + 1) / 2); ++y)
                for (int z = imax(0, c[2] - qs[2] / 2); z < imin(gz, c[2] + (qs[2] + 1) / 2); ++z) {
                    size_t col = (size_t)x * gy + y;
                    occ[col * gz + z] = 1;
                    near_id[col] = imin(near_id[col], z);
                    far_id[col] = imax(far_id[col], z);
                }
    }

    /* near_vox_full :332-362, rays in input order; the first ray of a column lists and marks it */
    for (int r = 0; r < R; ++r) {
        int px = pixel_idx[2 * r], py = pixel_idx[2 * r + 1];
        if (px < 0 || py < 0 || px / vscale[0] >= gx || py / vscale[1] >= gy) { ray_mask[r] = 0; counters[C_N_BAD_PIXEL]++; continue; }
        int vx = px / vscale[0], vy = py / vscale[1];
        size_t col = (size_t)vx * gy + vy;
        ray_mask[r] = far_id[col] > 0 ? 1 : 0;       /* F4 */
        if (pixel_map[col]) continue;
        pixel_map[col] = 1;
        int counter = 0, total = 0;
        for (int d = near_id[col]; d <= far_id[col]; ++d) total += occ[col * gz + d];
        if (total > SR) counters[C_N_CAPPED]++;
        for (int d = near_id[col]; d <= far_id[col]; ++d) {
            if (!occ[col * gz + d]) continue;
            list[col * SR + counter] = (int16_t)d;
            for (int x = imax(0, vx - qs[0] / 2); x < imin(gx, vx + (qs[0] + 1) / 2); ++x)
                for (int y = imax(0, vy - qs[1] / 2); y < imin(gy, vy + (qs[1] + 1) / 2); ++y)
                    for (int z = imax(0, d - qs[2] / 2); z < imin(gz, d + (qs[2] + 1) / 2); ++z) {
                        size_t v = ((size_t)x * gy + y) * gz + z;
                        if (loc[v] < 0) loc[v] = 1;
                    }
            if (counter >= SR - 1) break;            /* F5: the first SR */
            counter += 1;
        }
    }

    /* host glue :695-700: marked voxels numbered per column (int32 here; > 127 is the int8 wrap, F8) */
    int max_ord = -1;
    for (size_t col = 0; col < ncol; ++col) {
        int o = 0;
        for (int z = 0; z < gz; ++z) {
            size_t v = col * gz + z;
            ordv[v] = loc[v] > 0 ? o++ : -1;
            if (ordv[v] > max_ord) max_ord = ordv[v];
        }
    }
    int max_o = max_o_opt > 0 ? max_o_opt : max_ord + 1;
    if (max_o < 1) max_o = 1;
    counters[C_MAX_O] = max_o;
    if (max_ord + 1 > max_o || max_ord > 126) counters[C_OVERFLOW_O] = 1;

    /* insert_vox_points :384-410, ascending index, truncated voxel (F3), the first P kept (F2) */
    short* vcnt = calloc(ncol * (size_t)max_o, sizeof(short));
    int* cnt_full = calloc(ncol * (size_t)max_o, sizeof(int));
    int* vpt = malloc(ncol * (size_t)max_o * P * sizeof(int));
    if (!vcnt || !cnt_full || !vpt) return -1;
    for (int i = 0; i < N; ++i) {
        float q[3];
        for (int a = 0; a < 3; ++a) q[a] = (pers[3 * i + a] - lo[a]) / svs[a];
        if (!(q[0] > -1.0f && q[0] < (float)gx && q[1] > -1.0f && q[1] < (float)gy && q[2] > -1.0f && q[2] < (float)gz)) continue;
        int cx = (int)q[0], cy = (int)q[1], cz = (int)q[2];
        size_t col = (size_t)cx * gy + cy, v = col * gz + cz;
        if (ordv[v] < 0 || ordv[v] >= max_o) continue;
        size_t slot = col * max_o + ordv[v];
        int k = cnt_full[slot]++;
        if (k < P) { vpt[slot * P + k] = i; vcnt[slot] = (short)(k + 1); }
        else counters[C_OVERFLOW_P] = 1;
        if (cnt_full[slot] > counters[C_MAX_PTS]) counters[C_MAX_PTS] = cnt_full[slot];
    }

    /* compaction :689-693 */
    int R2 = 0;
    for (int r = 0; r < R; ++r)
        if (ray_mask[r]) { pixel_idx_cur[2 * R2] = pixel_idx[2 * r]; pixel_idx_cur[2 * R2 + 1] = pixel_idx[2 * r + 1]; ++R2; }
    counters[C_R2] = R2;

    /* query_neigh_along_ray_layered :522-597, NN 2 */
    for (int r = 0; r < R2; ++r)
        for (int s = 0; s < SR; ++s) {
            long idx = (long)r * SR + s;
            int px = pixel_idx_cur[2 * r], py = pixel_idx_cur[2 * r + 1];
            int fx = px / vscale[0], fy = py / vscale[1];
            size_t col = (size_t)fx * gy + fy;
            int fz = list[col * SR + s];
            float cx = (float)fma((double)(px % vscale[0]) + 0.5, (double)rvs[0], (double)fmaf((float)fx, svs[0], lo[0]));
            float cy = (float)fma((double)(py % vscale[1]) + 0.5, (double)rvs[1], (double)fmaf((float)fy, svs[1], lo[1]));
            float cz = (float)fma((double)fz + 0.5, (double)svs[2], (double)lo[2]);
            sample_loc[3 * idx] = cx;
            sample_loc[3 * idx + 1] = cy;
            sample_loc[3 * idx + 2] = cz;
            int* out = sample_pidx + idx * K;
            for (int k = 0; k < K; ++k) out[k] = -1;
            if (fz < 0) continue;
            float cxz = cx * cz, cyz = cy * cz;
            int kid = 0, far_ind = 0;
            float far2 = 0.0f, buf[64];
            for (int layer = 0; layer < (ks[0] + 1) / 2; ++layer) {
                int zlayer = imin((ks[2] + 1) / 2 - 1, layer);
                for (int x = imax(-fx, -layer); x < imin(gx - fx, layer + 1); ++x)
                    for (int y = imax(-fy, -layer); y < imin(gy - fy, layer + 1); ++y)
                        for (int z = imax(-fz, -zlayer); z < imin(gz - fz, zlayer + 1); ++z) {
                            if (imax(abs(x), abs(y)) != layer && ((zlayer == layer) ? (abs(z) != zlayer) : 1)) continue;
                            size_t c2 = (size_t)(fx + x) * gy + (fy + y), v = c2 * gz + (fz + z);
                            if (ordv[v] < 0 || ordv[v] >= max_o) continue;
                            size_t slot = c2 * max_o + ordv[v];
                            for (int g = 0; g < imin(P, vcnt[slot]); ++g) {
                                int pi = vpt[slot * P + g];
                                float qx = pers[3 * pi], qy = pers[3 * pi + 1], qz = pers[3 * pi + 2];
                                float xv = fmaf(qx, qz, -cxz), yv = fmaf(qy, qz, -cyz);
                                float xy2 = fmaf(xv, xv, yv * yv);
                                float z2 = (qz - cz) * (qz - cz);
                                float xyz2 = xy2 + z2;
                                if ((radius2 == 0.0f || xy2 <= radius2) && (depth2 == 0.0f || z2 <= depth2)) {
                                    if (kid++ < K) {
                                        out[kid - 1] = pi;
                                        buf[kid - 1] = xyz2;
                                        if (xyz2 > far2) { far2 = xyz2; far_ind = kid - 1; }
                                    } else if (xyz2 < far2) {
                                        out[far_ind] = pi;
                                        buf[far_ind] = xyz2;
                                        far2 = xyz2;
                                        for (int i2 = 0; i2 < K; ++i2)
                                            if (buf[i2] > far2) { far2 = buf[i2]; far_ind = i2; }
                                    }
                                }
                            }
                        }
            }
        }
    free(occ); free(loc); free(near_id); free(far_id); free(list); free(pixel_map); free(ordv); free(vcnt); free(cnt_full); free(vpt);
    return 0;
}
