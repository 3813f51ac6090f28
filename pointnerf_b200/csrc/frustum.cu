// Perspective-frustum neighbour query (wcoord_query 0, NN 2): deterministic per-view build + layered K-NN (DESIGN.md §5, F1-F9).
//
// Replaces the pycuda kernels of the reference's models/neural_points/query_point_indices.py:
//   get_occ_vox                      :263-312   -> k_fr_mark (occ_bits) + k_fr_columns (dilation, near/far)
//   near_vox_full                    :314-363   -> k_fr_columns (first SR depth ids per column) + k_fr_mask (ray_mask)
//   insert_vox_points                :366-411   -> k_fr_mark / k_fr_count / k_fr_scatter / k_fr_sort (CSR, first P by index)
//   query_neigh_along_ray_layered    :493-598   -> k_fr_knn
//   host glue                        :615-770   -> pnb_frustum_query (mask, R' scan) + pnb_frustum_export (compaction, K-NN)
// The build depends on the points and the camera only (F7), so a chunk loop over one view reuses it.  Layout:
//   pt_bits   voxels holding a point by TRUNCATED coordinates (insert_vox_points' bucket, F3); slot = word_rank + popc(below)
//   occ_bits  voxels holding a point by FLOORED coordinates (get_occ_vox's voxel; the only voxels the query searches, F7)
//   vox_start CSR offsets; spts[] = (x,y,z,index) by (voxel, ascending index)
//   col_list  [dim0*dim1, SR] first SR depth ids of the query_size dilation of occ_bits (-1 padded); col_far its last depth id
#include "common.cuh"

namespace pnb {

struct FrParams {
    float lo[3], svs[3], rvs[2];
    int dim[3], vs[2], ks[3], qs[3];
    int N, SR, P;
    uint32_t n_words;
};

// (p - lo) / svs with IEEE fp32 subtract and divide, as get_occ_vox :287-293 and insert_vox_points :389-393.
__device__ __forceinline__ float fr_q(float p, float lo, float svs) { return __fdiv_rn(__fsub_rn(p, lo), svs); }

// pass 1: truncated voxel of every point (pt_cell, pt_bits) and floored occupancy (occ_bits).
__global__ void __launch_bounds__(256) k_fr_mark(const float* __restrict__ xyz, FrParams p, uint32_t* pt_bits, uint32_t* occ_bits,
                                                 uint32_t* pt_cell, int* counters) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    bool tin = true, fin = true;
    int c3[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        float q = fr_q(xyz[3 * i + a], p.lo[a], p.svs[a]);
        tin &= (q > -1.0f) & (q < (float)p.dim[a]);   // (int)q in [0, dim): truncation toward zero
        fin &= (q >= 0.0f) & (q < (float)p.dim[a]);   // floorf(q) in [0, dim)
        c3[a] = tin ? (int)q : 0;
    }
    if (!tin) { pt_cell[i] = 0xffffffffu; return; }
    uint32_t c = cell_index(c3[0], c3[1], c3[2], p.dim);   // floor == trunc whenever fin
    pt_cell[i] = c;
    atomicOr(&pt_bits[c >> 5], 1u << (c & 31));
    atomicAdd(&counters[PNB_FB_N_INSERT], 1);
    if (fin) {
        atomicOr(&occ_bits[c >> 5], 1u << (c & 31));
        atomicAdd(&counters[PNB_FB_N_OCC], 1);
    }
}

// pass 2: voxel -> dense slot, points per slot.
__global__ void __launch_bounds__(256) k_fr_count(FrParams p, const uint32_t* __restrict__ pt_bits,
                                                  const uint32_t* __restrict__ word_rank, uint32_t* pt_cell, uint32_t* cnt) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    uint32_t c = pt_cell[i];
    if (c == 0xffffffffu) return;
    uint32_t slot = word_rank[c >> 5] + __popc(pt_bits[c >> 5] & ((1u << (c & 31)) - 1u));
    pt_cell[i] = slot;
    atomicAdd(&cnt[slot], 1u);
}

// pass 3: scatter into the CSR (order inside a voxel fixed by k_fr_sort).
__global__ void __launch_bounds__(256) k_fr_scatter(const float* __restrict__ xyz, FrParams p, const uint32_t* __restrict__ pt_cell,
                                                    const uint32_t* __restrict__ vox_start, uint32_t* fill, float4* spts) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.N) return;
    uint32_t slot = pt_cell[i];
    if (slot == 0xffffffffu) return;
    uint32_t pos = vox_start[slot] + atomicAdd(&fill[slot], 1u);
    spts[pos] = make_float4(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], __int_as_float(i));
}

// pass 4: ascending point index inside every voxel (F2), P statistics.
__global__ void __launch_bounds__(128) k_fr_sort(FrParams p, const uint32_t* __restrict__ word_rank, const uint32_t* __restrict__ vox_start,
                                                 float4* spts, int* counters) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= word_rank[p.n_words]) return;
    uint32_t a = vox_start[s], b = vox_start[s + 1];
    for (uint32_t i = a + 1; i < b; ++i) {
        float4 v = spts[i];
        int key = __float_as_int(v.w);
        uint32_t j = i;
        while (j > a && __float_as_int(spts[j - 1].w) > key) { spts[j] = spts[j - 1]; --j; }
        spts[j] = v;
    }
    int cnt = (int)(b - a);
    atomicMax(&counters[PNB_FB_MAX_PTS], cnt);
    if (cnt > p.P) atomicAdd(&counters[PNB_FB_OVERFLOW_P], 1);
}

// 32 bits of depth ids [start, start + 32) of the column whose bits begin at `base` (bits outside [0, gz) read as 0).
__device__ __forceinline__ uint32_t col_bits32(const uint32_t* __restrict__ bits, uint32_t n_words, uint64_t base, int start, int gz) {
    int lo = max(start, 0), hi = min(start + 32, gz);
    if (lo >= hi) return 0u;
    uint64_t b = base + (uint64_t)lo;
    uint32_t w = (uint32_t)(b >> 5), sh = (uint32_t)(b & 31);
    uint32_t v = bits[w] >> sh;
    if (sh && w + 1 < n_words) v |= bits[w + 1] << (32 - sh);
    int n = hi - lo;
    if (n < 32) v &= (1u << n) - 1u;
    return v << (lo - start);
}

// pass 5, one warp per column: the query_size dilation of occ_bits (get_occ_vox :299-309) in depth order, its first SR ids
// (near_vox_full :341-361), its last id (far_depth_id) and the number of occupied voxels of the column (the int8 numbering of F8).
__global__ void __launch_bounds__(256) k_fr_columns(FrParams p, const uint32_t* __restrict__ occ_bits, int16_t* col_list, int* col_far,
                                                    int* counters) {
    const int lane = threadIdx.x & 31;
    const uint32_t col = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t ncol = (uint32_t)p.dim[0] * (uint32_t)p.dim[1];
    if (col >= ncol) return;
    const int gz = p.dim[2], x = (int)(col / (uint32_t)p.dim[1]), y = (int)(col % (uint32_t)p.dim[1]);
    const int x0 = max(0, x - (p.qs[0] + 1) / 2 + 1), x1 = min(p.dim[0] - 1, x + p.qs[0] / 2);
    const int y0 = max(0, y - (p.qs[1] + 1) / 2 + 1), y1 = min(p.dim[1] - 1, y + p.qs[1] / 2);
    const int d0 = -((p.qs[2] + 1) / 2 - 1), d1 = p.qs[2] / 2;
    const int nwz = (gz + 31) / 32;
    int carry = 0, far = -1, own = 0;
    for (int k = 0; k < nwz; k += 32) {
        const int w = k + lane;
        uint32_t D = 0;
        if (w < nwz) {
            for (int cx = x0; cx <= x1; ++cx)
                for (int cy = y0; cy <= y1; ++cy) {
                    uint64_t base = ((uint64_t)cx * (uint64_t)p.dim[1] + (uint64_t)cy) * (uint64_t)gz;
                    for (int d = d0; d <= d1; ++d) D |= col_bits32(occ_bits, p.n_words, base, 32 * w + d, gz);
                }
            if (32 * w + 32 > gz) D &= (1u << (gz - 32 * w)) - 1u;   // a shift d < 0 moves depth gz - 1 to gz: not in the column
            own += __popc(col_bits32(occ_bits, p.n_words, (uint64_t)col * (uint64_t)gz, 32 * w, gz));
            if (D) far = 32 * w + 31 - __clz(D);
        }
        const int cnt = __popc(D);
        int incl = cnt;
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        int ord = carry + incl - cnt;
        for (uint32_t bits = D; bits && ord < p.SR; bits &= bits - 1, ++ord)
            col_list[(size_t)col * p.SR + ord] = (int16_t)(32 * w + __ffs(bits) - 1);
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    for (int o = 16; o > 0; o >>= 1) {
        far = max(far, __shfl_xor_sync(0xffffffffu, far, o));
        own += __shfl_xor_sync(0xffffffffu, own, o);
    }
    for (int ord = carry + lane; ord < p.SR; ord += 32) col_list[(size_t)col * p.SR + ord] = (int16_t)-1;
    if (lane == 0) {
        col_far[col] = far;
        atomicMax(&counters[PNB_FB_MAX_COL_VOX], own);
        atomicMax(&counters[PNB_FB_MAX_COL_SAMPLES], carry);
        if (carry > p.SR) atomicAdd(&counters[PNB_FB_N_COL_CAPPED], 1);
    }
}

// The reference numbers the marked voxels of a column with an int8 cumsum (:695-696) into a table of max_o slots per column
// (:698-703): a column with more occupied voxels than that can wrap or overrun it (F8).
__global__ void k_fr_finish(const uint32_t* word_rank, uint32_t n_words, int max_o, int* counters) {
    counters[PNB_FB_N_VOX] = (int)word_rank[n_words];
    const int limit = (max_o > 0 && max_o < 127) ? max_o : 127;
    counters[PNB_FB_OVERFLOW_O] = counters[PNB_FB_MAX_COL_VOX] > limit ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------------- query
__device__ __forceinline__ bool fr_column(const FrParams& p, int px, int py, uint32_t* col) {
    if (px < 0 || py < 0) return false;
    int fx = px / p.vs[0], fy = py / p.vs[1];
    if (fx >= p.dim[0] || fy >= p.dim[1]) return false;
    *col = (uint32_t)fx * (uint32_t)p.dim[1] + (uint32_t)fy;
    return true;
}

// ray_mask = far_id > 0 (near_vox_full :338, F4); pixels outside the grid are misses and are counted.
__global__ void __launch_bounds__(256) k_fr_mask(FrParams p, const int* __restrict__ pixel_idx, int R, const int* __restrict__ col_far,
                                                 int8_t* ray_mask, int* qcounters) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    uint32_t col;
    bool ok = fr_column(p, pixel_idx[2 * r], pixel_idx[2 * r + 1], &col);
    if (!ok) atomicAdd(&qcounters[PNB_FQ_N_BAD_PIXEL], 1);
    ray_mask[r] = (ok && col_far[col] > 0) ? (int8_t)1 : (int8_t)0;
}

__global__ void __launch_bounds__(256) k_fr_compact(const int* __restrict__ pixel_idx, int R, const int8_t* __restrict__ ray_mask,
                                                    const uint32_t* __restrict__ ray_rank, int* pixel_idx_cur) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R || !ray_mask[r]) return;
    uint32_t row = ray_rank[r];
    pixel_idx_cur[2 * row] = pixel_idx[2 * r];
    pixel_idx_cur[2 * row + 1] = pixel_idx[2 * r + 1];
}

// One thread per (compacted ray, sample slot): query_neigh_along_ray_layered :522-597 with NN = 2 and the canonical voxel order (F2).
// The contractions are those of the reference compiled with nvcc's defaults (F9).
template <int KMAX>
__global__ void __launch_bounds__(128) k_fr_knn(FrParams p, const int* __restrict__ pixel_idx_cur, int R2, int K, float radius2,
                                                float depth2, const uint32_t* __restrict__ pt_bits, const uint32_t* __restrict__ occ_bits,
                                                const uint32_t* __restrict__ word_rank, const uint32_t* __restrict__ vox_start,
                                                const float4* __restrict__ spts, const int16_t* __restrict__ col_list, int* sample_pidx,
                                                float* sample_loc) {
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)R2 * p.SR) return;
    const int r = (int)(idx / p.SR), s = (int)(idx - (long long)r * p.SR);
    const int px = pixel_idx_cur[2 * r], py = pixel_idx_cur[2 * r + 1];
    const int fx = px / p.vs[0], fy = py / p.vs[1];
    const uint32_t col = (uint32_t)fx * (uint32_t)p.dim[1] + (uint32_t)fy;
    const int fz = (int)col_list[(size_t)col * p.SR + s];
    const float cx = (float)fma((double)(px % p.vs[0]) + 0.5, (double)p.rvs[0], (double)fmaf((float)fx, p.svs[0], p.lo[0]));
    const float cy = (float)fma((double)(py % p.vs[1]) + 0.5, (double)p.rvs[1], (double)fmaf((float)fy, p.svs[1], p.lo[1]));
    const float cz = (float)fma((double)fz + 0.5, (double)p.svs[2], (double)p.lo[2]);
    sample_loc[3 * idx] = cx;
    sample_loc[3 * idx + 1] = cy;
    sample_loc[3 * idx + 2] = cz;
    int* out = sample_pidx + idx * K;
    for (int k = 0; k < K; ++k) out[k] = -1;
    if (fz < 0) return;
    const float cxz = __fmul_rn(cx, cz), cyz = __fmul_rn(cy, cz);
    int kid = 0, far_ind = 0;
    float far2 = 0.0f;
    float buf[KMAX];
    int ids[KMAX];
    const int nlayer = (p.ks[0] + 1) / 2;
    for (int layer = 0; layer < nlayer; ++layer) {
        const int zlayer = min((p.ks[2] + 1) / 2 - 1, layer);
        for (int x = max(-fx, -layer); x < min(p.dim[0] - fx, layer + 1); ++x)
            for (int y = max(-fy, -layer); y < min(p.dim[1] - fy, layer + 1); ++y)
                for (int z = max(-fz, -zlayer); z < min(p.dim[2] - fz, zlayer + 1); ++z) {
                    if (max(abs(x), abs(y)) != layer && ((zlayer == layer) ? (abs(z) != zlayer) : 1)) continue;
                    const uint32_t c = cell_index(fx + x, fy + y, fz + z, p.dim);
                    const uint32_t m = 1u << (c & 31);
                    if (!(occ_bits[c >> 5] & m)) continue;
                    const uint32_t slot = word_rank[c >> 5] + __popc(pt_bits[c >> 5] & (m - 1u));
                    const uint32_t a = vox_start[slot], b = min(vox_start[slot + 1], a + (uint32_t)p.P);
                    for (uint32_t g = a; g < b; ++g) {
                        const float4 q = spts[g];
                        const float xv = fmaf(q.x, q.z, -cxz);
                        const float yv = fmaf(q.y, q.z, -cyz);
                        const float xy2 = fmaf(xv, xv, __fmul_rn(yv, yv));
                        const float dz = __fsub_rn(q.z, cz);
                        const float z2 = __fmul_rn(dz, dz);
                        const float xyz2 = __fadd_rn(xy2, z2);
                        if ((radius2 == 0.0f || xy2 <= radius2) && (depth2 == 0.0f || z2 <= depth2)) {
                            if (kid++ < K) {
                                ids[kid - 1] = __float_as_int(q.w);
                                buf[kid - 1] = xyz2;
                                if (xyz2 > far2) { far2 = xyz2; far_ind = kid - 1; }
                            } else if (xyz2 < far2) {
                                ids[far_ind] = __float_as_int(q.w);
                                buf[far_ind] = xyz2;
                                far2 = xyz2;
#pragma unroll
                                for (int i = 0; i < KMAX; ++i)
                                    if (i < K && buf[i] > far2) { far2 = buf[i]; far_ind = i; }
                            }
                        }
                    }
                }
    }
    const int n = min(kid, K);
    for (int k = 0; k < n; ++k) out[k] = ids[k];
}

struct FrLayout {
    uint32_t *pt_bits, *occ_bits, *word_rank, *vox_start, *pt_cell, *fill, *scan_tmp;
    float4* spts;
    int16_t* col_list;
    int* col_far;
    int* counters;
    size_t bytes;
};

static FrLayout carve_frustum(void* buf, size_t cap, int N, const int32_t dim[3], int SR) {
    Carver c(buf, cap);
    FrLayout L;
    size_t vol = (size_t)dim[0] * dim[1] * dim[2], ncol = (size_t)dim[0] * dim[1];
    size_t nw = (vol + 31) / 32, nn = (size_t)(N > 0 ? N : 1);
    L.counters = c.take<int>(16);
    L.pt_bits = c.take<uint32_t>(nw);
    L.occ_bits = c.take<uint32_t>(nw);
    L.word_rank = c.take<uint32_t>(nw + 1);
    L.vox_start = c.take<uint32_t>(nn + 1);
    L.spts = c.take<float4>(nn);
    L.pt_cell = c.take<uint32_t>(nn);
    L.fill = c.take<uint32_t>(nn + 1);
    L.scan_tmp = c.take<uint32_t>(scan_tmp_elems(nw > nn ? nw : nn));
    L.col_list = c.take<int16_t>(ncol * (size_t)(SR > 0 ? SR : 1));
    L.col_far = c.take<int>(ncol);
    L.bytes = align_up(c.off);
    return L;
}

static FrParams fr_params(const pnb_frustum_t& f) {
    FrParams p;
    for (int i = 0; i < 3; ++i) {
        p.lo[i] = f.lo[i]; p.svs[i] = f.svs[i]; p.dim[i] = f.dim[i]; p.ks[i] = f.kernel_size[i]; p.qs[i] = f.query_size[i];
    }
    for (int i = 0; i < 2; ++i) { p.rvs[i] = f.rvs[i]; p.vs[i] = f.vscale[i]; }
    p.N = f.n_points; p.SR = f.SR; p.P = f.P; p.n_words = f.n_words;
    return p;
}

// query workspace: counters[16], ray_rank[R+1], scan scratch
struct FqLayout {
    int* counters;
    uint32_t *ray_rank, *scan_tmp;
    size_t bytes;
};

static FqLayout carve_fquery(void* ws, size_t cap, int R) {
    Carver c(ws, cap);
    FqLayout L;
    size_t nr = (size_t)(R > 0 ? R : 1);
    L.counters = c.take<int>(16);
    L.ray_rank = c.take<uint32_t>(nr + 1);
    L.scan_tmp = c.take<uint32_t>(scan_tmp_elems(nr));
    L.bytes = align_up(c.off);
    return L;
}

}  // namespace pnb

using namespace pnb;

extern "C" size_t pnb_frustum_bytes(int N, const int32_t dim[3], int SR) { return carve_frustum(nullptr, 0, N, dim, SR).bytes; }

extern "C" int pnb_frustum_build(pnb_frustum_t* fr, void* buf, size_t buf_bytes, const float* d_xyz_pers, int N, int B,
                                 const float lo[3], const float svs[3], const int32_t dim[3], const int32_t vscale[3],
                                 const int32_t kernel_size[3], const int32_t query_size[3], int SR, int K, int P, int max_o, int NN,
                                 int inverse, pnb_stream_t stream_, int32_t* h_counters) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(fr && buf && d_xyz_pers, PNB_ERR_INVALID, "pnb_frustum_build: null argument");
    PNB_REQUIRE(NN == 2, PNB_ERR_UNSUPPORTED, "pnb_frustum_build: NN=%d (only NN 2, the DTU scripts' value, is implemented)", NN);
    PNB_REQUIRE(inverse == 0, PNB_ERR_UNSUPPORTED, "pnb_frustum_build: inverse=%d (only 0 is implemented)", inverse);
    PNB_REQUIRE(B == 1, PNB_ERR_UNSUPPORTED, "pnb_frustum_build: B=%d (only 1 is implemented)", B);
    PNB_REQUIRE(K >= 1 && K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED, "pnb_frustum_build: K=%d outside 1..%d", K, PNB_MAX_K);
    PNB_REQUIRE(SR >= 1 && SR <= PNB_MAX_SR, PNB_ERR_UNSUPPORTED, "pnb_frustum_build: SR=%d outside 1..%d", SR, PNB_MAX_SR);
    PNB_REQUIRE(N > 0, PNB_ERR_INVALID, "pnb_frustum_build: N must be > 0 (got %d)", N);
    PNB_REQUIRE(P > 0, PNB_ERR_INVALID, "pnb_frustum_build: P must be > 0");
    PNB_REQUIRE(dim[0] > 0 && dim[1] > 0 && dim[2] > 0 && dim[2] <= 32767, PNB_ERR_INVALID, "pnb_frustum_build: bad dim %d %d %d",
                dim[0], dim[1], dim[2]);
    double vol = (double)dim[0] * dim[1] * dim[2];
    PNB_REQUIRE(vol < 4.0e9, PNB_ERR_UNSUPPORTED, "pnb_frustum_build: %g voxels exceed the 32-bit cell index", vol);
    PNB_REQUIRE(svs[0] > 0 && svs[1] > 0 && svs[2] > 0, PNB_ERR_INVALID, "pnb_frustum_build: voxel size must be > 0");
    PNB_REQUIRE(vscale[0] > 0 && vscale[1] > 0, PNB_ERR_INVALID, "pnb_frustum_build: vscale must be > 0");
    for (int a = 0; a < 3; ++a)
        PNB_REQUIRE(kernel_size[a] >= 1 && kernel_size[a] <= 15 && query_size[a] >= 1 && query_size[a] <= 15, PNB_ERR_UNSUPPORTED,
                    "pnb_frustum_build: kernel_size / query_size must be in 1..15");
    // F7: every voxel the layered search visits lies in the query_size box of the sample's own voxel, so the result of a ray does
    // not depend on the other rays of the call
    const int hxy = (kernel_size[0] + 1) / 2 - 1, hz = (kernel_size[2] + 1) / 2 - 1;
    for (int a = 0; a < 3; ++a) {
        const int h = a < 2 ? hxy : hz;
        PNB_REQUIRE(h <= query_size[a] / 2 && h <= (query_size[a] + 1) / 2 - 1, PNB_ERR_UNSUPPORTED,
                    "pnb_frustum_build: query_size %d %d %d does not cover the kernel_size %d %d %d search", query_size[0],
                    query_size[1], query_size[2], kernel_size[0], kernel_size[1], kernel_size[2]);
    }
    FrLayout L = carve_frustum(buf, buf_bytes, N, dim, SR);
    PNB_REQUIRE(L.bytes <= buf_bytes, PNB_ERR_WORKSPACE, "pnb_frustum_build: buffer %zu < required %zu", buf_bytes, L.bytes);

    pnb_frustum_t f;
    for (int i = 0; i < 3; ++i) {
        f.lo[i] = lo[i]; f.svs[i] = svs[i]; f.dim[i] = dim[i]; f.kernel_size[i] = kernel_size[i]; f.query_size[i] = query_size[i];
    }
    for (int i = 0; i < 2; ++i) {
        f.vscale[i] = vscale[i];
        f.rvs[i] = (float)((double)svs[i] / (double)vscale[i]);   // (scaled_vsize_gpu / vscale_gpu).astype(np.float32), :705
    }
    f.SR = SR; f.K = K; f.P = P; f.n_points = N;
    f.max_o = max_o;
    f.n_words = (uint32_t)(((size_t)vol + 31) / 32);
    f.pt_bits = L.pt_bits; f.occ_bits = L.occ_bits; f.word_rank = L.word_rank; f.vox_start = L.vox_start;
    f.spts = (float*)L.spts; f.col_list = L.col_list; f.col_far = L.col_far; f.counters = L.counters;
    const FrParams p = fr_params(f);
    const uint32_t nw = f.n_words, ncol = (uint32_t)dim[0] * (uint32_t)dim[1];

    PNB_CHECK_CUDA(cudaMemsetAsync(L.counters, 0, 16 * sizeof(int), stream));
    PNB_CHECK_CUDA(cudaMemsetAsync(L.pt_bits, 0, nw * sizeof(uint32_t), stream));
    PNB_CHECK_CUDA(cudaMemsetAsync(L.occ_bits, 0, nw * sizeof(uint32_t), stream));
    PNB_CHECK_CUDA(cudaMemsetAsync(L.fill, 0, ((size_t)N + 1) * sizeof(uint32_t), stream));
    const int nbN = (N + 255) / 256;
    k_fr_mark<<<nbN, 256, 0, stream>>>(d_xyz_pers, p, L.pt_bits, L.occ_bits, L.pt_cell, L.counters);
    int rc = exclusive_scan_u32(L.pt_bits, 1, L.word_rank, nw, L.scan_tmp, stream);
    if (rc) return rc;
    k_fr_count<<<nbN, 256, 0, stream>>>(p, L.pt_bits, L.word_rank, L.pt_cell, L.fill);
    rc = exclusive_scan_u32(L.fill, 0, L.vox_start, (uint32_t)N, L.scan_tmp, stream);
    if (rc) return rc;
    PNB_CHECK_CUDA(cudaMemsetAsync(L.fill, 0, ((size_t)N + 1) * sizeof(uint32_t), stream));
    k_fr_scatter<<<nbN, 256, 0, stream>>>(d_xyz_pers, p, L.pt_cell, L.vox_start, L.fill, L.spts);
    k_fr_sort<<<(N + 127) / 128, 128, 0, stream>>>(p, L.word_rank, L.vox_start, L.spts, L.counters);
    k_fr_columns<<<(unsigned)(((size_t)ncol * 32 + 255) / 256), 256, 0, stream>>>(p, L.occ_bits, L.col_list, L.col_far, L.counters);
    k_fr_finish<<<1, 1, 0, stream>>>(L.word_rank, nw, max_o, L.counters);
    PNB_CHECK_CUDA(cudaGetLastError());
    *fr = f;
    if (h_counters) {
        PNB_CHECK_CUDA(cudaMemcpyAsync(h_counters, L.counters, 16 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        PNB_CHECK_CUDA(cudaStreamSynchronize(stream));
    }
    return PNB_OK;
}

extern "C" size_t pnb_frustum_query_bytes(int R) { return carve_fquery(nullptr, 0, R).bytes; }

extern "C" int pnb_frustum_query(const pnb_frustum_t* fr, const int32_t* d_pixel_idx, int R, void* ws, size_t ws_bytes,
                                 int8_t* d_ray_mask, pnb_stream_t stream_, int32_t* h_counters) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(fr && ws && (d_pixel_idx || R == 0) && (d_ray_mask || R == 0), PNB_ERR_INVALID, "pnb_frustum_query: null argument");
    PNB_REQUIRE(R >= 0, PNB_ERR_INVALID, "pnb_frustum_query: R=%d", R);
    FqLayout L = carve_fquery(ws, ws_bytes, R);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_frustum_query: workspace %zu < required %zu", ws_bytes, L.bytes);
    const FrParams p = fr_params(*fr);
    PNB_CHECK_CUDA(cudaMemsetAsync(L.counters, 0, 16 * sizeof(int), stream));
    if (R > 0) k_fr_mask<<<(R + 255) / 256, 256, 0, stream>>>(p, d_pixel_idx, R, fr->col_far, d_ray_mask, L.counters);
    int rc = exclusive_scan_u32(d_ray_mask, 2, L.ray_rank, (uint32_t)R, L.scan_tmp, stream);
    if (rc) return rc;
    PNB_CHECK_CUDA(cudaMemcpyAsync(L.counters + PNB_FQ_R2, L.ray_rank + R, sizeof(int), cudaMemcpyDeviceToDevice, stream));
    PNB_CHECK_CUDA(cudaGetLastError());
    if (h_counters) {
        PNB_CHECK_CUDA(cudaMemcpyAsync(h_counters, L.counters, 16 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        PNB_CHECK_CUDA(cudaStreamSynchronize(stream));
    }
    return PNB_OK;
}

extern "C" int pnb_frustum_export(const pnb_frustum_t* fr, const int32_t* d_pixel_idx, int R, const void* ws, size_t ws_bytes,
                                  const int8_t* d_ray_mask, int R2, float radius_limit2, float depth_limit2, int32_t* d_pixel_idx_cur,
                                  int32_t* d_sample_pidx, float* d_sample_loc, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(fr && ws, PNB_ERR_INVALID, "pnb_frustum_export: null argument");
    PNB_REQUIRE(R2 >= 0 && R2 <= R, PNB_ERR_INVALID, "pnb_frustum_export: R2=%d outside 0..R=%d", R2, R);
    if (R2 == 0) return PNB_OK;
    PNB_REQUIRE(d_pixel_idx && d_ray_mask && d_pixel_idx_cur && d_sample_pidx && d_sample_loc, PNB_ERR_INVALID,
                "pnb_frustum_export: null argument");
    FqLayout L = carve_fquery((void*)ws, ws_bytes, R);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_frustum_export: workspace %zu < required %zu", ws_bytes, L.bytes);
    const FrParams p = fr_params(*fr);
    k_fr_compact<<<(R + 255) / 256, 256, 0, stream>>>(d_pixel_idx, R, d_ray_mask, L.ray_rank, d_pixel_idx_cur);
    const long long ns = (long long)R2 * p.SR;
    k_fr_knn<PNB_MAX_K><<<(unsigned)((ns + 127) / 128), 128, 0, stream>>>(
        p, d_pixel_idx_cur, R2, fr->K, radius_limit2, depth_limit2, fr->pt_bits, fr->occ_bits, fr->word_rank, fr->vox_start,
        (const float4*)fr->spts, fr->col_list, d_sample_pidx, d_sample_loc);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
