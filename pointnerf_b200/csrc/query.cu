// Ray march + first-SR sample selection + layered voxel K-NN, sample-compacted.
//
// Replaces (per call):
//   near_far_linear_ray_generation  /root/reference/models/rendering/diff_ray_marching.py:349-392
//        (raypos [1,R,400,3] is never materialised; positions are campos + raydir*t[d] in-kernel)
//   mask_raypos                     /root/reference/models/neural_points/cuda/query_worldcoords.cu:165-189
//   host glue (cumsum / first SR)   :381-391
//   get_shadingloc                  :192-214
//   query_neigh_along_ray_layered   :217-302
//   host glue (ray drop)            :425-429
// The integer decisions follow the canonical serial semantics of SURVEY.md 8(a) bit for bit: voxel index by
// IEEE sub+div+floor, distance fmaf(dz,dz,fmaf(dx,dx,dy*dy)), traversal x-major then y, z, list order,
// replace-farthest K buffer with strict '<', shell early-out once K candidates were seen.
#include "common.cuh"

namespace pnb {

struct QueryParams {
    GridDev g;
    float campos[3];
    const float* raydir;
    const float* t;
    int t_ray_stride;
    int R, D, SR, K;
    int ks0;  // kernel_size[0]
    float r2;
    int cap;
};

// One warp per ray: 32 march steps per iteration, ballot -> ordered slots.
__global__ void __launch_bounds__(256) k_march(QueryParams p, int* __restrict__ nsamp, uint16_t* __restrict__ steps) {
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (warp >= p.R) return;
    const int r = warp;
    const float dx = p.raydir[3 * r], dy = p.raydir[3 * r + 1], dz = p.raydir[3 * r + 2];
    const float* tr = p.t + (size_t)r * p.t_ray_stride;
    int count = 0;
    for (int base = 0; base < p.D; base += 32) {
        int d = base + lane;
        bool hit = false;
        if (d < p.D) {
            float t = tr[d];
            int x = vox1(raypos1(p.campos[0], dx, t), p.g.lo[0], p.g.svs[0]);
            int y = vox1(raypos1(p.campos[1], dy, t), p.g.lo[1], p.g.svs[1]);
            int z = vox1(raypos1(p.campos[2], dz, t), p.g.lo[2], p.g.svs[2]);
            if (in_grid(x, y, z, p.g.dim)) {
                uint32_t c = cell_index(x, y, z, p.g.dim);
                hit = (__ldg(&p.g.occ_bits[c >> 5]) >> (c & 31)) & 1u;
            }
        }
        uint32_t m = __ballot_sync(0xffffffffu, hit);
        int slot = count + __popc(m & ((1u << lane) - 1u));
        if (hit && slot < p.SR) steps[(size_t)r * p.SR + slot] = (uint16_t)d;
        count += __popc(m);
        if (count >= p.SR) break;
    }
    if (lane == 0) nsamp[r] = count < p.SR ? count : p.SR;
}

// candidate s -> packed (ray, slot)
__global__ void __launch_bounds__(256) k_expand(int R, int SR, int cap, const int* __restrict__ nsamp,
                                                const uint32_t* __restrict__ samp_off, uint32_t* __restrict__ samp_ray,
                                                int* counters) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R * SR) return;
    int r = i / SR, j = i - r * SR;
    if (j >= nsamp[r]) return;
    uint32_t s = samp_off[r] + j;
    if (s >= (uint32_t)cap) { counters[PNB_QC_OVERFLOW] = 1; return; }
    samp_ray[s] = ((uint32_t)r << 7) | (uint32_t)j;
    if (j == 0) atomicAdd(&counters[PNB_QC_R1], 1);
}

// One thread per candidate sample: canonical layered K-NN.
__global__ void __launch_bounds__(128) k_knn(QueryParams p, const uint32_t* __restrict__ samp_off,
                                             const uint32_t* __restrict__ samp_ray, const uint16_t* __restrict__ steps,
                                             int* __restrict__ cand_pidx, uint8_t* __restrict__ samp_nvalid,
                                             uint8_t* __restrict__ ray_hit, int* counters) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n_cand = min(samp_off[p.R], (uint32_t)p.cap);
    if (s >= n_cand) return;
    uint32_t pk = samp_ray[s];
    int r = (int)(pk >> 7), j = (int)(pk & 127u);
    int d = steps[(size_t)r * p.SR + j];
    float t = p.t[(size_t)r * p.t_ray_stride + d];
    const float cx = raypos1(p.campos[0], p.raydir[3 * r], t);
    const float cy = raypos1(p.campos[1], p.raydir[3 * r + 1], t);
    const float cz = raypos1(p.campos[2], p.raydir[3 * r + 2], t);
    const int fx = vox1(cx, p.g.lo[0], p.g.svs[0]);
    const int fy = vox1(cy, p.g.lo[1], p.g.svs[1]);
    const int fz = vox1(cz, p.g.lo[2], p.g.svs[2]);
    const int dead = p.g.parity_slot0 ? p.g.counters[PNB_GC_SLOT0_CELL] : -1;

    int idx[PNB_MAX_K];
    float buf[PNB_MAX_K];
#pragma unroll
    for (int m = 0; m < PNB_MAX_K; ++m) { idx[m] = -1; buf[m] = 0.f; }
    int kid = 0, far_ind = 0;
    float far2 = 0.f;
    const int nlayer = (p.ks0 + 1) / 2;
    for (int layer = 0; layer < nlayer; ++layer) {
        const int xa = max(-fx, -layer), xb = min(p.g.dim[0] - fx, layer + 1);
        const int ya = max(-fy, -layer), yb = min(p.g.dim[1] - fy, layer + 1);
        const int za = max(-fz, -layer), zb = min(p.g.dim[2] - fz, layer + 1);
        for (int x = xa; x < xb; ++x)
            for (int y = ya; y < yb; ++y)
                for (int z = za; z < zb; ++z) {
                    if (max(abs(z), max(abs(x), abs(y))) != layer) continue;
                    uint32_t c = cell_index(fx + x, fy + y, fz + z, p.g.dim);
                    uint32_t w = __ldg(&p.g.pt_bits[c >> 5]);
                    if (!((w >> (c & 31)) & 1u)) continue;
                    if ((int)c == dead) continue;  // query_worldcoords.cu:147 (slot 0 never filled)
                    uint32_t slot = __ldg(&p.g.word_rank[c >> 5]) + __popc(w & ((1u << (c & 31)) - 1u));
                    uint32_t a = __ldg(&p.g.cell_start[slot]), b = __ldg(&p.g.cell_start[slot + 1]);
                    if (b - a > (uint32_t)p.g.P) b = a + (uint32_t)p.g.P;
                    for (uint32_t g = a; g < b; ++g) {
                        float4 q = __ldg(&p.g.spts[g]);
                        float xv = __fsub_rn(q.x, cx), yv = __fsub_rn(q.y, cy), zv = __fsub_rn(q.z, cz);
                        float d2 = __fmaf_rn(zv, zv, __fmaf_rn(xv, xv, __fmul_rn(yv, yv)));
                        if (p.r2 == 0.f || d2 <= p.r2) {
                            int pi = __float_as_int(q.w);
                            if (kid++ < p.K) {
                                int slotk = kid - 1;
#pragma unroll
                                for (int m = 0; m < PNB_MAX_K; ++m)
                                    if (m == slotk) { idx[m] = pi; buf[m] = d2; }
                                if (d2 > far2) { far2 = d2; far_ind = slotk; }
                            } else if (d2 < far2) {
#pragma unroll
                                for (int m = 0; m < PNB_MAX_K; ++m)
                                    if (m == far_ind) { idx[m] = pi; buf[m] = d2; }
                                far2 = d2;
#pragma unroll
                                for (int m = 0; m < PNB_MAX_K; ++m)
                                    if (m < p.K && buf[m] > far2) { far2 = buf[m]; far_ind = m; }
                            }
                        }
                    }
                }
        if (kid >= p.K) break;
    }
    int nv = kid < p.K ? kid : p.K;
#pragma unroll
    for (int m = 0; m < PNB_MAX_K; ++m)
        if (m < p.K) cand_pidx[(size_t)s * p.K + m] = idx[m];
    samp_nvalid[s] = (uint8_t)nv;
    if (nv > 0) {
        ray_hit[r] = 1;
        atomicAdd(&counters[PNB_QC_N_PAIRS], nv);
    }
}

__global__ void __launch_bounds__(256) k_valid_list(int R, int cap, const uint32_t* __restrict__ samp_off,
                                                    const uint8_t* __restrict__ samp_nvalid,
                                                    const uint32_t* __restrict__ valid_rank, uint32_t* __restrict__ valid_list,
                                                    int* counters) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n_cand = min(samp_off[R], (uint32_t)cap);
    if (s == 0) {
        counters[PNB_QC_N_CAND] = (int)n_cand;
        counters[PNB_QC_N_VALID] = (int)valid_rank[n_cand];
    }
    if (s >= n_cand) return;
    if (samp_nvalid[s] > 0) valid_list[valid_rank[s]] = s;
}

__global__ void __launch_bounds__(256) k_count_rays(int R, const uint8_t* __restrict__ ray_hit, int* counters) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    int v = (r < R && ray_hit[r]) ? 1 : 0;
    uint32_t m = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(&counters[PNB_QC_R2], __popc(m));
}

// Dense reference layout: rows of rays with ray_hit, in ray order.
__global__ void __launch_bounds__(128) k_export(pnb_query_t q, float R00, float R10, float R20, float R01, float R11,
                                                float R21, float R02, float R12, float R22,
                                                const uint32_t* __restrict__ ray_rank, int32_t* __restrict__ ray_row,
                                                int8_t* __restrict__ ray_mask, int32_t* __restrict__ sample_pidx,
                                                float* __restrict__ sample_loc_w, float* __restrict__ sample_loc,
                                                float* __restrict__ sample_ray_dirs) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;  // (ray, slot)
    if (i >= q.R * q.SR) return;
    int r = i / q.SR, j = i - r * q.SR;
    bool hit = q.ray_hit[r] != 0;
    if (j == 0) { ray_mask[r] = hit ? 1 : 0; ray_row[r] = hit ? (int)ray_rank[r] : -1; }
    if (!hit) return;
    size_t row = (size_t)ray_rank[r] * q.SR + j;
    float lx = 0.f, ly = 0.f, lz = 0.f;
    int n = q.nsamp[r];
    if (j < n) {
        uint32_t s = q.samp_off[r] + j;
        int d = q.steps[(size_t)r * q.SR + j];
        float t = q.t[(size_t)r * q.t_ray_stride + d];
        lx = raypos1(q.campos[0], q.raydir[3 * r], t);
        ly = raypos1(q.campos[1], q.raydir[3 * r + 1], t);
        lz = raypos1(q.campos[2], q.raydir[3 * r + 2], t);
        for (int k = 0; k < q.K; ++k) sample_pidx[row * q.K + k] = q.cand_pidx[(size_t)s * q.K + k];
    } else {
        for (int k = 0; k < q.K; ++k) sample_pidx[row * q.K + k] = -1;
    }
    sample_loc_w[row * 3] = lx; sample_loc_w[row * 3 + 1] = ly; sample_loc_w[row * 3 + 2] = lz;
    if (sample_loc) {  // point_query.py:101-108
        float sx = lx - q.campos[0], sy = ly - q.campos[1], sz = lz - q.campos[2];
        float xc = sx * R00 + sy * R10 + sz * R20;
        float yc = sx * R01 + sy * R11 + sz * R21;
        float zc = sx * R02 + sy * R12 + sz * R22;
        sample_loc[row * 3] = xc / zc; sample_loc[row * 3 + 1] = yc / zc; sample_loc[row * 3 + 2] = zc;
    }
    if (sample_ray_dirs) {
        sample_ray_dirs[row * 3] = q.raydir[3 * r];
        sample_ray_dirs[row * 3 + 1] = q.raydir[3 * r + 1];
        sample_ray_dirs[row * 3 + 2] = q.raydir[3 * r + 2];
    }
}

// ------------------------------------------------------------------------------------------ frustum query -> compacted samples
// pnb_frustum_samples: one thread per (ray, slot).  A hit ray lists all SR slots as candidates, row ray_rank[r] of the dense tensors,
// so candidate s = ray_rank[r] * SR + j is entry s of [R',SR,...]; its neighbour count is the number of non-negative indices (the
// frustum export writes them first).
__global__ void __launch_bounds__(256) k_fs_rays(int R, int SR, const int8_t* __restrict__ ray_mask, int* __restrict__ nsamp,
                                                 uint8_t* __restrict__ ray_hit) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const bool hit = ray_mask[r] != 0;
    ray_hit[r] = hit ? 1 : 0;
    nsamp[r] = hit ? SR : 0;
}
__global__ void __launch_bounds__(256) k_fs_samples(int R, int SR, int K, const uint8_t* __restrict__ ray_hit,
                                                    const uint32_t* __restrict__ samp_off, const int32_t* __restrict__ pidx,
                                                    uint32_t* __restrict__ samp_ray, uint8_t* __restrict__ samp_nvalid, int* counters) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    int nv = 0;
    if (i < (long long)R * SR) {
        const int r = (int)(i / SR), j = (int)(i - (long long)r * SR);
        if (ray_hit[r]) {
            const uint32_t s = samp_off[r] + j;
            for (int k = 0; k < K; ++k) nv += pidx[(size_t)s * K + k] >= 0 ? 1 : 0;
            samp_ray[s] = ((uint32_t)r << 7) | (uint32_t)j;
            samp_nvalid[s] = (uint8_t)nv;
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) nv += __shfl_xor_sync(0xffffffffu, nv, d);
    if ((threadIdx.x & 31) == 0 && nv) atomicAdd(&counters[PNB_QC_N_PAIRS], nv);
}

struct QueryLayout {
    int* nsamp;
    uint32_t* samp_off;
    uint16_t* steps;
    uint32_t* samp_ray;
    int* cand_pidx;
    uint8_t* samp_nvalid;
    uint32_t* valid_list;
    uint32_t* valid_rank;
    uint8_t* ray_hit;
    int* counters;
    uint32_t* scan_tmp;
    uint32_t* ray_rank;
    size_t bytes;
};

static QueryLayout carve_query(void* ws, size_t cap_bytes, int R, int SR, int K, int cap) {
    Carver c(ws, cap_bytes);
    QueryLayout L;
    size_t r = (size_t)(R > 0 ? R : 1), cs = (size_t)(cap > 0 ? cap : 1);
    L.counters = c.take<int>(16);
    L.nsamp = c.take<int>(r);
    L.samp_off = c.take<uint32_t>(r + 1);
    L.steps = c.take<uint16_t>(r * SR);
    L.samp_ray = c.take<uint32_t>(cs);
    L.cand_pidx = c.take<int>(cs * K);
    L.samp_nvalid = c.take<uint8_t>(cs);
    L.valid_list = c.take<uint32_t>(cs);
    L.valid_rank = c.take<uint32_t>(cs + 1);
    L.ray_hit = c.take<uint8_t>(r);
    L.ray_rank = c.take<uint32_t>(r + 1);
    L.scan_tmp = c.take<uint32_t>(scan_tmp_elems(cs > r ? cs : r));
    L.bytes = align_up(c.off);
    return L;
}

}  // namespace pnb

using namespace pnb;

static inline int default_cap(int R, int SR, int cap) { return cap > 0 ? cap : R * SR; }

extern "C" size_t pnb_query_bytes(int R, int SR, int K, int cap_samples) {
    return carve_query(nullptr, 0, R, SR, K, default_cap(R, SR, cap_samples)).bytes;
}

extern "C" int pnb_query(pnb_query_t* q, void* ws, size_t ws_bytes, const pnb_grid_t* grid, const float campos[3],
                         const float* d_raydir, int R, const float* d_t, int t_ray_stride, int D, int SR, int K,
                         float radius_limit, const int32_t kernel_size[3], int cap_samples, pnb_stream_t stream_,
                         int32_t* h_counters) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && ws && grid && d_raydir && d_t, PNB_ERR_INVALID, "pnb_query: null argument");
    PNB_REQUIRE(R > 0 && R < (1 << 25), PNB_ERR_INVALID, "pnb_query: R=%d out of range [1, 2^25)", R);
    PNB_REQUIRE(K >= 1 && K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED,
                "pnb_query: K=%d unsupported (reference kernel buffer is KN=8, query_worldcoords.cu:14)", K);
    PNB_REQUIRE(SR >= 1 && SR <= PNB_MAX_SR, PNB_ERR_UNSUPPORTED, "pnb_query: SR=%d unsupported (1..%d)", SR, PNB_MAX_SR);
    PNB_REQUIRE(D >= 1 && D <= 65535, PNB_ERR_UNSUPPORTED, "pnb_query: D=%d unsupported (1..65535)", D);
    PNB_REQUIRE(t_ray_stride == 0 || t_ray_stride >= D, PNB_ERR_INVALID, "pnb_query: bad t_ray_stride");
    PNB_REQUIRE((long long)R * SR < (1ll << 31), PNB_ERR_UNSUPPORTED, "pnb_query: R*SR too large");
    int cap = default_cap(R, SR, cap_samples);
    QueryLayout L = carve_query(ws, ws_bytes, R, SR, K, cap);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_query: workspace %zu < required %zu", ws_bytes, L.bytes);

    QueryParams p;
    p.g = to_dev(*grid);
    for (int i = 0; i < 3; ++i) p.campos[i] = campos[i];
    p.raydir = d_raydir; p.t = d_t; p.t_ray_stride = t_ray_stride;
    p.R = R; p.D = D; p.SR = SR; p.K = K; p.ks0 = kernel_size[0];
    p.r2 = radius_limit * radius_limit;  // query_worldcoords.cu:410
    p.cap = cap;

    PNB_CHECK_CUDA(cudaMemsetAsync(L.counters, 0, 16 * sizeof(int), stream));
    PNB_CHECK_CUDA(cudaMemsetAsync(L.ray_hit, 0, (size_t)R, stream));
    PNB_CHECK_CUDA(cudaMemsetAsync(L.samp_nvalid, 0, (size_t)cap, stream));  // tail beyond n_cand must scan as 0
    {
        long long threads = (long long)R * 32;
        k_march<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(p, L.nsamp, L.steps);
    }
    int rc;
    rc = exclusive_scan_u32(L.nsamp, 3, L.samp_off, (uint32_t)R, L.scan_tmp, stream);
    if (rc) return rc;
    k_expand<<<(R * SR + 255) / 256, 256, 0, stream>>>(R, SR, cap, L.nsamp, L.samp_off, L.samp_ray, L.counters);
    k_knn<<<(cap + 127) / 128, 128, 0, stream>>>(p, L.samp_off, L.samp_ray, L.steps, L.cand_pidx, L.samp_nvalid,
                                                  L.ray_hit, L.counters);
    PNB_CHECK_CUDA(cudaGetLastError());
    // valid-sample list (ascending candidate id)
    rc = exclusive_scan_u32(L.samp_nvalid, 2, L.valid_rank, (uint32_t)cap, L.scan_tmp, stream);
    if (rc) return rc;
    k_valid_list<<<(cap + 255) / 256, 256, 0, stream>>>(R, cap, L.samp_off, L.samp_nvalid, L.valid_rank, L.valid_list,
                                                         L.counters);
    k_count_rays<<<(R + 255) / 256, 256, 0, stream>>>(R, L.ray_hit, L.counters);
    PNB_CHECK_CUDA(cudaGetLastError());

    q->R = R; q->SR = SR; q->K = K; q->D = D; q->cap_samples = cap;
    q->nsamp = L.nsamp; q->samp_off = L.samp_off; q->steps = L.steps; q->samp_ray = L.samp_ray;
    q->cand_pidx = L.cand_pidx; q->samp_nvalid = L.samp_nvalid; q->valid_list = L.valid_list;
    q->valid_rank = L.valid_rank; q->ray_hit = L.ray_hit; q->counters = L.counters;
    q->ray_rank = L.ray_rank; q->scan_tmp = L.scan_tmp;
    q->raydir = d_raydir; q->t = d_t; q->t_ray_stride = t_ray_stride;
    for (int i = 0; i < 3; ++i) q->campos[i] = campos[i];
    if (h_counters) {
        PNB_CHECK_CUDA(cudaMemcpyAsync(h_counters, L.counters, 16 * sizeof(int), cudaMemcpyDeviceToHost, stream));
        PNB_CHECK_CUDA(cudaStreamSynchronize(stream));
    }
    return PNB_OK;
}

extern "C" int pnb_query_export(const pnb_query_t* q, const pnb_shade_opts_t* cam, int32_t* d_ray_row, int8_t* d_ray_mask,
                                int32_t* d_sample_pidx, float* d_sample_loc_w, float* d_sample_loc,
                                float* d_sample_ray_dirs, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && cam && d_ray_row && d_ray_mask && d_sample_pidx && d_sample_loc_w, PNB_ERR_INVALID,
                "pnb_query_export: null argument");
    int rc = exclusive_scan_u32(q->ray_hit, 2, q->ray_rank, (uint32_t)q->R, q->scan_tmp, stream);
    if (rc) return rc;
    const float* M = cam->camrotc2w;
    k_export<<<(q->R * q->SR + 127) / 128, 128, 0, stream>>>(*q, M[0], M[3], M[6], M[1], M[4], M[7], M[2], M[5], M[8],
                                                              q->ray_rank, d_ray_row, d_ray_mask, d_sample_pidx,
                                                              d_sample_loc_w, d_sample_loc, d_sample_ray_dirs);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

// The per-candidate arrays of pnb_query over a frustum query's dense result (cand_pidx is not carved: the shading reads the
// caller's [R2,SR,K] indices in place).
extern "C" size_t pnb_frustum_samples_bytes(int R, int R2, int SR) {
    return carve_query(nullptr, 0, R, SR, 0, R2 * SR).bytes;
}

extern "C" int pnb_frustum_samples(pnb_query_t* q, void* ws, size_t ws_bytes, const int8_t* d_ray_mask, int R, int R2, int SR, int K,
                                   const int32_t* d_sample_pidx, const float* d_sample_loc_w, const float* d_sample_loc,
                                   const float* d_sample_ray_dirs, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && ws && d_ray_mask && (R2 == 0 || (d_sample_pidx && d_sample_loc_w && d_sample_loc && d_sample_ray_dirs)),
                PNB_ERR_INVALID, "pnb_frustum_samples: null argument");
    PNB_REQUIRE(R > 0 && R < (1 << 25), PNB_ERR_INVALID, "pnb_frustum_samples: R=%d out of range [1, 2^25)", R);
    PNB_REQUIRE(R2 >= 0 && R2 <= R, PNB_ERR_INVALID, "pnb_frustum_samples: R2=%d outside 0..R=%d", R2, R);
    PNB_REQUIRE(K >= 1 && K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED, "pnb_frustum_samples: K=%d unsupported", K);
    PNB_REQUIRE(SR >= 1 && SR <= PNB_MAX_SR, PNB_ERR_UNSUPPORTED, "pnb_frustum_samples: SR=%d unsupported (1..%d)", SR, PNB_MAX_SR);
    PNB_REQUIRE((long long)R * SR < (1ll << 31), PNB_ERR_UNSUPPORTED, "pnb_frustum_samples: R*SR too large");
    const int cap = R2 * SR;
    QueryLayout L = carve_query(ws, ws_bytes, R, SR, 0, cap);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_frustum_samples: workspace %zu < required %zu", ws_bytes, L.bytes);
    const uint32_t cs = (uint32_t)(cap > 0 ? cap : 1);
    PNB_CHECK_CUDA(cudaMemsetAsync(L.counters, 0, 16 * sizeof(int), stream));
    PNB_CHECK_CUDA(cudaMemsetAsync(L.samp_nvalid, 0, cs, stream));
    k_fs_rays<<<(R + 255) / 256, 256, 0, stream>>>(R, SR, d_ray_mask, L.nsamp, L.ray_hit);
    int rc = exclusive_scan_u32(L.nsamp, 3, L.samp_off, (uint32_t)R, L.scan_tmp, stream);
    if (rc) return rc;
    rc = exclusive_scan_u32(L.ray_hit, 2, L.ray_rank, (uint32_t)R, L.scan_tmp, stream);
    if (rc) return rc;
    const long long n = (long long)R * SR;
    k_fs_samples<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(R, SR, K, L.ray_hit, L.samp_off, d_sample_pidx, L.samp_ray,
                                                                  L.samp_nvalid, L.counters);
    PNB_CHECK_CUDA(cudaGetLastError());
    rc = exclusive_scan_u32(L.samp_nvalid, 2, L.valid_rank, cs, L.scan_tmp, stream);
    if (rc) return rc;
    k_valid_list<<<(cs + 255) / 256, 256, 0, stream>>>(R, cap, L.samp_off, L.samp_nvalid, L.valid_rank, L.valid_list, L.counters);
    k_count_rays<<<(R + 255) / 256, 256, 0, stream>>>(R, L.ray_hit, L.counters);
    PNB_CHECK_CUDA(cudaGetLastError());

    *q = pnb_query_t{};
    q->R = R; q->SR = SR; q->K = K; q->D = 0; q->cap_samples = cap;
    q->nsamp = L.nsamp; q->samp_off = L.samp_off; q->steps = nullptr; q->samp_ray = L.samp_ray;
    q->cand_pidx = const_cast<int32_t*>(d_sample_pidx); q->samp_nvalid = L.samp_nvalid; q->valid_list = L.valid_list;
    q->valid_rank = L.valid_rank; q->ray_hit = L.ray_hit; q->counters = L.counters;
    q->ray_rank = L.ray_rank; q->scan_tmp = L.scan_tmp;
    q->xs_loc_w = d_sample_loc_w; q->xs_loc = d_sample_loc; q->xs_dir = d_sample_ray_dirs;
    return PNB_OK;
}
