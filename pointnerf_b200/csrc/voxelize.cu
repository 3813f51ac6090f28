// Voxel down-sampling of a point cloud (pnb_vox_build / pnb_vox_outputs): the construct_vox_points{,_closest,_ind,_xyz} family of
// models/mvs/mvs_utils.py:484-561 with canonical, run-to-run identical results (DESIGN.md §5 "Voxel down-sampling").
//
//   keys     voxel index floorf((p - space_min) / vox_sz) per axis (IEEE fp32 subtract, true fp32 divide), packed into a key that
//            sorts as torch.unique(dim=0) orders rows: 32 bits (10 per axis, indices in [0, 1024)) or 64 bits (21 per axis, biased
//            by 2^20, indices in [-2^20, 2^20)).  An index outside the key's range fails the call (PNB_VC_N_OUT_OF_KEY), never mis-sorts.
//   sort     CUB's stable LSD radix sort of (key, point index): voxels in lexicographic (x, y, z) order, ascending index inside each.
//   segments head flags + exclusive scan: M, the first sorted position of every voxel, inv_idx.  One host synchronise returns M.
//   outputs  per voxel: its index, the first point, the centroid (fp64 tree below, one rounding to fp32), the closest point.
//
// Centroid tree (restated by oracle/voxelize_oracle.py): a voxel's c points x_0..x_{c-1} in ascending point index feed W = 256 lanes;
// lane t < min(c, W) starts from x_t and adds x_{t+256}, x_{t+512}, ... in order (fp64).  Then for off = 128, 64, ..., 1 every lane
// t < off with t + off < min(c, W) adds lane t + off.  The centroid is fp32(lane 0 / c), the divide in fp64.  A warp reduces a voxel of
// <= 256 points, a 256-thread block a larger one; both run exactly this tree.
#include <cub/cub.cuh>

#include "common.cuh"

namespace pnb {
namespace {

constexpr int kLanes = 256;        // width of the centroid tree; also the block of k_vox_big
constexpr int kBias64 = 1 << 20;   // 64-bit key: 21 bits per axis, index + 2^20

struct VoxLayout {
    int* counters;
    void *keys_a, *keys_b;
    uint32_t *idx_a, *idx_b, *rank, *seg_start, *big_list, *scan_tmp;
    uint8_t* head;
    void* sort_tmp;
    size_t sort_tmp_bytes, bytes;
};

template <typename K>
size_t sort_tmp_bytes(int N) {
    size_t b = 0;
    cub::DoubleBuffer<K> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    cub::DeviceRadixSort::SortPairs(nullptr, b, k, v, N, 0, (int)sizeof(K) * 8 - 1);
    return b;
}

VoxLayout carve_vox(void* buf, size_t cap, int N, int key_bits) {
    Carver c(buf, cap);
    VoxLayout L;
    const size_t nn = (size_t)(N > 0 ? N : 1);
    const size_t kb = key_bits == 32 ? 4 : 8;
    L.counters = c.take<int>(16);
    L.keys_a = c.take<char>(nn * kb);
    L.keys_b = c.take<char>(nn * kb);
    L.idx_a = c.take<uint32_t>(nn);
    L.idx_b = c.take<uint32_t>(nn);
    L.head = c.take<uint8_t>(nn);
    L.rank = c.take<uint32_t>(nn + 1);
    L.seg_start = c.take<uint32_t>(nn + 1);
    L.big_list = c.take<uint32_t>(nn / (kLanes + 1) + 1);
    L.scan_tmp = c.take<uint32_t>(scan_tmp_elems(nn));
    L.sort_tmp_bytes = key_bits == 32 ? sort_tmp_bytes<uint32_t>(N) : sort_tmp_bytes<unsigned long long>(N);
    L.sort_tmp = c.take<char>(L.sort_tmp_bytes);
    L.bytes = align_up(c.off);
    return L;
}

__device__ __forceinline__ int vox_axis(float p, float lo, float sz) {
    return __float2int_rz(floorf(__fdiv_rn(__fsub_rn(p, lo), sz)));   // saturating, NaN -> 0: torch's CUDA float -> int32
}

template <typename K>
__device__ __forceinline__ bool pack_key(int x, int y, int z, K* key);
template <>
__device__ __forceinline__ bool pack_key<uint32_t>(int x, int y, int z, uint32_t* key) {
    const bool ok = (unsigned)x < 1024u && (unsigned)y < 1024u && (unsigned)z < 1024u;
    *key = ok ? ((uint32_t)x << 20) | ((uint32_t)y << 10) | (uint32_t)z : 0u;
    return ok;
}
template <>
__device__ __forceinline__ bool pack_key<unsigned long long>(int x, int y, int z, unsigned long long* key) {
    const unsigned lim = 2u * kBias64;
    const unsigned ux = (unsigned)(x + kBias64), uy = (unsigned)(y + kBias64), uz = (unsigned)(z + kBias64);
    const bool ok = ux < lim && uy < lim && uz < lim;
    *key = ok ? ((unsigned long long)ux << 42) | ((unsigned long long)uy << 21) | (unsigned long long)uz : 0ull;
    return ok;
}
__device__ __forceinline__ void unpack_key(uint32_t k, int* v) {
    v[0] = (int)(k >> 20); v[1] = (int)((k >> 10) & 1023u); v[2] = (int)(k & 1023u);
}
__device__ __forceinline__ void unpack_key(unsigned long long k, int* v) {
    v[0] = (int)(k >> 42) - kBias64; v[1] = (int)((k >> 21) & 0x1fffffull) - kBias64; v[2] = (int)(k & 0x1fffffull) - kBias64;
}

template <typename K>
__global__ void __launch_bounds__(256) k_vox_keys(const float* __restrict__ xyz, int N, const float* __restrict__ space_min,
                                                  const float* __restrict__ vox_sz, K* keys, uint32_t* idx, int* counters) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    int v[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) v[a] = vox_axis(xyz[3 * (size_t)i + a], space_min[a], vox_sz[a]);
    K key;
    if (!pack_key<K>(v[0], v[1], v[2], &key)) atomicAdd(&counters[PNB_VC_N_OUT_OF_KEY], 1);
    keys[i] = key;
    idx[i] = (uint32_t)i;
}

template <typename K>
__global__ void __launch_bounds__(256) k_vox_heads(const K* __restrict__ keys, int N, uint8_t* head) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < N) head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// seg_start[s] = first sorted position of voxel s (seg_start[M] = N); inv_idx[point] = its voxel.
__global__ void __launch_bounds__(256) k_vox_segments(const uint8_t* __restrict__ head, const uint32_t* __restrict__ rank,
                                                      const uint32_t* __restrict__ idx, int N, uint32_t* seg_start,
                                                      long long* inv_idx, int* counters) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    if (head[i]) seg_start[rank[i]] = (uint32_t)i;
    if (inv_idx) inv_idx[idx[i]] = (long long)(rank[i] + head[i]) - 1;
    if (i == 0) {
        seg_start[rank[N]] = (uint32_t)N;
        counters[PNB_VC_N_VOX] = (int)rank[N];
    }
}

// Voxels of more than kLanes points go to the block kernel (list order is immaterial: each voxel's result depends on it alone).
__global__ void __launch_bounds__(256) k_vox_sizes(const uint32_t* __restrict__ seg_start, int N, uint32_t* big_list, int* counters) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= N || s >= counters[PNB_VC_N_VOX]) return;
    const int c = (int)(seg_start[s + 1] - seg_start[s]);
    atomicMax(&counters[PNB_VC_MAX_PTS], c);
    if (c > kLanes) big_list[atomicAdd(&counters[PNB_VC_N_BIG], 1)] = (uint32_t)s;
}

struct VoxOut {
    const float* val;
    const uint32_t* idx;
    const uint32_t* seg_start;
    const void* keys;
    int key_bits;
    int M;
    int closest;
    int* grid_idx;
    float* centroid;
    long long* min_idx;
};

__device__ __forceinline__ float residual(const float* p, const float* c) {
    const float dx = __fsub_rn(p[0], c[0]), dy = __fsub_rn(p[1], c[1]), dz = __fsub_rn(p[2], c[2]);
    return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
}
__device__ __forceinline__ void load3(const float* val, uint32_t i, float* p) {
    p[0] = val[3 * (size_t)i]; p[1] = val[3 * (size_t)i + 1]; p[2] = val[3 * (size_t)i + 2];
}
// (residual bits, point index): residuals are >= 0, so the bits order as the values; ties go to the lower index.
__device__ __forceinline__ unsigned long long rkey(float r, uint32_t i) {
    return ((unsigned long long)__float_as_uint(r) << 32) | i;
}

// One warp per voxel: grid index and first point of every voxel; centroid and closest point of the voxels of <= kLanes points.
__global__ void __launch_bounds__(256) k_vox_small(VoxOut o) {
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (blockDim.x >> 5);
    for (int s = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); s < o.M; s += warps) {
        const uint32_t a = o.seg_start[s];
        const int c = (int)(o.seg_start[s + 1] - a);
        if (lane == 0) {
            if (o.grid_idx) {
                int v[3];
                if (o.key_bits == 32) unpack_key(((const uint32_t*)o.keys)[a], v);
                else unpack_key(((const unsigned long long*)o.keys)[a], v);
                for (int k = 0; k < 3; ++k) o.grid_idx[3 * (size_t)s + k] = v[k];
            }
            if (o.min_idx && !o.closest) o.min_idx[s] = (long long)o.idx[a];
        }
        if (!o.centroid || c > kLanes) continue;
        double p[8][3];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int t = lane + 32 * j;
            float q[3] = {0.f, 0.f, 0.f};
            if (t < c) load3(o.val, o.idx[a + t], q);
            for (int k = 0; k < 3; ++k) p[j][k] = (double)q[k];
        }
#pragma unroll
        for (int off = 4; off >= 1; off >>= 1)       // tree steps 128, 64, 32: lane-local
#pragma unroll
            for (int j = 0; j < off; ++j)
                if (lane + 32 * (j + off) < c)
                    for (int k = 0; k < 3; ++k) p[j][k] = __dadd_rn(p[j][k], p[j + off][k]);
#pragma unroll
        for (int off = 16; off >= 1; off >>= 1)
            for (int k = 0; k < 3; ++k) {
                const double y = __shfl_down_sync(0xffffffffu, p[0][k], off);
                if (lane < off && lane + off < c) p[0][k] = __dadd_rn(p[0][k], y);
            }
        float cen[3];
        for (int k = 0; k < 3; ++k) cen[k] = __shfl_sync(0xffffffffu, __double2float_rn(__ddiv_rn(p[0][k], (double)c)), 0);
        if (lane == 0)
            for (int k = 0; k < 3; ++k) o.centroid[3 * (size_t)s + k] = cen[k];
        if (!o.closest) continue;
        unsigned long long best = ~0ull;
        for (int t = lane; t < c; t += 32) {
            const uint32_t i = o.idx[a + t];
            float q[3];
            load3(o.val, i, q);
            best = min(best, rkey(residual(q, cen), i));
        }
        for (int off = 16; off >= 1; off >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, off));
        if (lane == 0) o.min_idx[s] = (long long)(uint32_t)best;
    }
}

// One 256-thread block per voxel of more than kLanes points (the same tree, every lane present).
__global__ void __launch_bounds__(kLanes) k_vox_big(VoxOut o, const uint32_t* __restrict__ big_list, int n_big) {
    __shared__ double sh[kLanes][3];
    __shared__ unsigned long long shb[kLanes / 32];
    __shared__ float cen[3];
    const int t = threadIdx.x, lane = t & 31;
    for (int b = blockIdx.x; b < n_big; b += gridDim.x) {
        const uint32_t s = big_list[b];
        const uint32_t a = o.seg_start[s];
        const int c = (int)(o.seg_start[s + 1] - a);
        double p[3];
        float q[3];
        load3(o.val, o.idx[a + t], q);
        for (int k = 0; k < 3; ++k) p[k] = (double)q[k];
        for (int r = t + kLanes; r < c; r += kLanes) {
            load3(o.val, o.idx[a + r], q);
            for (int k = 0; k < 3; ++k) p[k] = __dadd_rn(p[k], (double)q[k]);
        }
        for (int k = 0; k < 3; ++k) sh[t][k] = p[k];
        __syncthreads();
        for (int off = kLanes / 2; off >= 32; off >>= 1) {
            if (t < off)
                for (int k = 0; k < 3; ++k) sh[t][k] = __dadd_rn(sh[t][k], sh[t + off][k]);
            __syncthreads();
        }
        if (t < 32) {
            for (int k = 0; k < 3; ++k) p[k] = sh[t][k];
            for (int off = 16; off >= 1; off >>= 1)
                for (int k = 0; k < 3; ++k) {
                    const double y = __shfl_down_sync(0xffffffffu, p[k], off);
                    if (lane < off) p[k] = __dadd_rn(p[k], y);
                }
            if (t == 0)
                for (int k = 0; k < 3; ++k) {
                    cen[k] = __double2float_rn(__ddiv_rn(p[k], (double)c));
                    o.centroid[3 * (size_t)s + k] = cen[k];
                }
        }
        __syncthreads();
        if (o.closest) {
            const float cc[3] = {cen[0], cen[1], cen[2]};
            unsigned long long best = ~0ull;
            for (int r = t; r < c; r += kLanes) {
                const uint32_t i = o.idx[a + r];
                load3(o.val, i, q);
                best = min(best, rkey(residual(q, cc), i));
            }
            for (int off = 16; off >= 1; off >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, off));
            if (lane == 0) shb[t >> 5] = best;
            __syncthreads();
            if (t == 0) {
                for (int w = 1; w < kLanes / 32; ++w) best = min(best, shb[w]);
                o.min_idx[s] = (long long)(uint32_t)best;
            }
        }
        __syncthreads();
    }
}

template <typename K>
int vox_sort_and_segment(const VoxLayout& L, const float* d_xyz, int N, const float* d_space_min, const float* d_vox_sz,
                         long long* d_inv_idx, cudaStream_t stream, const void** sorted_keys, const uint32_t** sorted_idx) {
    const int nb = (N + 255) / 256;
    k_vox_keys<K><<<nb, 256, 0, stream>>>(d_xyz, N, d_space_min, d_vox_sz, (K*)L.keys_a, L.idx_a, L.counters);
    cub::DoubleBuffer<K> keys((K*)L.keys_a, (K*)L.keys_b);
    cub::DoubleBuffer<uint32_t> vals(L.idx_a, L.idx_b);
    size_t tb = L.sort_tmp_bytes;
    PNB_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(L.sort_tmp, tb, keys, vals, N, 0, sizeof(K) == 4 ? 30 : 63, stream));
    k_vox_heads<K><<<nb, 256, 0, stream>>>(keys.Current(), N, L.head);
    int rc = exclusive_scan_u32(L.head, 2, L.rank, (uint32_t)N, L.scan_tmp, stream);
    if (rc) return rc;
    k_vox_segments<<<nb, 256, 0, stream>>>(L.head, L.rank, vals.Current(), N, L.seg_start, d_inv_idx, L.counters);
    k_vox_sizes<<<nb, 256, 0, stream>>>(L.seg_start, N, L.big_list, L.counters);
    PNB_CHECK_CUDA(cudaGetLastError());
    *sorted_keys = keys.Current();
    *sorted_idx = vals.Current();
    return PNB_OK;
}

}  // namespace
}  // namespace pnb

using namespace pnb;

extern "C" size_t pnb_vox_bytes(int N, int key_bits) {
    if (N < 0 || (key_bits != 32 && key_bits != 64)) return 0;
    return carve_vox(nullptr, 0, N, key_bits).bytes;
}

extern "C" int pnb_vox_build(pnb_vox_t* v, void* ws, size_t ws_bytes, const float* d_xyz, int N, const float* d_space_min,
                             const float* d_vox_sz, int key_bits, long long* d_inv_idx, pnb_stream_t stream_, int32_t* h_counters) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(v && ws && h_counters && d_space_min && d_vox_sz, PNB_ERR_INVALID, "pnb_vox_build: null argument");
    PNB_REQUIRE(N >= 0, PNB_ERR_INVALID, "pnb_vox_build: N must be >= 0 (got %d)", N);
    PNB_REQUIRE(N == 0 || d_xyz, PNB_ERR_INVALID, "pnb_vox_build: null argument");
    PNB_REQUIRE(key_bits == 32 || key_bits == 64, PNB_ERR_INVALID, "pnb_vox_build: key_bits must be 32 or 64 (got %d)", key_bits);
    VoxLayout L = carve_vox(ws, ws_bytes, N, key_bits);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_vox_build: workspace %zu < required %zu", ws_bytes, L.bytes);
    PNB_CHECK_CUDA(cudaMemsetAsync(L.counters, 0, 16 * sizeof(int), stream));
    const void* keys = L.keys_a;
    const uint32_t* idx = L.idx_a;
    if (N > 0) {
        int rc = key_bits == 32
                     ? vox_sort_and_segment<uint32_t>(L, d_xyz, N, d_space_min, d_vox_sz, d_inv_idx, stream, &keys, &idx)
                     : vox_sort_and_segment<unsigned long long>(L, d_xyz, N, d_space_min, d_vox_sz, d_inv_idx, stream, &keys, &idx);
        if (rc) return rc;
    }
    PNB_CHECK_CUDA(cudaMemcpyAsync(h_counters, L.counters, 16 * sizeof(int), cudaMemcpyDeviceToHost, stream));
    PNB_CHECK_CUDA(cudaStreamSynchronize(stream));
    PNB_REQUIRE(h_counters[PNB_VC_N_OUT_OF_KEY] == 0, PNB_ERR_UNSUPPORTED,
                "pnb_vox_build: %d points have a voxel index outside the %d-bit key's range ([0, 1024) per axis for 32 bits, "
                "[-2^20, 2^20) for 64 bits)", h_counters[PNB_VC_N_OUT_OF_KEY], key_bits);
    v->n_points = N;
    v->key_bits = key_bits;
    v->n_vox = h_counters[PNB_VC_N_VOX];
    v->n_big = h_counters[PNB_VC_N_BIG];
    v->sorted_keys = keys;
    v->sorted_idx = idx;
    v->seg_start = L.seg_start;
    v->big_list = L.big_list;
    v->counters = L.counters;
    return PNB_OK;
}

extern "C" int pnb_vox_outputs(const pnb_vox_t* v, const float* d_val, int32_t* d_grid_idx, float* d_centroid, long long* d_min_idx,
                               int closest, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(v, PNB_ERR_INVALID, "pnb_vox_outputs: null argument");
    if (v->n_vox == 0) return PNB_OK;                    // an empty cloud: nothing to write (its outputs may be NULL)
    PNB_REQUIRE(!d_centroid || d_val, PNB_ERR_INVALID, "pnb_vox_outputs: the centroid needs the value points");
    PNB_REQUIRE(!closest || (d_centroid && d_min_idx), PNB_ERR_INVALID, "pnb_vox_outputs: the closest point needs centroid and min_idx");
    VoxOut o;
    o.val = d_val; o.idx = v->sorted_idx; o.seg_start = v->seg_start; o.keys = v->sorted_keys; o.key_bits = v->key_bits;
    o.M = v->n_vox; o.closest = closest; o.grid_idx = d_grid_idx; o.centroid = d_centroid; o.min_idx = d_min_idx;
    k_vox_small<<<(unsigned)((v->n_vox + 7LL) / 8), 256, 0, stream>>>(o);
    if (d_centroid && v->n_big > 0) {
        int dev = 0, sms = 0;
        PNB_CHECK_CUDA(cudaGetDevice(&dev));
        PNB_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        const int nb = v->n_big < 8 * sms ? v->n_big : 8 * sms;
        k_vox_big<<<nb, kLanes, 0, stream>>>(o, v->big_list, v->n_big);
    }
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
