// Shared device/host helpers of libpnb200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <type_traits>
#include <vector>

#include "../../include/pnb200.h"

namespace pnb {

void set_error(const char* fmt, ...);

#define PNB_CHECK_CUDA(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            pnb::set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, #expr,          \
                           cudaGetErrorString(_e));                                       \
            return PNB_ERR_CUDA;                                                          \
        }                                                                                 \
    } while (0)

#define PNB_REQUIRE(cond, code, ...)                                                      \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            pnb::set_error(__VA_ARGS__);                                                  \
            return code;                                                                  \
        }                                                                                 \
    } while (0)

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ---- point_features_dim F: 32 (most shipped scripts) or 63 (the DTU scripts), each a compile-time instantiation of the kernels
// F (0 read as 32) or -1 when the width has no instantiation
static inline int feat_of(int32_t f) { return f == 0 ? PNB_FEAT : (f == PNB_FEAT || f == PNB_FEAT_DTU) ? (int)f : -1; }
// block1.0 inputs [f (F), PE3(f) (6F), PE5(dists) (60)] = 7F + 60, padded to whole K = 32 blocks: 288 | 512
__host__ __device__ constexpr int kpad1_of(int F) { return F == PNB_FEAT ? 288 : 512; }

// ---- the run-time inputs that select a shading kernel's instantiation
struct Variant {
    int F;      // point_features_dim
    bool pp;    // per-point frames (pts->rw2c != NULL)
    bool xs;    // explicit samples (the frustum query, q->xs_loc_w != NULL)
};
// What an entry point requires of explicit samples
enum class XsRule {
    none,     // nothing (k_aux_outputs)
    feat63,   // F = 63 (k_probe_outputs)
    frames,   // F = 63, a uniform Rw2c and xs_loc / xs_dir given: the kernels that read the points' frames
};
// The points' F (0 read as 32), which must have an instantiation and, with an MLP, equal the MLP's; then explicit samples (q may be
// NULL) by `rule`.  Sets the error text on failure.
static inline int resolve_variant(const char* fn, const pnb_points_t* pts, const pnb_mlp_t* mlp, const pnb_query_t* q, XsRule rule,
                                  Variant* v) {
    const int F = feat_of(pts->feat_dim);
    PNB_REQUIRE(F > 0, PNB_ERR_UNSUPPORTED, "%s: point_features_dim %d unsupported (32 or 63)", fn, (int)pts->feat_dim);
    if (mlp)
        PNB_REQUIRE(feat_of(mlp->feat_dim) == F, PNB_ERR_INVALID, "%s: the MLP was built for point_features_dim %d, the points have %d",
                    fn, (int)(mlp->feat_dim ? mlp->feat_dim : PNB_FEAT), F);
    *v = Variant{F, pts->rw2c != nullptr, q && q->xs_loc_w};
    if (v->xs && rule == XsRule::frames) {
        PNB_REQUIRE(q->xs_loc && q->xs_dir, PNB_ERR_INVALID, "%s: explicit samples need xs_loc_w, xs_loc and xs_dir", fn);
        PNB_REQUIRE(F == PNB_FEAT_DTU && !v->pp, PNB_ERR_UNSUPPORTED,
                    "%s: the frustum query's samples are shaded with point_features_dim 63 and a uniform Rw2c only", fn);
    }
    if (v->xs && rule == XsRule::feat63)
        PNB_REQUIRE(F == PNB_FEAT_DTU, PNB_ERR_UNSUPPORTED, "%s: the frustum query's samples need point_features_dim 63", fn);
    return PNB_OK;
}

// ---- run-time values as template arguments.  Each helper calls f with std::integral_constant arguments, which convert to their
// values in a template argument list, so that f names the instantiation: [](auto PP, auto F, auto XS) { return k<PP, F, XS>; }.
// Only the combinations a helper passes are instantiated.
template <bool B> using Bool = std::integral_constant<bool, B>;
template <int I> using Int = std::integral_constant<int, I>;
template <class Fn> static inline auto with_bool(bool b, Fn&& f) { return b ? f(Bool<true>{}) : f(Bool<false>{}); }
template <class Fn> static inline auto with_feat(int F, Fn&& f) { return F == PNB_FEAT ? f(Int<PNB_FEAT>{}) : f(Int<PNB_FEAT_DTU>{}); }
// f(F, XS) of k_probe_outputs: explicit samples at F = 63 only
template <class Fn> static inline auto with_feat_xs(const Variant& v, Fn&& f) {
    return v.xs ? f(Int<PNB_FEAT_DTU>{}, Bool<true>{}) : with_feat(v.F, [&](auto F) { return f(F, Bool<false>{}); });
}
// f(PP, F, XS) of the kernels that read the points' frames: explicit samples at F = 63 with a uniform Rw2c only
template <class Fn> static inline auto with_frames(const Variant& v, Fn&& f) {
    return v.xs ? f(Bool<false>{}, Int<PNB_FEAT_DTU>{}, Bool<true>{})
                : with_bool(v.pp, [&](auto PP) { return with_feat(v.F, [&](auto F) { return f(PP, F, Bool<false>{}); }); });
}

// Prepares the launch of `kern` on the current device: opts it into `smem` bytes of dynamic shared memory the first time it is
// launched there, and gives the device's SM count (n_sm may be NULL).  Call it for the selected kernel just before its launch.  The
// state is per device, for one host thread per device.
static inline int prepare_launch(const void* kern, size_t smem, int* n_sm, const char* fn) {
    static std::vector<const void*> opted_in[64];
    static int sm_count[64];
    int dev = 0;
    PNB_CHECK_CUDA(cudaGetDevice(&dev));
    PNB_REQUIRE(dev >= 0 && dev < 64, PNB_ERR_UNSUPPORTED, "%s: device ordinal %d", fn, dev);
    std::vector<const void*>& done = opted_in[dev];
    if (std::find(done.begin(), done.end(), kern) == done.end()) {
        PNB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        done.push_back(kern);
    }
    if (!sm_count[dev]) PNB_CHECK_CUDA(cudaDeviceGetAttribute(&sm_count[dev], cudaDevAttrMultiProcessorCount, dev));
    if (n_sm) *n_sm = sm_count[dev];
    return PNB_OK;
}

// Bump allocator over a caller-provided workspace.
struct Carver {
    char* base;
    size_t off, cap;
    Carver(void* p, size_t bytes) : base((char*)p), off(0), cap(bytes) {}
    template <typename T>
    T* take(size_t n) {
        size_t o = align_up(off);
        off = o + n * sizeof(T);
        return (T*)(base ? base + o : nullptr);
    }
    bool ok() const { return off <= cap; }
};

// Grid parameters by value for kernels.
struct GridDev {
    float lo[3];
    float svs[3];
    int dim[3];
    int P;
    int parity_slot0;
    const uint32_t* occ_bits;
    const uint32_t* pt_bits;
    const uint32_t* word_rank;
    const uint32_t* cell_start;
    const float4* spts;
    const int* counters;
};

static inline GridDev to_dev(const pnb_grid_t& g) {
    GridDev d;
    for (int i = 0; i < 3; ++i) { d.lo[i] = g.lo[i]; d.svs[i] = g.svs[i]; d.dim[i] = g.dim[i]; }
    d.P = g.P; d.parity_slot0 = g.parity_slot0;
    d.occ_bits = g.occ_bits; d.pt_bits = g.pt_bits; d.word_rank = g.word_rank;
    d.cell_start = g.cell_start; d.spts = (const float4*)g.spts; d.counters = g.counters;
    return d;
}

#ifdef __CUDACC__
// Voxel coordinate exactly as query_worldcoords.cu:40-42: IEEE fp32 subtract, IEEE fp32 divide, floor.
__device__ __forceinline__ int vox1(float p, float lo, float svs) {
    return (int)floorf(__fdiv_rn(__fsub_rn(p, lo), svs));
}
// Sample position as the reference's torch ops form it (diff_ray_marching.py:386): mul, then add, no FMA.
__device__ __forceinline__ float raypos1(float c, float dir, float t) {
    return __fadd_rn(c, __fmul_rn(dir, t));
}
__device__ __forceinline__ bool in_grid(int x, int y, int z, const int* dim) {
    return (x >= 0) & (x < dim[0]) & (y >= 0) & (y < dim[1]) & (z >= 0) & (z < dim[2]);
}
__device__ __forceinline__ uint32_t cell_index(int x, int y, int z, const int* dim) {
    return ((uint32_t)x * (uint32_t)dim[1] + (uint32_t)y) * (uint32_t)dim[2] + (uint32_t)z;
}
#endif

// Device-wide exclusive scan of uint32 (3 small kernels; build-time / per-call bookkeeping, not a hot loop).
// mode 0: in[i];  mode 1: popc(in[i]);  mode 2: (in_u8[i] > 0);  mode 3: in_i32[i]
int exclusive_scan_u32(const void* in, int mode, uint32_t* out /* n+1 */, uint32_t n, uint32_t* tmp /* >= n/1024+2 */,
                       cudaStream_t stream);
static inline size_t scan_tmp_elems(size_t n) { return n / 1024 + 4; }

}  // namespace pnb
