// Fused per-pair shading on the Hopper tensor cores (wgmma), sm_90a.
//
//   gather + weights + positional encoding  ->  block1 (284->256->256)  ->  cat extras  ->  block3 (263->256->256)
//   ->  alpha branch + K-reduction  ->  colour branch (280->128->128->128->3)
//   (reference: models/aggregators/point_aggregators.py:488-644, 727-814; gather models/neural_points/neural_points.py:706-717)
//
// Kernels of this file:
//   k_pack_*      row packing: the valid (sample, neighbour) pairs -> 32-row quadrants of 128-row MMA tiles (first fit)
//   k_shade_wg    pair MLPs, one packed 128-row tile per iteration of a persistent CTA: every layer D[128x256] = A[128xK] * W[256xK]^T
//                 on wgmma (BF16 operands in shared memory, FP32 accumulators in registers), K-reduction, writes h-bar + sigma.
//                 FROZEN (rendering a point cloud whose parameters need no gradient): the 224 point-only inputs of block1.0 are
//                 hoisted into a per-point table (k_point_pre) and layer 1 runs on the 64 sample-dependent inputs only
//   k_color_wg    colour branch per 128 valid samples, fed by h-bar in its own operand format (one bulk copy per tile)
// The reference computes these layers in fp32 and the parity bar is 1e-4 on the rendered radiance, which a single BF16/TF32
// pass misses (SURVEY.md section 7) -> error-compensated split:
//   A = A_hi + A_lo, W = W_hi + W_lo (bf16 each);   D = A_hi*W_hi + A_lo*W_hi + A_hi*W_lo    (3 MMAs per k-step)
// Weight images are pre-packed per K = 16 step in the wgmma operand layout (pnb_mlp_pack) and streamed L2 -> shared memory with
// cp.async.bulk (TMA engine) through a 4-stage mbarrier ring.
#include "pair_inputs.cuh"
#include "wgmma.cuh"

namespace pnb {
using namespace wg;

namespace tc {
constexpr int LAYOUT = LAYOUT_NONE;
constexpr int TM = 128;                 // pair rows per tile
constexpr int ABLK = 128 * 64;          // bytes of one A block ([128 x 32] bf16)
constexpr int NKB_MAX = 9;
// K blocks of block1.0 (9 | 16 for F = 32 | 63), of layer l, and the first K block of layer l in the packed images
__host__ __device__ constexpr int nkb0_of(int F) { return kpad1_of(F) / 32; }
__host__ __device__ constexpr int nkb_of(int l, int F = PNB_FEAT) { return l == 0 ? nkb0_of(F) : l == 2 ? 9 : 8; }
__host__ __device__ constexpr int img_base(int l, int F = PNB_FEAT) { return l == 0 ? 0 : l == 1 ? nkb0_of(F) : l == 2 ? nkb0_of(F) + 8 : nkb0_of(F) + 17; }
__host__ __device__ constexpr int nblk_total(int F) { return nkb0_of(F) + 25; }
// F = 63: the 512 block1.0 inputs are built and multiplied in two halves of 256 operand columns (the whole row, 128 rows x hi / lo,
// would take 256 KB).  Operand column order (the packer maps the W^T rows to it, w1_row_f63):
//   half 0:  PE5(dists) (60) + 4 zeros | PE3 of channels 0..31 (6 per channel: 2j + {sin, cos})
//   half 1:  raw features 0..62 + 1 zero | PE3 of channels 32..62 + 6 zeros
// so that the frozen kernel's distance-only layer 1 is K steps 0..3, and the second half needs no pair geometry.
__host__ __device__ inline int w1_row_f63(int k) {     // W^T row (reference input order) of operand column k; -1: zero
    if (k < 64) return k < 60 ? 7 * PNB_FEAT_DTU + k : -1;
    if (k < 256) return PNB_FEAT_DTU + (k - 64);
    if (k < 320) return k - 256 < PNB_FEAT_DTU ? k - 256 : -1;
    return 32 + (k - 320) / 6 < PNB_FEAT_DTU ? PNB_FEAT_DTU + 6 * 32 + (k - 320) : -1;
}
constexpr int STEP = 2 * 256 * 32;      // one weight stage: hi + lo image ([256 x 16] bf16 each) of one K = 16 step
constexpr float LEAKY = 0.01f;
constexpr int XE = 128 * 32;            // bytes of one [128 x 16] bf16 extras operand (SBO = 256)
__device__ __forceinline__ uint32_t xe_offset(int r, int k) { return k16_offset_bytes(r, k); }
}  // namespace tc

struct ShadeTcParams {
    pnb_query_t q;
    pnb_points_t pts;
    pnb_shade_opts_t o;
    const unsigned char* wimg;   // packed weight images (N = 256 per image)
    const float* bias[4];
    const float* wa;             // alpha_branch.0 weight [256]
    const float* ba;             // alpha_branch.0 bias [1]
    float* hbar;                 // h-bar as bf16 hi/lo A-operand blocks of k_color_wg (per 128 samples: 8 K blocks x {hi,lo} x [128x32])
    float* sigma;                // [n_valid]
    int hbar_cap;
    int* err;
    const unsigned char* vcnt;   // row packing: neighbours per PACKED position [n_valid] (vcntp of k_pack_quads)
    const uint32_t* vorder;      // valid-sample index of every packed position [n_valid]
    const uint32_t* quad_first;  // first valid sample of every 32-row quadrant [n_quads + 1]
    const int* pack_cnt;         // [0] = n_quads
    const float* pre;            // FROZEN: per-point hoisted layer-1 pre-activation [N][256] (k_point_pre)
};

// sin/cos of x*2^j, j = 0..NF-1: one accurate sincosf + angle doubling (abs error < 1e-6 after 4 doublings; the
// fp32 kernel keeps NF independent sincosf calls).  out[2j] = sin, out[2j+1] = cos  (networks.py:175-190 layout).
template <int NF>
__device__ __forceinline__ void pe_doubling(float x, float* out) {
    float s, c;
    sincosf(x, &s, &c);
    out[0] = s; out[1] = c;
#pragma unroll
    for (int j = 1; j < NF; ++j) {
        float s2 = 2.0f * s * c, c2 = fmaf(c, c, -s * s);
        s = s2; c = c2;
        out[2 * j] = s; out[2 * j + 1] = c;
    }
}

template <class SmemT>
__device__ __forceinline__ void store_chunk8_a1(SmemT& sm, int r, int kb, int k8, const float* v) {
    uint32_t h[4], l[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split_bf16x2(v[2 * i], v[2 * i + 1], h[i], l[i]);
    uint32_t off = (uint32_t)kb * tc::ABLK + tile_offset_bytes<tc::LAYOUT>(r, k8);
    *reinterpret_cast<uint4*>(sm.a_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(sm.a_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
}

// Sum of v over the lanes st .. st+cnt-1 of the warp (cnt <= 8; every lane calls it, lanes outside any segment pass st = lane,
// cnt = 1).  The order of the additions depends on cnt only, not on where the segment sits in the warp.
__device__ __forceinline__ float seg_scan8(float v, int lane, int st) {          // inclusive scan within the segment
#pragma unroll
    for (int d = 1; d <= 4; d <<= 1) {
        const float tv = __shfl_up_sync(0xffffffffu, v, d);
        if (lane - d >= st) v += tv;
    }
    return v;
}
__device__ __forceinline__ float seg_sum8(float v, int lane, int st, int cnt) {
    return __shfl_sync(0xffffffffu, seg_scan8(v, lane, st), st + cnt - 1);
}

// One pair row of the layer-1 operand (gather, distance weights, PE by angle doubling, hi/lo split -> shared memory).  The caller
// has packed only the valid (sample, neighbour) pairs into the rows: row `row` is neighbour `pk` of valid sample `pvi` (pvi < 0:
// unused row), and the rows of that sample are lanes pst .. pst+pcnt-1 of this warp.  Two builder threads per row:
//   part 0 = operand columns 0..151   (raw features, PE of features 0..19)
//   part 1 = operand columns 152..287 (PE of features 20..31, PE of the 6 distances), extras operand, weight*conf
// FROZEN (part 1 only, one builder thread per row): the feature columns come from the per-point table, so the row is part 1
// without the feature PE and with the distance PE at operand columns 0..63 (K blocks 0, 1); it also records the row's point.
// PP: per-point frames (pair_inputs.cuh, point_frame).  XSAMP: explicit samples (the frustum query, pair_inputs.cuh).
// F = 63 (not FROZEN; column order at tc::w1_row_f63), half HALF of the row:
//   half 0: part 0 = PE of features 0..23; part 1 = PE of features 24..31, PE of the distances, extras, weight*conf, the row's point
//   half 1: part 0 = raw features, PE of features 32..43; part 1 = PE of features 44..62 (the point is read back from sm.prow)
// emb rows of 63 floats are not 16-byte aligned: scalar loads.
template <int PART, bool FROZEN, bool PP, int F = PNB_FEAT, int HALF = 0, bool XSAMP = false, class SmemT>
__device__ __forceinline__ void build_pair_part(SmemT& sm, const ShadeTcParams& p, int row, int n_valid, int pvi, int pk, int pst, int pcnt) {
    using namespace tc;
    static_assert(PART == 0 || PART == 1, "two parts per row");
    static_assert(!FROZEN || PART == 1, "the frozen row is a part-1 row");
    constexpr bool W = F != PNB_FEAT;                                   // the 512-wide row of F = 63
    static_assert(!W || (F == PNB_FEAT_DTU && !FROZEN && (HALF == 0 || HALF == 1)), "F = 63: two halves, not frozen");
    static_assert(W || HALF == 0, "F = 32: one row");
    constexpr bool P0 = PART == 0, P1 = PART == 1;
    constexpr bool GEO = P1 && HALF == 0;                               // forms the pair geometry: dist PE, extras, weight*conf
    constexpr bool RAW = P0 && (!W || HALF == 1);                       // writes the raw features
    constexpr int G_LO = !W ? (P0 ? 0 : 5) : HALF == 0 ? (P0 ? 0 : 6) : (P0 ? 8 : 11);   // feature groups (4 features each) whose
    constexpr int G_HI = !W ? ((P1 && !FROZEN) ? 8 : 5) : HALF == 0 ? (P0 ? 6 : 8) : (P0 ? 11 : 16);   // PE this part builds
    constexpr int GCOL0 = !W ? 32 : 64 - 192 * HALF;                    // operand column of group gi: GCOL0 + 24 gi
    constexpr int NRAW = W ? 8 : 4;                                     // 16-byte chunks of raw features
    constexpr int DCOL = (FROZEN || W) ? 0 : 224;                       // first operand column of the distance PE
    constexpr int C_LO = P1 && !FROZEN ? 19 : 0, C_HI = P0 ? 19 : FROZEN ? 8 : 36;   // 16-byte chunks (column / 8) of this part (F = 32)
    const pnb_query_t& q = p.q;
    int pidx = -1, p0 = 0;
    CandSample cs = {};
    float3 lp = make_float3(0.f, 0.f, 0.f);
    if (W && HALF == 1) {
        pidx = sm.prow[row];
    } else if (pvi >= 0 && pvi < n_valid) {
        const uint32_t s = q.valid_list[pvi];
        if (GEO) { cs = cand_sample<XSAMP>(q, s); p0 = view_point<PP>(q, s); if (XSAMP) lp = cand_pers<XSAMP>(q, s); }
        if (pk < q.K) pidx = q.cand_pidx[(size_t)s * q.K + pk];
    }
    if (FROZEN || (W && GEO)) sm.prow[row] = pidx;
    const bool valid = pidx >= 0;
    const int pi = valid ? pidx : 0;
    PairGeom g;
    float3 ov;
    if (GEO) {
        ov = view_in_points<PP>(p.pts, p.o, p0, cs.dir);
        g = pair_geom<PP, XSAMP>(p.pts, p.o, pidx, cs.pos, lp);
        const float wsum = seg_sum8(g.w, row & 31, pst, pcnt);   // every lane takes part in the shuffles
        sm.wc[row] = valid ? norm_weight(g.w, wsum) * g.cc : 0.f;
    }
    float ex[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (valid) {
        const float4* ep = (const float4*)&p.pts.emb[(size_t)pi * F];
        const float* es = &p.pts.emb[(size_t)pi * F];
#pragma unroll
        for (int gi = G_LO; gi < G_HI; ++gi) {  // 4 features per step
            float f[4];
            if (!W) {
                float4 fv = __ldg(ep + gi);
                f[0] = fv.x; f[1] = fv.y; f[2] = fv.z; f[3] = fv.w;
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) f[e] = 4 * gi + e < F ? __ldg(es + 4 * gi + e) : 0.f;
            }
            float pe[24];
#pragma unroll
            for (int e = 0; e < 4; ++e) pe_doubling<3>(f[e], pe + e * 6);
            const int col = GCOL0 + 24 * gi;
#pragma unroll
            for (int c = 0; c < 3; ++c) store_chunk8_a1(sm, row, (col + 8 * c) >> 5, (col + 8 * c) & 31, pe + 8 * c);
        }
        if (RAW) {
#pragma unroll
            for (int gi = 0; gi < NRAW; ++gi) {    // raw features, 8 per chunk (re-read: L1 hit)
                float f8[8];
                if (!W) {
                    float4 a = __ldg(ep + 2 * gi), b = __ldg(ep + 2 * gi + 1);
                    f8[0] = a.x; f8[1] = a.y; f8[2] = a.z; f8[3] = a.w; f8[4] = b.x; f8[5] = b.y; f8[6] = b.z; f8[7] = b.w;
                } else {
#pragma unroll
                    for (int e = 0; e < 8; ++e) f8[e] = 8 * gi + e < F ? __ldg(es + 8 * gi + e) : 0.f;
                }
                store_chunk8_a1(sm, row, (8 * gi) >> 5, (8 * gi) & 31, f8);
            }
        }
        if (GEO) {
            float dp[64];
#pragma unroll
            for (int e = 0; e < 6; ++e) pe_doubling<5>(g.dist[e], dp + 10 * e);
            dp[60] = dp[61] = dp[62] = dp[63] = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) store_chunk8_a1(sm, row, (DCOL + 8 * c) >> 5, (DCOL + 8 * c) & 31, dp + 8 * c);
            point_extras<PP>(p.pts, p.o, pi, ov, ex);
        }
    } else {
        float z8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (!W) {
            for (int c = C_LO; c < C_HI; ++c) store_chunk8_a1(sm, row, c >> 2, (c & 3) * 8, z8);
        } else {
#pragma unroll
            for (int c = 3 * G_LO; c < 3 * G_HI; ++c) store_chunk8_a1(sm, row, (GCOL0 + 8 * c) >> 5, (GCOL0 + 8 * c) & 31, z8);
            if (RAW)
#pragma unroll
                for (int c = 0; c < NRAW; ++c) store_chunk8_a1(sm, row, (8 * c) >> 5, (8 * c) & 31, z8);
            if (GEO)
#pragma unroll
                for (int c = 0; c < 8; ++c) store_chunk8_a1(sm, row, (DCOL + 8 * c) >> 5, (DCOL + 8 * c) & 31, z8);
        }
    }
    if (GEO) {   // block3 extras operand [128 x 16]: chunk 0 = extras, chunk 1 = 0
        uint32_t h[4], l[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_bf16x2(ex[2 * i], ex[2 * i + 1], h[i], l[i]);
        uint32_t off = tc::xe_offset(row, 0);
        *reinterpret_cast<uint4*>(sm.xe_hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
        *reinterpret_cast<uint4*>(sm.xe_lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
        *reinterpret_cast<uint4*>(sm.xe_hi + off + 128) = make_uint4(0u, 0u, 0u, 0u);
        *reinterpret_cast<uint4*>(sm.xe_lo + off + 128) = make_uint4(0u, 0u, 0u, 0u);
    }
}
// ------------------------------------------------------------------------------------------ weight packing
// W^T fp32 [Kpad][N] (rows >= Kpad read as zero) -> per K = 16 step: hi image then lo image, each [N x 16] bf16 in the wgmma
// operand layout (k16_offset_bytes): one contiguous weight stage per step.
__global__ void __launch_bounds__(256) k_pack_weights(const float* __restrict__ wt, int Kpad, int nks, int N, unsigned char* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (ks, n, k)
    if (i >= nks * N * 16) return;
    const int ks = i / (N * 16), rem = i - ks * N * 16;
    const int n = rem >> 4, k = rem & 15;
    const int kg = ks * 16 + k;
    const float v = kg < Kpad ? wt[(size_t)kg * N + n] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    const uint32_t off = k16_offset_bytes(n, k);
    const size_t img = (size_t)N * 32;
    *(__nv_bfloat16*)(out + (size_t)(2 * ks) * img + off) = h;
    *(__nv_bfloat16*)(out + (size_t)(2 * ks + 1) * img + off) = l;
}
// block1.0 of F = 63: the same images, operand column kg taken from W^T row tc::w1_row_f63(kg)
__global__ void __launch_bounds__(256) k_pack_block1_f63(const float* __restrict__ wt, int nks, int N, unsigned char* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;   // (ks, n, k)
    if (i >= nks * N * 16) return;
    const int ks = i / (N * 16), rem = i - ks * N * 16;
    const int n = rem >> 4, k = rem & 15;
    const int src = tc::w1_row_f63(ks * 16 + k);
    const float v = src >= 0 ? wt[(size_t)src * N + n] : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    const uint32_t off = k16_offset_bytes(n, k);
    const size_t img = (size_t)N * 32;
    *(__nv_bfloat16*)(out + (size_t)(2 * ks) * img + off) = h;
    *(__nv_bfloat16*)(out + (size_t)(2 * ks + 1) * img + off) = l;
}

// Weight ring of the pair and colour kernels.  Consumption m (one K = 16 step, counted over the CTA's whole tile sequence) uses
// stage m % NSTAGE.  One producer thread, outside the consumer warpgroups, runs the whole sequence: it waits until the 8 consumer
// warps have released the stage's previous consumption and refills it.  A consumer warp only waits for `full` and releases a stage
// once the wgmma group that read it has retired (a predicated arrive of lane 0): nothing divergent sits between its wgmma, so ptxas
// keeps them asynchronous.  The weights do not depend on the tile, so the ring runs ahead across tile boundaries.
template <int NSTAGE, int STEP, class ImgOf>
struct Ring {
    static constexpr uint32_t CONSUMER_WARPS = 8;         // arrivals that empty a stage
    unsigned char (*buf)[STEP];
    uint64_t* full;
    uint64_t* empty;
    const unsigned char* src;
    uint32_t total;
    ImgOf img_of;
    int* err;
    __device__ __forceinline__ void init() {              // one thread, before the CTA-wide barrier that publishes the ring
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], CONSUMER_WARPS); }
    }
    // the producer thread; after a failed (timed-out) wait it stops refilling and the consumers' waits report their own time-out
    __device__ __forceinline__ void produce() {
#pragma unroll 1
        for (uint32_t m = 0; m < total; ++m) {
            const uint32_t s = m % NSTAGE;
            if (m >= (uint32_t)NSTAGE && !mbar_wait(&empty[s], (m / NSTAGE - 1u) & 1u, err, 92)) return;
            mbar_arrive_expect_tx(&full[s], STEP);
            bulk_g2s(buf[s], src + (size_t)img_of(m) * STEP, STEP, &full[s]);
        }
    }
    // after a failed (timed-out) wait `ok` stays false: later waits are skipped, every barrier is still reached, the error flag is set
    __device__ __forceinline__ bool acquire(uint32_t m, bool ok) {
        return ok && mbar_wait(&full[m % NSTAGE], (m / NSTAGE) & 1u, err, 91);
    }
    __device__ __forceinline__ void release(uint32_t m) { mbar_arrive_if(&empty[m % NSTAGE], (threadIdx.x & 31) == 0); }
};

// ------------------------------------------------------------------------------------------ row packing
namespace pk {
constexpr int PACK_S = 512;             // samples per independently packed super-chunk (its last quadrant may stay partly empty)
constexpr int PACK_WIN = 64;            // look-ahead of the first-fit packing
}  // namespace pk

// ---- row packing (runs before the pair kernel; all sizes come from device counters, nothing synchronises)
// First-fit packing of the valid samples (1..8 rows each = their neighbour count) into 32-row quadrants, independently per
// super-chunk of PACK_S samples: samples are taken in order while they fit; a sample that does not fit stays first in line for
// the next quadrant while up to PACK_WIN later, smaller samples may fill the remaining rows (so the order inside a super-chunk
// becomes a permutation, vorder).  tests/test_host_logic.py restates the algorithm in Python; tests/test_gpu_shade.py compares
// the tables of these kernels with that restatement.
//   k_pack_quads  one WARP per super-chunk (counts in shared memory; the sequential "take while it fits" loop over the 64-entry
//                 window becomes <= 32 rounds of one warp scan each: a round takes the maximal prefix of still-fitting
//                 candidates and rejects the first one that does not fit).  Writes vorder / vcntp (final positions: the
//                 packing only permutes inside a super-chunk) and the quadrant boundaries super-chunk-locally.
//   k_pack_scan   exclusive scan of the per-super-chunk quadrant counts (one block), n_quads, sentinel
//   k_pack_place  quadrant boundaries -> their global position (fully parallel)
__global__ void __launch_bounds__(256) k_pack_quads(pnb_query_t q, int cap, uint32_t* __restrict__ sc_quads, uint32_t* __restrict__ quad_local,
                                                    uint32_t* __restrict__ vorder, unsigned char* __restrict__ vcntp,
                                                    float4* __restrict__ sigma_rgb) {
    __shared__ unsigned char cnt[8][pk::PACK_S];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sc = blockIdx.x * 8 + wib;
    const int n_all = q.counters[PNB_QC_N_VALID];
    const int n_valid = min(n_all, cap);
    if (n_all > cap) {
        // workspace overflow (flagged as err 9 by the pair kernel): the samples that are dropped must not reach the compositing
        // kernel uninitialised -> they contribute nothing (sigma = 0)
        for (int vi = cap + blockIdx.x * blockDim.x + threadIdx.x; vi < n_all; vi += gridDim.x * blockDim.x)
            sigma_rgb[q.valid_list[vi]] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const int i0 = sc * pk::PACK_S;
    if (i0 >= n_valid) return;
    const int n = min(pk::PACK_S, n_valid - i0);
    unsigned char* c = cnt[wib];                  // neighbour counts of this super-chunk; 0 = already placed
    for (int i = lane; i < n; i += 32) c[i] = q.samp_nvalid[q.valid_list[i0 + i]];
    __syncwarp();
    const uint32_t lt = (1u << lane) - 1u;
    int pos = 0, emitted = 0, nq = 0;
    while (pos < n) {                             // one quadrant per iteration (warp-uniform)
        if (lane == 0) quad_local[i0 + nq] = (uint32_t)(i0 + emitted);     // nq <= emitted: every quadrant holds >= 1 sample
        const int lim = min(n, pos + pk::PACK_WIN);
        const int ia = pos + lane, ib = pos + 32 + lane;
        int ca = ia < lim ? (int)c[ia] : 0, cb = ib < lim ? (int)c[ib] : 0;
        int rows = 0, start = 0;                  // candidates with window index < start have been decided for this quadrant
        for (;;) {
            const int room = 32 - rows;
            const int va = (lane >= start && ca <= room) ? ca : 0, vb = (32 + lane >= start && cb <= room) ? cb : 0;
            int pa = va, pb = vb;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int ta = __shfl_up_sync(0xffffffffu, pa, d), tb = __shfl_up_sync(0xffffffffu, pb, d);
                if (lane >= d) { pa += ta; pb += tb; }
            }
            pb += __shfl_sync(0xffffffffu, pa, 31);
            const bool fa = va != 0 && pa <= room, fb = vb != 0 && pb <= room;
            const uint32_t ma = __ballot_sync(0xffffffffu, fa), mb = __ballot_sync(0xffffffffu, fb);
            const uint32_t na = __ballot_sync(0xffffffffu, va != 0 && pa > room), nb = __ballot_sync(0xffffffffu, vb != 0 && pb > room);
            const int cnt_a = __popc(ma);
            if (fa) { const int e = i0 + emitted + __popc(ma & lt); vorder[e] = (uint32_t)(i0 + ia); vcntp[e] = (unsigned char)ca; c[ia] = 0; }
            if (fb) { const int e = i0 + emitted + cnt_a + __popc(mb & lt); vorder[e] = (uint32_t)(i0 + ib); vcntp[e] = (unsigned char)cb; c[ib] = 0; }
            // rows taken this round = the largest fitting prefix sum
            int took = fb ? pb : (fa ? pa : 0);
#pragma unroll
            for (int d = 16; d >= 1; d >>= 1) took = max(took, __shfl_xor_sync(0xffffffffu, took, d));
            if (fa) ca = 0;
            if (fb) cb = 0;
            emitted += cnt_a + __popc(mb);
            rows += took;
            if (rows >= 32 || (na | nb) == 0u) break;
            start = na ? __ffs(na) : 32 + __ffs(nb);          // first rejected candidate + 1
            if (start >= 64) break;
        }
        __syncwarp();
        // first entry still unplaced (the window's entries keep their order; everything beyond the window is untouched)
        const uint32_t ra = __ballot_sync(0xffffffffu, ca != 0), rb = __ballot_sync(0xffffffffu, cb != 0);
        pos = ra ? pos + __ffs(ra) - 1 : (rb ? pos + 32 + __ffs(rb) - 1 : lim);
        ++nq;
    }
    if (lane == 0) sc_quads[sc] = (uint32_t)nq;
}
// exclusive scan of the per-super-chunk quadrant counts (one block): sc_quads[0 .. n_sc] (last = total), total -> pack_cnt[0],
// sentinel quad_first[n_quads] = n_valid
__global__ void __launch_bounds__(1024) k_pack_scan(pnb_query_t q, int cap, uint32_t* __restrict__ sc_quads, uint32_t* __restrict__ quad_first,
                                                    int* __restrict__ pack_cnt) {
    __shared__ uint32_t wsum[32];
    const int n_valid = min(q.counters[PNB_QC_N_VALID], cap);
    const int n_sc = (n_valid + pk::PACK_S - 1) / pk::PACK_S;
    const int per = (n_sc + 1023) / 1024;
    const int b0 = threadIdx.x * per, b1 = min(b0 + per, n_sc);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    uint32_t sum = 0;
    for (int i = b0; i < b1; ++i) sum += sc_quads[i];
    uint32_t incl = sum;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
    if (lane == 31) wsum[w] = incl;
    __syncthreads();
    if (w == 0) {
        uint32_t v = wsum[lane], iv = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, iv, d); if (lane >= d) iv += t; }
        wsum[lane] = iv - v;
        if (lane == 31) { pack_cnt[0] = (int)iv; quad_first[iv] = (uint32_t)n_valid; sc_quads[n_sc] = iv; }
    }
    __syncthreads();
    uint32_t run = wsum[w] + incl - sum;
    for (int i = b0; i < b1; ++i) { const uint32_t v = sc_quads[i]; sc_quads[i] = run; run += v; }
}
__global__ void __launch_bounds__(256) k_pack_place(pnb_query_t q, int cap, const uint32_t* __restrict__ sc_quads, const uint32_t* __restrict__ quad_local,
                                                    uint32_t* __restrict__ quad_first) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_valid = min(q.counters[PNB_QC_N_VALID], cap);
    if (i >= n_valid) return;
    const int sc = i / pk::PACK_S, j = i - sc * pk::PACK_S;
    const uint32_t first = sc_quads[sc], nq = sc_quads[sc + 1] - first;
    if ((uint32_t)j < nq) quad_first[first + j] = quad_local[i];
}

// One 16-column chunk of the last epilogue: columns c0 .. c0+15 of this lane's row (raw layer-4 accumulator in v): + bias, LeakyReLU,
// partial alpha dot product, weight*conf scaling, the K-reduction over the rows of each sample as a segmented inclusive scan
// (segments = samples, <= 8 lanes, first lane st); the last row of a sample (swrite) holds the sums and writes h-bar in the
// colour kernel's operand format (bf16 hi / lo, core-matrix layout).
template <bool O1>
__device__ __forceinline__ void last_chunk_from_regs(const ShadeTcParams& p, int c0, const uint32_t* v, float wrow, int st, bool swrite, int sidx, int lane,
                                                     float& apart) {
    using namespace tc;
    const float* bias = p.bias[3];
    constexpr bool order1 = O1;
    float z[16];
#pragma unroll
    for (int e4 = 0; e4 < 4; ++e4) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + c0) + e4), ww = __ldg(reinterpret_cast<const float4*>(p.wa + c0) + e4);
        const float bq[4] = {bb.x, bb.y, bb.z, bb.w}, wq[4] = {ww.x, ww.y, ww.z, ww.w};
#pragma unroll
        for (int e1 = 0; e1 < 4; ++e1) {
            const int e = 4 * e4 + e1;
            float y = __uint_as_float(v[e]) + bq[e1];
            y = fmaxf(y, LEAKY * y);
            if (!order1) apart = fmaf(y, wq[e1], apart);
            z[e] = y * wrow;
        }
    }
#pragma unroll
    for (int e = 0; e < 16; ++e) z[e] = seg_scan8(z[e], lane, st);
    if (order1) {
#pragma unroll
        for (int e = 0; e < 16; ++e) apart = fmaf(z[e], __ldg(p.wa + c0 + e), apart);
    }
    if (swrite) {
        uint32_t hh[8], ll[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) split_bf16x2(z[2 * e], z[2 * e + 1], hh[e], ll[e]);
        unsigned char* dst = reinterpret_cast<unsigned char*>(p.hbar) + ((size_t)(sidx >> 7) * 8 + (c0 >> 5)) * (2 * 8192) +
                             tile_offset_bytes<LAYOUT_NONE>(sidx & 127, c0 & 31);
        *reinterpret_cast<uint4*>(dst) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
        *reinterpret_cast<uint4*>(dst + 128) = make_uint4(hh[4], hh[5], hh[6], hh[7]);
        *reinterpret_cast<uint4*>(dst + 8192) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
        *reinterpret_cast<uint4*>(dst + 8192 + 128) = make_uint4(ll[4], ll[5], ll[6], ll[7]);
    }
}
// segment bookkeeping of one quadrant row: first row / index of its sample, whether it is the sample's last row
struct QuadRow { int st, j; bool live, is_end; };
__device__ __forceinline__ QuadRow quad_row(uint32_t head, int tot, int lane) {
    QuadRow r;
    r.live = lane < tot;
    const uint32_t below = head & (0xffffffffu >> (31 - lane));
    r.st = r.live ? 31 - __clz(below) : lane;
    r.j = r.live ? __popc(below) - 1 : 0;
    const uint32_t nxt = lane < 31 ? (head >> (lane + 1)) : 0u;
    r.is_end = r.live && lane == (nxt ? lane + __ffs(nxt) - 1 : tot - 1);
    return r;
}

// pre[n][c] = b1[c] + sum_{k<7F} W1^T[k][c] * x_n[k],  x_n = [f (F), PE3(f) (6F, column F + 6*feature + 2*j + {sin, cos})]: the
// point-only inputs of block1.0 (F = 32: exactly the first 7 K blocks of the operand build_pair_part writes).  fp32 FMAs in ascending k.
// Block = NP points x 256 columns (F = 63: 16 points, the 441 inputs padded to 444 with zeros).
__host__ __device__ constexpr int point_pre_np(int F) { return F == PNB_FEAT ? 32 : 16; }   // points per block
template <int F>
__global__ void __launch_bounds__(256) k_point_pre(const float* __restrict__ emb, int N, const float* __restrict__ w1t, const float* __restrict__ b1,
                                                   float* __restrict__ pre) {
    constexpr int NP = point_pre_np(F);
    constexpr int KX = (7 * F + 3) / 4 * 4;               // inputs, whole float4: 224 | 444
    __shared__ __align__(16) float x[NP][KX + 4];
    const int n0 = blockIdx.x * NP;
    for (int i = threadIdx.x; i < NP * F; i += 256) {
        const int pl = F == PNB_FEAT ? i >> 5 : i / F, f = F == PNB_FEAT ? i & 31 : i - pl * F, n = n0 + pl;
        const float v = n < N ? __ldg(&emb[(size_t)n * F + f]) : 0.f;
        float pe[6];
        pe_doubling<3>(v, pe);
        x[pl][f] = v;
#pragma unroll
        for (int e = 0; e < 6; ++e) x[pl][F + 6 * f + e] = pe[e];
    }
    if (KX > 7 * F)
        for (int i = threadIdx.x; i < NP * (KX - 7 * F); i += 256) x[i / (KX - 7 * F)][7 * F + i % (KX - 7 * F)] = 0.f;
    __syncthreads();
    const int c = threadIdx.x;
    float acc[NP];
    const float bc = __ldg(&b1[c]);
#pragma unroll
    for (int i = 0; i < NP; ++i) acc[i] = 0.f;
    for (int k = 0; k < KX; k += 4) {
        const float w0 = __ldg(&w1t[(size_t)k * 256 + c]), w1 = __ldg(&w1t[(size_t)(k + 1) * 256 + c]);
        const float w2 = __ldg(&w1t[(size_t)(k + 2) * 256 + c]), w3 = __ldg(&w1t[(size_t)(k + 3) * 256 + c]);
#pragma unroll
        for (int i = 0; i < NP; ++i) {
            const float4 xv = *reinterpret_cast<const float4*>(&x[i][k]);
            acc[i] = fmaf(xv.w, w3, fmaf(xv.z, w2, fmaf(xv.y, w1, fmaf(xv.x, w0, acc[i]))));
        }
    }
#pragma unroll
    for (int i = 0; i < NP; ++i)
        if (n0 + i < N) pre[(size_t)(n0 + i) * 256 + c] = acc[i] + bc;
}

// =====================================================================================================================
// k_shade_wg: the pair MLPs of the packed 128-row tiles (a tile is four 32-row quadrants, each holding whole samples back to back,
// only their valid neighbours: 99 % of the rows carry a pair on the lego frame).  One persistent CTA per SM, 384 threads = two
// consumer warpgroups + a producer warpgroup (one thread of warp 8 runs the weight ring; it hands its registers to the consumers
// with setmaxnreg); warpgroup c < 2 owns tile rows 64c .. 64c+63 of every layer (wgmma M = 64, N = 256: a 128-register fp32
// accumulator per thread).  Per tile:
//   build     two threads per row (operand columns 0..151 | 152..287 of block1.0; FROZEN: one thread per row, PE5(dists) only) write
//             the layer-1 operand (bf16 hi / lo, core-matrix layout) and the block3 extras operand into shared memory
//   layers    per K = 16 step: wait for the weight stage, 3 wgmma (A_hi W_hi, A_lo W_hi, A_hi W_lo), one wgmma group in flight; the
//             epilogue (+ bias or + pre[point], LeakyReLU, bf16 hi / lo split) writes the next layer's operand over this layer's.
//             A warpgroup reads and writes only its own 64 rows, so the two warpgroups only meet at the weight ring.
//   last      the layer-4 accumulators go to shared memory (fp32, over the dead operand) and are reduced over the rows of each
//             sample with lane = row (segmented warp scan; its addition order depends on the neighbour count only, so a ray's colour
//             does not depend on which rays share the call): h-bar + sigma
namespace hw {
constexpr int NTHR = 256;                 // the two consumer warpgroups
constexpr int NTHR_CTA = NTHR + 128;      // + warpgroup 2: the weight-ring producer (one thread of warp 8)
// setmaxnreg budgets: the launch gives 168 registers per thread (65,536 / 384, rounded down to 8); the CTA's 64,512 are
// redistributed as 2 x 128 x REGS_CONSUMER + 128 x REGS_PRODUCER.  At 232 consumer registers the frozen per-point-frame
// instantiations spill; the producer loop fits in 24.
constexpr uint32_t REGS_CONSUMER = 240, REGS_PRODUCER = 24;
static_assert(2 * 128 * REGS_CONSUMER + 128 * REGS_PRODUCER <= 168 * NTHR_CTA, "register budgets exceed the launch allocation");
constexpr int NSTAGE = 4;
constexpr int YLD = 260;                  // fp32 row stride of the last-epilogue buffer: lane = row float4 reads are conflict-free
// first K step of the frozen layer 1: the distance PE (F = 32: operand columns 224..287 of block1.0; F = 63: 0..63, tc::w1_row_f63)
__host__ __device__ constexpr int ks_frozen0(int F) { return F == PNB_FEAT ? 14 : 0; }
struct Smem {
    unsigned char a_hi[tc::NKB_MAX * tc::ABLK];   // layer operand; a_hi + a_lo also hold the fp32 [128 x YLD] rows of the last epilogue
    unsigned char a_lo[tc::NKB_MAX * tc::ABLK];
    unsigned char b[NSTAGE][tc::STEP];
    unsigned char xe_hi[tc::XE];
    unsigned char xe_lo[tc::XE];
    float wc[tc::TM];
    int prow[tc::TM];                     // FROZEN: point index of every row (-1: unused row)
    float alpha_part[2][tc::TM];
    uint32_t qhead[4], qfirst[4], qtotal[4];   // per quadrant: segment heads, first packed position, rows
    uint64_t bar_full[NSTAGE], bar_empty[NSTAGE];
};
static_assert(tc::TM * YLD * 4 <= 2 * tc::NKB_MAX * tc::ABLK, "last-epilogue rows exceed the operand region");
// K = 16 steps of a tile: layer 1 (18 | F = 63: 32 | FROZEN 4), layer 2 (16), layer 3 (16 + the extras step), layer 4 (16)
__host__ __device__ constexpr int steps_of(int l, bool frozen, int F = PNB_FEAT) { return l == 0 ? (frozen ? 4 : kpad1_of(F) / 16) : l == 2 ? 17 : 16; }
// weight image (index in K = 16 steps of the packed pair images) of step j of a tile
template <int F = PNB_FEAT>
__device__ __forceinline__ uint32_t step_image(uint32_t j, bool frozen) {
    const uint32_t s0 = (uint32_t)steps_of(0, frozen, F);
    if (j < s0) return (frozen ? (uint32_t)ks_frozen0(F) : 0u) + j;
    j -= s0;
    if (j < 16u) return 2u * tc::img_base(1, F) + j;
    j -= 16u;
    if (j < 17u) return 2u * tc::img_base(2, F) + j;
    return 2u * tc::img_base(3, F) + (j - 17u);
}
}  // namespace hw

// O1: agg_intrp_order == 1 as a compile-time flag (the alpha dot product over the K-aggregated feature); PP: per-point frames
// (pts.rw2c != NULL), compile-time as well, so that the uniform-frame builds keep their registers; F: point_features_dim (32 | 63);
// XSAMP: explicit samples (the frustum query, pair_inputs.cuh), instantiated for F = 63 with uniform frames.
// F = 63, not FROZEN: layer 1 runs over 512 operand columns in two halves of 16 K steps; after the first half every wgmma that read it
// retires (both warpgroups), the builders write the second half over it and the accumulator carries on.  FROZEN does not read the
// features: only its layer-1 weight images differ.
template <bool FROZEN, bool O1, bool PP, int F, bool XSAMP = false>
__global__ void __launch_bounds__(hw::NTHR_CTA, 1) k_shade_wg(ShadeTcParams p) {
    using namespace tc;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    hw::Smem& sm = *reinterpret_cast<hw::Smem*>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int wgi = warp >> 2;                                   // consumer warpgroup
    const pnb_query_t& q = p.q;
    const int n_valid = min(q.counters[PNB_QC_N_VALID], p.hbar_cap);
    const int n_quads = p.pack_cnt[0];
    const int n_tiles = (n_quads + 3) >> 2;
    const int my_tiles = n_tiles > (int)blockIdx.x ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    constexpr bool SPLIT = F != PNB_FEAT && !FROZEN;              // layer 1 in two halves
    constexpr uint32_t ST = (uint32_t)(hw::steps_of(0, FROZEN, F) + 16 + 17 + 16);
    auto img_of = [](uint32_t m) { return hw::step_image<F>(m % ST, FROZEN); };
    Ring<hw::NSTAGE, STEP, decltype(img_of)> ring{sm.b, sm.bar_full, sm.bar_empty, p.wimg, (uint32_t)my_tiles * ST, img_of, p.err};

    if (tid == 0) {
        ring.init();
        mbar_fence_init();
        if (blockIdx.x == 0 && q.counters[PNB_QC_N_VALID] > p.hbar_cap) atomicExch(p.err, 9);
    }
    __syncthreads();
    if (wgi == 2) {                                              // producer warpgroup
        setmaxnreg_dec<hw::REGS_PRODUCER>();
        if (tid == hw::NTHR) ring.produce();
        return;
    }
    setmaxnreg_inc<hw::REGS_CONSUMER>();

    const uint32_t a_hi0 = smem_u32(sm.a_hi) + (uint32_t)wgi * 4096u, a_lo0 = smem_u32(sm.a_lo) + (uint32_t)wgi * 4096u;
    const uint32_t xe_hi0 = smem_u32(sm.xe_hi) + (uint32_t)wgi * 2048u, xe_lo0 = smem_u32(sm.xe_lo) + (uint32_t)wgi * 2048u;
    const uint32_t b0 = smem_u32(sm.b[0]);
    const int r0 = 64 * wgi + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);   // fragment: rows r0, r0 + 8; columns 8j + cq, +1
    float* ybuf = reinterpret_cast<float*>(sm.a_hi);
    uint32_t m = 0;
    bool ok = true;
    float acc[128];
    for (int t = 0; t < my_tiles; ++t) {
        const int tile = (int)blockIdx.x + t * (int)gridDim.x;
        named_bar_sync(1, hw::NTHR);                             // the previous tile's last epilogue is done with shared memory
        // ---------------- build: quadrant qw = warp % 4; part = warp / 4 (FROZEN: warps 0-3 only)
        {
            const int qw = warp & 3, part = warp >> 2, row = qw * 32 + lane;
            if (!FROZEN || part == 0) {
                const int qd = tile * 4 + qw;
                uint32_t first = 0, nsamp = 0;
                if (qd < n_quads) { first = p.quad_first[qd]; nsamp = p.quad_first[qd + 1] - first; }
                const int c = lane < (int)nsamp ? (int)p.vcnt[first + lane] : 0;
                int incl = c;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += v; }
                const uint32_t head = __reduce_or_sync(0xffffffffu, lane < (int)nsamp ? (1u << (incl - c)) : 0u);
                const int total = __shfl_sync(0xffffffffu, incl, 31);
                const QuadRow qr = quad_row(head, total, lane);
                const int cj = __shfl_sync(0xffffffffu, c, qr.j);
                if (lane == 0 && part == 0) { sm.qhead[qw] = head; sm.qfirst[qw] = first; sm.qtotal[qw] = (uint32_t)total; }
                const int pvi = qr.live ? (int)p.vorder[first + qr.j] : -1;
                if (FROZEN) build_pair_part<1, true, PP, PNB_FEAT, 0, XSAMP>(sm, p, row, n_valid, pvi, lane - qr.st, qr.st, qr.live ? cj : 1);
                else if (part == 0) build_pair_part<0, false, PP, F, 0, XSAMP>(sm, p, row, n_valid, pvi, lane - qr.st, qr.st, qr.live ? cj : 1);
                else build_pair_part<1, false, PP, F, 0, XSAMP>(sm, p, row, n_valid, pvi, lane - qr.st, qr.st, qr.live ? cj : 1);
            }
            fence_proxy_async();
            named_bar_sync(1, hw::NTHR);
        }
        // ---------------- the four layers
        for (int l = 0; l < 4; ++l) {
            const int nst = hw::steps_of(l, FROZEN, F);
            wg::fence();
            for (int kk = 0; kk < nst; ++kk, ++m) {
                if constexpr (SPLIT) {
                    if (l == 0 && kk == 16) {
                        // second half of the layer-1 operand: the first half's wgmma have retired in both warpgroups before it is
                        // overwritten (its last weight stage is released after the next step, as usual)
                        wg::wait<0>();
                        pin<128>(acc);
                        named_bar_sync(1, hw::NTHR);
                        const int row = (warp & 3) * 32 + lane;
                        if (warp < 4) build_pair_part<0, false, PP, F, 1, XSAMP>(sm, p, row, n_valid, -1, 0, 0, 1);
                        else build_pair_part<1, false, PP, F, 1, XSAMP>(sm, p, row, n_valid, -1, 0, 0, 1);
                        fence_proxy_async();
                        named_bar_sync(1, hw::NTHR);
                        wg::fence();
                    }
                }
                ok = ring.acquire(m, ok);
                const uint32_t bs = b0 + (m % hw::NSTAGE) * (uint32_t)STEP;
                const uint64_t bh = desc_k16(bs), bl = desc_k16(bs + STEP / 2);
                uint64_t ah, al;
                if (l == 2 && kk == 16) {
                    ah = desc_k16(xe_hi0); al = desc_k16(xe_lo0);
                } else {
                    const int ka = SPLIT && l == 0 ? (kk & 15) : kk;      // K step within the operand in shared memory
                    const uint32_t off = (uint32_t)(ka >> 1) * ABLK + (uint32_t)(ka & 1) * 256u;
                    ah = desc_none(a_hi0 + off); al = desc_none(a_lo0 + off);
                }
                mma_n256(acc, ah, bh, kk ? 1u : 0u);
                mma_n256(acc, al, bh, 1u);
                mma_n256(acc, ah, bl, 1u);
                wg::commit();
                wg::wait<1>();
                if (kk > 0) ring.release(m - 1);
            }
            wg::wait<0>();
            pin<128>(acc);
            ring.release(m - 1);
            if (l == 3) break;
            // epilogue: + bias (FROZEN layer 1: + pre[point of the row], which includes the bias), LeakyReLU, bf16 hi / lo split
            const float* bias = p.bias[l];
            const float* pre0 = nullptr;
            const float* pre1 = nullptr;
            if (FROZEN && l == 0) {                                  // unused rows (prow < 0): any finite values
                pre0 = p.pre + (size_t)max(sm.prow[r0], 0) * 256;
                pre1 = p.pre + (size_t)max(sm.prow[r0 + 8], 0) * 256;
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const int col = 8 * j + cq;
                float2 u0, u1;
                if (FROZEN && l == 0) {
                    u0 = __ldg(reinterpret_cast<const float2*>(pre0 + col));
                    u1 = __ldg(reinterpret_cast<const float2*>(pre1 + col));
                } else {
                    u0 = __ldg(reinterpret_cast<const float2*>(bias + col));
                    u1 = u0;
                }
                float y0 = acc[4 * j] + u0.x, y1 = acc[4 * j + 1] + u0.y, y2 = acc[4 * j + 2] + u1.x, y3 = acc[4 * j + 3] + u1.y;
                y0 = fmaxf(y0, LEAKY * y0); y1 = fmaxf(y1, LEAKY * y1); y2 = fmaxf(y2, LEAKY * y2); y3 = fmaxf(y3, LEAKY * y3);
                uint32_t h0, l0, h1, l1;
                split_bf16x2(y0, y1, h0, l0);
                split_bf16x2(y2, y3, h1, l1);
                const uint32_t o = (uint32_t)(col >> 5) * ABLK + tile_offset_bytes<LAYOUT>(r0, col & 31);   // row r0 + 8: + 512
                *reinterpret_cast<uint32_t*>(sm.a_hi + o) = h0;
                *reinterpret_cast<uint32_t*>(sm.a_lo + o) = l0;
                *reinterpret_cast<uint32_t*>(sm.a_hi + o + 512) = h1;
                *reinterpret_cast<uint32_t*>(sm.a_lo + o + 512) = l1;
            }
            fence_proxy_async();
            named_bar_sync(2 + wgi, 128);
        }
        // ---------------- last epilogue: raw layer-4 accumulators -> fp32 rows in shared memory -> K-reduction with lane = row
        named_bar_sync(1, hw::NTHR);                             // both warpgroups' layer-4 wgmma have completed
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            const int col = 8 * j + cq;
            *reinterpret_cast<float2*>(ybuf + r0 * hw::YLD + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
            *reinterpret_cast<float2*>(ybuf + (r0 + 8) * hw::YLD + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
        }
        named_bar_sync(1, hw::NTHR);
        {
            const int qd = warp & 3, half = warp >> 2, row = qd * 32 + lane;      // columns 128 half .. 128 half + 127 of the row
            const QuadRow qr = quad_row(sm.qhead[qd], (int)sm.qtotal[qd], lane);
            const int sidx = qr.live ? (int)p.vorder[sm.qfirst[qd] + qr.j] : 0;
            const bool swrite = qr.is_end && sidx < n_valid;
            const float wrow = sm.wc[row];
            const float* yr = ybuf + row * hw::YLD + 128 * half;
            float apart = 0.f;
#pragma unroll 1
            for (int i = 0; i < 8; ++i) {
                uint32_t v[16];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const uint4 u = *reinterpret_cast<const uint4*>(yr + 16 * i + 4 * e);
                    v[4 * e] = u.x; v[4 * e + 1] = u.y; v[4 * e + 2] = u.z; v[4 * e + 3] = u.w;
                }
                last_chunk_from_regs<O1>(p, 128 * half + 16 * i, v, wrow, qr.st, swrite, sidx, lane, apart);
            }
            sm.alpha_part[half][row] = apart;
            named_bar_sync(1, hw::NTHR);
            if (half == 0) {
                // sigma = softplus(alpha dot product - 1): order 2 per neighbour, weighted sum over the sample's rows; order 1: `a` is
                // already the sample's value (its last row).  The two column halves are added in a fixed order: deterministic.
                const float sp = softplus_m1((sm.alpha_part[0][row] + sm.alpha_part[1][row]) + __ldg(p.ba));
                const float zz = O1 ? sp : seg_scan8(sp * wrow, lane, qr.st);
                if (swrite) p.sigma[sidx] = zz;
            }
        }
    }
}

// =====================================================================================================================
// Colour branch: packed weight images of colour_branch.{0,2,4} and the kernel parameters.
namespace ctc {
constexpr int NBLK = 9 + 4 + 4;               // K blocks of the three layers
__host__ __device__ constexpr int nkb_of(int l) { return l == 0 ? 9 : 4; }
__host__ __device__ constexpr int img_base(int l) { return l == 0 ? 0 : l == 1 ? 9 : 13; }
}  // namespace ctc

struct ColorTcParams {
    pnb_query_t q;
    pnb_shade_opts_t o;
    const unsigned char* wimg;      // packed colour_branch.{0,2,4} images
    const float* bias[3];
    const float* w3t;               // colour_branch.6 W^T [128][3]
    const float* b3;
    const float* hbar;
    const float* sigma;
    int hbar_cap;
    float4* sigma_rgb;
    int* err;
    pnb_points_t pts;               // PP: the per-point frames of the view direction
};

// =====================================================================================================================
// k_color_wg: the colour branch per 128 consecutive valid samples.  The pair kernel writes h-bar already split into bf16 hi / lo
// and laid out as this kernel's A-operand blocks (per 128 samples 8 K blocks x {hi, lo} x [128 x 32], one contiguous 128 KB region),
// so the layer-1 operand is one bulk copy per tile; threads 0-127 add the PE(view) K block.  Two consumer warpgroups of 64 rows
// (wgmma N = 128), the same producer warpgroup, weight ring and in-place operand epilogues as k_shade_wg; the last layer
// (128 -> 3 + sigmoid) runs on CUDA cores straight from the accumulator fragments.
namespace hcw {
constexpr int NTHR = 256, NSTAGE = 4;         // consumer threads
constexpr int NTHR_CTA = NTHR + 128;          // + the producer warpgroup, as in k_shade_wg
constexpr uint32_t REGS_CONSUMER = hw::REGS_CONSUMER, REGS_PRODUCER = hw::REGS_PRODUCER;
constexpr int BLK = 128 * 64;                 // [128 x 32] bf16 block
constexpr int STEP = 2 * 128 * 32;            // hi + lo image ([128 x 16] bf16 each) of one K = 16 step
constexpr int TILE_BYTES = 8 * 2 * BLK;       // h-bar operand of one tile in global memory
constexpr uint32_t ST = 18 + 8 + 8;           // K = 16 steps per tile
struct Smem {
    unsigned char a[9][2][BLK];               // layer operand: K block, hi / lo (layer 1: blocks 0-7 h-bar, 8 PE(view))
    unsigned char b[NSTAGE][STEP];
    uint64_t bar_full[NSTAGE], bar_empty[NSTAGE], bar_a;
};
}  // namespace hcw

// PP: per-point frames (the view direction in the frame of each sample's slot-0 point); XSAMP: explicit samples (pair_inputs.cuh)
template <bool PP, bool XSAMP = false>
__global__ void __launch_bounds__(hcw::NTHR_CTA, 1) k_color_wg(ColorTcParams p) {
    using namespace hcw;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    Smem& sm = *reinterpret_cast<Smem*>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;
    const pnb_query_t& q = p.q;
    const int n_valid = min(q.counters[PNB_QC_N_VALID], p.hbar_cap);
    const int n_tiles = (n_valid + 127) / 128;
    const int my_tiles = n_tiles > (int)blockIdx.x ? (n_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    auto img_of = [](uint32_t m) { return m % ST; };
    Ring<NSTAGE, STEP, decltype(img_of)> ring{sm.b, sm.bar_full, sm.bar_empty, p.wimg, (uint32_t)my_tiles * ST, img_of, p.err};
    if (tid == 0) {
        ring.init();
        mbar_init(&sm.bar_a, 1);
        mbar_fence_init();
    }
    __syncthreads();
    if (wgi == 2) {                                              // producer warpgroup
        setmaxnreg_dec<REGS_PRODUCER>();
        if (tid == NTHR) ring.produce();
        return;
    }
    setmaxnreg_inc<REGS_CONSUMER>();

    const uint32_t a0 = smem_u32(sm.a[0][0]) + (uint32_t)wgi * 4096u, b0 = smem_u32(sm.b[0]);
    const int r0 = 64 * wgi + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
    uint32_t m = 0;
    bool ok = true;
    float acc[64];
    for (int t = 0; t < my_tiles; ++t) {
        const int tile = (int)blockIdx.x + t * (int)gridDim.x;
        named_bar_sync(1, NTHR);                                 // the previous tile's wgmma have completed in both warpgroups
        if (tid == 0) {
            mbar_arrive_expect_tx(&sm.bar_a, TILE_BYTES);
            const unsigned char* src = reinterpret_cast<const unsigned char*>(p.hbar) + (size_t)tile * TILE_BYTES;
#pragma unroll 1
            for (int c = 0; c < 8; ++c) bulk_g2s(sm.a[c][0], src + (size_t)c * 2 * BLK, 2 * BLK, &sm.bar_a);
        }
        if (tid < 128) {                                         // PE(view) K block, thread = sample row
            const int row = tid, vi = tile * 128 + row;
            float pe[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) pe[i] = 0.f;
            if (vi < n_valid) {
                const uint32_t s = q.valid_list[vi];
                const float3 v = view_in_points<PP>(p.pts, p.o, view_point<PP>(q, s), cand_view_dir<XSAMP>(q, s));
                const float ov[3] = {v.x, v.y, v.z};
#pragma unroll
                for (int d = 0; d < 3; ++d) {     // ori=True layout: sin block (d*4+j) then cos block
                    float sc[8];
                    pe_doubling<4>(ov[d], sc);
#pragma unroll
                    for (int j = 0; j < 4; ++j) { pe[d * 4 + j] = sc[2 * j]; pe[12 + d * 4 + j] = sc[2 * j + 1]; }
                }
            }
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                uint32_t h[4], l[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) split_bf16x2(pe[8 * c + 2 * i], pe[8 * c + 2 * i + 1], h[i], l[i]);
                const uint32_t off = tile_offset_bytes<tc::LAYOUT>(row, 8 * c);
                *reinterpret_cast<uint4*>(sm.a[8][0] + off) = make_uint4(h[0], h[1], h[2], h[3]);
                *reinterpret_cast<uint4*>(sm.a[8][1] + off) = make_uint4(l[0], l[1], l[2], l[3]);
            }
        }
        fence_proxy_async();
        ok = ok && mbar_wait(&sm.bar_a, (uint32_t)t & 1u, p.err, 84);
        named_bar_sync(1, NTHR);
        for (int l = 0; l < 3; ++l) {
            const int nst = l == 0 ? 18 : 8;
            wg::fence();
            for (int kk = 0; kk < nst; ++kk, ++m) {
                ok = ring.acquire(m, ok);
                const uint32_t bs = b0 + (m % NSTAGE) * (uint32_t)STEP;
                const uint64_t bh = desc_k16(bs), bl = desc_k16(bs + STEP / 2);
                const uint32_t off = (uint32_t)(kk >> 1) * 2u * BLK + (uint32_t)(kk & 1) * 256u;
                const uint64_t ah = desc_none(a0 + off), al = desc_none(a0 + off + BLK);
                mma_n128(acc, ah, bh, kk ? 1u : 0u);
                mma_n128(acc, al, bh, 1u);
                mma_n128(acc, ah, bl, 1u);
                wg::commit();
                wg::wait<1>();
                if (kk > 0) ring.release(m - 1);
            }
            wg::wait<0>();
            pin<64>(acc);
            ring.release(m - 1);
            const float* bias = p.bias[l];
            if (l < 2) {
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = 8 * j + cq;
                    const float2 u = __ldg(reinterpret_cast<const float2*>(bias + col));
                    float y0 = acc[4 * j] + u.x, y1 = acc[4 * j + 1] + u.y, y2 = acc[4 * j + 2] + u.x, y3 = acc[4 * j + 3] + u.y;
                    y0 = fmaxf(y0, tc::LEAKY * y0); y1 = fmaxf(y1, tc::LEAKY * y1); y2 = fmaxf(y2, tc::LEAKY * y2); y3 = fmaxf(y3, tc::LEAKY * y3);
                    uint32_t h0, l0, h1, l1;
                    split_bf16x2(y0, y1, h0, l0);
                    split_bf16x2(y2, y3, h1, l1);
                    unsigned char* blk = sm.a[col >> 5][0];
                    const uint32_t o = tile_offset_bytes<tc::LAYOUT>(r0, col & 31);      // row r0 + 8: + 512
                    *reinterpret_cast<uint32_t*>(blk + o) = h0;
                    *reinterpret_cast<uint32_t*>(blk + BLK + o) = l0;
                    *reinterpret_cast<uint32_t*>(blk + o + 512) = h1;
                    *reinterpret_cast<uint32_t*>(blk + BLK + o + 512) = l1;
                }
                fence_proxy_async();
                named_bar_sync(2 + wgi, 128);
            } else {
                // colour_branch.6 (128 -> 3) on CUDA cores: this thread's 32 columns of rows r0, r0 + 8, then the 4 lanes of a row
                // (fixed butterfly order)
                float d[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
                for (int j = 0; j < 16; ++j) {
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int c = 8 * j + cq + e;
                        const float bc = __ldg(bias + c);
                        const float* wr = p.w3t + c * 3;
                        const float w0 = __ldg(wr), w1 = __ldg(wr + 1), w2 = __ldg(wr + 2);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            float y = acc[4 * j + 2 * h + e] + bc;
                            y = fmaxf(y, tc::LEAKY * y);
                            d[h][0] = fmaf(y, w0, d[h][0]); d[h][1] = fmaf(y, w1, d[h][1]); d[h][2] = fmaf(y, w2, d[h][2]);
                        }
                    }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int o = 0; o < 3; ++o) {
                        d[h][o] += __shfl_xor_sync(0xffffffffu, d[h][o], 1);
                        d[h][o] += __shfl_xor_sync(0xffffffffu, d[h][o], 2);
                    }
                if ((lane & 3) == 0) {
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int vi = tile * 128 + r0 + 8 * h;
                        if (vi < n_valid) {
                            const uint32_t s = q.valid_list[vi];
                            float4 o4;
                            o4.x = p.sigma[vi];
                            o4.y = raw2out_color(d[h][0] + __ldg(p.b3));
                            o4.z = raw2out_color(d[h][1] + __ldg(p.b3 + 1));
                            o4.w = raw2out_color(d[h][2] + __ldg(p.b3 + 2));
                            p.sigma_rgb[s] = o4;
                        }
                    }
                }
            }
        }
    }
}

}  // namespace pnb

using namespace pnb;

static size_t pack_pairs_bytes(int F) { return (size_t)tc::nblk_total(F) * 2 * tc::STEP; }
static size_t pack_color_bytes() { return (size_t)ctc::NBLK * 2 * hcw::STEP; }
extern "C" size_t pnb_mlp_pack_bytes(int feat_dim) {
    const int F = feat_of(feat_dim);
    return F > 0 ? pack_pairs_bytes(F) + pack_color_bytes() : 0;
}

// Packs block1/block3 and colour_branch.{0,2,4} weights (pnb_mlp_t W^T buffers, fp32) into wgmma operand images, one hi + lo
// pair per K = 16 step.  Call once per weight version.
extern "C" int pnb_mlp_pack(const pnb_mlp_t* mlp, void* d_out, size_t out_bytes, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(mlp && d_out, PNB_ERR_INVALID, "pnb_mlp_pack: null argument");
    const int F = feat_of(mlp->feat_dim);
    PNB_REQUIRE(F > 0, PNB_ERR_UNSUPPORTED, "pnb_mlp_pack: point_features_dim %d unsupported (32 or 63)", (int)mlp->feat_dim);
    PNB_REQUIRE(out_bytes >= pnb_mlp_pack_bytes(F), PNB_ERR_WORKSPACE, "pnb_mlp_pack: buffer too small");
    const int kpad[4] = {kpad1_of(F), 256, 272, 256};
    for (int l = 0; l < 4; ++l) {
        const int nks = 2 * tc::nkb_of(l, F), n = nks * 256 * 16;
        unsigned char* dst = (unsigned char*)d_out + (size_t)tc::img_base(l, F) * 2 * tc::STEP;
        if (l == 0 && F != PNB_FEAT) k_pack_block1_f63<<<(n + 255) / 256, 256, 0, stream>>>(mlp->w[0], nks, 256, dst);
        else k_pack_weights<<<(n + 255) / 256, 256, 0, stream>>>(mlp->w[l], kpad[l], nks, 256, dst);
    }
    const int ckpad[3] = {288, 128, 128};   // colour_branch.{0,2,4}: W^T [K_pad][128]
    for (int l = 0; l < 3; ++l) {
        const int nks = 2 * ctc::nkb_of(l), n = nks * 128 * 16;
        k_pack_weights<<<(n + 255) / 256, 256, 0, stream>>>(mlp->w[5 + l], ckpad[l], nks, 128,
                                                            (unsigned char*)d_out + pack_pairs_bytes(F) + (size_t)ctc::img_base(l) * 2 * hcw::STEP);
    }
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

// Hoisted layer-1 table of a frozen point cloud (k_point_pre): d_pre [N][256] fp32.
extern "C" size_t pnb_point_pre_bytes(int N) { return (size_t)(N > 0 ? N : 0) * 256 * sizeof(float); }
extern "C" int pnb_point_pre(const pnb_points_t* pts, const pnb_mlp_t* mlp, float* d_pre, size_t pre_bytes, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(pts && mlp && d_pre, PNB_ERR_INVALID, "pnb_point_pre: null argument");
    PNB_REQUIRE(pre_bytes >= pnb_point_pre_bytes(pts->N), PNB_ERR_WORKSPACE, "pnb_point_pre: buffer too small");
    Variant v;
    { const int rc = resolve_variant("pnb_point_pre", pts, mlp, nullptr, XsRule::none, &v); if (rc) return rc; }
    const int np = point_pre_np(v.F);
    const auto kern = with_feat(v.F, [](auto F) { return k_point_pre<F>; });
    if (pts->N > 0) kern<<<(pts->N + np - 1) / np, 256, 0, stream>>>(pts->emb, pts->N, mlp->w[0], mlp->b[0], d_pre);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

static size_t pack_sc_max(int cap) { return (size_t)cap / pk::PACK_S + 3; }
namespace {
struct TcWs {   // carve-up of the caller's workspace (all sizes from max_valid_samples; the kernels read the live counts on the device)
    float* hbar; float* sigma; uint32_t* sc_quads; uint32_t* quad_local; uint32_t* quad_first; uint32_t* vorder; unsigned char* vcntp; int* pack_cnt;
    TcWs(void* ws, size_t ws_bytes, int cap) {
        Carver c(ws, ws_bytes);
        hbar = c.take<float>(((size_t)cap + 127) / 128 * 128 * 256);   // whole 128-sample colour tiles
        sigma = c.take<float>((size_t)cap);
        sc_quads = c.take<uint32_t>(pack_sc_max(cap));
        quad_local = c.take<uint32_t>((size_t)cap + 2);
        quad_first = c.take<uint32_t>((size_t)cap + 2);
        vorder = c.take<uint32_t>((size_t)cap + 2);
        vcntp = c.take<unsigned char>((size_t)cap + 16);
        pack_cnt = c.take<int>(4);
    }
};
}  // namespace
extern "C" size_t pnb_shade_tc_bytes(int max_valid_samples) {
    const size_t cap = (size_t)max_valid_samples;
    return align_up((cap + 127) / 128 * 128 * 256 * sizeof(float)) + align_up(cap * sizeof(float)) + align_up(pack_sc_max(max_valid_samples) * 4) +
           3 * align_up((cap + 2) * 4) + align_up(cap + 16) + align_up(16) + 256;
}
// diagnostics / tests: device pointers of the row-packing tables inside a workspace laid out for max_valid_samples
extern "C" int pnb_shade_tc_tables(void* ws, size_t ws_bytes, int max_valid_samples, void** vorder, void** vcntp, void** quad_first, void** pack_cnt) {
    PNB_REQUIRE(ws && ws_bytes >= pnb_shade_tc_bytes(max_valid_samples), PNB_ERR_WORKSPACE, "pnb_shade_tc_tables: workspace too small");
    TcWs w(ws, ws_bytes, max_valid_samples);
    if (vorder) *vorder = w.vorder;
    if (vcntp) *vcntp = w.vcntp;
    if (quad_first) *quad_first = w.quad_first;
    if (pack_cnt) *pack_cnt = w.pack_cnt;
    return PNB_OK;
}
// tests: device pointers of the pair kernel's products inside a workspace laid out for max_valid_samples (h-bar operand blocks, sigma)
extern "C" int pnb_shade_tc_buffers(void* ws, size_t ws_bytes, int max_valid_samples, void** hbar, void** sigma) {
    PNB_REQUIRE(ws && ws_bytes >= pnb_shade_tc_bytes(max_valid_samples), PNB_ERR_WORKSPACE, "pnb_shade_tc_buffers: workspace too small");
    TcWs w(ws, ws_bytes, max_valid_samples);
    if (hbar) *hbar = w.hbar;
    if (sigma) *sigma = w.sigma;
    return PNB_OK;
}

// Tensor-core forward: row packing, per-pair MLPs and colour branch on wgmma (BF16x3).  ws: >= pnb_shade_tc_bytes.
extern "C" int pnb_shade_forward_tc(const pnb_query_t* q, const pnb_points_t* pts, const pnb_mlp_t* mlp, const void* d_packed,
                                    const float* d_point_pre, const pnb_shade_opts_t* opts, float* d_sigma_rgb, void* ws, size_t ws_bytes,
                                    int max_valid_samples, int flags, int* d_err, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && pts && mlp && d_packed && opts && d_sigma_rgb && ws && d_err, PNB_ERR_INVALID, "pnb_shade_forward_tc: null argument");
    PNB_REQUIRE(q->K >= 1 && q->K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED, "pnb_shade_forward_tc: K=%d unsupported", q->K);
    PNB_REQUIRE(max_valid_samples > 0, PNB_ERR_INVALID, "pnb_shade_forward_tc: max_valid_samples must be positive");
    PNB_REQUIRE(ws_bytes >= pnb_shade_tc_bytes(max_valid_samples), PNB_ERR_WORKSPACE, "pnb_shade_forward_tc: workspace too small");
    const bool frozen = (flags & PNB_TC_FROZEN) != 0;
    PNB_REQUIRE(!frozen || d_point_pre, PNB_ERR_INVALID, "pnb_shade_forward_tc: PNB_TC_FROZEN needs the table of pnb_point_pre");
    Variant v;
    { const int rc = resolve_variant("pnb_shade_forward_tc", pts, mlp, q, XsRule::frames, &v); if (rc) return rc; }
    // interleaved (non-swizzled) operand layout: 128-byte alignment of the carve-out is sufficient
    constexpr size_t kSmemMax = 232448;   // 227 KB opt-in limit per block on sm_90
    const size_t smem_pair = sizeof(hw::Smem) + 128, smem_color = sizeof(hcw::Smem) + 128;
    static_assert(sizeof(hw::Smem) + 128 <= kSmemMax, "pair kernel shared-memory carve-out exceeds the per-block limit");
    static_assert(sizeof(hcw::Smem) + 128 <= kSmemMax, "colour kernel shared-memory carve-out exceeds the per-block limit");
    // PNB_TC_FEW_CTAS (test of the persistent tile loop): one CTA per 8 SMs, so every CTA runs many tiles
    const auto ctas = [flags](int n_sm) { return (flags & PNB_TC_FEW_CTAS) ? (n_sm + 7) / 8 : n_sm; };
    TcWs w(ws, ws_bytes, max_valid_samples);
    ShadeTcParams p;
    p.q = *q; p.pts = *pts; p.o = *opts; p.wimg = (const unsigned char*)d_packed;
    for (int l = 0; l < 4; ++l) p.bias[l] = mlp->b[l];
    p.wa = mlp->w[4];
    p.ba = mlp->b[4];
    p.hbar = w.hbar; p.sigma = w.sigma; p.hbar_cap = max_valid_samples; p.err = d_err;
    p.vcnt = w.vcntp; p.vorder = w.vorder; p.quad_first = w.quad_first; p.pack_cnt = w.pack_cnt;
    p.pre = d_point_pre;
    if (flags & PNB_TC_PAIRS) {
        const auto kern = with_bool(frozen, [&](auto FROZEN) {
            return with_bool(opts->agg_intrp_order == 1, [&](auto O1) {
                return with_frames(v, [&](auto PP, auto F, auto XS) { return k_shade_wg<FROZEN, O1, PP, F, XS>; });
            });
        });
        int n_sm = 0;
        { const int rc = prepare_launch((const void*)kern, smem_pair, &n_sm, "pnb_shade_forward_tc"); if (rc) return rc; }
        const int cap = max_valid_samples, n_sc = (int)pack_sc_max(cap);
        k_pack_quads<<<(n_sc + 7) / 8, 256, 0, stream>>>(p.q, cap, w.sc_quads, w.quad_local, w.vorder, w.vcntp, (float4*)d_sigma_rgb);
        k_pack_scan<<<1, 1024, 0, stream>>>(p.q, cap, w.sc_quads, w.quad_first, w.pack_cnt);
        k_pack_place<<<(cap + 255) / 256, 256, 0, stream>>>(p.q, cap, w.sc_quads, w.quad_local, w.quad_first);
        kern<<<ctas(n_sm), hw::NTHR_CTA, smem_pair, stream>>>(p);
    }
    if (flags & PNB_TC_COLOR) {
        ColorTcParams ct;
        ct.q = *q; ct.o = *opts; ct.wimg = (const unsigned char*)d_packed + pack_pairs_bytes(v.F);
        for (int i = 0; i < 3; ++i) ct.bias[i] = mlp->b[5 + i];
        ct.w3t = mlp->w[8]; ct.b3 = mlp->b[8];
        ct.hbar = w.hbar; ct.sigma = w.sigma; ct.hbar_cap = max_valid_samples; ct.sigma_rgb = (float4*)d_sigma_rgb; ct.err = d_err;
        ct.pts = *pts;
        const auto kern = with_frames(v, [](auto PP, auto F, auto XS) { return k_color_wg<PP, XS>; });
        int n_sm = 0;
        { const int rc = prepare_launch((const void*)kern, smem_color, &n_sm, "pnb_shade_forward_tc"); if (rc) return rc; }
        kern<<<ctas(n_sm), hcw::NTHR_CTA, smem_color, stream>>>(ct);
    }
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
