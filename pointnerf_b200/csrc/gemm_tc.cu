// Generic fp32-in / fp32-out GEMM on the Hopper tensor cores (wgmma) with the BF16x3 error-compensated split of shade_tc.cu --
// the GEMM engine of the BACKWARD pass (backward.cu): forward recompute, dX = dZ . W and dW = X^T . dZ.
//
//   C[M x N] = op( sum_k A(m,k) * B(n,k) + bias[n] )        A(m,k) = A[m*a_rs + k*a_ks],  B(n,k) = B[n*b_rs + k*b_ks]
//
// Either stride of an operand may be the unit one: operands whose reduction index is NOT contiguous in memory (W^T buffers,
// the activations of dW = X^T dZ) are transposed on the way into shared memory, so the tensor cores only ever see the K-major
// core-matrix layout of wgmma.cuh (tests/test_gpu_umma.py).  One CTA = one 128 x 128 output tile, two warpgroups of 64 rows each
// (wgmma M = 64, N = 128, fp32 accumulators in registers), K blocks of 32 through a 2-stage shared-memory ring:
//   warps 0-3  load the fp32 rows of A, split into bf16 hi / lo and store them in the operand layout; the next K block is already in
//              registers while the current one is converted.  Lane mapping of a K block of 32 rows x 32 k per warp:
//                * reduction index contiguous (ks == 1): load i of 8, lane l -> row 8(i/2) + (l/2)%8, floats 16(i%2) + 8(l/16) + 4(l%2) .. +3:
//                  8 lines per LDG.128 (thread = row would touch 32 lines per request), and the 8-byte stores of a half warp fill one
//                  128-byte run of the core-matrix layout;
//                * row index contiguous (transposing operands): thread = row, one coalesced LDG.32 per k
//   warps 4-7  the same for the rows of B
//   all warps  then issue the wgmma of the block (A_hi B_hi, A_lo B_hi, A_hi B_lo for the two K = 16 steps; one group in flight)
//              and finally run the epilogue from their accumulator fragments
// PRECISE mode (forward recompute only): three bf16 parts per operand and the six products of total order <= 2 (a0b0, a1b0, a0b1,
// a2b0, a1b1, a0b2): fp32-level pre-activations, so that the LeakyReLU masks of the backward are those of an fp32 forward (with the
// BF16x3 recompute ~1e-5 of the units land on the other side of zero and each such flip changes a pair's gradient by ~1/256).
// Split-K (dW: the reduction runs over the ~1e5 pair rows of a training batch): blockIdx.z owns a K range and writes its partial
// tile to a workspace; k_splitk_reduce adds the partials in split order (deterministic, no atomics).
#include "common.cuh"
#include "gemm_tc.cuh"
#include "wgmma.cuh"

namespace pnb {
using namespace wg;

namespace gtc {
constexpr int TM = 128, TN = 128, NSTAGE = 2;
constexpr int BLK = 128 * 64;             // [128 x 32] bf16 block
constexpr int NTHR = 256;                 // warps 0-3: A loaders, 4-7: B loaders; two wgmma warpgroups of 64 rows
template <int NPART>
struct Smem {
    unsigned char a[NPART][NSTAGE][BLK], b[NPART][NSTAGE][BLK];     // part 0 = hi, 1 = lo (mid), 2 = lo of the 3-part split
};
// One K block (32 rows x 32 k of one loader warp) of an operand into registers / from registers into the NPART bf16 blocks of stage s.
// COOP (ks == 1): v[4 i + c] = P(row 8(i/2) + (lane/2)%8, k0 + 16(i%2) + 8(lane/16) + 4(lane%2) + c); else v[e] = P(row lane, k0 + e).
// w = first tile row of the warp (32 * loader warp), R0 = first global row of the tile, nrows = rows of the operand.
template <bool COOP>
__device__ __forceinline__ void fetch_blk(const float* __restrict__ P, long rs, long ks, long R0, int w, int lane, long nrows, int k0, int kend, float* v) {
    if (COOP) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const long r = R0 + w + 8 * (i >> 1) + ((lane >> 1) & 7);
            const int k = k0 + 16 * (i & 1) + 8 * (lane >> 4) + 4 * (lane & 1);
            if (r < nrows && k + 4 <= kend) {
                const float4 x = __ldg(reinterpret_cast<const float4*>(P + r * rs + k));
                v[4 * i] = x.x; v[4 * i + 1] = x.y; v[4 * i + 2] = x.z; v[4 * i + 3] = x.w;
            } else {
#pragma unroll
                for (int c = 0; c < 4; ++c) v[4 * i + c] = (r < nrows && k + c < kend) ? __ldg(P + r * rs + k + c) : 0.f;
            }
        }
    } else {
        const long r = R0 + w + lane;
#pragma unroll
        for (int e = 0; e < 32; ++e) v[e] = (r < nrows && k0 + e < kend) ? __ldg(P + r * rs + (long)(k0 + e) * ks) : 0.f;
    }
}
template <int NPART, bool COOP>
__device__ __forceinline__ void store_blk(float* v, unsigned char (*blk)[NSTAGE][BLK], int s, int w, int lane) {
    if (COOP) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int t = w + 8 * (i >> 1) + ((lane >> 1) & 7);
            const uint32_t off = tile_offset_bytes<LAYOUT_NONE>(t, 16 * (i & 1) + 8 * (lane >> 4)) + 8u * (uint32_t)(lane & 1);
#pragma unroll
            for (int part = 0; part < NPART; ++part) {
                uint32_t ww[2];
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const __nv_bfloat162 h = __floats2bfloat162_rn(v[4 * i + 2 * c], v[4 * i + 2 * c + 1]);
                    v[4 * i + 2 * c] -= __low2float(h); v[4 * i + 2 * c + 1] -= __high2float(h);      // the residual feeds the next part
                    ww[c] = *reinterpret_cast<const uint32_t*>(&h);
                }
                *reinterpret_cast<uint2*>(blk[part][s] + off) = make_uint2(ww[0], ww[1]);
            }
        }
    } else {
        const int t = w + lane;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const uint32_t off = tile_offset_bytes<LAYOUT_NONE>(t, 8 * c);
#pragma unroll
            for (int part = 0; part < NPART; ++part) {
                uint32_t ww[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const __nv_bfloat162 h = __floats2bfloat162_rn(v[8 * c + 2 * i], v[8 * c + 2 * i + 1]);
                    v[8 * c + 2 * i] -= __low2float(h); v[8 * c + 2 * i + 1] -= __high2float(h);
                    ww[i] = *reinterpret_cast<const uint32_t*>(&h);
                }
                *reinterpret_cast<uint4*>(blk[part][s] + off) = make_uint4(ww[0], ww[1], ww[2], ww[3]);
            }
        }
    }
}
}  // namespace gtc

template <bool PRECISE>
__global__ void __launch_bounds__(gtc::NTHR, 1) k_gemm_tc(GemmTc g) {
    using namespace gtc;
    constexpr int NPART = PRECISE ? 3 : 2;
    using SmemT = Smem<NPART>;
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    SmemT& sm = *reinterpret_cast<SmemT*>(smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u));
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;
    const int m0 = blockIdx.y * TM, n0 = blockIdx.x * TN;
    const int kbeg = blockIdx.z * g.kchunk, kend = min(g.K, kbeg + g.kchunk);
    const int nkb = (kend - kbeg + 31) >> 5;

    // loaders: warps 0-3 own the A rows, warps 4-7 the B rows (32 rows per warp); the NEXT K block is fetched into registers before
    // the current one is converted and stored, so a full K block of loads is in flight per thread
    const bool isB = warp >= 4;
    const float* P = isB ? g.B : g.A;
    const long rs = isB ? g.b_rs : g.a_rs, ks = isB ? g.b_ks : g.a_ks;
    const long R0 = isB ? n0 : m0, nrows = isB ? g.N : g.M;
    const int w32 = (tid & 127) & ~31;
    const bool coop = ks == 1;
    unsigned char (*blk)[NSTAGE][BLK] = isB ? sm.b : sm.a;
    float cur[32], nxt[32];
    if (coop) fetch_blk<true>(P, rs, ks, R0, w32, lane, nrows, kbeg, kend, cur);
    else fetch_blk<false>(P, rs, ks, R0, w32, lane, nrows, kbeg, kend, cur);

    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    const uint32_t a0 = smem_u32(sm.a[0][0]) + (uint32_t)wgi * 4096u, b0 = smem_u32(sm.b[0][0]);
    constexpr uint32_t PART = NSTAGE * BLK;                  // byte distance between the parts of an operand
    for (int kb = 0; kb < nkb; ++kb) {
        const int s = kb & (NSTAGE - 1);
        if (kb + 1 < nkb) {
            if (coop) fetch_blk<true>(P, rs, ks, R0, w32, lane, nrows, kbeg + 32 * (kb + 1), kend, nxt);
            else fetch_blk<false>(P, rs, ks, R0, w32, lane, nrows, kbeg + 32 * (kb + 1), kend, nxt);
        }
        named_bar_sync(1, NTHR);                     // both warpgroups have retired the wgmma group of block kb - 2 (stage s)
        if (coop) store_blk<NPART, true>(cur, blk, s, w32, lane);
        else store_blk<NPART, false>(cur, blk, s, w32, lane);
        fence_proxy_async();
        named_bar_sync(1, NTHR);
        wg::fence();
#pragma unroll
        for (int i = 0; i < NPART; ++i)
#pragma unroll
            for (int j = 0; j < NPART; ++j) {
                if (i + j >= NPART) continue;          // products of total order < NPART: 3 (BF16x3) or 6 (3-part split)
                const uint32_t ad = a0 + (uint32_t)i * PART + (uint32_t)s * BLK, bd = b0 + (uint32_t)j * PART + (uint32_t)s * BLK;
                mma_n128(acc, desc_none(ad), desc_none(bd), (kb > 0 || i + j > 0) ? 1u : 0u);
                mma_n128(acc, desc_none(ad + 256u), desc_none(bd + 256u), 1u);
            }
        wg::commit();
        wg::wait<1>();
#pragma unroll
        for (int e = 0; e < 32; ++e) cur[e] = nxt[e];
    }
    wg::wait<0>();
    pin<64>(acc);
    if (nkb == 0) return;
    // ---------------- epilogue from the accumulator fragments: rows r0, r0 + 8, columns n0 + 8j + cq, +1
    const long r0 = (long)m0 + 64 * wgi + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const long ra = r0 + 8 * h;
        if (ra >= g.M) continue;
        float* crow = g.part ? g.part + ((size_t)blockIdx.z * g.M + (size_t)ra) * g.N : g.C + ra * g.ldc;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            const int n = n0 + 8 * j + cq;
            if (n >= g.N) continue;
            float y0 = acc[4 * j + 2 * h], y1 = acc[4 * j + 2 * h + 1];
            if (!g.part) {
                if (g.bias) { y0 += __ldg(g.bias + n); y1 += __ldg(g.bias + n + 1); }
                if (g.act) { y0 = fmaxf(y0, 0.01f * y0); y1 = fmaxf(y1, 0.01f * y1); }
                if (g.dact && n < g.dact_n) {            // backward of the LeakyReLU below: * (Y > 0 ? 1 : 0.01)
                    const float2 yy = __ldg(reinterpret_cast<const float2*>(g.dact + ra * g.ldd + n));
                    y0 *= yy.x > 0.f ? 1.0f : 0.01f; y1 *= yy.y > 0.f ? 1.0f : 0.01f;
                }
            }
            *reinterpret_cast<float2*>(crow + n) = make_float2(y0, y1);
        }
    }
}

// C[m][n] (+)= sum_z part[z][m][n], z ascending
__global__ void __launch_bounds__(256) k_splitk_reduce(const float* __restrict__ part, int splits, int M, int N, float* __restrict__ C, long ldc, int accumulate) {
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)M * N) return;
    const int m = (int)(i / N), n = (int)(i - (long)m * N);
    float s = accumulate ? C[m * ldc + n] : 0.f;
    for (int z = 0; z < splits; ++z) s += part[(size_t)z * M * N + i];
    C[m * ldc + n] = s;
}

int gemm_tc(const GemmTc& g0, int splits, float* part_ws, size_t part_bytes, int accumulate, cudaStream_t st) {
    GemmTc g = g0;
    if (g.M <= 0 || g.N <= 0 || g.K <= 0) return PNB_OK;
    PNB_REQUIRE(g.N % 16 == 0 && g.ldc % 4 == 0, PNB_ERR_INVALID, "gemm_tc: N (%d) must be a multiple of 16 and ldc (%ld) of 4", g.N, g.ldc);
    PNB_REQUIRE((g.a_rs == 1) != (g.a_ks == 1) || g.K == 1 || g.M == 1, PNB_ERR_INVALID, "gemm_tc: one stride of A must be 1");
    PNB_REQUIRE(g.a_ks != 1 || g.a_rs % 4 == 0, PNB_ERR_INVALID, "gemm_tc: leading dimension of A must be a multiple of 4");
    PNB_REQUIRE(g.b_ks != 1 || g.b_rs % 4 == 0, PNB_ERR_INVALID, "gemm_tc: leading dimension of B must be a multiple of 4");
    PNB_REQUIRE(g.dact == nullptr || g.ldd % 2 == 0, PNB_ERR_INVALID, "gemm_tc: leading dimension of dact must be even");
    const bool precise = g.precise != 0;
    const size_t smem = (precise ? sizeof(gtc::Smem<3>) : sizeof(gtc::Smem<2>)) + 128;
    static_assert(sizeof(gtc::Smem<3>) + 128 <= 232448, "precise GEMM tile exceeds the shared memory of an SM");
    const auto kern = with_bool(precise, [](auto PRECISE) { return k_gemm_tc<PRECISE>; });
    { const int rc = prepare_launch((const void*)kern, smem, nullptr, "gemm_tc"); if (rc) return rc; }
    if (splits <= 1) {
        g.kchunk = g.K; g.part = nullptr;
        dim3 grid((g.N + gtc::TN - 1) / gtc::TN, (g.M + gtc::TM - 1) / gtc::TM, 1);
        PNB_REQUIRE(!accumulate, PNB_ERR_INVALID, "gemm_tc: accumulation needs the split-K path");
        kern<<<grid, gtc::NTHR, smem, st>>>(g);
    } else {
        int kchunk = ((g.K + splits - 1) / splits + 31) / 32 * 32;
        splits = (g.K + kchunk - 1) / kchunk;
        PNB_REQUIRE(part_ws && part_bytes >= (size_t)splits * g.M * g.N * sizeof(float), PNB_ERR_WORKSPACE, "gemm_tc: split-K workspace too small");
        g.kchunk = kchunk; g.part = part_ws;
        dim3 grid((g.N + gtc::TN - 1) / gtc::TN, (g.M + gtc::TM - 1) / gtc::TM, splits);
        kern<<<grid, gtc::NTHR, smem, st>>>(g);
        const long n = (long)g.M * g.N;
        k_splitk_reduce<<<(int)((n + 255) / 256), 256, 0, st>>>(part_ws, splits, g.M, g.N, g.C, g.ldc, accumulate);
    }
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

}  // namespace pnb
