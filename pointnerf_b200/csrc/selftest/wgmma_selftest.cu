// Self-test of the wgmma building blocks used by the fused shading kernels: one CTA (two warpgroups of 64 rows) computes
//   D[128 x N] = A[128 x K] * W[N x K]^T    with the BF16x3 error-compensated split
//   (A_hi*W_hi + A_lo*W_hi + A_hi*W_lo, fp32 accumulation in registers)
// from fp32 inputs, operands staged in shared memory in the selected K-major layout (W zero padded to 256 rows: one wgmma N).
// tests/test_gpu_umma.py compares D against an fp64 matmul: this pins descriptors, layouts, the accumulator fragment and the
// split accuracy on the real hardware before the big kernels depend on them.  Two more forms of the same product: the A operand
// from registers (wgmma "RS", optionally mixed with a shared-memory K step) and a cluster of two CTAs (M = 256) in which each CTA
// converts half of B and writes it into both CTAs' shared memory (distributed shared memory, cluster barriers).
//
// TEST-ONLY library (libpnb200_selftest.so): these entry points are not part of the product ABI (include/pnb200.h); they are
// declared in pnb200_selftest.h next to this file and used by tests/test_gpu_umma.py.
#include <stdarg.h>

#include "../common.cuh"
#include "../wgmma.cuh"
#include "pnb200_selftest.h"

namespace pnb {
static thread_local char g_selftest_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_selftest_err, sizeof(g_selftest_err), fmt, ap);
    va_end(ap);
}
}  // namespace pnb
extern "C" const char* pnb_selftest_last_error(void) { return pnb::g_selftest_err; }

namespace pnb {
using namespace wg;

template <int LAYOUT>
__device__ __forceinline__ uint64_t op_desc(uint32_t addr) { return LAYOUT == LAYOUT_NONE ? desc_none(addr) : desc_sw64(addr); }
template <int LAYOUT>
__device__ __forceinline__ uint32_t kstep_bytes(int ks) { return LAYOUT == LAYOUT_NONE ? (uint32_t)ks * 256u : (uint32_t)ks * 32u; }

template <int LAYOUT>
__global__ void __launch_bounds__(256, 1) k_umma_selftest(const float* __restrict__ A, const float* __restrict__ W,
                                                          float* __restrict__ D, int K, int N) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // swizzle atoms need 1 KB alignment
    // A_hi | A_lo : nkb blocks of [128 x 32] (8 KB each);  B_hi | B_lo : one block of [256 x 32] (16 KB each)
    const int nkb = (K + BK - 1) / BK;
    unsigned char* a_hi = smem;
    unsigned char* a_lo = a_hi + nkb * 8192;
    unsigned char* b_hi = a_lo + nkb * 8192;
    unsigned char* b_lo = b_hi + 256 * 64;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;

    for (int i = tid; i < 128 * nkb * BK; i += 256) {          // stage A (all K blocks)
        const int r = i / (nkb * BK), k = i - r * (nkb * BK);
        const float v = k < K ? A[(size_t)r * K + k] : 0.f;
        __nv_bfloat16 h, l;
        split_bf16(v, h, l);
        const uint32_t off = (uint32_t)(k / BK) * 8192u + tile_offset_bytes<LAYOUT>(r, k % BK);
        *(__nv_bfloat16*)(a_hi + off) = h;
        *(__nv_bfloat16*)(a_lo + off) = l;
    }
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    const uint32_t arow = (uint32_t)wgi * 64u * 64u;            // this warpgroup's 64 rows (64 bytes per row in both layouts)
    for (int kb = 0; kb < nkb; ++kb) {
        for (int i = tid; i < 256 * BK; i += 256) {
            const int n = i / BK, k = i - n * BK, kg = kb * BK + k;
            const float v = (n < N && kg < K) ? W[(size_t)n * K + kg] : 0.f;
            __nv_bfloat16 h, l;
            split_bf16(v, h, l);
            const uint32_t off = tile_offset_bytes<LAYOUT>(n, k);
            *(__nv_bfloat16*)(b_hi + off) = h;
            *(__nv_bfloat16*)(b_lo + off) = l;
        }
        fence_proxy_async();
        __syncthreads();
        wg::fence();
        const int nks = (min(K - kb * BK, BK) + 15) / 16;
        for (int ks = 0; ks < nks; ++ks) {
            const uint32_t adv = kstep_bytes<LAYOUT>(ks);
            const uint64_t dah = op_desc<LAYOUT>(smem_u32(a_hi + kb * 8192) + arow + adv);
            const uint64_t dal = op_desc<LAYOUT>(smem_u32(a_lo + kb * 8192) + arow + adv);
            const uint64_t dbh = op_desc<LAYOUT>(smem_u32(b_hi) + adv), dbl = op_desc<LAYOUT>(smem_u32(b_lo) + adv);
            mma_n256(acc, dah, dbh, 1u);
            mma_n256(acc, dal, dbh, 1u);
            mma_n256(acc, dah, dbl, 1u);
        }
        wg::commit();
        wg::wait<0>();                                           // everyone's wgmma of this block are done before B is overwritten
        pin<128>(acc);
        __syncthreads();
    }
    const int r0 = 64 * wgi + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 32; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int r = r0 + 8 * (e >> 1), n = 8 * j + cq + (e & 1);
            if (n < N) D[(size_t)r * N + n] = acc[4 * j + e];
        }
}

// D[64 x 256] (+)= A[64 x 16] * B[256 x 16]^T with A from REGISTERS (the "RS" form): per warp of the warpgroup its 16 rows in the
// mma.m16n8k16 A-fragment layout (a[0] = row l/4, k 2(l%4) + {0,1}; a[1] = row + 8; a[2], a[3] = the same at k + 8).
__device__ __forceinline__ void mma_n256_rs(float* d, const uint32_t* a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %133, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, {%128, %129, %130, %131}, %132, p, 1, 1, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(accumulate));
}

// ---- A operand in registers (RS form) and a cluster of two CTAs sharing B through distributed shared memory ---------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// shared::cluster address of the same variable in CTA `rank` of the cluster
__device__ __forceinline__ uint32_t map_to_cta(const void* local_smem, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(local_smem)), "r"(rank));
    return r;
}
__device__ __forceinline__ void st_cluster_b16(uint32_t addr, __nv_bfloat16 v) {
    asm volatile("st.shared::cluster.b16 [%0], %1;" ::"r"(addr), "h"(__bfloat16_as_ushort(v)) : "memory");
}

// D[128 x N] = A[128 x K] * W[N x K]^T (BF16x3) per CTA, operands in the interleaved layout, W zero padded to 256 rows.
// A_REGS: the first K - 16*ss_tail columns of A reach the tensor cores from registers (fragments loaded and split per K step); the
// last K step comes from shared memory when ss_tail (both forms on one accumulator).  CLUSTER: two CTAs (rows 0..127 | 128..255 of A
// and D); CTA r converts rows 128r .. 128r+127 of the padded W block and stores them into its own AND its peer's shared memory.
template <bool A_REGS, bool CLUSTER>
__global__ void __launch_bounds__(256, 1) k_wgmma_selftest_x(const float* __restrict__ A, const float* __restrict__ W,
                                                             float* __restrict__ D, int K, int N, int ss_tail) {
    extern __shared__ __align__(1024) unsigned char smem_raw[];
    unsigned char* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int nkb = (K + BK - 1) / BK;
    unsigned char* a_hi = smem;
    unsigned char* a_lo = a_hi + nkb * 8192;
    unsigned char* b_hi = a_lo + nkb * 8192;
    unsigned char* b_lo = b_hi + 256 * 64;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;
    const uint32_t rank = CLUSTER ? cluster_ctarank() : 0u, peer = rank ^ 1u;
    A += (size_t)rank * 128 * K;
    D += (size_t)rank * 128 * N;
    const int k_regs = A_REGS ? K - 16 * ss_tail : 0;          // K columns served from registers

    for (int i = tid; i < 128 * nkb * BK; i += 256) {          // A -> shared memory (used by the SS steps)
        const int r = i / (nkb * BK), k = i - r * (nkb * BK);
        const float v = k < K ? A[(size_t)r * K + k] : 0.f;
        __nv_bfloat16 h, l;
        split_bf16(v, h, l);
        const uint32_t off = (uint32_t)(k / BK) * 8192u + tile_offset_bytes<LAYOUT_NONE>(r, k % BK);
        *(__nv_bfloat16*)(a_hi + off) = h;
        *(__nv_bfloat16*)(a_lo + off) = l;
    }
    float acc[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) acc[i] = 0.f;
    const int g = lane >> 2, q = lane & 3, fr = 64 * wgi + 16 * (warp & 3) + g;      // fragment rows fr, fr + 8
    const int n_lo = CLUSTER ? 128 * (int)rank : 0, n_cnt = CLUSTER ? 128 : 256;
    for (int kb = 0; kb < nkb; ++kb) {
        if (CLUSTER) cluster_sync_all();                       // both CTAs' wgmma of the previous block have completed
        else __syncthreads();
        for (int i = tid; i < n_cnt * BK; i += 256) {
            const int n = n_lo + i / BK, k = i % BK, kg = kb * BK + k;
            const float v = (n < N && kg < K) ? W[(size_t)n * K + kg] : 0.f;
            __nv_bfloat16 h, l;
            split_bf16(v, h, l);
            const uint32_t off = tile_offset_bytes<LAYOUT_NONE>(n, k);
            *(__nv_bfloat16*)(b_hi + off) = h;
            *(__nv_bfloat16*)(b_lo + off) = l;
            if (CLUSTER) {
                st_cluster_b16(map_to_cta(b_hi + off, peer), h);
                st_cluster_b16(map_to_cta(b_lo + off, peer), l);
            }
        }
        asm volatile("fence.proxy.async;" ::: "memory");        // generic-proxy stores (own and peer's) -> wgmma operand reads
        if (CLUSTER) cluster_sync_all();
        else __syncthreads();
        const int nks = (min(K - kb * BK, BK) + 15) / 16;
        for (int ks = 0; ks < nks; ++ks) {
            const int k0 = kb * BK + 16 * ks;
            const uint64_t dbh = desc_none(smem_u32(b_hi) + 256u * ks), dbl = desc_none(smem_u32(b_lo) + 256u * ks);
            if (A_REGS && k0 < k_regs) {
                uint32_t ah[4], al[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int r = fr + 8 * (e & 1), k = k0 + 2 * q + 8 * (e >> 1);
                    const float x0 = k < K ? A[(size_t)r * K + k] : 0.f, x1 = k + 1 < K ? A[(size_t)r * K + k + 1] : 0.f;
                    split_bf16x2(x0, x1, ah[e], al[e]);
                }
                wg::fence();                                    // the fragment registers were just written
                mma_n256_rs(acc, ah, dbh, 1u);
                mma_n256_rs(acc, al, dbh, 1u);
                mma_n256_rs(acc, ah, dbl, 1u);
            } else {
                const uint32_t arow = (uint32_t)wgi * 4096u + 256u * ks;
                const uint64_t dah = desc_none(smem_u32(a_hi + kb * 8192) + arow), dal = desc_none(smem_u32(a_lo + kb * 8192) + arow);
                wg::fence();
                mma_n256(acc, dah, dbh, 1u);
                mma_n256(acc, dal, dbh, 1u);
                mma_n256(acc, dah, dbl, 1u);
            }
        }
        wg::commit();
        wg::wait<0>();
        pin<128>(acc);
    }
    if (CLUSTER) cluster_sync_all();                           // no CTA leaves while its peer may still write its shared memory
    const int cq = 2 * q;
#pragma unroll
    for (int j = 0; j < 32; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int r = fr + 8 * (e >> 1), n = 8 * j + cq + (e & 1);
            if (n < N) D[(size_t)r * N + n] = acc[4 * j + e];
        }
}

}  // namespace pnb

using namespace pnb;

extern "C" int pnb_umma_selftest(const float* d_A, const float* d_W, float* d_D, int K, int N, int layout, int* d_err,
                                 pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(d_A && d_W && d_D && d_err, PNB_ERR_INVALID, "pnb_umma_selftest: null argument");
    PNB_REQUIRE(K >= 1 && K <= 288 && N >= 16 && N <= 256 && N % 16 == 0, PNB_ERR_INVALID, "pnb_umma_selftest: bad K/N");
    const int nkb = (K + 31) / 32;
    const size_t smem = (size_t)nkb * 8192 * 2 + 256 * 64 * 2 + 1024;
    if (layout == wg::LAYOUT_NONE) {
        PNB_CHECK_CUDA(cudaFuncSetAttribute(k_umma_selftest<wg::LAYOUT_NONE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_umma_selftest<wg::LAYOUT_NONE><<<1, 256, smem, stream>>>(d_A, d_W, d_D, K, N);
    } else if (layout == wg::LAYOUT_SW64) {
        PNB_CHECK_CUDA(cudaFuncSetAttribute(k_umma_selftest<wg::LAYOUT_SW64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_umma_selftest<wg::LAYOUT_SW64><<<1, 256, smem, stream>>>(d_A, d_W, d_D, K, N);
    } else if (layout == 100 || layout == 101) {                 // A from registers; 101: the last K step from shared memory
        PNB_REQUIRE(layout == 100 || (K % 16 == 0 && K >= 32), PNB_ERR_INVALID, "pnb_umma_selftest: mode 101 needs K %% 16 == 0, K >= 32");
        PNB_CHECK_CUDA(cudaFuncSetAttribute(k_wgmma_selftest_x<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k_wgmma_selftest_x<true, false><<<1, 256, smem, stream>>>(d_A, d_W, d_D, K, N, layout - 100);
    } else {
        PNB_REQUIRE(false, PNB_ERR_INVALID, "pnb_umma_selftest: layout %d unsupported", layout);
    }
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

extern "C" int pnb_umma_selftest2(const float* d_A, const float* d_W, float* d_D, int K, int N, int mode, int* d_err, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(d_A && d_W && d_D && d_err, PNB_ERR_INVALID, "pnb_umma_selftest2: null argument");
    PNB_REQUIRE(K >= 1 && K <= 288 && N >= 16 && N <= 256 && N % 16 == 0 && (mode == 0 || mode == 1), PNB_ERR_INVALID,
                "pnb_umma_selftest2: bad K/N/mode");
    const int nkb = (K + 31) / 32;
    const size_t smem = (size_t)nkb * 8192 * 2 + 256 * 64 * 2 + 1024;
    auto kern = mode ? k_wgmma_selftest_x<true, true> : k_wgmma_selftest_x<false, true>;
    PNB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2, 1, 1);
    cfg.blockDim = dim3(256, 1, 1);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
    PNB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, d_A, d_W, d_D, K, N, 0));
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
