// Hopper (sm_90a) tensor-core building blocks: wgmma descriptors and instructions, mbarrier, bulk async copy (TMA engine),
// BF16x3 split.  Inline PTX, no CUTLASS.  Encodings follow the PTX ISA "Asynchronous Warpgroup Level Matrix" chapter.
//
// Operand layouts in shared memory (K-major, 16-bit elements).  An operand block is [rows][BK = 32 k]:
//   LAYOUT_NONE  8 x 16-byte core matrices:  byte(r, k) = (r/8)*SBO + (k/8)*LBO + (r%8)*16 + (k%8)*2, LBO = 128, SBO = 512;
//                no swizzle, conflict-free 16-byte stores.  One K = 16 step of a block starts 256 bytes further.
//   LAYOUT_SW64  64-byte rows, 16-byte chunks XOR-swizzled with bits (r/2)%4 (8-row atom = 512 B); a K = 16 step starts 32 bytes
//                further.  Only the self-test uses it.
// [rows x 16] operands (weight images of one K step, the extras operand of block3) use the same core matrices with SBO = 256.
// A warpgroup's m64 slice of a [128 x K] operand block starts 64 rows = 4096 bytes (LAYOUT_NONE, [128 x 32]) further.
//
// Accumulator fragment of wgmma m64nNk16 (fp32): register 4j + 2h + e of thread (warp w of the warpgroup, lane l) holds
//   row 16w + l/4 + 8h, column 8j + 2(l%4) + e.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace pnb {
namespace wg {

enum { LAYOUT_NONE = 0, LAYOUT_SW64 = 4 };
constexpr int BK = 32;  // K elements per operand block

template <int LAYOUT>
__host__ __device__ __forceinline__ uint32_t tile_offset_bytes(int r, int k) {  // k in [0, BK)
    if (LAYOUT == LAYOUT_NONE) return (uint32_t)((r >> 3) * 512 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
    return (uint32_t)(r * 64 + ((((k >> 3) ^ (r >> 1)) & 3) * 16) + (k & 7) * 2);
}
// [rows x 16] operand (SBO = 256)
__host__ __device__ __forceinline__ uint32_t k16_offset_bytes(int r, int k) {
    return (uint32_t)((r >> 3) * 256 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2);
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 64-bit wgmma matrix descriptor: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46), swizzle [62,64) (0 none, 2 = 64 B).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo, uint32_t sbo, uint32_t swizzle = 0) {
    return (uint64_t)((smem_addr >> 4) & 0x3fffu) | ((uint64_t)((lbo >> 4) & 0x3fffu) << 16) | ((uint64_t)((sbo >> 4) & 0x3fffu) << 32) |
           ((uint64_t)swizzle << 62);
}
__device__ __forceinline__ uint64_t desc_none(uint32_t smem_addr) { return make_desc(smem_addr, 128, 512); }      // [rows x 32] block
__device__ __forceinline__ uint64_t desc_k16(uint32_t smem_addr) { return make_desc(smem_addr, 128, 256); }       // [rows x 16] operand
__device__ __forceinline__ uint64_t desc_sw64(uint32_t smem_addr) { return make_desc(smem_addr, 16, 512, 2); }

// ---- wgmma (whole warpgroup, convergent) --------------------------------------------------------------------------
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Registers the asynchronous wgmma writes are pinned after its wait (no copy of them may be scheduled before it).
template <int N>
__device__ __forceinline__ void pin(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T, both operands K-major in shared memory, BF16 in, FP32 accumulate in registers.
// accumulate = 0 overwrites D.
__device__ __forceinline__ void mma_n256(float* d, uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(accumulate));
}

__device__ __forceinline__ void mma_n128(float* d, uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
}

// ---- mbarrier ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// arrive of the threads with pred set, as a predicated instruction: no branch, so it may sit between wgmma without serialising them
__device__ __forceinline__ void mbar_arrive_if(uint64_t* bar, bool pred) {
    asm volatile("{\n\t.reg .pred p;\n\t.reg .b64 st;\n\tsetp.ne.b32 p, %1, 0;\n\t@p mbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)),
                 "r"((uint32_t)pred)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}
// Bounded wait (2 s wall clock): a protocol bug must surface as an error flag, never as a hung GPU.
__device__ __forceinline__ bool mbar_wait(uint64_t* bar, uint32_t parity, int* err_flag, int code) {
    if (mbar_try_wait(bar, parity)) return true;
    const uint64_t t0 = globaltimer_ns();
    for (;;) {
        if (mbar_try_wait(bar, parity)) return true;
        if (globaltimer_ns() - t0 > 2000000000ull) break;
    }
    if (err_flag) atomicCAS(err_flag, 0, code);      // the FIRST time-out is the diagnostic one (the others follow from it)
    return false;
}

// ---- 1-D bulk async copy global -> shared (TMA engine), completes on an mbarrier -----------------------------------
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// generic-proxy stores to shared memory -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---- register reallocation between warpgroups (whole warpgroup, convergent): the launch gives every thread the same count, a
// producer warpgroup hands its share to the consumers.  The counts of a CTA must add up to at most what the launch allocated.
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }

// ---- fp32 -> (hi, lo) bf16 split: x ~= hi + lo with |x - hi - lo| <= 2^-17 |x| ------------------------------------
__device__ __forceinline__ void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(x);
    lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}
// two floats -> packed hi pair / lo pair (element 0 in the low half)
__device__ __forceinline__ void split_bf16x2(float a, float b, uint32_t& hi, uint32_t& lo) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    float ra = a - __low2float(h), rb = b - __high2float(h);
    __nv_bfloat162 l = __floats2bfloat162_rn(ra, rb);
    hi = *reinterpret_cast<uint32_t*>(&h);
    lo = *reinterpret_cast<uint32_t*>(&l);
}

}  // namespace wg
}  // namespace pnb
