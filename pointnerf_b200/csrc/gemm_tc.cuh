// wgmma BF16x3 GEMM of the backward pass (gemm_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace pnb {

struct GemmTc {
    const float* A; long a_rs, a_ks;   // A(m,k) = A[m*a_rs + k*a_ks]   (one of the strides is 1)
    const float* B; long b_rs, b_ks;   // B(n,k) = B[n*b_rs + k*b_ks]
    float* C; long ldc;                // C[m*ldc + n]
    int M, N, K;
    const float* bias;                 // [N] or null
    int act;                           // 1: LeakyReLU(0.01) on the result
    const float* dact; long ldd;       // not null: result *= (dact[m*ldd + n] > 0 ? 1 : 0.01) for n < dact_n  (backward of the LeakyReLU below)
    int dact_n;
    int precise;                       // 1: three bf16 parts per operand, six products (fp32-level result); 0: BF16x3 (two parts, three products)
    int* err;                          // device int: set non-zero if a bounded pipeline wait expires
    // filled by gemm_tc():
    int kchunk; float* part;
};

// C = A B^T (+ bias, activation).  splits > 1: split-K over blockIdx.z with partial tiles in part_ws
// (>= splits * M * N floats), reduced in split order; accumulate != 0 adds to C instead of overwriting (split-K path only).
int gemm_tc(const GemmTc& g, int splits, float* part_ws, size_t part_bytes, int accumulate, cudaStream_t st);

}  // namespace pnb
