/*
 * libpnb200_selftest.so -- TEST-ONLY diagnostics of the wgmma building blocks (wgmma.cuh) and of the backward GEMM engine.
 * Not part of the product ABI (include/pnb200.h); built next to libpnb200.so by pointnerf_b200/build.py, used by
 * tests/test_gpu_umma.py.
 */
#ifndef PNB200_SELFTEST_H
#define PNB200_SELFTEST_H
#include "../../../include/pnb200.h"
#ifdef __cplusplus
extern "C" {
#endif
const char* pnb_selftest_last_error(void);
/* One-CTA wgmma self-test: D[128,N] = A[128,K] * W[N,K]^T with the BF16x3 split used by the fused kernels.
 * layout: 0 = interleaved core matrices, 4 = 64-byte swizzle, 100 = A from registers (interleaved B), 101 = A from registers
 * except the last K step (shared memory; K % 16 == 0).  d_err: device int (kept for the ABI; the test has no waits). */
int pnb_umma_selftest(const float* d_A, const float* d_W, float* d_D, int K, int N, int layout, int* d_err,
                      pnb_stream_t stream);
/* Cluster of two CTAs: D[256,N] = A[256,K] * W[N,K]^T, CTA r computes rows 128r.., converts rows 128r.. of W (zero padded to 256)
 * and stores them into both CTAs' shared memory.  mode 0: A from shared memory, 1: A from registers. */
int pnb_umma_selftest2(const float* d_A, const float* d_W, float* d_D, int K, int N, int mode, int* d_err, pnb_stream_t stream);
/* The wgmma GEMM engine of the backward pass (csrc/gemm_tc.cu): C[M,N] = op(A B^T + bias), A(m,k) = A[m*a_rs + k*a_ks],
 * B(n,k) = B[n*b_rs + k*b_ks]; dact / dact_n: multiply by LeakyReLU'(dact) for n < dact_n; splits > 1: split-K through `part`
 * (>= splits*M*N floats), accumulate != 0 adds to C. */
int pnb_gemm_tc_test(const float* A, long a_rs, long a_ks, const float* B, long b_rs, long b_ks, float* C, long ldc, int M, int N, int K,
                     const float* bias, int act, const float* dact, long ldd, int dact_n, int splits, float* part, size_t part_bytes,
                     int accumulate, int precise /* 3-part split, 6 products */, int* d_err, pnb_stream_t stream);
#ifdef __cplusplus
}
#endif
#endif
