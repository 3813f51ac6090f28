// TEST-ONLY (libpnb200_selftest.so): C entry point over the wgmma GEMM engine of the backward pass (../gemm_tc.cu, compiled
// into this library a second time) so that tests/test_gpu_umma.py can compare every operand form with a torch matmul.
#include "../gemm_tc.cu"
#include "pnb200_selftest.h"

extern "C" int pnb_gemm_tc_test(const float* A, long a_rs, long a_ks, const float* B, long b_rs, long b_ks, float* C, long ldc, int M, int N, int K,
                                const float* bias, int act, const float* dact, long ldd, int dact_n, int splits, float* part, size_t part_bytes,
                                int accumulate, int precise, int* d_err, pnb_stream_t stream) {
    pnb::GemmTc g{};
    g.A = A; g.a_rs = a_rs; g.a_ks = a_ks; g.B = B; g.b_rs = b_rs; g.b_ks = b_ks; g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
    g.bias = bias; g.act = act; g.dact = dact; g.ldd = ldd; g.dact_n = dact_n; g.precise = precise; g.err = d_err;
    return pnb::gemm_tc(g, splits, part, part_bytes, accumulate, (cudaStream_t)stream);
}
