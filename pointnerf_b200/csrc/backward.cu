// Backward of the shading + compositing path for per-scene optimisation batches (run/train_ft.py: 3600 rays/step).
//
// Reference: loss.backward() through autograd (/root/reference/models/mvs_points_volumetric_model.py:98-118) over
//   ray_march        /root/reference/models/rendering/diff_ray_marching.py:508-554
//   viewmlp          /root/reference/models/aggregators/point_aggregators.py:488-644
//   index_select     /root/reference/models/neural_points/neural_points.py:706-717 (backward = index_add into [1,N,.])
// Gradients consumed: d loss / d ray_color [R,3], d loss / d opacity [R,SR] and d loss / d bg_T [R] (the outputs ray_march keeps in the
// autograd graph, returned as coarse_raycolor / coarse_point_opacity / coarse_is_background, neural_points_volumetric_model.py:312-324),
// each optional.  Gradients produced: points_embeding [N,F] (F = 32 | 63), points_color [N,3], points_dir [N,3], points_conf [N] (through
// weight*conf_coefficient, straight-through clamp :722-724), and the 18 MLP tensors (in the W^T layout of pnb_mlp_t).
// xyz receives no gradient (xyz_grad = 0 in every shipped script).
//
// Training batches are small (~2e4 valid samples), so the per-layer activations are recomputed into an HBM workspace and the
// layer gradients are plain GEMMs: forward recompute  H = act(X W^T + b),  dX = (dZ W) * act'  and  dW += X^T dZ  all run on
// the tensor cores (gemm_tc.cu: wgmma, BF16x3 split, fp32 accumulate; the activation derivative is fused into the
// dX epilogue, dW is a deterministic split-K).
// LeakyReLU masks: the recomputed pre-activations carry the BF16x3 error (~1e-5 relative), so ~1e-6 of the units (those whose
// pre-activation is that close to zero) get the other mask than an fp32 forward would give them; each such unit changes ONE pair's
// gradient by ~1/256 (measure-zero for the optimisation, visible in a max-abs comparison with fp32 autograd,
// tests/test_gpu_backward.py bounds them).  A fix-up of the near-zero units cannot help - the perturbation comes from the inputs of the layer - and a three-part split
// stops at ~1e-6 (tests/test_gpu_umma.py).  PNB_BWD_FP32_RECOMPUTE keeps the recompute on the fp32 CUDA-core tiles (fp32-faithful
// masks, dX / dW still on the tensor cores); PNB_BWD_FP32_GEMM selects the hand-written fp32 CUDA-core tiles instead
// (the parity reference of the tensor-core path; always used for the 128 -> 3 colour head).
#include "pair_inputs.cuh"
#include "gemm_tc.cuh"

namespace pnb {
namespace bw {

constexpr float LEAKY = 0.01f;

// ------------------------------------------------------------------------------------------ generic fp32 GEMM
// C[M x N] (+)= sum_k Aeff[m][k] * Beff[k][n],  Aeff[m][k] = A[m*sam + k*sak],  Beff[k][n] = B[k*sbk + n*sbn].
// 128 x 64 tile, 256 threads, 8 x 4 outputs per thread (float4 shared-memory reads: 32 FMA per 3 LDS.128).
// blockIdx.z splits the reduction (ATOMIC accumulation).
template <bool ATOMIC>
__global__ void __launch_bounds__(256) k_gemm(const float* __restrict__ A, long sam, long sak, const float* __restrict__ B,
                                              long sbk, long sbn, float* __restrict__ C, long ldc, int M, int N, int K,
                                              int kchunk, const float* __restrict__ bias, int act) {
    __shared__ __align__(16) float As[16][132];
    __shared__ __align__(16) float Bs[16][68];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * 128, n0 = blockIdx.x * 64;
    const int kbeg = blockIdx.z * kchunk, kend = min(K, kbeg + kchunk);
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    for (int k0 = kbeg; k0 < kend; k0 += 16) {
        // load tiles: the thread->element map follows the unit-stride direction of each operand
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            int idx = tid + e * 256;           // 0..2047
            int am, ak;
            if (sak == 1) { ak = idx & 15; am = idx >> 4; } else { am = idx & 127; ak = idx >> 7; }
            int gm = m0 + am, gk = k0 + ak;
            As[ak][am] = (gm < M && gk < kend) ? A[gm * sam + gk * sak] : 0.f;
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            int idx = tid + e * 256;           // 0..1023
            int bn, bk;
            if (sbn == 1) { bn = idx & 63; bk = idx >> 6; } else { bk = idx & 15; bn = idx >> 4; }
            int gn = n0 + bn, gk2 = k0 + bk;
            Bs[bk][bn] = (gn < N && gk2 < kend) ? B[gk2 * sbk + gn * sbn] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * 8 + 4]);
            const float4 b4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int gm = m0 + ty * 8 + i;
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int gn = n0 + tx * 4 + j;
            if (gn >= N) continue;
            float v = acc[i][j];
            if (ATOMIC) {
                atomicAdd(&C[gm * ldc + gn], v);
            } else {
                if (bias) v += bias[gn];
                if (act) v = v > 0.f ? v : LEAKY * v;
                C[gm * ldc + gn] = v;
            }
        }
    }
}

struct GemmCtx {
    bool precise_all;   // diagnostic (flags & 2): three-part split in every tensor-core GEMM
    bool tc;            // tensor-core GEMMs (default) or the fp32 CUDA-core tiles
    float* part;        // split-K workspace of the tensor-core dW GEMMs
    size_t part_bytes;
    int* err;
    cudaStream_t st;
    bool fp32_recompute;   // PNB_BWD_FP32_RECOMPUTE: the forward recompute on the fp32 CUDA-core tiles (fp32-faithful LeakyReLU masks)
};
constexpr int SPLITK_MAX = 64;
// split-K partials of the widest dW GEMM (block1.0: kpad1_of(F) x 256)
static size_t part_floats(int F) { return (size_t)SPLITK_MAX * kpad1_of(F) * 256; }

__global__ void __launch_bounds__(256) k_lrelu_bwd(float* __restrict__ dY, const float* __restrict__ Y, long ldy, long ldd, int M, int N);

// C[M x N] = act(A[M x K] * Bt[K x N] + bias)
static int gemm_nn(const GemmCtx& cx, const float* A, long lda, const float* Bt, long ldb, float* C, long ldc, int M, int N, int K,
                   const float* bias, int act) {
    if (M <= 0) return PNB_OK;
    if (cx.tc && !cx.fp32_recompute && N % 16 == 0) {
        GemmTc g{};
        g.A = A; g.a_rs = lda; g.a_ks = 1; g.B = Bt; g.b_rs = 1; g.b_ks = ldb; g.C = C; g.ldc = ldc; g.M = M; g.N = N; g.K = K;
        g.bias = bias; g.act = act; g.dact = nullptr; g.ldd = 0; g.dact_n = 0; g.err = cx.err; g.precise = cx.precise_all;
        return gemm_tc(g, 1, cx.part, cx.part_bytes, 0, cx.st);
    }
    dim3 g((N + 63) / 64, (M + 127) / 128, 1);
    k_gemm<false><<<g, 256, 0, cx.st>>>(A, lda, 1, Bt, ldb, 1, C, ldc, M, N, K, K, bias, act);
    return PNB_OK;
}
// dX[M x Kin] = (dZ[M x Nout] * Wt[Kin x Nout]^T) * leaky'(Y[:, :ny])      (Y == nullptr: no activation below)
static int gemm_nt(const GemmCtx& cx, const float* dZ, long ldz, const float* Wt, long ldw, float* dX, long ldx, int M, int Kin, int Nout,
                   const float* Y = nullptr, long ldy = 0, int ny = 0) {
    if (M <= 0) return PNB_OK;
    if (cx.tc && Kin % 16 == 0 && ldw % 4 == 0 && ldz % 4 == 0) {
        // a few columns beyond a 256-wide tile (the 16 extras of block3.0) would cost a second pass over dZ on the tensor cores:
        // they go to the fp32 tiles instead (no activation below them)
        const int tail = (Kin > 256 && Kin - 256 <= 32 && ny <= 256) ? Kin - 256 : 0;
        GemmTc g{};
        g.A = dZ; g.a_rs = ldz; g.a_ks = 1; g.B = Wt; g.b_rs = ldw; g.b_ks = 1; g.C = dX; g.ldc = ldx; g.M = M; g.N = Kin - tail; g.K = Nout;
        g.bias = nullptr; g.act = 0; g.dact = Y; g.ldd = ldy; g.dact_n = ny; g.err = cx.err; g.precise = cx.precise_all;
        int rc = gemm_tc(g, 1, cx.part, cx.part_bytes, 0, cx.st);
        if (rc || !tail) return rc;
        dim3 gt((tail + 63) / 64, (M + 127) / 128, 1);
        k_gemm<false><<<gt, 256, 0, cx.st>>>(dZ, ldz, 1, Wt + (size_t)256 * ldw, 1, ldw, dX + 256, ldx, M, tail, Nout, Nout, nullptr, 0);
        return PNB_OK;
    }
    dim3 g((Kin + 63) / 64, (M + 127) / 128, 1);
    k_gemm<false><<<g, 256, 0, cx.st>>>(dZ, ldz, 1, Wt, 1, ldw, dX, ldx, M, Kin, Nout, Nout, nullptr, 0);
    if (Y) k_lrelu_bwd<<<(int)(((long)M * ny + 255) / 256), 256, 0, cx.st>>>(dX, Y, ldy, ldx, M, ny);
    return PNB_OK;
}
// dWt[Kin x Nout] += X[M x Kin]^T * dZ[M x Nout]   (reduction over the M rows: deterministic split-K on the tensor cores,
// atomics on the CUDA-core path)
static int gemm_tn_acc(const GemmCtx& cx, const float* X, long ldx, const float* dZ, long ldz, float* dWt, long ldw, int M, int Kin, int Nout) {
    if (M <= 0) return PNB_OK;
    if (cx.tc && Nout % 16 == 0 && ldw % 4 == 0) {
        GemmTc g{};
        g.A = X; g.a_rs = 1; g.a_ks = ldx; g.B = dZ; g.b_rs = 1; g.b_ks = ldz; g.C = dWt; g.ldc = ldw; g.M = Kin; g.N = Nout; g.K = M;
        g.bias = nullptr; g.act = 0; g.dact = nullptr; g.ldd = 0; g.dact_n = 0; g.err = cx.err; g.precise = cx.precise_all;
        int splits = (M + 2047) / 2048;
        splits = splits < 2 ? 2 : (splits > SPLITK_MAX ? SPLITK_MAX : splits);
        return gemm_tc(g, splits, cx.part, cx.part_bytes, 1, cx.st);
    }
    const int chunk = 2048;
    dim3 g((Nout + 63) / 64, (Kin + 127) / 128, (M + chunk - 1) / chunk);
    k_gemm<true><<<g, 256, 0, cx.st>>>(X, 1, ldx, dZ, ldz, 1, dWt, ldw, Kin, Nout, M, chunk, nullptr, 0);
    return PNB_OK;
}

__global__ void __launch_bounds__(256) k_lrelu_bwd(float* __restrict__ dY, const float* __restrict__ Y, long ldy, long ldd, int M, int N) {
    long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)M * N) return;
    int m = (int)(i / N), n = (int)(i - (long)m * N);
    float y = Y[m * ldy + n];
    dY[m * ldd + n] *= (y > 0.f ? 1.0f : LEAKY);
}

// db[n] += sum_m dZ[m][n]   (N <= 4: the colour head)
__global__ void __launch_bounds__(256) k_colsum(const float* __restrict__ dZ, long ld, int M, int N, float* __restrict__ db) {
    int n = blockIdx.x * 32 + (threadIdx.x & 31);
    int r0 = blockIdx.y * 2048 + (threadIdx.x >> 5);
    float s = 0.f;
    if (n < N)
        for (int m = r0; m < min(M, (int)(blockIdx.y + 1) * 2048); m += 8) s += dZ[(long)m * ld + n];
    __shared__ float red[8][33];
    red[threadIdx.x >> 5][threadIdx.x & 31] = s;
    __syncthreads();
    if (threadIdx.x < 32 && n < N) {
        float t = 0.f;
        for (int w = 0; w < 8; ++w) t += red[w][threadIdx.x];
        atomicAdd(&db[n], t);
    }
}
// the same for N % 128 == 0: a warp reads 512 contiguous bytes of a row (float4 per lane), 8 warps stride the rows of a 512-row slab
__global__ void __launch_bounds__(256) k_colsum4(const float* __restrict__ dZ, long ld, int M, int N, float* __restrict__ db) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int n = blockIdx.x * 128 + 4 * lane;
    const int m1 = min(M, (int)(blockIdx.y + 1) * 512);
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int m = blockIdx.y * 512 + w; m < m1; m += 8) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(dZ + (long)m * ld + n));
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    __shared__ float4 red[8][32];
    red[w][lane] = s;
    __syncthreads();
    if (w == 0) {
        float4 t = red[0][lane];
        for (int i = 1; i < 8; ++i) { t.x += red[i][lane].x; t.y += red[i][lane].y; t.z += red[i][lane].z; t.w += red[i][lane].w; }
        atomicAdd(&db[n], t.x); atomicAdd(&db[n + 1], t.y); atomicAdd(&db[n + 2], t.z); atomicAdd(&db[n + 3], t.w);
    }
}
static void colsum(const float* dZ, long ld, int M, int N, float* db, cudaStream_t st) {
    if (M <= 0) return;
    if (N % 128 == 0 && ld % 4 == 0) k_colsum4<<<dim3(N / 128, (M + 511) / 512), 256, 0, st>>>(dZ, ld, M, N, db);
    else k_colsum<<<dim3((N + 31) / 32, (M + 2047) / 2048), 256, 0, st>>>(dZ, ld, M, N, db);
}

// ------------------------------------------------------------------------------------------ path-specific kernels
struct BwdParams {
    pnb_query_t q;
    pnb_points_t pts;
    pnb_shade_opts_t o;
    int n_valid;        // S
    int n_rows;         // P = number of valid (sample, neighbour) pairs: the rows of the pair-level buffers are PACKED (no rows for empty slots)
    const uint32_t* pair_off;   // [S+1] first row of every valid sample
    int* row_samp;      // [P] valid-sample index of every row
    // forward recompute buffers
    float* X1;          // [P x kpad1_of(F)]  block1.0 inputs
    float* H1;          // [P x 256]
    float* X3;          // [P x 272]  (H2 | extras | 0)
    float* H3;          // [P x 256]
    float* H4;          // [P x 256]
    float* wc;          // [P]   weight * conf_coefficient
    float* wn;          // [P]   normalised distance weight (no conf)
    float* sp;          // [P]   softplus(alpha_raw - 1)
    float* sg;          // [P]   sigmoid(alpha_raw - 1)   (= d softplus)
    int* pidx;          // [P]   point index or -1
    float* CX;          // [S x 288]  (hbar | PE(view) | 0)
    float* C1; float* C2; float* C3;   // [S x 128]
    float* O3;          // [S x 4]   raw colour outputs (3 used)
    // gradient buffers
    float* G1;          // [P x kpad1_of(F)]  (also scratch of ld 288 for the block3 gradients)
    float* G2;          // [P x 272]
    float* G3;          // [P x 256]
    float* GS1;         // [S x 288]
    float* GS2;         // [S x 128]
    float* GS3;         // [S x 128]
    float* dO3;         // [S x 4]
    float* dsig;        // [S]
    const float4* d_sigma_rgb;   // per candidate (from k_composite_bwd)
    const float* wa; const float* ba;
};

// neighbour count of every valid sample (its exclusive prefix = the first packed row of the sample)
__global__ void __launch_bounds__(256) k_bwd_counts(pnb_query_t q, int n_valid, uint32_t* __restrict__ nv) {
    const int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi < n_valid) nv[vi] = q.samp_nvalid[q.valid_list[vi]];
}
// One warp per valid sample, 4 lanes per pair row: the fp32 forward's row builder, writing the dense block1 input, the block3 extras
// and the view PE to the recompute buffers.
template <bool PP, int F, bool XSAMP = false>
__global__ void __launch_bounds__(256) k_bwd_build(BwdParams p) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= p.n_valid) return;
    const pnb_query_t& q = p.q;
    const int vi = warp, k = lane >> 2, part = lane & 3;
    const uint32_t s = q.valid_list[vi];
    const long row = (long)p.pair_off[vi] + k;               // packed: only the sample's neighbours (its first slots) own a row
    float* cx = p.CX + (long)vi * 288;
    float* er = p.X3 + row * 272 + 256;
    const Fp32Pair pr = fp32_pair<PP, XSAMP>(q, p.pts, p.o, true, s, min((int)q.samp_nvalid[s], q.K), lane, cx + 256);
    if (lane < 8) cx[280 + lane] = 0.f;
    if (!pr.g.valid) return;
    if (part == 0) { p.wc[row] = pr.wc; p.wn[row] = pr.wn; p.pidx[row] = pr.pidx; p.row_samp[row] = vi; }
    fp32_pair_row<PP, F>(p.pts, p.o, pr, lane, p.X1 + row * kpad1_of(F), er);
    if (part == 1)
        for (int e = 7; e < 16; ++e) er[e] = 0.f;
}

// alpha branch + K-reduction forward (dense): one warp per sample.
__global__ void __launch_bounds__(256) k_bwd_reduce_fwd(BwdParams p) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= p.n_valid) return;
    const long r0 = (long)p.pair_off[warp];
    const int nrow = (int)(p.pair_off[warp + 1] - p.pair_off[warp]);
    float hb[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) hb[c] = 0.f;
    for (int k = 0; k < nrow; ++k) {
        const float* h = p.H4 + (r0 + k) * 256;
        float wck = p.wc[r0 + k];
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            float v = h[lane + 32 * c];
            a = fmaf(v, __ldg(&p.wa[lane + 32 * c]), a);
            hb[c] = fmaf(v, wck, hb[c]);
        }
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0 && p.o.agg_intrp_order != 1) {
            const float x = a + __ldg(p.ba);
            p.sp[r0 + k] = softplus_m1(x);
            p.sg[r0 + k] = 1.0f / (1.0f + expf(-(x - 1.0f)));   // its derivative
        }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) p.CX[(long)warp * 288 + lane + 32 * c] = hb[c];
    if (p.o.agg_intrp_order == 1 && nrow > 0) {
        // agg_intrp_order 1 (point_aggregators.py:573-587): the density comes from the aggregated feature; its softplus / sigmoid are
        // kept in the slot of the sample's FIRST row
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) a = fmaf(hb[c], __ldg(&p.wa[lane + 32 * c]), a);
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) {
            const float x = a + __ldg(p.ba);
            p.sp[r0] = softplus_m1(x);
            p.sg[r0] = 1.0f / (1.0f + expf(-(x - 1.0f)));
        }
    }
}

// colour head: O3 raw -> d(raw) ; sigma gradient per valid sample
__global__ void __launch_bounds__(256) k_bwd_head(BwdParams p) {
    int vi = blockIdx.x * blockDim.x + threadIdx.x;
    if (vi >= p.n_valid) return;
    uint32_t s = p.q.valid_list[vi];
    float4 g = p.d_sigma_rgb[s];
    p.dsig[vi] = g.x;
    float gr[3] = {g.y, g.z, g.w};
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        float sgm = 1.0f / (1.0f + expf(-p.O3[(long)vi * 4 + c]));
        p.dO3[(long)vi * 4 + c] = gr[c] * (1.0f + 2.0f * 0.001f) * sgm * (1.0f - sgm);
    }
    p.dO3[(long)vi * 4 + 3] = 0.f;
}

// dH4[p][c] = wc[p] * dhbar[s][c] + dalpha_raw[p] * wa[c] ;  dwc[p] = <dhbar[s], H4[p]> + dsigma[s] * sp[p]
// output dH4 in G3 (then lrelu' applied separately), dwc into G1[row*288] scratch column 0 (consumed by k_bwd_scatter)
__global__ void __launch_bounds__(256) k_bwd_reduce_bwd(BwdParams p, float* __restrict__ dwc) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= p.n_valid) return;
    const long r0 = (long)p.pair_off[warp];
    const int nrow = (int)(p.pair_off[warp + 1] - p.pair_off[warp]);
    float dh[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) dh[c] = p.GS1[(long)warp * 288 + lane + 32 * c];
    const float ds = p.dsig[warp];
    if (p.o.agg_intrp_order == 1) {
        // order 1: sigma = softplus(<wa, hbar> + ba - 1): the density gradient joins the colour branch's d hbar; dwc = <d hbar, H4>
        if (nrow > 0) {
            const float dar = ds * p.sg[r0];
#pragma unroll
            for (int c = 0; c < 8; ++c) dh[c] = fmaf(dar, __ldg(&p.wa[lane + 32 * c]), dh[c]);
        }
        for (int k = 0; k < nrow; ++k) {
            const long row = r0 + k;
            const float wck = p.wc[row];
            const float* h = p.H4 + row * 256;
            float dot = 0.f;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                dot = fmaf(dh[c], h[lane + 32 * c], dot);
                p.G3[row * 256 + lane + 32 * c] = wck * dh[c];
            }
            for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
            if (lane == 0) dwc[row] = dot;
        }
        return;
    }
    for (int k = 0; k < nrow; ++k) {
        const long row = r0 + k;
        const float wck = p.wc[row];
        const float dar = ds * wck * p.sg[row];     // d alpha_raw
        const float* h = p.H4 + row * 256;
        float dot = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            dot = fmaf(dh[c], h[lane + 32 * c], dot);
            p.G3[row * 256 + lane + 32 * c] = wck * dh[c] + dar * __ldg(&p.wa[lane + 32 * c]);
        }
        for (int o = 16; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
        if (lane == 0) dwc[row] = dot + ds * p.sp[row];
    }
}

// alpha-branch parameter gradients: dwa[c] += sum_p dalpha_raw[p] * H4[p][c] ; dba += sum_p dalpha_raw[p]
__global__ void __launch_bounds__(256) k_bwd_alpha_params(BwdParams p, float* __restrict__ dwa, float* __restrict__ dba) {
    const int c = threadIdx.x;
    const long P = (long)p.n_rows;
    // 256-row slabs (a 1024-row slab left most SMs of a 1e5-row batch without a block); the row factors are computed once per block
    __shared__ float dar_s[256];
    const long r0 = (long)blockIdx.x * 256, r1 = min(P, r0 + 256);
    const long mine = r0 + c;
    dar_s[c] = mine < r1 ? p.dsig[p.row_samp[mine]] * p.wc[mine] * p.sg[mine] : 0.f;
    __syncthreads();
    float acc = 0.f, accb = 0.f;
    const int n = (int)(r1 - r0);
#pragma unroll 4
    for (int i = 0; i < n; ++i) {
        const float dar = dar_s[i];
        acc = fmaf(dar, p.H4[(r0 + i) * 256 + c], acc);
        accb += dar;
    }
    atomicAdd(&dwa[c], acc);
    if (c == 0) atomicAdd(dba, accb);
}

// agg_intrp_order 1: dwa[c] += sum_s dalpha_raw[s] * hbar[s][c] ; dba += sum_s dalpha_raw[s]   (per valid sample, hbar = CX[:, :256])
__global__ void __launch_bounds__(256) k_bwd_alpha_params_o1(BwdParams p, float* __restrict__ dwa, float* __restrict__ dba) {
    const int c = threadIdx.x;
    const long S = (long)p.n_valid;
    __shared__ float dar_s[256];
    const long s0 = (long)blockIdx.x * 256, s1 = min(S, s0 + 256);
    const long mine = s0 + c;
    dar_s[c] = (mine < s1 && p.pair_off[mine + 1] > p.pair_off[mine]) ? p.dsig[mine] * p.sg[p.pair_off[mine]] : 0.f;
    __syncthreads();
    float acc = 0.f, accb = 0.f;
    const int n = (int)(s1 - s0);
#pragma unroll 4
    for (int i = 0; i < n; ++i) {
        const float dar = dar_s[i];
        acc = fmaf(dar, p.CX[(s0 + i) * 288 + c], acc);
        accb += dar;
    }
    atomicAdd(&dwa[c], acc);
    if (c == 0) atomicAdd(dba, accb);
}

// dWt[Kin x Nout] += X^T dZ and db[n] += sum_m dZ[m][n] for a tiny Nout (the 128 -> 3 colour head): thread = input column, 256-row slabs
template <int NOUT>
__global__ void __launch_bounds__(128) k_dw_small(const float* __restrict__ X, long ldx, const float* __restrict__ dZ, long ldz, float* __restrict__ dWt,
                                                  long ldw, float* __restrict__ db, int M, int Kin) {
    __shared__ float dz_s[256][NOUT];
    const int c = threadIdx.x;
    const long r0 = (long)blockIdx.x * 256;
    const int n = (int)min((long)256, (long)M - r0);
    for (int i = c; i < n * NOUT; i += 128) dz_s[i / NOUT][i % NOUT] = dZ[(r0 + i / NOUT) * ldz + (i % NOUT)];
    __syncthreads();
    float acc[NOUT];
#pragma unroll
    for (int j = 0; j < NOUT; ++j) acc[j] = 0.f;
    if (c < Kin) {
#pragma unroll 4
        for (int i = 0; i < n; ++i) {
            const float x = X[(r0 + i) * ldx + c];
#pragma unroll
            for (int j = 0; j < NOUT; ++j) acc[j] = fmaf(x, dz_s[i][j], acc[j]);
        }
#pragma unroll
        for (int j = 0; j < NOUT; ++j) atomicAdd(&dWt[(long)c * ldw + j], acc[j]);
    }
    if (db && c < NOUT) {
        float sb = 0.f;
        for (int i = 0; i < n; ++i) sb += dz_s[i][c];
        atomicAdd(&db[c], sb);
    }
}

// Scatter to the points: embedding (through PE), colour, dir, conf.  4 lanes per pair row (8 embedding channels per lane, 16 for F = 63).
template <bool PP, int F, bool XSAMP = false>
__global__ void __launch_bounds__(256) k_bwd_scatter(BwdParams p, const float* __restrict__ dwc, float* __restrict__ d_emb,
                                                     float* __restrict__ d_color, float* __restrict__ d_dir, float* __restrict__ d_conf) {
    constexpr int CPL = F == PNB_FEAT ? 8 : 16;
    const long gt = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const long row = gt >> 2;
    const int part = (int)(gt & 3);
    const long P = (long)p.n_rows;
    if (row >= P) return;
    const int pi = p.pidx[row];
    if (pi < 0) return;
    const float* x = p.X1 + row * kpad1_of(F);
    const float* g = p.G1 + row * kpad1_of(F);
    if (d_emb) {
#pragma unroll
        for (int e = 0; e < CPL; ++e) {
            int c = part * CPL + e;
            if (F != PNB_FEAT && c >= F) continue;
            float acc = g[c];
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                float sn = x[F + (c * 3 + j) * 2], cs = x[F + (c * 3 + j) * 2 + 1];
                float gs = g[F + (c * 3 + j) * 2], gc = g[F + (c * 3 + j) * 2 + 1];
                acc = fmaf((float)(1 << j), cs * gs - sn * gc, acc);
            }
            atomicAdd(&d_emb[(size_t)pi * F + c], acc);
        }
    }
    if (part == 0) {
        const float* ge = p.G2 + row * 272 + 256;
        if (d_color) { atomicAdd(&d_color[3 * pi], ge[0]); atomicAdd(&d_color[3 * pi + 1], ge[1]); atomicAdd(&d_color[3 * pi + 2], ge[2]); }
        if (d_dir) {
            // extras: (dir' - view')[3], <dir', view'>  with dir' = M_p dir (the point's frame) and view' in the frame of the sample's
            // slot-0 point  ->  d dir = M_p^T (g[3:6] + g[6] * view')
            const uint32_t s = p.q.valid_list[p.row_samp[row]];
            const float3 ov = view_in_points<PP>(p.pts, p.o, view_point<PP>(p.q, s), cand_view_dir<XSAMP>(p.q, s));
            float gx = ge[3] + ge[6] * ov.x, gy = ge[4] + ge[6] * ov.y, gz = ge[5] + ge[6] * ov.z;
            float ox, oy, oz;
            rot3T(point_frame<PP>(p.pts, p.o, pi), gx, gy, gz, ox, oy, oz);
            atomicAdd(&d_dir[3 * pi], ox); atomicAdd(&d_dir[3 * pi + 1], oy); atomicAdd(&d_dir[3 * pi + 2], oz);
        }
        if (d_conf) atomicAdd(&d_conf[pi], dwc[row] * p.wn[row]);   // straight-through clamp (gradiant_clamp :722-724)
    }
}

// Composite backward: per ray, d ray_color, d opacity and d bg_T -> d(sigma, rgb) of each of its candidate samples.
struct CompBwdParams {
    pnb_query_t q;
    pnb_shade_opts_t o;
    const float4* sigma_rgb;
    const float* d_ray_color;   // [R,3]; NULL (EXT only): no colour term
    float4* d_sigma_rgb;        // [cap]
    const float* d_opacity;     // [R,SR] or NULL (EXT only)
    const float* d_bg_T;        // [R] or NULL (EXT only)
};

// EXT: the upstream gradients of opacity and bg_T (each optional, as is the colour's); without it the kernel reads d ray_color only.
// With T_{j+1} = T_j (1 - o_j + 1e-10) and bg_T = T_end, the bg_T gradient enters the suffix beside g.bg, and the opacity gradient
// adds to d o_j directly.  XSAMP: explicit samples (pair_inputs.cuh).
template <bool EXT, bool XSAMP = false>
__global__ void __launch_bounds__(128) k_composite_bwd(CompBwdParams p) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    const pnb_query_t& q = p.q;
    if (r >= q.R) return;
    const int n = q.nsamp[r];
    const uint32_t s0 = q.samp_off[r];
    if (n == 0) return;
    if (!q.ray_hit[r]) {
        for (int j = 0; j < n; ++j) p.d_sigma_rgb[s0 + j] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    const float3 dir = XSAMP ? make_float3(0.f, 0.f, 0.f) : ray_dir(q, r);
    const bool col = !EXT || p.d_ray_color;
    const float gR = col ? p.d_ray_color[3 * r] : 0.f, gG = col ? p.d_ray_color[3 * r + 1] : 0.f,
                gB = col ? p.d_ray_color[3 * r + 2] : 0.f;
    const float* g_o = EXT && p.d_opacity ? p.d_opacity + (size_t)r * q.SR : nullptr;
    // pass 1 (front to back): opacity, ray distance and transmittance of every candidate (local arrays, SR <= 128)
    float o_[PNB_MAX_SR], rd_[PNB_MAX_SR], T_[PNB_MAX_SR];
    float Tend;
    {
        float cm = slot_depth<XSAMP>(q, p.o, r, n, 0, dir), T = 1.0f;
        for (int j = 0; j < n; ++j) {
            const float rd = ray_dist_step<XSAMP>(q, p.o, r, n, j, dir, cm);
            float o1 = 0.f;
            if (q.samp_nvalid[s0 + j] > 0) o1 = 1.0f - expf(-p.sigma_rgb[s0 + j].x * rd);
            o_[j] = o1; rd_[j] = rd; T_[j] = T;
            T = T * (1.0f - o1 + 1e-10f);
        }
        Tend = T;
    }
    // pass 2 (back to front): suffix_j = (g.bg + g_T) T_end + sum_{i>j} g.rgb_i o_i T_i   (no cancellation)
    float gbg = gR * p.o.bg_color[0] + gG * p.o.bg_color[1] + gB * p.o.bg_color[2];
    if (EXT && p.d_bg_T) gbg += p.d_bg_T[r];
    float suffix = gbg * Tend;
    for (int j = n - 1; j >= 0; --j) {
        float4 out = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q.samp_nvalid[s0 + j] > 0) {
            float4 v = p.sigma_rgb[s0 + j];
            float o1 = o_[j], T = T_[j];
            float gdot = gR * v.y + gG * v.z + gB * v.w;
            float bw = o1 * T;
            float d_o = gdot * T - suffix / (1.0f - o1 + 1e-10f);
            if (EXT && g_o) d_o += g_o[j];               // added last: a zero g_o leaves the colour-only bits unchanged
            out.x = d_o * rd_[j] * (1.0f - o1);              // d o / d sigma = rd * exp(-sigma rd)
            out.y = gR * bw; out.z = gG * bw; out.w = gB * bw;
            suffix += gdot * bw;
        }
        p.d_sigma_rgb[s0 + j] = out;
    }
}

struct Layout {
    float *X1, *H1, *X3, *H3, *H4, *wc, *wn, *sp, *sg, *CX, *C1, *C2, *C3, *O3, *G1, *G2, *G3, *GS1, *GS2, *GS3, *dO3, *dsig, *dwc;
    int* pidx;
    float4* d_sigma_rgb;
    float* part;
    uint32_t *nv, *pair_off, *scan_tmp;
    int* row_samp;
    size_t bytes;
};
static Layout carve(void* ws, size_t cap, int max_valid, int cap_samples, int F) {
    Carver c(ws, cap);
    Layout L;
    size_t S = (size_t)(max_valid > 0 ? max_valid : 1), P = S * PNB_MAX_K;
    L.X1 = c.take<float>(P * kpad1_of(F)); L.H1 = c.take<float>(P * 256); L.X3 = c.take<float>(P * 272);
    L.H3 = c.take<float>(P * 256); L.H4 = c.take<float>(P * 256);
    L.wc = c.take<float>(P); L.wn = c.take<float>(P); L.sp = c.take<float>(P); L.sg = c.take<float>(P); L.dwc = c.take<float>(P);
    L.pidx = c.take<int>(P);
    L.CX = c.take<float>(S * 288); L.C1 = c.take<float>(S * 128); L.C2 = c.take<float>(S * 128); L.C3 = c.take<float>(S * 128);
    L.O3 = c.take<float>(S * 4);
    L.G1 = c.take<float>(P * kpad1_of(F)); L.G2 = c.take<float>(P * 272); L.G3 = c.take<float>(P * 256);
    L.GS1 = c.take<float>(S * 288); L.GS2 = c.take<float>(S * 128); L.GS3 = c.take<float>(S * 128);
    L.dO3 = c.take<float>(S * 4); L.dsig = c.take<float>(S);
    L.d_sigma_rgb = c.take<float4>((size_t)(cap_samples > 0 ? cap_samples : 1));
    L.part = c.take<float>(part_floats(F));
    L.nv = c.take<uint32_t>(S); L.pair_off = c.take<uint32_t>(S + 1); L.scan_tmp = c.take<uint32_t>(scan_tmp_elems(S)); L.row_samp = c.take<int>(P);
    L.bytes = align_up(c.off);
    return L;
}

}  // namespace bw
}  // namespace pnb

using namespace pnb;
using namespace pnb::bw;

extern "C" size_t pnb_backward_bytes(int n_valid, int cap_samples, int feat_dim) {
    const int F = feat_of(feat_dim);
    return F > 0 ? carve(nullptr, 0, n_valid, cap_samples, F).bytes : 0;
}

// tests: device pointers of the recompute buffers inside a workspace pnb_shade_backward used with the same n_valid / cap_samples / F
extern "C" int pnb_backward_tables(void* ws, size_t ws_bytes, int n_valid, int cap_samples, int feat_dim, void** out) {
    const int F = feat_of(feat_dim);
    PNB_REQUIRE(ws && out, PNB_ERR_INVALID, "pnb_backward_tables: null argument");
    PNB_REQUIRE(F > 0, PNB_ERR_UNSUPPORTED, "pnb_backward_tables: point_features_dim %d unsupported", feat_dim);
    const Layout L = carve(ws, ws_bytes, n_valid, cap_samples, F);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_backward_tables: workspace %zu < required %zu", ws_bytes, L.bytes);
    void* const t[10] = {L.H1, L.X3, L.H3, L.H4, L.C1, L.C2, L.C3, L.pair_off, L.row_samp, L.pidx};
    for (int i = 0; i < 10; ++i) out[i] = t[i];
    return PNB_OK;
}

// d_mlp_w[i] / d_mlp_b[i]: gradient accumulators in the layout of pnb_mlp_t (W^T [K_pad][N], bias [N]); the caller
// zero-initialises them.  Point gradients are accumulated (atomicAdd) into d_emb/d_color/d_dir/d_conf (caller zeroes);
// any of them may be NULL.  Upstream gradients: d_ray_color [R,3], d_opacity [R,SR], d_bg_T [R], each may be NULL (at least one is
// given).  n_valid: host copy of counters[PNB_QC_N_VALID] of the query.
extern "C" int pnb_shade_backward(const pnb_query_t* q, const pnb_points_t* pts, const pnb_mlp_t* mlp,
                                  const pnb_shade_opts_t* opts, const float* d_sigma_rgb_fwd, const float* d_ray_color,
                                  const float* d_opacity, const float* d_bg_T, int n_valid, int n_pairs, float* d_emb, float* d_color,
                                  float* d_dir, float* d_conf, float* const* d_mlp_w, float* const* d_mlp_b, void* ws, size_t ws_bytes,
                                  int flags, int* d_err, pnb_stream_t stream_) {
    cudaStream_t st = (cudaStream_t)stream_;
    PNB_REQUIRE(q && pts && mlp && opts && d_sigma_rgb_fwd && d_mlp_w && d_mlp_b && ws, PNB_ERR_INVALID,
                "pnb_shade_backward: null argument");
    PNB_REQUIRE(d_ray_color || d_opacity || d_bg_T, PNB_ERR_INVALID,
                "pnb_shade_backward: no upstream gradient (d_ray_color, d_opacity and d_bg_T are all NULL)");
    Variant v;
    { const int rc = resolve_variant("pnb_shade_backward", pts, mlp, q, XsRule::frames, &v); if (rc) return rc; }
    const int F = v.F, KP1 = kpad1_of(F);
    Layout L = carve(ws, ws_bytes, n_valid, q->cap_samples, F);
    PNB_REQUIRE(L.bytes <= ws_bytes, PNB_ERR_WORKSPACE, "pnb_shade_backward: workspace %zu < required %zu", ws_bytes, L.bytes);
    // composite backward first (also covers n_valid == 0)
    CompBwdParams cp;
    cp.q = *q; cp.o = *opts; cp.sigma_rgb = (const float4*)d_sigma_rgb_fwd; cp.d_ray_color = d_ray_color; cp.d_sigma_rgb = L.d_sigma_rgb;
    cp.d_opacity = d_opacity; cp.d_bg_T = d_bg_T;
    const bool colour_only = d_ray_color && !d_opacity && !d_bg_T;   // colour-only loss
    const auto comp = with_bool(!colour_only, [&](auto EXT) {
        return with_bool(v.xs, [&](auto XS) { return k_composite_bwd<EXT, XS>; });
    });
    comp<<<(q->R + 127) / 128, 128, 0, st>>>(cp);
    if (n_valid <= 0) { PNB_CHECK_CUDA(cudaGetLastError()); return PNB_OK; }
    PNB_REQUIRE(n_pairs >= n_valid && n_pairs <= n_valid * PNB_MAX_K, PNB_ERR_INVALID, "pnb_shade_backward: n_pairs %d inconsistent with n_valid %d", n_pairs, n_valid);
    const int S = n_valid, P = n_pairs;      // pair-level buffers hold one row per VALID (sample, neighbour) pair
    BwdParams p;
    p.q = *q; p.pts = *pts; p.o = *opts; p.n_valid = n_valid;
    p.n_rows = P; p.pair_off = L.pair_off; p.row_samp = L.row_samp;
    k_bwd_counts<<<(S + 255) / 256, 256, 0, st>>>(*q, S, L.nv);
    { int rc = exclusive_scan_u32(L.nv, 0, L.pair_off, (uint32_t)S, L.scan_tmp, st); if (rc) return rc; }
    p.X1 = L.X1; p.H1 = L.H1; p.X3 = L.X3; p.H3 = L.H3; p.H4 = L.H4; p.wc = L.wc; p.wn = L.wn; p.sp = L.sp; p.sg = L.sg; p.pidx = L.pidx;
    p.CX = L.CX; p.C1 = L.C1; p.C2 = L.C2; p.C3 = L.C3; p.O3 = L.O3; p.G1 = L.G1; p.G2 = L.G2; p.G3 = L.G3;
    p.GS1 = L.GS1; p.GS2 = L.GS2; p.GS3 = L.GS3; p.dO3 = L.dO3; p.dsig = L.dsig; p.d_sigma_rgb = L.d_sigma_rgb;
    p.wa = mlp->w[4]; p.ba = mlp->b[4];
    const int wb = (S * 32 + 255) / 256;   // one warp per sample
    GemmCtx cx{(flags & 2) != 0, (flags & PNB_BWD_FP32_GEMM) == 0, L.part, part_floats(F) * sizeof(float), d_err, st, (flags & PNB_BWD_FP32_RECOMPUTE) != 0};
    PNB_REQUIRE(!cx.tc || d_err, PNB_ERR_INVALID, "pnb_shade_backward: the tensor-core path needs d_err");
    // ---------------- forward recompute ----------------
    const auto build = with_frames(v, [](auto PP, auto F, auto XS) { return k_bwd_build<PP, F, XS>; });
    build<<<wb, 256, 0, st>>>(p);
    gemm_nn(cx, L.X1, KP1, mlp->w[0], 256, L.H1, 256, P, 256, KP1, mlp->b[0], 1);
    gemm_nn(cx, L.H1, 256, mlp->w[1], 256, L.X3, 272, P, 256, 256, mlp->b[1], 1);   // H2 into X3[:, :256]
    gemm_nn(cx, L.X3, 272, mlp->w[2], 256, L.H3, 256, P, 256, 272, mlp->b[2], 1);
    gemm_nn(cx, L.H3, 256, mlp->w[3], 256, L.H4, 256, P, 256, 256, mlp->b[3], 1);
    k_bwd_reduce_fwd<<<wb, 256, 0, st>>>(p);
    gemm_nn(cx, L.CX, 288, mlp->w[5], 128, L.C1, 128, S, 128, 288, mlp->b[5], 1);
    gemm_nn(cx, L.C1, 128, mlp->w[6], 128, L.C2, 128, S, 128, 128, mlp->b[6], 1);
    gemm_nn(cx, L.C2, 128, mlp->w[7], 128, L.C3, 128, S, 128, 128, mlp->b[7], 1);
    gemm_nn(cx, L.C3, 128, mlp->w[8], 3, L.O3, 4, S, 3, 128, mlp->b[8], 0);          // N = 3: CUDA cores
    // ---------------- backward ----------------
    k_bwd_head<<<(S + 255) / 256, 256, 0, st>>>(p);
    // colour branch (each dX GEMM applies the derivative of the LeakyReLU below it in its epilogue)
    k_dw_small<3><<<(S + 255) / 256, 128, 0, st>>>(L.C3, 128, L.dO3, 4, d_mlp_w[8], 3, d_mlp_b[8], S, 128);     // colour head 128 -> 3 (+ its bias)
    gemm_nt(cx, L.dO3, 4, mlp->w[8], 3, L.GS3, 128, S, 128, 3, L.C3, 128, 128);       // dC3
    gemm_tn_acc(cx, L.C2, 128, L.GS3, 128, d_mlp_w[7], 128, S, 128, 128);
    colsum(L.GS3, 128, S, 128, d_mlp_b[7], st);
    gemm_nt(cx, L.GS3, 128, mlp->w[7], 128, L.GS2, 128, S, 128, 128, L.C2, 128, 128); // dC2
    gemm_tn_acc(cx, L.C1, 128, L.GS2, 128, d_mlp_w[6], 128, S, 128, 128);
    colsum(L.GS2, 128, S, 128, d_mlp_b[6], st);
    gemm_nt(cx, L.GS2, 128, mlp->w[6], 128, L.GS3, 128, S, 128, 128, L.C1, 128, 128); // dC1 (reuse GS3)
    gemm_tn_acc(cx, L.CX, 288, L.GS3, 128, d_mlp_w[5], 128, S, 288, 128);
    colsum(L.GS3, 128, S, 128, d_mlp_b[5], st);
    gemm_nt(cx, L.GS3, 128, mlp->w[5], 128, L.GS1, 288, S, 288, 128);                 // d(hbar | view PE)
    // K-reduction + alpha branch
    k_bwd_reduce_bwd<<<wb, 256, 0, st>>>(p, L.dwc);
    if (p.o.agg_intrp_order == 1) k_bwd_alpha_params_o1<<<(S + 255) / 256, 256, 0, st>>>(p, d_mlp_w[4], d_mlp_b[4]);
    else k_bwd_alpha_params<<<(P + 255) / 256, 256, 0, st>>>(p, d_mlp_w[4], d_mlp_b[4]);
    // block3.2
    k_lrelu_bwd<<<(int)(((long)P * 256 + 255) / 256), 256, 0, st>>>(L.G3, L.H4, 256, 256, P, 256);
    gemm_tn_acc(cx, L.H3, 256, L.G3, 256, d_mlp_w[3], 256, P, 256, 256);
    colsum(L.G3, 256, P, 256, d_mlp_b[3], st);
    gemm_nt(cx, L.G3, 256, mlp->w[3], 256, L.G1, 288, P, 256, 256, L.H3, 256, 256);   // dH3 in G1[:, :256] (ld 288)
    // block3.0
    gemm_tn_acc(cx, L.X3, 272, L.G1, 288, d_mlp_w[2], 256, P, 272, 256);
    colsum(L.G1, 288, P, 256, d_mlp_b[2], st);
    gemm_nt(cx, L.G1, 288, mlp->w[2], 256, L.G2, 272, P, 272, 256, L.X3, 272, 256);   // dX3 = (dH2 | d extras); the extras have no activation
    // block1.2
    gemm_tn_acc(cx, L.H1, 256, L.G2, 272, d_mlp_w[1], 256, P, 256, 256);
    colsum(L.G2, 272, P, 256, d_mlp_b[1], st);
    gemm_nt(cx, L.G2, 272, mlp->w[1], 256, L.G3, 256, P, 256, 256, L.H1, 256, 256);   // dH1 in G3
    // block1.0
    gemm_tn_acc(cx, L.X1, KP1, L.G3, 256, d_mlp_w[0], 256, P, KP1, 256);
    colsum(L.G3, 256, P, 256, d_mlp_b[0], st);
    // dX1: only the 7F feature columns are consumed (k_bwd_scatter; no xyz gradient), rounded up to 16: 224 | 448
    gemm_nt(cx, L.G3, 256, mlp->w[0], 256, L.G1, KP1, P, (7 * F + 15) / 16 * 16, 256);
    // scatter to the points
    const auto scatter = with_frames(v, [](auto PP, auto F, auto XS) { return k_bwd_scatter<PP, F, XS>; });
    scatter<<<(int)(((long)P * 4 + 255) / 256), 256, 0, st>>>(p, L.dwc, d_emb, d_color, d_dir, d_conf);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
