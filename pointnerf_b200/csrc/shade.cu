// Fused gather + distance weights + positional encoding + MLP chain + K-reduction + colour branch (forward),
// fp32 CUDA-core version ("v1": the exact-fp32 path; the wgmma BF16x3 path lives in shade_tc.cu).
//
// Replaces, per valid sample tile, what the reference does with ~40 eager torch kernels and HBM round trips:
//   gather                     /root/reference/models/neural_points/neural_points.py:706-717
//   dists / linear weights     /root/reference/models/aggregators/point_aggregators.py:727-814, :421-429
//   viewmlp (intrp order 2)    /root/reference/models/aggregators/point_aggregators.py:488-644
//   positional_encoding        /root/reference/models/helpers/networks.py:175-190
//   raw2out_density / _color   /root/reference/models/aggregators/point_aggregators.py:262-273
// and, in k_composite, ray distances + alpha compositing + fill_invalid:
//   /root/reference/models/neural_points_volumetric_model.py:271-305, :87-123
//   /root/reference/models/rendering/diff_ray_marching.py:508-554
//
// Tile = 8 valid samples x 8 neighbour slots = 64 (sample,k) pair rows; one warp builds one sample's rows.
// Activations never leave shared memory; weights (W^T, zero padded to multiples of 16 rows) stream from L2
// through a cp.async double buffer.
// F = 63 (point_features_dim of the DTU scripts): the 512-wide block1.0 input rows (stride XS1) overlay X and H, which are contiguous;
// layer 1 writes H only after its last read of the rows (gemm64x256 synchronises before its epilogue).
#include "pair_inputs.cuh"

namespace pnb {

constexpr int TS = 8;             // samples per tile
constexpr int TR = TS * PNB_MAX_K;  // 64 pair rows
constexpr int XS = 292;           // X row stride (floats): 284 inputs padded to 288, +4 against bank conflicts
constexpr int HS = 284;           // H row stride: holds 280 colour-branch inputs (256 + 24) and 272 block3 inputs
constexpr int XS1 = 516;          // F = 63: block1.0 input row stride (512 inputs + 4), over X and H
constexpr int KC = 16;            // weight rows per pipeline stage
constexpr int NTHREADS = 256;
constexpr float LEAKY = 0.01f;

struct ShadeParams {
    pnb_query_t q;
    pnb_points_t pts;
    pnb_mlp_t mlp;
    pnb_shade_opts_t o;
    float4* sigma_rgb;
};

struct __align__(16) ShadeSmem {
    float X[TR * XS];
    float H[TR * HS];
    float W[2][KC * 256];
    float E[TR][8];       // block3 extras: colour(3), dir - view(3), <dir,view>(1)
    float wc[TR];         // weight * conf_coefficient per pair (0 for empty slots)
    float alpha[TR];
    float view[TS][28];   // per sample: ori_viewdirs(3) + PE4 (sin 12, cos 12)
    uint32_t samp[TS];    // candidate id of each tile sample (0xffffffff = padding)
};

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ float lrelu(float x) { return x > 0.f ? x : LEAKY * x; }

// C[64 x 256] = act(A[64 x Kp] * Wt[Kp x 256] + b);  A, C in shared memory (row strides sa, sc).
// Thread (ty, tx): rows ty*4..+3, columns tx*4 + 64*j .. +3  (j = 0..3).
__device__ __forceinline__ void gemm64x256(const float* __restrict__ A, int sa, float* __restrict__ C, int sc,
                                           const float* __restrict__ Wt, const float* __restrict__ bias, int Kp,
                                           float (*Wst)[KC * 256], bool act) {
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    float acc[4][16];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[i][j] = 0.f;
    const int nchunk = Kp / KC;
    // stage 0
    {
        const float4* src = (const float4*)Wt;
#pragma unroll
        for (int i = 0; i < 4; ++i) cp_async16(&Wst[0][(tid + i * NTHREADS) * 4], src + tid + i * NTHREADS);
        cp_async_commit();
    }
    for (int c = 0; c < nchunk; ++c) {
        if (c + 1 < nchunk) {
            const float4* src = (const float4*)(Wt + (size_t)(c + 1) * KC * 256);
#pragma unroll
            for (int i = 0; i < 4; ++i) cp_async16(&Wst[(c + 1) & 1][(tid + i * NTHREADS) * 4], src + tid + i * NTHREADS);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float* Wc = Wst[c & 1];
#pragma unroll
        for (int k4 = 0; k4 < KC; k4 += 4) {
            float4 a[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = *(const float4*)&A[(ty * 4 + i) * sa + c * KC + k4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                float4 w[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) w[j] = *(const float4*)&Wc[(k4 + kk) * 256 + tx * 4 + 64 * j];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    float av = kk == 0 ? a[i].x : kk == 1 ? a[i].y : kk == 2 ? a[i].z : a[i].w;
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        acc[i][j * 4 + 0] = fmaf(av, w[j].x, acc[i][j * 4 + 0]);
                        acc[i][j * 4 + 1] = fmaf(av, w[j].y, acc[i][j * 4 + 1]);
                        acc[i][j * 4 + 2] = fmaf(av, w[j].z, acc[i][j * 4 + 2]);
                        acc[i][j * 4 + 3] = fmaf(av, w[j].w, acc[i][j * 4 + 3]);
                    }
                }
            }
        }
        __syncthreads();
    }
    // epilogue (A may alias nothing written here: C is the other buffer)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float4 b = *(const float4*)&bias[tx * 4 + 64 * j];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            float4 v;
            v.x = acc[i][j * 4 + 0] + b.x; v.y = acc[i][j * 4 + 1] + b.y;
            v.z = acc[i][j * 4 + 2] + b.z; v.w = acc[i][j * 4 + 3] + b.w;
            if (act) { v.x = lrelu(v.x); v.y = lrelu(v.y); v.z = lrelu(v.z); v.w = lrelu(v.w); }
            *(float4*)&C[(ty * 4 + i) * sc + tx * 4 + 64 * j] = v;
        }
    }
    __syncthreads();
}

// Small dense layer for the colour branch: out[s][n] = act(sum_k in[s][k] * Wt[k][n] + b[n]),  s < 8, n < Nout.
__device__ __forceinline__ void dense8(const float* __restrict__ in, int sin_, float* __restrict__ out, int sout,
                                       const float* __restrict__ Wt, const float* __restrict__ bias, int Kin, int Nout,
                                       bool act) {
    const int tid = threadIdx.x;
    // 256 threads: n = tid % 128, sample half = tid / 128 (4 samples each)
    const int n = tid & 127, s0 = (tid >> 7) * 4;
    if (n < Nout) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (int k = 0; k < Kin; ++k) {
            float w = __ldg(&Wt[(size_t)k * Nout + n]);
            a0 = fmaf(in[(s0 + 0) * sin_ + k], w, a0);
            a1 = fmaf(in[(s0 + 1) * sin_ + k], w, a1);
            a2 = fmaf(in[(s0 + 2) * sin_ + k], w, a2);
            a3 = fmaf(in[(s0 + 3) * sin_ + k], w, a3);
        }
        float b = __ldg(&bias[n]);
        a0 += b; a1 += b; a2 += b; a3 += b;
        if (act) { a0 = lrelu(a0); a1 = lrelu(a1); a2 = lrelu(a2); a3 = lrelu(a3); }
        out[(s0 + 0) * sout + n] = a0; out[(s0 + 1) * sout + n] = a1;
        out[(s0 + 2) * sout + n] = a2; out[(s0 + 3) * sout + n] = a3;
    }
    __syncthreads();
}

static_assert(offsetof(ShadeSmem, H) == sizeof(float) * TR * XS && TR * XS1 <= TR * (XS + HS), "F = 63 rows overlay X and H");

// PP: per-point frames (pts.rw2c != NULL); F: point_features_dim (32 | 63); XSAMP: explicit samples (the frustum query,
// pair_inputs.cuh); all compile-time parameters
template <bool PP, int F, bool XSAMP = false>
__global__ void __launch_bounds__(NTHREADS, 1) k_shade_fwd(ShadeParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    ShadeSmem& sm = *reinterpret_cast<ShadeSmem*>(smem_raw);
    constexpr int KP1 = kpad1_of(F), XS_1 = F == PNB_FEAT ? XS : XS1;    // block1.0 inputs: width, row stride
    float* const X1 = reinterpret_cast<float*>(smem_raw);                  // == sm.X (F = 63: over sm.H as well)
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_valid = p.q.counters[PNB_QC_N_VALID];
    const int n_tiles = (n_valid + TS - 1) / TS;
    const pnb_query_t& q = p.q;

    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        // ------------------------------------------------------------------ phase A: inputs (warp = sample)
        {
            const int vi = tile * TS + warp;
            const int k = lane >> 2, part = lane & 3;  // neighbour slot, quarter of the feature vector
            const int row = warp * PNB_MAX_K + k;
            const bool have = vi < n_valid;
            const uint32_t s = have ? q.valid_list[vi] : 0xffffffffu;
            float* xr = &X1[row * XS_1];
            if (lane == 0) sm.samp[warp] = s;
            const Fp32Pair pr = fp32_pair<PP, XSAMP>(q, p.pts, p.o, have, s, q.K, lane, &sm.view[warp][3]);
            if (lane < 3) sm.view[warp][lane] = lane == 0 ? pr.ov.x : lane == 1 ? pr.ov.y : pr.ov.z;
            if (part == 0) sm.wc[row] = pr.wc;
            if (pr.g.valid) {
                fp32_pair_row<PP, F>(p.pts, p.o, pr, lane, xr, sm.E[row]);
            } else {
                for (int c = part; c < KP1; c += 4) xr[c] = 0.f;
                if (part == 1)
                    for (int e = 0; e < 7; ++e) sm.E[row][e] = 0.f;
            }
            if (part == 1) sm.E[row][7] = 0.f;
        }
        __syncthreads();
        // ------------------------------------------------------------------ phase B: per-pair MLPs
        gemm64x256(X1, XS_1, sm.H, HS, p.mlp.w[0], p.mlp.b[0], KP1, sm.W, true);   // block1.0  7F + 60 -> 256
        gemm64x256(sm.H, HS, sm.X, XS, p.mlp.w[1], p.mlp.b[1], 256, sm.W, true);   // block1.2  256 -> 256
        for (int i = tid; i < TR * 16; i += NTHREADS) {                             // cat extras, zero pad to 272
            int row = i >> 4, c = i & 15;
            sm.X[row * XS + 256 + c] = c < 7 ? sm.E[row][c] : 0.f;
        }
        __syncthreads();
        gemm64x256(sm.X, XS, sm.H, HS, p.mlp.w[2], p.mlp.b[2], 272, sm.W, true);   // block3.0  263 -> 256
        gemm64x256(sm.H, HS, sm.X, XS, p.mlp.w[3], p.mlp.b[3], 256, sm.W, true);   // block3.2  256 -> 256
        // alpha branch: 4 lanes per row
        {
            const int row = tid >> 2, part = tid & 3;
            float a = 0.f;
            const float* wa = p.mlp.w[4];
            for (int c = part; c < 256; c += 4) a = fmaf(sm.X[row * XS + c], __ldg(&wa[c]), a);
            a += __shfl_xor_sync(0xffffffffu, a, 1);
            a += __shfl_xor_sync(0xffffffffu, a, 2);
            if (part == 0) sm.alpha[row] = softplus_m1(a + __ldg(&p.mlp.b[4][0]));
        }
        __syncthreads();
        // ------------------------------------------------------------------ phase C: K-reduction -> colour input
        for (int i = tid; i < TS * 256; i += NTHREADS) {
            int s = i >> 8, c = i & 255;
            float acc = 0.f;
#pragma unroll
            for (int k = 0; k < PNB_MAX_K; ++k) acc += sm.X[(s * PNB_MAX_K + k) * XS + c] * sm.wc[s * PNB_MAX_K + k];
            sm.H[s * HS + c] = acc;
        }
        for (int i = tid; i < TS * 24; i += NTHREADS) {
            int s = i / 24, c = i - s * 24;
            sm.H[s * HS + 256 + c] = sm.view[s][3 + c];
        }
        __syncthreads();
        // ------------------------------------------------------------------ phase D: colour branch (8 samples)
        float* B0 = sm.X;            // scratch rows (stride XS)
        float* B1 = sm.X + 8 * XS;
        dense8(sm.H, HS, B0, XS, p.mlp.w[5], p.mlp.b[5], 280, 128, true);
        dense8(B0, XS, B1, XS, p.mlp.w[6], p.mlp.b[6], 128, 128, true);
        dense8(B1, XS, B0, XS, p.mlp.w[7], p.mlp.b[7], 128, 128, true);
        dense8(B0, XS, B1, XS, p.mlp.w[8], p.mlp.b[8], 128, 3, false);
        if (tid < TS) {
            uint32_t s = sm.samp[tid];
            if (s != 0xffffffffu) {
                float sg = 0.f;
                if (p.o.agg_intrp_order == 1) {
                    // agg_intrp_order 1 (point_aggregators.py:573-587): density from the K-aggregated feature (still in sm.H)
                    const float* wa = p.mlp.w[4];
                    float a = 0.f;
                    for (int c = 0; c < 256; ++c) a = fmaf(sm.H[tid * HS + c], __ldg(&wa[c]), a);
                    sg = softplus_m1(a + __ldg(&p.mlp.b[4][0]));
                } else {
#pragma unroll
                    for (int k = 0; k < PNB_MAX_K; ++k) sg += sm.alpha[tid * PNB_MAX_K + k] * sm.wc[tid * PNB_MAX_K + k];
                }
                float4 o4;
                o4.x = sg;
                o4.y = raw2out_color(B1[tid * XS + 0]);
                o4.z = raw2out_color(B1[tid * XS + 1]);
                o4.w = raw2out_color(B1[tid * XS + 2]);
                p.sigma_rgb[s] = o4;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------ composite
struct CompositeParams {
    pnb_query_t q;
    pnb_shade_opts_t o;
    const float4* sigma_rgb;
    float* ray_color;
    float* opacity;
    float* bg_T;
    int8_t* ray_mask;
    const float* bg_ray;   // BGR: [R,3]
};

// XSAMP: explicit samples (pair_inputs.cuh); BGR: per-ray background bg_ray instead of bg_color, added as the reference's fill_invalid
// adds it (coarse_is_background * bg_ray, then + colour: each rounded, no contraction)
template <bool XSAMP = false, bool BGR = false>
__global__ void __launch_bounds__(128) k_composite(CompositeParams p) {
    int r = blockIdx.x * blockDim.x + threadIdx.x;
    const pnb_query_t& q = p.q;
    if (r >= q.R) return;
    const int SR = q.SR;
    const bool hit = q.ray_hit[r] != 0;
    if (p.ray_mask) p.ray_mask[r] = hit ? 1 : 0;
    float* op = p.opacity ? p.opacity + (size_t)r * SR : nullptr;
    if (!hit) {  // fill_invalid: background colour, zero opacity, is_background 1
        if (BGR) {
            p.ray_color[3 * r] = p.bg_ray[3 * r]; p.ray_color[3 * r + 1] = p.bg_ray[3 * r + 1]; p.ray_color[3 * r + 2] = p.bg_ray[3 * r + 2];
        } else {
            p.ray_color[3 * r] = p.o.bg_color[0]; p.ray_color[3 * r + 1] = p.o.bg_color[1]; p.ray_color[3 * r + 2] = p.o.bg_color[2];
        }
        if (p.bg_T) p.bg_T[r] = 1.0f;
        if (op) for (int j = 0; j < SR; ++j) op[j] = 0.f;
        return;
    }
    const int n = q.nsamp[r];
    const uint32_t s0 = q.samp_off[r];
    const float3 dir = XSAMP ? make_float3(0.f, 0.f, 0.f) : ray_dir(q, r);
    float cm = slot_depth<XSAMP>(q, p.o, r, n, 0, dir);  // cummax so far
    float T = 1.0f, cr = 0.f, cg = 0.f, cb = 0.f;
    for (int j = 0; j < SR; ++j) {
        float rd = ray_dist_step<XSAMP>(q, p.o, r, n, j, dir, cm);
        float sg = 0.f, rr = 0.f, gg = 0.f, bb = 0.f;
        bool valid = false;
        if (j < n && q.samp_nvalid[s0 + j] > 0) {
            float4 v = p.sigma_rgb[s0 + j];
            sg = v.x; rr = v.y; gg = v.z; bb = v.w;
            valid = true;
        }
        rd = valid ? rd : 0.f;
        float o1 = 1.0f - expf(-sg * rd);
        float bw = o1 * T;
        cr += rr * bw; cg += gg * bw; cb += bb * bw;
        T = T * (1.0f - o1 + 1e-10f);
        if (op) op[j] = o1;
    }
    if (BGR) {
        p.ray_color[3 * r] = __fadd_rn(__fmul_rn(T, p.bg_ray[3 * r]), cr);
        p.ray_color[3 * r + 1] = __fadd_rn(__fmul_rn(T, p.bg_ray[3 * r + 1]), cg);
        p.ray_color[3 * r + 2] = __fadd_rn(__fmul_rn(T, p.bg_ray[3 * r + 2]), cb);
    } else {
        p.ray_color[3 * r] = cr + p.o.bg_color[0] * T;
        p.ray_color[3 * r + 1] = cg + p.o.bg_color[1] * T;
        p.ray_color[3 * r + 2] = cb + p.o.bg_color[2] * T;
    }
    if (p.bg_T) p.bg_T[r] = T;
}

// ------------------------------------------------------------------------------------------ auxiliary training outputs
// `weight`, `conf_coefficient`, `blend_weight` of the reference's output dict (neural_points_volumetric_model.py:325-329 with
// point_aggregators.py:421-429, 727-732 and neural_points.py:706-717) in the dense [R', SR, K] layout of the R' hit rays, straight from
// the sample-compacted query: one thread per (hit ray, sample slot).  Unfilled slots follow the reference: position 0, indices -1 ->
// weight 0, and conf_coefficient = clamp(points_conf[0]) (the reference gathers with the index clamped to 0, neural_points.py:707).
struct AuxParams {
    pnb_query_t q;
    const float* xyz;
    const float* conf;
    const long long* rows;     // [n_rows] ray ids of the hit rays, ascending
    int n_rows;
    const float* opacity;      // [R, SR] as written by k_composite
    float* weight;             // [n_rows, SR, K]
    float* cc;                 // [n_rows, SR, K]
    float* blend;              // [n_rows, SR]
    const float* grad_cc;      // backward: [n_rows, SR, K]
    float* grad_conf;          // backward: [N], accumulated into
};

template <bool XSAMP = false>
__global__ void __launch_bounds__(128) k_aux_outputs(AuxParams p) {
    const pnb_query_t& q = p.q;
    const int SR = q.SR, K = q.K;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (long long)p.n_rows * SR) return;
    const int rr = (int)(idx / SR), j = (int)(idx - (long long)rr * SR);
    const int r = (int)p.rows[rr];
    const int n = q.nsamp[r];
    float3 l = make_float3(0.f, 0.f, 0.f);
    const int32_t* pid = nullptr;
    if (j < n) {
        l = slot_pos<XSAMP>(q, r, j);
        pid = q.cand_pidx + (size_t)(q.samp_off[r] + j) * K;
    }
    float w[PNB_MAX_K], wsum = 0.f;
    const float c_first = conf_coef(__ldg(p.conf));
    float* cc = p.cc + (size_t)idx * K;
    for (int k = 0; k < K; ++k) {
        const int pi = pid ? pid[k] : -1;
        w[k] = 0.f;
        float c = c_first;
        if (pi >= 0) {
            w[k] = inv_dist_weight(__ldg(&p.xyz[3 * pi]) - l.x, __ldg(&p.xyz[3 * pi + 1]) - l.y, __ldg(&p.xyz[3 * pi + 2]) - l.z);
            c = conf_coef(__ldg(&p.conf[pi]));
        }
        wsum += w[k];
        cc[k] = c;
    }
    float* wo = p.weight + (size_t)idx * K;
    for (int k = 0; k < K; ++k) wo[k] = norm_weight(w[k], wsum);
    // blend_weight = opacity * exclusive cumprod(1 - opacity + 1e-10)   (diff_ray_marching.py:536-541)
    const float* op = p.opacity + (size_t)r * SR;
    float T = 1.0f;
    for (int i = 0; i < j; ++i) T *= (1.0f - op[i] + 1e-10f);
    p.blend[idx] = op[j] * T;
}

// d loss / d points_conf through conf_coefficient: the clamp is a straight-through estimator (value clamp(c), gradient 1,
// neural_points.py:713), so every entry adds its gradient to the conf of its (clamped) index; the entries of empty slots all land on
// point 0: summed per warp first, one atomic per warp.
__global__ void __launch_bounds__(128) k_aux_conf_bwd(AuxParams p) {
    const pnb_query_t& q = p.q;
    const int SR = q.SR, K = q.K;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float g0 = 0.f;
    if (idx < (long long)p.n_rows * SR) {
        const int rr = (int)(idx / SR), j = (int)(idx - (long long)rr * SR);
        const int r = (int)p.rows[rr];
        const int32_t* pid = j < q.nsamp[r] ? q.cand_pidx + (size_t)(q.samp_off[r] + j) * K : nullptr;
        const float* g = p.grad_cc + (size_t)idx * K;
        for (int k = 0; k < K; ++k) {
            const int pi = pid ? pid[k] : -1;
            if (pi > 0) atomicAdd(&p.grad_conf[pi], g[k]);
            else g0 += g[k];
        }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) g0 += __shfl_xor_sync(0xffffffffu, g0, d);
    if ((threadIdx.x & 31) == 0 && g0 != 0.f) atomicAdd(&p.grad_conf[0], g0);
}

// ------------------------------------------------------------------------------------------ probe outputs (point growing)
// The opt.prob == 1 outputs of neural_points_volumetric_model.py:331-351, straight from the compacted query and the [R, SR] opacity
// of k_composite: one warp per ray.
//   arg-max slot oi   torch.max(opacity, -1): the first maximal slot wins a tie; slots past nsamp hold opacity 0
//   position          the sample at oi as pnb_query_export writes it (slot_t / ray_pos; 0 past nsamp)
//   weights           w_k = weight_k * conf_coefficient_k at oi, formed as k_aux_outputs forms both factors (same bits)
//   far_dist          min over the K slots of |xyz[max(pidx_k, 0)] - loc|: an empty slot measures point 0 (the reference's clamp)
//   averages          sum_k w_k * attr[max(pidx_k, 0)] in k order, lanes over the 7 + F channels (colour, dir, conf, embedding)
// rows: the R' hit rays (compacted outputs), or NULL for all R rays (full-R outputs, zeros for a ray that missed, as unmask fills
// them, :120-131).  Per-point frames play no part.
struct ProbeParams {
    pnb_query_t q;
    pnb_points_t pts;
    const long long* rows;     // [n_rows] ray ids, ascending, or NULL (row = ray)
    int n_rows;
    const float* opacity;      // [R, SR]
    float* max_opacity;        // [n_rows]
    float* max_loc;            // [n_rows, 3]
    float* far_dist;           // [n_rows]
    float* avg_color;          // [n_rows, 3]
    float* avg_dir;            // [n_rows, 3]
    float* avg_conf;           // [n_rows]
    float* avg_emb;            // [n_rows, F]
    int32_t* slot;             // [n_rows] or NULL (tests): oi
    float* weight;             // [n_rows, K] or NULL (tests): w_k
};

template <int F, bool XSAMP = false>
__global__ void __launch_bounds__(128) k_probe_outputs(ProbeParams p) {
    const pnb_query_t& q = p.q;
    const int SR = q.SR, K = q.K, lane = threadIdx.x & 31;
    const long long rr = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (rr >= p.n_rows) return;
    const int r = p.rows ? (int)p.rows[rr] : (int)rr;
    constexpr int NC = 7 + F;   // colour 3, dir 3, conf 1, embedding F
    if (!p.rows && !q.ray_hit[r]) {
        for (int c = lane; c < NC; c += 32) {
            if (c < 3) p.avg_color[rr * 3 + c] = 0.f;
            else if (c < 6) p.avg_dir[rr * 3 + c - 3] = 0.f;
            else if (c == 6) p.avg_conf[rr] = 0.f;
            else p.avg_emb[rr * F + c - 7] = 0.f;
        }
        if (lane < 3) p.max_loc[rr * 3 + lane] = 0.f;
        if (lane == 0) { p.max_opacity[rr] = 0.f; p.far_dist[rr] = 0.f; if (p.slot) p.slot[rr] = 0; }
        if (p.weight && lane < K) p.weight[rr * K + lane] = 0.f;
        return;
    }
    // first maximum: ascending slots within a lane keep the first (strict >), the butterfly keeps the lower slot of equal values
    const float* op = p.opacity + (size_t)r * SR;
    float best = -INFINITY;
    int bj = SR;
    for (int j = lane; j < SR; j += 32) {
        const float v = op[j];
        if (v > best) { best = v; bj = j; }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) {
        const float v = __shfl_xor_sync(0xffffffffu, best, d);
        const int j = __shfl_xor_sync(0xffffffffu, bj, d);
        if (v > best || (v == best && j < bj)) { best = v; bj = j; }
    }
    const int oi = bj;
    const int n = q.nsamp[r];
    float3 l = make_float3(0.f, 0.f, 0.f);
    const int32_t* pid = nullptr;
    if (oi < n) {
        l = slot_pos<XSAMP>(q, r, oi);
        pid = q.cand_pidx + (size_t)(q.samp_off[r] + oi) * K;
    }
    // the K weights and distances, every lane the same (K <= 8 points): k_aux_outputs' expressions in its k order
    const float c_first = conf_coef(__ldg(p.pts.conf));
    float w[PNB_MAX_K], c[PNB_MAX_K];
    int pi[PNB_MAX_K];
    float wsum = 0.f, far = INFINITY;
#pragma unroll
    for (int k = 0; k < PNB_MAX_K; ++k) {
        if (k >= K) break;
        const int pk = pid ? pid[k] : -1;
        pi[k] = max(pk, 0);
        const float dx = __ldg(&p.pts.xyz[3 * pi[k]]) - l.x, dy = __ldg(&p.pts.xyz[3 * pi[k] + 1]) - l.y,
                    dz = __ldg(&p.pts.xyz[3 * pi[k] + 2]) - l.z;
        w[k] = pk >= 0 ? inv_dist_weight(dx, dy, dz) : 0.f;
        c[k] = pk >= 0 ? conf_coef(__ldg(&p.pts.conf[pk])) : c_first;
        wsum += w[k];
        far = fminf(far, sqrtf(dx * dx + dy * dy + dz * dz));
    }
#pragma unroll
    for (int k = 0; k < PNB_MAX_K; ++k) {
        if (k >= K) break;
        w[k] = __fmul_rn(norm_weight(w[k], wsum), c[k]);
    }
    // lanes over channels: products rounded, then summed in k order (no contraction)
    for (int ch = lane; ch < NC; ch += 32) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < PNB_MAX_K; ++k) {
            if (k >= K) break;
            const float a = ch < 3 ? __ldg(&p.pts.color[3 * pi[k] + ch])
                          : ch < 6 ? __ldg(&p.pts.dir[3 * pi[k] + ch - 3])
                          : ch == 6 ? __ldg(&p.pts.conf[pi[k]])
                          : __ldg(&p.pts.emb[(size_t)pi[k] * F + ch - 7]);
            s = __fadd_rn(s, __fmul_rn(a, w[k]));
        }
        if (ch < 3) p.avg_color[rr * 3 + ch] = s;
        else if (ch < 6) p.avg_dir[rr * 3 + ch - 3] = s;
        else if (ch == 6) p.avg_conf[rr] = s;
        else p.avg_emb[rr * F + ch - 7] = s;
    }
    if (lane < 3) p.max_loc[rr * 3 + lane] = lane == 0 ? l.x : lane == 1 ? l.y : l.z;
    if (lane == 0) { p.max_opacity[rr] = best; p.far_dist[rr] = far; if (p.slot) p.slot[rr] = oi; }
    if (p.weight) {
#pragma unroll
        for (int k = 0; k < PNB_MAX_K; ++k)
            if (k < K && lane == k) p.weight[rr * K + k] = w[k];
    }
}

}  // namespace pnb

using namespace pnb;

extern "C" size_t pnb_shade_bytes(int cap_samples) {
    (void)cap_samples;
    return 256;
}

extern "C" int pnb_shade_forward(const pnb_query_t* q, const pnb_points_t* pts, const pnb_mlp_t* mlp,
                                 const pnb_shade_opts_t* opts, float* d_sigma_rgb, void* ws, size_t ws_bytes,
                                 pnb_stream_t stream_) {
    (void)ws; (void)ws_bytes;
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && pts && mlp && opts && d_sigma_rgb, PNB_ERR_INVALID, "pnb_shade_forward: null argument");
    PNB_REQUIRE(q->K >= 1 && q->K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED, "pnb_shade_forward: K=%d unsupported", q->K);
    for (int i = 0; i < 9; ++i)
        PNB_REQUIRE(mlp->w[i] && mlp->b[i], PNB_ERR_INVALID, "pnb_shade_forward: MLP tensor %d is null", i);
    Variant v;
    { const int rc = resolve_variant("pnb_shade_forward", pts, mlp, q, XsRule::frames, &v); if (rc) return rc; }
    ShadeParams p;
    p.q = *q; p.pts = *pts; p.mlp = *mlp; p.o = *opts; p.sigma_rgb = (float4*)d_sigma_rgb;
    const auto kern = with_frames(v, [](auto PP, auto F, auto XS) { return k_shade_fwd<PP, F, XS>; });
    int n_sm = 0;
    { const int rc = prepare_launch((const void*)kern, sizeof(ShadeSmem), &n_sm, "pnb_shade_forward"); if (rc) return rc; }
    kern<<<n_sm, NTHREADS, sizeof(ShadeSmem), stream>>>(p);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

static int composite(const pnb_query_t* q, const pnb_shade_opts_t* opts, const float* d_sigma_rgb, const float* d_bg_ray,
                     float* d_ray_color, float* d_opacity, float* d_bg_T, int8_t* d_ray_mask, cudaStream_t stream) {
    CompositeParams p;
    p.q = *q; p.o = *opts; p.sigma_rgb = (const float4*)d_sigma_rgb;
    p.ray_color = d_ray_color; p.opacity = d_opacity; p.bg_T = d_bg_T; p.ray_mask = d_ray_mask; p.bg_ray = d_bg_ray;
    const auto kern = with_bool(q->xs_loc_w != nullptr, [&](auto XS) {
        return with_bool(d_bg_ray != nullptr, [&](auto BGR) { return k_composite<XS, BGR>; });
    });
    kern<<<(q->R + 127) / 128, 128, 0, stream>>>(p);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

extern "C" int pnb_composite_forward(const pnb_query_t* q, const pnb_shade_opts_t* opts, const float* d_sigma_rgb,
                                     float* d_ray_color, float* d_opacity, float* d_bg_T, int8_t* d_ray_mask,
                                     pnb_stream_t stream_) {
    PNB_REQUIRE(q && opts && d_sigma_rgb && d_ray_color, PNB_ERR_INVALID, "pnb_composite_forward: null argument");
    return composite(q, opts, d_sigma_rgb, nullptr, d_ray_color, d_opacity, d_bg_T, d_ray_mask, (cudaStream_t)stream_);
}

extern "C" int pnb_composite_forward_bg_ray(const pnb_query_t* q, const pnb_shade_opts_t* opts, const float* d_sigma_rgb,
                                            const float* d_bg_ray, float* d_ray_color, float* d_opacity, float* d_bg_T,
                                            int8_t* d_ray_mask, pnb_stream_t stream_) {
    PNB_REQUIRE(q && opts && d_sigma_rgb && d_bg_ray && d_ray_color, PNB_ERR_INVALID, "pnb_composite_forward_bg_ray: null argument");
    return composite(q, opts, d_sigma_rgb, d_bg_ray, d_ray_color, d_opacity, d_bg_T, d_ray_mask, (cudaStream_t)stream_);
}

extern "C" int pnb_aux_outputs(const pnb_query_t* q, const pnb_points_t* pts, const long long* d_rows, int n_rows, const float* d_opacity,
                               float* d_weight, float* d_conf_coefficient, float* d_blend_weight, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && pts && d_opacity && d_weight && d_conf_coefficient && d_blend_weight, PNB_ERR_INVALID, "pnb_aux_outputs: null argument");
    PNB_REQUIRE(q->K >= 1 && q->K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED, "pnb_aux_outputs: K=%d unsupported", q->K);
    Variant v;
    { const int rc = resolve_variant("pnb_aux_outputs", pts, nullptr, q, XsRule::none, &v); if (rc) return rc; }
    if (n_rows <= 0) return PNB_OK;
    PNB_REQUIRE(d_rows, PNB_ERR_INVALID, "pnb_aux_outputs: null row list");
    AuxParams p;
    p.q = *q; p.xyz = pts->xyz; p.conf = pts->conf; p.rows = d_rows; p.n_rows = n_rows; p.opacity = d_opacity;
    p.weight = d_weight; p.cc = d_conf_coefficient; p.blend = d_blend_weight; p.grad_cc = nullptr; p.grad_conf = nullptr;
    const long long n = (long long)n_rows * q->SR;
    const auto kern = with_bool(v.xs, [](auto XS) { return k_aux_outputs<XS>; });
    kern<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(p);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

extern "C" int pnb_probe_outputs(const pnb_query_t* q, const pnb_points_t* pts, const long long* d_rows, int n_rows, const float* d_opacity,
                                 float* d_max_opacity, float* d_max_loc, float* d_far_dist, float* d_avg_color, float* d_avg_dir,
                                 float* d_avg_conf, float* d_avg_emb, int32_t* d_slot, float* d_weight, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && pts && d_opacity && d_max_opacity && d_max_loc && d_far_dist && d_avg_color && d_avg_dir && d_avg_conf && d_avg_emb,
                PNB_ERR_INVALID, "pnb_probe_outputs: null argument");
    PNB_REQUIRE(q->K >= 1 && q->K <= PNB_MAX_K, PNB_ERR_UNSUPPORTED, "pnb_probe_outputs: K=%d unsupported", q->K);
    PNB_REQUIRE(q->SR >= 1 && q->SR <= PNB_MAX_SR, PNB_ERR_UNSUPPORTED, "pnb_probe_outputs: SR=%d unsupported (1..%d)", q->SR, PNB_MAX_SR);
    Variant v;     // the check on explicit samples runs only when there are rows to launch for
    { const int rc = resolve_variant("pnb_probe_outputs", pts, nullptr, q, n_rows > 0 ? XsRule::feat63 : XsRule::none, &v); if (rc) return rc; }
    PNB_REQUIRE(d_rows || n_rows == q->R, PNB_ERR_INVALID, "pnb_probe_outputs: without a row list n_rows must be R (%d), got %d", q->R, n_rows);
    if (n_rows <= 0) return PNB_OK;
    ProbeParams p;
    p.q = *q; p.pts = *pts; p.rows = d_rows; p.n_rows = n_rows; p.opacity = d_opacity;
    p.max_opacity = d_max_opacity; p.max_loc = d_max_loc; p.far_dist = d_far_dist; p.avg_color = d_avg_color; p.avg_dir = d_avg_dir;
    p.avg_conf = d_avg_conf; p.avg_emb = d_avg_emb; p.slot = d_slot; p.weight = d_weight;
    const unsigned blocks = (unsigned)((n_rows + 3) / 4);   // 4 rays (warps) per block
    const auto kern = with_feat_xs(v, [](auto F, auto XS) { return k_probe_outputs<F, XS>; });
    kern<<<blocks, 128, 0, stream>>>(p);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

extern "C" int pnb_aux_conf_backward(const pnb_query_t* q, const long long* d_rows, int n_rows, const float* d_grad_conf_coefficient,
                                     float* d_grad_conf, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(q && d_grad_conf_coefficient && d_grad_conf, PNB_ERR_INVALID, "pnb_aux_conf_backward: null argument");
    if (n_rows <= 0) return PNB_OK;
    PNB_REQUIRE(d_rows, PNB_ERR_INVALID, "pnb_aux_conf_backward: null row list");
    AuxParams p;
    p.q = *q; p.xyz = nullptr; p.conf = nullptr; p.rows = d_rows; p.n_rows = n_rows; p.opacity = nullptr;
    p.weight = nullptr; p.cc = nullptr; p.blend = nullptr; p.grad_cc = d_grad_conf_coefficient; p.grad_conf = d_grad_conf;
    const long long n = (long long)n_rows * q->SR;
    k_aux_conf_bwd<<<(unsigned)((n + 127) / 128), 128, 0, stream>>>(p);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
