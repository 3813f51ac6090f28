// The initial point cloud's geometric steps (pnb_depth_filter_* / pnb_alpha_mask): filter_utils.filter_by_masks_gpu with
// reproject_with_depth_gpu and check_geometric_consistency_gpu, and mvs_utils.alpha_masking (models/mvs/filter_utils.py:157-291,
// models/mvs/mvs_utils.py:573-607) for pointnerf_b200.depth_filter (DESIGN.md §5 "Depth filter and visual hull").  One thread per
// (ref view, pixel) or per point; the compaction counts fixed row-major chunks and scans them, so no atomic decides an order.
//
// Matrices (formed once per call on the host, float64 from the fp32 inputs, rounded once to fp32): K_v, Kinv_v = inv(K_v),
// c2w_v = rows 0..2 of inv(E_v), pair(r, s) = rows 0..2 of E_s inv(E_r).
// Every fp32 operation is an explicit round-to-nearest intrinsic, in this order (oracle/depth_filter_oracle.py restates it bit for bit);
// dot(a, b) = (a0 b0 + a1 b1) + a2 b2, aff(A, b) = dot(A_i, b) + A_i3:
//   ref point   p = (x d, y d, d) (x, y the integer pixel as fp32, d the depth);  q = dot(Kinv_r rows, p)
//   per src s != r, ascending:
//     project   c = aff(pair(r, s), q);  k = dot(K_s rows, c);  xs = k0 / k2, ys = k1 / k2
//     sample    gx = (xs * 2) / (W - 1) - 1;  sx = (gx + 1) * ((W - 1) / 2), clamped to [0, W - 1] (border), likewise y;
//               x0 = floor sx, a = sx - x0, e = 1 - a, b = sy - y0, t = 1 - b;  weights nw = t e, ne = t a, sw = b e, se = b a;
//               ds = ((v_nw nw + v_ne ne) + v_sw sw) + v_se se, a corner outside the image reads 0
//     back      c2 = dot(Kinv_s rows, (xs ds, ys ds, ds));  e = aff(pair(s, r), c2);  dre = e2;  k = dot(K_r rows, e);
//               dx = k0 / k2 - x, dy = k1 / k2 - y
//     test      match = sqrt(dx dx + dy dy) < 1 && |dre - d| / d < 0.01f;  geo += match;  dsum = dsum + (match ? dre : 0)
//   avg = (dsum + d) / (geo + 1);  final = conf > thresh && mask && (V == 1 || geo >= geo_cnsst_num)
//   world = aff(c2w_r, (x_cam, y_cam, avg)) (x_cam, y_cam: the input's raw camera x, y);  kept: final && (no ranges ||
//   lo_j <= world_j <= hi_j for j = 0..2)
// A pixel that fails conf > thresh && mask skips the source loop: nothing it would compute is read.
//
// Visual hull, per point p and view v (all views ANDed):  c = aff(w2c_v rows 0..2, p);  near/far (when given): c2 >= lo && c2 <= hi;
//   k = dot(K_v rows, c);  ix = (int64) floor(k0 / k2), iy likewise (saturating);  in = 0 <= ix < W && 0 <= iy < H (only when the range
//   test is on);  a = alpha_v[clamp(iy, 0, H-1), clamp(ix, 0, W-1)];  test (a + (in ? 0 : 1)) > 0.1f with the range test on,
//   a > 0.1f without.
#include "common.cuh"

namespace pnb {
namespace {

constexpr int TX = 32, TY = 8;        // the consistency kernel's pixel patch: neighbouring src taps share cache lines
constexpr int SRC_CHUNK = 32;         // src views whose matrices one shared-memory stage holds
constexpr int PAIR_F = 42;            // per src: pair(r, s) 12, pair(s, r) 12, K_s 9, Kinv_s 9
constexpr int CHUNK = 1024;           // the compaction's row-major chunk (one block, one pixel per thread)
constexpr int VIEW_CHUNK = 64;        // views whose matrices one stage of the visual-hull kernel holds

__device__ __forceinline__ float dot3(const float* a, float b0, float b1, float b2) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b0), __fmul_rn(a[1], b1)), __fmul_rn(a[2], b2));
}
__device__ __forceinline__ float aff(const float* a, float b0, float b1, float b2) { return __fadd_rn(dot3(a, b0, b1, b2), a[3]); }

__device__ __forceinline__ float tap(const float* __restrict__ p, int H, int W, int ix, int iy) {
    return (ix >= 0 && ix < W && iy >= 0 && iy < H) ? __ldg(p + (size_t)iy * W + ix) : 0.f;
}

__device__ __forceinline__ void world_of(const float* __restrict__ c2w, float x, float y, float z, float* w) {
#pragma unroll
    for (int i = 0; i < 3; ++i) w[i] = aff(c2w + 4 * i, x, y, z);
}

__global__ void __launch_bounds__(TX* TY) k_consistency(int V, int H, int W, int r0, const float* __restrict__ depth,
                                                        const float* const* __restrict__ conf, const uint8_t* const* __restrict__ mask,
                                                        const float* const* __restrict__ xyz, const float* __restrict__ Kall,
                                                        const float* __restrict__ Kinv_all, const float* __restrict__ c2w_all,
                                                        const float* __restrict__ pair, const float* __restrict__ ranges, float thresh,
                                                        int geo_n, uint8_t* __restrict__ flag, float* __restrict__ avg_out) {
    __shared__ float sm[SRC_CHUNK * PAIR_F];
    const int li = blockIdx.z, r = r0 + li;
    const int x = blockIdx.x * TX + threadIdx.x, y = blockIdx.y * TY + threadIdx.y;
    const bool inside = x < W && y < H;
    const size_t HW = (size_t)H * W, pix = (size_t)y * W + x;
    float d = 0.f;
    bool live = false;
    if (inside) {
        d = __ldg(depth + (size_t)r * HW + pix);
        live = __ldg(conf[li] + pix) > thresh && __ldg(mask[li] + pix) != 0;
    }
    const float fx = (float)x, fy = (float)y;
    float Kr[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) Kr[i] = __ldg(Kall + 9 * r + i);
    float q[3];
    {
        const float p0 = __fmul_rn(fx, d), p1 = __fmul_rn(fy, d);
#pragma unroll
        for (int i = 0; i < 3; ++i) q[i] = dot3(Kinv_all + 9 * r + 3 * i, p0, p1, d);
    }
    const float sfW = (float)(W - 1) * 0.5f, sfH = (float)(H - 1) * 0.5f;   // exact: halving
    const float dW = (float)(W - 1), dH = (float)(H - 1);
    int geo = 0;
    float dsum = 0.f;
    const int tid = threadIdx.y * TX + threadIdx.x;
    const bool any_live = __syncthreads_or(live) != 0;
    for (int s0 = 0; any_live && s0 < V; s0 += SRC_CHUNK) {
        const int ns = min(SRC_CHUNK, V - s0);
        __syncthreads();
        for (int k = tid; k < ns * PAIR_F; k += TX * TY) {
            const int j = k / PAIR_F, f = k - j * PAIR_F, s = s0 + j;
            float v;
            if (f < 12) v = __ldg(pair + ((size_t)r * V + s) * 12 + f);
            else if (f < 24) v = __ldg(pair + ((size_t)s * V + r) * 12 + f - 12);
            else if (f < 33) v = __ldg(Kall + 9 * s + f - 24);
            else v = __ldg(Kinv_all + 9 * s + f - 33);
            sm[k] = v;
        }
        __syncthreads();
        if (!live) continue;
        for (int j = 0; j < ns; ++j) {
            const int s = s0 + j;
            if (s == r) continue;
            const float* A = sm + j * PAIR_F;
            const float* B = A + 12;
            const float* Ks = A + 24;
            const float* Kis = A + 33;
            const float c0 = aff(A, q[0], q[1], q[2]), c1 = aff(A + 4, q[0], q[1], q[2]), c2 = aff(A + 8, q[0], q[1], q[2]);
            const float k0 = dot3(Ks, c0, c1, c2), k1 = dot3(Ks + 3, c0, c1, c2), k2 = dot3(Ks + 6, c0, c1, c2);
            const float xs = __fdiv_rn(k0, k2), ys = __fdiv_rn(k1, k2);
            const float gx = __fsub_rn(__fdiv_rn(__fmul_rn(xs, 2.f), dW), 1.f);
            const float gy = __fsub_rn(__fdiv_rn(__fmul_rn(ys, 2.f), dH), 1.f);
            const float sx = fminf(fmaxf(__fmul_rn(__fadd_rn(gx, 1.f), sfW), 0.f), dW);
            const float sy = fminf(fmaxf(__fmul_rn(__fadd_rn(gy, 1.f), sfH), 0.f), dH);
            const float x0 = floorf(sx), y0 = floorf(sy);
            const float a = __fsub_rn(sx, x0), e = __fsub_rn(1.f, a), b = __fsub_rn(sy, y0), t = __fsub_rn(1.f, b);
            const int ix = (int)x0, iy = (int)y0;
            const float* ps = depth + (size_t)s * HW;
            const float ds = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(tap(ps, H, W, ix, iy), __fmul_rn(t, e)),
                                                           __fmul_rn(tap(ps, H, W, ix + 1, iy), __fmul_rn(t, a))),
                                                 __fmul_rn(tap(ps, H, W, ix, iy + 1), __fmul_rn(b, e))),
                                       __fmul_rn(tap(ps, H, W, ix + 1, iy + 1), __fmul_rn(b, a)));
            const float m0 = __fmul_rn(xs, ds), m1 = __fmul_rn(ys, ds);
            const float h0 = dot3(Kis, m0, m1, ds), h1 = dot3(Kis + 3, m0, m1, ds), h2 = dot3(Kis + 6, m0, m1, ds);
            const float e0 = aff(B, h0, h1, h2), e1 = aff(B + 4, h0, h1, h2), e2 = aff(B + 8, h0, h1, h2);
            const float u0 = dot3(Kr, e0, e1, e2), u1 = dot3(Kr + 3, e0, e1, e2), u2 = dot3(Kr + 6, e0, e1, e2);
            const float ddx = __fsub_rn(__fdiv_rn(u0, u2), fx), ddy = __fsub_rn(__fdiv_rn(u1, u2), fy);
            const float dist = __fsqrt_rn(__fadd_rn(__fmul_rn(ddx, ddx), __fmul_rn(ddy, ddy)));
            const float rel = __fdiv_rn(fabsf(__fsub_rn(e2, d)), d);
            const bool match = dist < 1.f && rel < 0.01f;
            geo += match;
            dsum = __fadd_rn(dsum, match ? e2 : 0.f);
        }
    }
    if (!inside) return;
    bool keep = live && (V == 1 || geo >= geo_n);
    const float avg = __fdiv_rn(__fadd_rn(dsum, d), (float)(geo + 1));
    if (keep && ranges) {
        const float* pc = xyz[li] + 3 * pix;
        float w[3];
        world_of(c2w_all + 12 * r, __ldg(pc), __ldg(pc + 1), avg, w);
#pragma unroll
        for (int j = 0; j < 3; ++j) keep = keep && w[j] >= __ldg(ranges + j) && w[j] <= __ldg(ranges + 3 + j);
    }
    flag[(size_t)li * HW + pix] = keep;
    avg_out[(size_t)li * HW + pix] = avg;
}

// blockIdx.x: chunk of view blockIdx.y
__global__ void __launch_bounds__(CHUNK) k_chunk_count(size_t HW, int ncpv, const uint8_t* __restrict__ flag, long long* __restrict__ cnt) {
    const size_t p = (size_t)blockIdx.x * CHUNK + threadIdx.x;
    const int f = p < HW ? flag[(size_t)blockIdx.y * HW + p] : 0;
    const int n = __syncthreads_count(f);
    if (threadIdx.x == 0) cnt[(size_t)blockIdx.y * ncpv + blockIdx.x] = n;
}

// One block: off[i] = sum of cnt[0..i), off[n] = the total.  Each thread scans a contiguous run, then the runs' totals are scanned.
__global__ void __launch_bounds__(1024) k_scan(const long long* __restrict__ cnt, long long n, long long* __restrict__ off) {
    __shared__ long long part[1024];
    const long long per = (n + 1023) / 1024, b = threadIdx.x * per, e = min(n, b + per);
    long long s = 0;
    for (long long i = b; i < e; ++i) s += cnt[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int k = 1; k < 1024; k <<= 1) {
        const long long v = threadIdx.x >= k ? part[threadIdx.x - k] : 0;
        __syncthreads();
        part[threadIdx.x] += v;
        __syncthreads();
    }
    long long run = threadIdx.x ? part[threadIdx.x - 1] : 0;
    for (long long i = b; i < e; ++i) {
        off[i] = run;
        run += cnt[i];
    }
    if (threadIdx.x == 1023) off[n] = part[1023];
}

__global__ void __launch_bounds__(CHUNK) k_scatter(size_t HW, int ncpv, int r0, const uint8_t* __restrict__ flag,
                                                   const float* __restrict__ avg, const long long* __restrict__ off,
                                                   const float* const* __restrict__ xyz, const float* const* __restrict__ conf,
                                                   const float* __restrict__ c2w_all, float* __restrict__ out_cam,
                                                   float* __restrict__ out_world, float* __restrict__ out_conf) {
    __shared__ int wsum[CHUNK / 32];
    const int li = blockIdx.y;
    const size_t p = (size_t)blockIdx.x * CHUNK + threadIdx.x;
    const bool f = p < HW && flag[(size_t)li * HW + p];
    const unsigned bal = __ballot_sync(0xffffffffu, f);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) wsum[wid] = __popc(bal);
    __syncthreads();
    if (!f) return;
    int before = __popc(bal & ((1u << lane) - 1u));
    for (int k = 0; k < wid; ++k) before += wsum[k];
    const long long o = off[(size_t)li * ncpv + blockIdx.x] + before;
    const float* pc = xyz[li] + 3 * p;
    const float x = __ldg(pc), y = __ldg(pc + 1), z = avg[(size_t)li * HW + p];
    float w[3];
    world_of(c2w_all + 12 * (r0 + li), x, y, z, w);
    out_cam[3 * o] = x;
    out_cam[3 * o + 1] = y;
    out_cam[3 * o + 2] = z;
    out_world[3 * o] = w[0];
    out_world[3 * o + 1] = w[1];
    out_world[3 * o + 2] = w[2];
    out_conf[o] = __ldg(conf[li] + p);
}

__global__ void __launch_bounds__(256) k_alpha_mask(const float* __restrict__ pts, long long N, int V, const float* __restrict__ w2c,
                                                    const float* __restrict__ K, const float* __restrict__ alpha, int H, int W,
                                                    int use_near_far, float lo, float hi, int range_test, uint8_t* __restrict__ out) {
    __shared__ float sm[VIEW_CHUNK * 21];
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float x = 0.f, y = 0.f, z = 0.f;
    if (i < N) {
        x = pts[3 * i];
        y = pts[3 * i + 1];
        z = pts[3 * i + 2];
    }
    bool keep = i < N;
    const size_t HW = (size_t)H * W;
    for (int v0 = 0; v0 < V; v0 += VIEW_CHUNK) {
        const int nv = min(VIEW_CHUNK, V - v0);
        __syncthreads();
        for (int k = threadIdx.x; k < nv * 21; k += blockDim.x) {
            const int j = k / 21, f = k - j * 21;
            sm[k] = f < 12 ? __ldg(w2c + 12 * (v0 + j) + f) : __ldg(K + 9 * (v0 + j) + f - 12);
        }
        __syncthreads();
        for (int j = 0; keep && j < nv; ++j) {
            const float* A = sm + 21 * j;
            const float c0 = aff(A, x, y, z), c1 = aff(A + 4, x, y, z), c2 = aff(A + 8, x, y, z);
            const bool nf = !use_near_far || (c2 >= lo && c2 <= hi);
            const float k0 = dot3(A + 12, c0, c1, c2), k1 = dot3(A + 15, c0, c1, c2), k2 = dot3(A + 18, c0, c1, c2);
            const long long ix = (long long)floorf(__fdiv_rn(k0, k2)), iy = (long long)floorf(__fdiv_rn(k1, k2));
            const bool in = ix >= 0 && ix < W && iy >= 0 && iy < H;
            const long long cx = ix < 0 ? 0 : ix > W - 1 ? W - 1 : ix, cy = iy < 0 ? 0 : iy > H - 1 ? H - 1 : iy;
            float a = __ldg(alpha + (size_t)(v0 + j) * HW + (size_t)cy * W + cx);
            if (range_test) a = __fadd_rn(a, in ? 0.f : 1.f);
            keep = nf && a > 0.1f;
        }
    }
    if (i < N) out[i] = keep;
}

struct Ws {
    uint8_t* flag;
    float* avg;
    long long* cnt;
    long long* off;
};

size_t ws_layout(int nr, int H, int W, void* base, Ws* w) {
    const size_t HW = (size_t)H * W, ncpv = (HW + CHUNK - 1) / CHUNK, n = (size_t)nr * ncpv;
    size_t o = 0;
    char* b = (char*)base;
    if (w) w->flag = (uint8_t*)(b + o);
    o = align_up(o + (size_t)nr * HW);
    if (w) w->avg = (float*)(b + o);
    o = align_up(o + (size_t)nr * HW * 4);
    if (w) w->cnt = (long long*)(b + o);
    o = align_up(o + n * 8);
    if (w) w->off = (long long*)(b + o);
    return align_up(o + (n + 1) * 8);
}

}  // namespace
}  // namespace pnb

using namespace pnb;

extern "C" size_t pnb_depth_filter_bytes(int nr, int H, int W) {
    if (nr < 1 || H < 1 || W < 1) return 0;
    return ws_layout(nr, H, W, nullptr, nullptr);
}

extern "C" int pnb_depth_filter_build(void* ws, size_t ws_bytes, int V, int H, int W, int r0, int nr, const float* d_depth,
                                      const float* const* d_conf, const uint8_t* const* d_mask, const float* const* d_xyz,
                                      const float* d_K, const float* d_Kinv, const float* d_c2w, const float* d_pair,
                                      const float* d_ranges, float conf_thresh, int geo_cnsst_num, pnb_stream_t stream_,
                                      long long* h_counts) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(V >= 1 && H >= 2 && W >= 2 && nr >= 1 && r0 >= 0 && r0 + nr <= V && nr <= 65535, PNB_ERR_INVALID,
                "pnb_depth_filter_build: need V >= 1, H, W >= 2 and 0 <= r0 < r0 + nr <= V, nr <= 65535 (got %d, %d, %d, %d, %d)", V, H, W,
                r0, nr);
    PNB_REQUIRE(ws && d_depth && d_conf && d_mask && d_xyz && d_K && d_Kinv && d_c2w && d_pair && h_counts, PNB_ERR_INVALID,
                "pnb_depth_filter_build: null argument");
    Ws w;
    const size_t need = ws_layout(nr, H, W, ws, &w);
    PNB_REQUIRE(ws_bytes >= need, PNB_ERR_WORKSPACE, "pnb_depth_filter_build: workspace %zu < %zu bytes", ws_bytes, need);
    const size_t HW = (size_t)H * W;
    const int ncpv = (int)((HW + CHUNK - 1) / CHUNK);
    const long long n = (long long)nr * ncpv;
    k_consistency<<<dim3((unsigned)((W + TX - 1) / TX), (unsigned)((H + TY - 1) / TY), (unsigned)nr), dim3(TX, TY), 0, stream>>>(
        V, H, W, r0, d_depth, d_conf, d_mask, d_xyz, d_K, d_Kinv, d_c2w, d_pair, d_ranges, conf_thresh, geo_cnsst_num, w.flag, w.avg);
    PNB_CHECK_CUDA(cudaGetLastError());
    k_chunk_count<<<dim3((unsigned)ncpv, (unsigned)nr), CHUNK, 0, stream>>>(HW, ncpv, w.flag, w.cnt);
    PNB_CHECK_CUDA(cudaGetLastError());
    k_scan<<<1, 1024, 0, stream>>>(w.cnt, n, w.off);
    PNB_CHECK_CUDA(cudaGetLastError());
    std::vector<long long> bound((size_t)nr + 1);
    PNB_CHECK_CUDA(cudaMemcpy2DAsync(bound.data(), sizeof(long long), w.off, (size_t)ncpv * sizeof(long long), sizeof(long long),
                                     (size_t)nr + 1, cudaMemcpyDeviceToHost, stream));
    PNB_CHECK_CUDA(cudaStreamSynchronize(stream));
    for (int i = 0; i < nr; ++i) h_counts[i] = bound[i + 1] - bound[i];
    return PNB_OK;
}

extern "C" int pnb_depth_filter_outputs(const void* ws, size_t ws_bytes, int H, int W, int r0, int nr, const float* const* d_xyz,
                                        const float* const* d_conf, const float* d_c2w, float* d_xyz_cam, float* d_xyz_world,
                                        float* d_conf_out, pnb_stream_t stream) {
    PNB_REQUIRE(H >= 2 && W >= 2 && nr >= 1 && nr <= 65535 && r0 >= 0, PNB_ERR_INVALID,
                "pnb_depth_filter_outputs: need H, W >= 2, 1 <= nr <= 65535, r0 >= 0 (got %d, %d, %d, %d)", H, W, nr, r0);
    PNB_REQUIRE(ws && d_xyz && d_conf && d_c2w && d_xyz_cam && d_xyz_world && d_conf_out, PNB_ERR_INVALID,
                "pnb_depth_filter_outputs: null argument");
    Ws w;
    const size_t need = ws_layout(nr, H, W, (void*)ws, &w);
    PNB_REQUIRE(ws_bytes >= need, PNB_ERR_WORKSPACE, "pnb_depth_filter_outputs: workspace %zu < %zu bytes", ws_bytes, need);
    const size_t HW = (size_t)H * W;
    const int ncpv = (int)((HW + CHUNK - 1) / CHUNK);
    k_scatter<<<dim3((unsigned)ncpv, (unsigned)nr), CHUNK, 0, (cudaStream_t)stream>>>(HW, ncpv, r0, w.flag, w.avg, w.off, d_xyz, d_conf,
                                                                                     d_c2w, d_xyz_cam, d_xyz_world, d_conf_out);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

extern "C" int pnb_alpha_mask(const float* d_points, long long N, int V, const float* d_w2c, const float* d_K, const float* d_alpha,
                              int H, int W, const float* h_near_far, int range_test, uint8_t* d_mask, pnb_stream_t stream) {
    PNB_REQUIRE(N >= 0 && V >= 1 && H >= 1 && W >= 1, PNB_ERR_INVALID,
                "pnb_alpha_mask: need N >= 0, V >= 1, H >= 1, W >= 1 (got %lld, %d, %d, %d)", N, V, H, W);
    if (N == 0) return PNB_OK;
    PNB_REQUIRE(d_points && d_w2c && d_K && d_alpha && d_mask, PNB_ERR_INVALID, "pnb_alpha_mask: null argument");
    PNB_REQUIRE((N + 255) / 256 <= 0x7fffffffLL, PNB_ERR_INVALID, "pnb_alpha_mask: N = %lld is too large", N);
    k_alpha_mask<<<(unsigned)((N + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        d_points, N, V, d_w2c, d_K, d_alpha, H, W, h_near_far != nullptr, h_near_far ? h_near_far[0] : 0.f,
        h_near_far ? h_near_far[1] : 0.f, range_test, d_mask);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
