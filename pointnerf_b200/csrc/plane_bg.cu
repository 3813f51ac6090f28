// The plane background of bgmodel plane (pnb_plane_cross / pnb_plane_fg_masks / pnb_plane_bg): mvs_utils.get_rayplane_cross and
// MvsPointsVolumetricModel.set_bg (models/mvs/mvs_utils.py:299-421, models/mvs_points_volumetric_model.py:272-310) for
// pointnerf_b200.plane_bg (DESIGN.md §5 "Plane background").  One thread per ray or per (point, view); no reductions across threads,
// so every result is a function of its inputs alone.
//
// Every fp32 operation is an explicit round-to-nearest intrinsic, in this order (oracle/plane_bg_oracle.py restates it bit for bit):
//   cross      dot = (n0 d0 + n1 d1) + n2 d2;  dot >= 0.001f: p = c + d * (-((n0 w0 + n1 w1) + n2 w2) / dot), w = c - plane point;
//              otherwise p = (0, 0, 0)
//   project    c_i = ((W_i0 x + W_i1 y) + W_i2 z) + W_i3 (rows 0..2 of w2c);  (px, py, pz) = (c0 / c2, c1 / c2, c2 / c2);
//              u = (px K00 + py K01) + pz K02,  v = (px K10 + py K11) + pz K12;
//              in bounds: x, y, z finite and 0 <= u <= WD-1, 0 <= v <= HD-1 (no depth test);  cell (ceil v, ceil u)
//   sample     gx = u / ((WD-1)/2) - 1,  x = (gx + 1) * ((W-1)/2) (W: the image's width), likewise y with HD and H;
//              x0 = floor x, a = x - x0, e = 1 - a, b = y - y0, s = 1 - b;  weights nw = s e, ne = s a, sw = b e, se = b a;
//              value = ((v_nw nw + v_ne ne) + v_sw sw) + v_se se, a corner outside the image reads 0
//   fit        every channel in [c - 0.03f, c + 0.03f] (both bounds rounded to fp32), else the view gives 0
//   bg         view 0's value, then per channel: the later view's value where it is greater
#include "common.cuh"

namespace pnb {
namespace {

__device__ __forceinline__ float dot3(float a0, float a1, float a2, float b0, float b1, float b2) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a0, b0), __fmul_rn(a1, b1)), __fmul_rn(a2, b2));
}

// (u, v) of world point (x, y, z) in view g; true when it lands in bounds.  A non-finite coordinate never does: the reference's
// identity c2w product turns it into NaN in all four homogeneous components.
__device__ __forceinline__ bool project(const float* __restrict__ w2c, const float* __restrict__ K, int HD, int WD, float x, float y,
                                        float z, float* u, float* v) {
    float c[3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
        c[i] = __fadd_rn(dot3(__ldg(w2c + 4 * i), __ldg(w2c + 4 * i + 1), __ldg(w2c + 4 * i + 2), x, y, z), __ldg(w2c + 4 * i + 3));
    const float px = __fdiv_rn(c[0], c[2]), py = __fdiv_rn(c[1], c[2]), pz = __fdiv_rn(c[2], c[2]);
    *u = dot3(px, py, pz, __ldg(K + 0), __ldg(K + 1), __ldg(K + 2));
    *v = dot3(px, py, pz, __ldg(K + 3), __ldg(K + 4), __ldg(K + 5));
    return isfinite(x) && isfinite(y) && isfinite(z) && *u >= 0.f && *u <= (float)(WD - 1) && *v >= 0.f && *v <= (float)(HD - 1);
}

__global__ void __launch_bounds__(256) k_plane_cross(const float* __restrict__ campos, const float* __restrict__ raydir,
                                                     const float* __restrict__ pnt, const float* __restrict__ nrm, int R,
                                                     float* __restrict__ out) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float d0 = raydir[3 * (size_t)r], d1 = raydir[3 * (size_t)r + 1], d2 = raydir[3 * (size_t)r + 2];
    const float n0 = __ldg(nrm), n1 = __ldg(nrm + 1), n2 = __ldg(nrm + 2);
    const float c0 = __ldg(campos), c1 = __ldg(campos + 1), c2 = __ldg(campos + 2);
    const float dot = dot3(n0, n1, n2, d0, d1, d2);
    float p0 = 0.f, p1 = 0.f, p2 = 0.f;
    if (dot >= 1e-3f) {
        const float nw = dot3(n0, n1, n2, __fsub_rn(c0, __ldg(pnt)), __fsub_rn(c1, __ldg(pnt + 1)), __fsub_rn(c2, __ldg(pnt + 2)));
        const float fac = __fdiv_rn(-nw, dot);
        p0 = __fadd_rn(c0, __fmul_rn(d0, fac));
        p1 = __fadd_rn(c1, __fmul_rn(d1, fac));
        p2 = __fadd_rn(c2, __fmul_rn(d2, fac));
    }
    out[3 * (size_t)r] = p0;
    out[3 * (size_t)r + 1] = p1;
    out[3 * (size_t)r + 2] = p2;
}

// blockIdx.y: the view.  Only 1 is ever written, so concurrent writes to one cell agree.
__global__ void __launch_bounds__(256) k_plane_fg_masks(const float* __restrict__ xyz, int N, const float* __restrict__ w2c,
                                                        const float* __restrict__ K, const int32_t* __restrict__ hdwd,
                                                        const long long* __restrict__ mask_off, int8_t* __restrict__ masks) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int g = blockIdx.y;
    if (i >= N) return;
    const int HD = __ldg(hdwd + 2 * g), WD = __ldg(hdwd + 2 * g + 1);
    float u, v;
    if (project(w2c + 16 * g, K + 9 * g, HD, WD, xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2], &u, &v))
        masks[__ldg(mask_off + g) + (long long)ceilf(v) * WD + (long long)ceilf(u)] = 1;
}

__device__ __forceinline__ float texel(const float* __restrict__ p, int H, int W, int ix, int iy) {
    return (ix >= 0 && ix < W && iy >= 0 && iy < H) ? __ldg(p + (size_t)iy * W + ix) : 0.f;
}

__global__ void __launch_bounds__(256) k_plane_bg(const float* __restrict__ xyz, int R, int G, const float* __restrict__ w2c,
                                                  const float* __restrict__ K, const int32_t* __restrict__ hdwd,
                                                  const long long* __restrict__ mask_off, const int8_t* __restrict__ masks,
                                                  const float* __restrict__ img, int H, int W, const float* __restrict__ color,
                                                  float* __restrict__ bg) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const float x = xyz[3 * (size_t)r], y = xyz[3 * (size_t)r + 1], z = xyz[3 * (size_t)r + 2];
    float lo[3], hi[3], best[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        lo[c] = __fsub_rn(__ldg(color + c), 0.03f);
        hi[c] = __fadd_rn(__ldg(color + c), 0.03f);
    }
    const float sfW = (float)(W - 1) * 0.5f, sfH = (float)(H - 1) * 0.5f;   // exact: halving
    const size_t plane = (size_t)H * W;
    for (int g = 0; g < G; ++g) {
        const int HD = __ldg(hdwd + 2 * g), WD = __ldg(hdwd + 2 * g + 1);
        float s[3] = {0.f, 0.f, 0.f};
        float u, v;
        if (project(w2c + 16 * g, K + 9 * g, HD, WD, x, y, z, &u, &v) &&
            __ldg(masks + __ldg(mask_off + g) + (long long)ceilf(v) * WD + (long long)ceilf(u)) < 1) {
            const float gx = __fsub_rn(__fdiv_rn(u, (float)(WD - 1) * 0.5f), 1.f);
            const float gy = __fsub_rn(__fdiv_rn(v, (float)(HD - 1) * 0.5f), 1.f);
            const float sx = __fmul_rn(__fadd_rn(gx, 1.f), sfW), sy = __fmul_rn(__fadd_rn(gy, 1.f), sfH);
            const float x0 = floorf(sx), y0 = floorf(sy);
            const float a = __fsub_rn(sx, x0), e = __fsub_rn(1.f, a), b = __fsub_rn(sy, y0), so = __fsub_rn(1.f, b);
            const float wnw = __fmul_rn(so, e), wne = __fmul_rn(so, a), wsw = __fmul_rn(b, e), wse = __fmul_rn(b, a);
            const int ix = (int)x0, iy = (int)y0;
            float val[3];
            bool fit = true;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float* p = img + ((size_t)g * 3 + c) * plane;
                val[c] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(texel(p, H, W, ix, iy), wnw), __fmul_rn(texel(p, H, W, ix + 1, iy), wne)),
                                             __fmul_rn(texel(p, H, W, ix, iy + 1), wsw)),
                                   __fmul_rn(texel(p, H, W, ix + 1, iy + 1), wse));
                fit = fit && val[c] >= lo[c] && val[c] <= hi[c];
            }
            if (fit)
#pragma unroll
                for (int c = 0; c < 3; ++c) s[c] = val[c];
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) best[c] = (g == 0 || s[c] > best[c]) ? s[c] : best[c];
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) bg[3 * (size_t)r + c] = best[c];
}

}  // namespace
}  // namespace pnb

using namespace pnb;

extern "C" int pnb_plane_cross(const float* d_campos, const float* d_raydir, const float* d_plane_pnt, const float* d_plane_normal, int R,
                               float* d_xyz, pnb_stream_t stream) {
    PNB_REQUIRE(R >= 0, PNB_ERR_INVALID, "pnb_plane_cross: R must be >= 0 (got %d)", R);
    if (R == 0) return PNB_OK;
    PNB_REQUIRE(d_campos && d_raydir && d_plane_pnt && d_plane_normal && d_xyz, PNB_ERR_INVALID, "pnb_plane_cross: null argument");
    k_plane_cross<<<(unsigned)((R + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_campos, d_raydir, d_plane_pnt, d_plane_normal, R,
                                                                                  d_xyz);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}

extern "C" int pnb_plane_fg_masks(const float* d_xyz, int N, int G, const float* d_w2c, const float* d_K, const int32_t* d_hdwd,
                                  const long long* d_mask_off, int8_t* d_masks, size_t mask_bytes, pnb_stream_t stream_) {
    cudaStream_t stream = (cudaStream_t)stream_;
    PNB_REQUIRE(N >= 0 && G >= 1 && G <= 65535, PNB_ERR_INVALID, "pnb_plane_fg_masks: need N >= 0 and 1 <= G <= 65535 (got %d, %d)",
                N, G);
    PNB_REQUIRE(d_w2c && d_K && d_hdwd && d_mask_off && d_masks && (N == 0 || d_xyz), PNB_ERR_INVALID,
                "pnb_plane_fg_masks: null argument");
    PNB_CHECK_CUDA(cudaMemsetAsync(d_masks, 0, mask_bytes, stream));
    if (N > 0) {
        k_plane_fg_masks<<<dim3((unsigned)((N + 255) / 256), (unsigned)G), 256, 0, stream>>>(d_xyz, N, d_w2c, d_K, d_hdwd, d_mask_off,
                                                                                            d_masks);
        PNB_CHECK_CUDA(cudaGetLastError());
    }
    return PNB_OK;
}

extern "C" int pnb_plane_bg(const float* d_xyz, int R, int G, const float* d_w2c, const float* d_K, const int32_t* d_hdwd,
                            const long long* d_mask_off, const int8_t* d_masks, const float* d_img, int H, int W,
                            const float* d_plane_color, float* d_bg, pnb_stream_t stream) {
    PNB_REQUIRE(R >= 0 && G >= 1 && H >= 1 && W >= 1, PNB_ERR_INVALID,
                "pnb_plane_bg: need R >= 0, G >= 1, H >= 1, W >= 1 (got %d, %d, %d, %d)", R, G, H, W);
    if (R == 0) return PNB_OK;
    PNB_REQUIRE(d_xyz && d_w2c && d_K && d_hdwd && d_mask_off && d_masks && d_img && d_plane_color && d_bg, PNB_ERR_INVALID,
                "pnb_plane_bg: null argument");
    k_plane_bg<<<(unsigned)((R + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_xyz, R, G, d_w2c, d_K, d_hdwd, d_mask_off, d_masks,
                                                                               d_img, H, W, d_plane_color, d_bg);
    PNB_CHECK_CUDA(cudaGetLastError());
    return PNB_OK;
}
