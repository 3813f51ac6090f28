// The reference's per-pair shading inputs, defined once for every kernel that builds or reads them: the fp32 forward
// (k_shade_fwd), the tensor-core builders (k_shade_wg), the backward's recompute (k_bwd_build), and the kernels that need one
// piece (k_color_wg, k_aux_outputs, k_composite, k_composite_bwd, k_bwd_scatter, k_bwd_reduce_fwd).
//   sample position          diff_ray_marching.py:386 (world query); the frustum querier's tuple (XSAMP, below)
//   point frames (Rw2c)      neural_points.py:717, point_aggregators.py:491-496 (uniform [3,3], or per point [N,3,3]: the pair's point
//                            for dists and dir, the sample's slot-0 point for the view direction, :506, :526, :566)
//   dists / linear weights   point_aggregators.py:727-814, :421-429 (conf_coefficient: neural_points.py:706-717, :722-724)
//   block3 extras            point_aggregators.py:560-571
//   raw2out_density / _color point_aggregators.py:262-273
//   ray distances            neural_points_volumetric_model.py:271-277
// Under --fmad=true the FMA contraction follows the expression tree, so every kernel that inlines one of these expressions gets the
// same bits: the backward's recompute agrees with the fp32 forward by construction.  What deliberately differs between the kernels
// stays with them: the positional encoding (sincosf per frequency in the fp32 kernels, angle doubling on the tensor-core path) and
// the order of the weight sum (32-lane butterfly, or the tensor-core path's segmented scan).
#pragma once
#include "common.cuh"

namespace pnb {

// v @ M^T (row vector times the transpose) == M v
__device__ __forceinline__ void rot3(const float* M, float x, float y, float z, float& ox, float& oy, float& oz) {
    ox = x * M[0] + y * M[1] + z * M[2];
    oy = x * M[3] + y * M[4] + z * M[5];
    oz = x * M[6] + y * M[7] + z * M[8];
}
// M^T v
__device__ __forceinline__ void rot3T(const float* M, float x, float y, float z, float& ox, float& oy, float& oz) {
    ox = x * M[0] + y * M[3] + z * M[6];
    oy = x * M[1] + y * M[4] + z * M[7];
    oz = x * M[2] + y * M[5] + z * M[8];
}
// neural_points.py:604-610 : xyz_c[j] = sum_i shift[i] * camrotc2w[i][j];  perspective (x / z, y / z, z)
__device__ __forceinline__ void w2pers(const pnb_shade_opts_t& o, float px, float py, float pz, float& xp, float& yp, float& zp) {
    float xc, yc, zc;
    rot3T(o.camrotc2w, px - o.campos[0], py - o.campos[1], pz - o.campos[2], xc, yc, zc);
    xp = xc / zc; yp = yc / zc; zp = zc;
}
// camera-space depth of a world position (z of w2pers), rounded as the reference's torch.sum(shift[..., :, None] * camrotc2w, -2):
// each product rounded, then summed in order, never contracted to FMAs.  The ray distances are differences of these depths, and the
// raydist_mode_unit test (> 2 vsize_z) decides on their last bit where consecutive samples lie exactly 2 vsize_z apart in depth; there,
// one rounding apart replaces a step by vsize_z and moves the ray's colour by a few 1e-2 (rotated cameras; the identity's products are
// exact, so there any order gives the same bits).
__device__ __forceinline__ float cam_depth(const pnb_shade_opts_t& o, float3 x) {
    const float* M = o.camrotc2w;
    const float sx = x.x - o.campos[0], sy = x.y - o.campos[1], sz = x.z - o.campos[2];
    return __fadd_rn(__fadd_rn(__fmul_rn(sx, M[2]), __fmul_rn(sy, M[5])), __fmul_rn(sz, M[8]));
}

// ------------------------------------------------------------------------------------------ samples
__device__ __forceinline__ float3 ray_dir(const pnb_query_t& q, int r) {
    return make_float3(q.raydir[3 * r], q.raydir[3 * r + 1], q.raydir[3 * r + 2]);
}
// ray parameter of slot j of ray r
__device__ __forceinline__ float slot_t(const pnb_query_t& q, int r, int j) {
    return q.t[(size_t)r * q.t_ray_stride + q.steps[(size_t)r * q.SR + j]];
}
__device__ __forceinline__ float3 ray_pos(const pnb_query_t& q, float3 dir, float t) {
    return make_float3(raypos1(q.campos[0], dir.x, t), raypos1(q.campos[1], dir.y, t), raypos1(q.campos[2], dir.z, t));
}
// the ray of candidate sample s (samp_ray = ray << 7 | slot)
__device__ __forceinline__ int cand_ray(const pnb_query_t& q, uint32_t s) { return (int)(q.samp_ray[s] >> 7); }
// Sample source, a compile-time parameter XSAMP of every helper and kernel that reads a sample's geometry.  World query (XSAMP false):
// slot j of ray r lies at campos + raydir * t[steps], is seen along its ray's direction, and its perspective position is w2pers of
// that.  Explicit samples (XSAMP true, the perspective-frustum query, pnb_frustum_samples): the querier's [R',SR,3] tensors give the
// world position (sample_loc_w), the perspective position with its jitter (sample_loc) and the view direction (sample_ray_dirs) of
// every slot (neural_points_volumetric_model.py:268-277, point_aggregators.py:773-781).  There every slot of a hit ray is a candidate,
// so candidate s is entry s of those tensors, and slot j of ray r is entry samp_off[r] + j.
__device__ __forceinline__ float3 ld_f3(const float* v, size_t i) { return make_float3(__ldg(&v[3 * i]), __ldg(&v[3 * i + 1]), __ldg(&v[3 * i + 2])); }
struct CandSample {
    float3 dir;   // view direction: its ray's direction (XSAMP: the sample's own)
    float3 pos;   // world position
};
template <bool XSAMP = false>
__device__ __forceinline__ CandSample cand_sample(const pnb_query_t& q, uint32_t s) {
    CandSample c;
    if (XSAMP) {
        c.dir = ld_f3(q.xs_dir, s);
        c.pos = ld_f3(q.xs_loc_w, s);
        return c;
    }
    const uint32_t rj = q.samp_ray[s];
    const int r = (int)(rj >> 7);
    const float t = slot_t(q, r, (int)(rj & 127u));
    c.dir = ray_dir(q, r);
    c.pos = ray_pos(q, c.dir, t);
    return c;
}
// perspective position of candidate sample s for pair_geom: the querier's (XSAMP); the world query forms it from the world position there
template <bool XSAMP = false>
__device__ __forceinline__ float3 cand_pers(const pnb_query_t& q, uint32_t s) {
    return XSAMP ? ld_f3(q.xs_loc, s) : make_float3(0.f, 0.f, 0.f);
}
// view direction of candidate sample s
template <bool XSAMP = false>
__device__ __forceinline__ float3 cand_view_dir(const pnb_query_t& q, uint32_t s) {
    return XSAMP ? ld_f3(q.xs_dir, s) : ray_dir(q, cand_ray(q, s));
}
// world position of slot j < nsamp of ray r
template <bool XSAMP = false>
__device__ __forceinline__ float3 slot_pos(const pnb_query_t& q, int r, int j) {
    return XSAMP ? ld_f3(q.xs_loc_w, q.samp_off[r] + j) : ray_pos(q, ray_dir(q, r), slot_t(q, r, j));
}
// ------------------------------------------------------------------------------------------ point frames
// World -> canonical rotation of point pi, row-major (neural_points.Rw2c, gathered per neighbour: neural_points.py:717).  PP (per-point
// frames, a compile-time parameter of every kernel that reads a frame): row pi of pts.rw2c [N][9], read in place; otherwise the one
// uniform opts.Rw2c, and pi is not read.
template <bool PP>
__device__ __forceinline__ const float* point_frame(const pnb_points_t& pts, const pnb_shade_opts_t& o, int pi) {
    if (PP) return pts.rw2c + (size_t)pi * 9;
    return o.Rw2c;
}
// The point whose frame a sample's view direction is rotated into: its slot-0 neighbour (sampled_Rw2c[:,:,:,0], :495).  A sample
// with a neighbour always has one in slot 0; an empty slot 0 (padding) reads point 0, as the reference's clamped gather.  Uniform
// frames: no read.
template <bool PP>
__device__ __forceinline__ int view_point(const pnb_query_t& q, uint32_t s) {
    return PP ? max(q.cand_pidx[(size_t)s * q.K], 0) : 0;
}
// the view direction in the frame of point p0 (the sample's view_point) (:506)
template <bool PP>
__device__ __forceinline__ float3 view_in_points(const pnb_points_t& pts, const pnb_shade_opts_t& o, int p0, float3 dir) {
    float3 v;
    rot3(point_frame<PP>(pts, o, p0), dir.x, dir.y, dir.z, v.x, v.y, v.z);
    return v;
}

// ------------------------------------------------------------------------------------------ pairs
// inverse-distance weight of a world offset (linear :424, :427), before the normalisation over the sample's neighbours
__device__ __forceinline__ float inv_dist_weight(float dx, float dy, float dz) {
    return 1.0f / fmaxf(sqrtf(dx * dx + dy * dy + dz * dz), 1e-6f);
}
// :801-802
__device__ __forceinline__ float norm_weight(float w, float wsum) { return w / fmaxf(wsum, 1e-8f); }
// conf_coefficient: the forward value of gradiant_clamp (:722-724)
__device__ __forceinline__ float conf_coef(float conf) { return fminf(fmaxf(conf, 1e-4f), 1.0f); }

// Geometry of one (sample at l, point pidx) pair; pidx < 0 is an empty slot, read as point 0 with weight 0.
struct PairGeom {
    bool valid;
    int pi;          // point index (0 for an empty slot)
    float w;         // inverse-distance weight, not normalised
    float cc;        // conf_coefficient
    float dist[6];   // world offset + perspective terms (:782-784); the offset rotated into the point's frame
};
// l: the sample's world position; lp (XSAMP): its perspective position, which the world query forms as w2pers(l)
template <bool PP, bool XSAMP = false>
__device__ __forceinline__ PairGeom pair_geom(const pnb_points_t& pts, const pnb_shade_opts_t& o, int pidx, float3 l,
                                              float3 lp = make_float3(0.f, 0.f, 0.f)) {
    PairGeom g;
    g.valid = pidx >= 0;
    g.pi = g.valid ? pidx : 0;
    const float px = __ldg(&pts.xyz[3 * g.pi]), py = __ldg(&pts.xyz[3 * g.pi + 1]), pz = __ldg(&pts.xyz[3 * g.pi + 2]);
    const float dx = px - l.x, dy = py - l.y, dz = pz - l.z;
    float xpp, ypp, zpp, xsp, ysp, zsp;
    w2pers(o, px, py, pz, xpp, ypp, zpp);
    if (XSAMP) { xsp = lp.x; ysp = lp.y; zsp = lp.z; }
    else w2pers(o, l.x, l.y, l.z, xsp, ysp, zsp);
    g.dist[3] = xpp * zpp - xsp * zsp;
    g.dist[4] = ypp * zpp - ysp * zsp;
    g.dist[5] = zpp - zsp;
    g.w = g.valid ? inv_dist_weight(dx, dy, dz) : 0.f;
    g.cc = conf_coef(__ldg(&pts.conf[g.pi]));
    rot3(point_frame<PP>(pts, o, g.pi), dx, dy, dz, g.dist[0], g.dist[1], g.dist[2]);
    return g;
}
// block3 extras of point pi seen along the view direction ov (the sample's view frame): colour (3), dir - view (3), <dir, view> (1);
// dir is rotated into the point's own frame (:566)
template <bool PP>
__device__ __forceinline__ void point_extras(const pnb_points_t& pts, const pnb_shade_opts_t& o, int pi, float3 ov, float* ex) {
    float ddx, ddy, ddz;
    rot3(point_frame<PP>(pts, o, pi), __ldg(&pts.dir[3 * pi]), __ldg(&pts.dir[3 * pi + 1]), __ldg(&pts.dir[3 * pi + 2]), ddx, ddy, ddz);
    ex[0] = __ldg(&pts.color[3 * pi]); ex[1] = __ldg(&pts.color[3 * pi + 1]); ex[2] = __ldg(&pts.color[3 * pi + 2]);
    ex[3] = ddx - ov.x; ex[4] = ddy - ov.y; ex[5] = ddz - ov.z;
    ex[6] = ddx * ov.x + ddy * ov.y + ddz * ov.z;
}

// ------------------------------------------------------------------------------------------ outputs
// raw2out_density: Softplus(a - 1), threshold 20
__device__ __forceinline__ float softplus_m1(float a) {
    const float x = a - 1.0f;
    return x > 20.f ? x : log1pf(expf(x));
}
// raw2out_color: sigmoid scaled to (-0.001, 1.001)
__device__ __forceinline__ float raw2out_color(float x) { return 1.0f / (1.0f + expf(-x)) * (1.0f + 2.0f * 0.001f) - 0.001f; }

// ------------------------------------------------------------------------------------------ ray distances
// camera depth of slot j of ray r (n filled slots); an unfilled slot holds the world origin (SURVEY a17).  XSAMP: the z of the querier's
// sample_loc, written for every slot (an empty one sits at near - vsize_z / 2, DESIGN.md §5 F6); dir is not read.
template <bool XSAMP = false>
__device__ __forceinline__ float slot_depth(const pnb_query_t& q, const pnb_shade_opts_t& o, int r, int n, int j, float3 dir) {
    if (XSAMP) return __ldg(&q.xs_loc[3 * ((size_t)q.samp_off[r] + j) + 2]);
    if (j < n) return cam_depth(o, ray_pos(q, dir, slot_t(q, r, j)));
    return cam_depth(o, make_float3(0.f, 0.f, 0.f));
}
// Ray distance of slot j: the step of the cumulative maximum of the slot depths to slot j + 1 (vsize_z for the last slot), replaced
// by vsize_z below 1e-8 or, with raydist_mode_unit, above 2 vsize_z.  cm: the cumulative maximum up to slot j (start: slot_depth
// of slot 0), advanced to slot j + 1.
template <bool XSAMP = false>
__device__ __forceinline__ float ray_dist_step(const pnb_query_t& q, const pnb_shade_opts_t& o, int r, int n, int j, float3 dir, float& cm) {
    const float vz = o.vsize_z;
    float rd;
    if (j + 1 < q.SR) {
        const float cmn = fmaxf(cm, slot_depth<XSAMP>(q, o, r, n, j + 1, dir));
        rd = cmn - cm;
        cm = cmn;
    } else {
        rd = vz;
    }
    bool m = rd < 1e-8f;
    if (o.raydist_mode_unit > 0) m = m || (rd > 2.0f * vz);
    return m ? vz : rd;
}

// ------------------------------------------------------------------------------------------ fp32 row builder
// The pair rows of the fp32 kernels (k_shade_fwd, k_bwd_build): one warp per sample, 4 lanes per row, lane = 4 * slot + part.
// Two steps, so that a caller can store the row's scalars before the row itself (the backward's stores to global memory keep
// their order, and the scalars need not stay live across the row):
//   fp32_pair      the sample, the pair geometry and the weights; lanes 0-11 write the sample's view encoding PE4 (ori=True
//                  layout, index d*4 + j: networks.py:183): sin to vpe[0..11], cos to vpe[12..23].  have: the warp has a sample s;
//                  nk: slots k < nk are read from cand_pidx
//   fp32_pair_row  for a non-empty slot, the row's four lanes write the kpad1_of(F) block1.0 inputs to xr (features (F), PE3 of the
//                  features (6F, index F + (c*3 + j)*2 + {sin, cos}), PE5 of the dists (60, from column 7F), zeros up to 288 | 512);
//                  part 1 writes the 7 block3 extras to ex.  F = 63: emb rows are not 16-byte aligned (scalar loads), 16 channels
//                  per lane
struct Fp32Pair {
    PairGeom g;
    int pidx;
    float wn;     // normalised weight
    float wc;     // weight * conf_coefficient (0 for an empty slot)
    float3 ov;    // view direction in the sample's view frame
};
template <bool PP, bool XSAMP = false>
__device__ __forceinline__ Fp32Pair fp32_pair(const pnb_query_t& q, const pnb_points_t& pts, const pnb_shade_opts_t& o, bool have,
                                              uint32_t s, int nk, int lane, float* vpe) {
    const int k = lane >> 2, part = lane & 3;   // neighbour slot, quarter of the feature vector
    CandSample cs = {};
    float3 lp = make_float3(0.f, 0.f, 0.f);
    Fp32Pair r;
    r.pidx = -1;
    int p0 = 0;
    if (have) {
        cs = cand_sample<XSAMP>(q, s);
        if (XSAMP) lp = cand_pers<XSAMP>(q, s);
        if (k < nk) r.pidx = q.cand_pidx[(size_t)s * q.K + k];
        p0 = view_point<PP>(q, s);
    }
    r.ov = view_in_points<PP>(pts, o, p0, cs.dir);
    if (lane < 12) {
        const int dd = lane >> 2, jj = lane & 3;
        float sn, cn;
        sincosf((dd == 0 ? r.ov.x : dd == 1 ? r.ov.y : r.ov.z) * (float)(1 << jj), &sn, &cn);
        vpe[lane] = sn;
        vpe[12 + lane] = cn;
    }
    r.g = pair_geom<PP, XSAMP>(pts, o, r.pidx, cs.pos, lp);
    float wsum = part == 0 ? r.g.w : 0.f;       // sum over the 8 slots
    for (int d = 16; d > 0; d >>= 1) wsum += __shfl_xor_sync(0xffffffffu, wsum, d);
    r.wn = norm_weight(r.g.w, wsum);
    r.wc = r.g.valid ? r.wn * r.g.cc : 0.f;
    return r;
}
template <bool PP, int F = PNB_FEAT>
__device__ __forceinline__ void fp32_pair_row(const pnb_points_t& pts, const pnb_shade_opts_t& o, const Fp32Pair& r, int lane, float* xr,
                                              float* ex) {
    static_assert(F == PNB_FEAT || F == PNB_FEAT_DTU, "point_features_dim 32 or 63");
    constexpr int CPL = F == PNB_FEAT ? 8 : 16;   // channels per lane
    constexpr int DC = 7 * F;                     // first column of the distance PE
    const int part = lane & 3;
    const PairGeom& g = r.g;
    // features: this lane's channels + their PE (3 freqs)
    float f[CPL];
    if (F == PNB_FEAT) {
        const float4* ep = (const float4*)&pts.emb[(size_t)g.pi * F + part * 8];
        const float4 f0 = __ldg(ep), f1 = __ldg(ep + 1);
        f[0] = f0.x; f[1] = f0.y; f[2] = f0.z; f[3] = f0.w; f[4] = f1.x; f[5] = f1.y; f[6] = f1.z; f[7] = f1.w;
    } else {
#pragma unroll
        for (int e = 0; e < CPL; ++e) {
            const int c = part * CPL + e;
            f[e] = c < F ? __ldg(&pts.emb[(size_t)g.pi * F + c]) : 0.f;
        }
    }
#pragma unroll
    for (int e = 0; e < CPL; ++e) {
        const int c = part * CPL + e;
        if (F != PNB_FEAT && c >= F) continue;
        xr[c] = f[e];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float sn, cn;
            sincosf(f[e] * (float)(1 << j), &sn, &cn);
            xr[F + (c * 3 + j) * 2] = sn;
            xr[F + (c * 3 + j) * 2 + 1] = cn;
        }
    }
    // distance PE (5 freqs): 30 (d, j) pairs split over the 4 lanes
    const float dist[6] = {g.dist[0], g.dist[1], g.dist[2], g.dist[3], g.dist[4], g.dist[5]};
    for (int i = part; i < 30; i += 4) {
        const int dd = i / 5, jj = i - dd * 5;
        float sn, cn;
        sincosf(dist[dd] * (float)(1 << jj), &sn, &cn);
        xr[DC + i * 2] = sn;
        xr[DC + i * 2 + 1] = cn;
    }
    if (F == PNB_FEAT) {
        if (part == 0) { xr[284] = 0.f; xr[285] = 0.f; xr[286] = 0.f; xr[287] = 0.f; }
    } else {
        for (int c = DC + 60 + part; c < kpad1_of(F); c += 4) xr[c] = 0.f;
    }
    if (part == 1) point_extras<PP>(pts, o, g.pi, r.ov, ex);
}

}  // namespace pnb
