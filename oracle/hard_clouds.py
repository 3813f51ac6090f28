"""TEST INFRASTRUCTURE ONLY -- seeded adversarial inputs for the two neighbour queries: the world query (wcoord_query -1, oracle/query_oracle.c,
csrc/grid.cu + csrc/query.cu) and the perspective-frustum query (wcoord_query 0 / NN 2, oracle/frustum_oracle.c, csrc/frustum.cu).  The CPU
tests of the C oracles and the GPU tests of libpnb200 share them.

A smooth random cloud never reaches the inputs where a query is decided by one integer or IEEE choice.  The families here do:
  ties        dyadic lattice points, rays whose directions have exact zero components and a dyadic t table: samples land on lattice planes
              and candidate distances tie exactly, often four ways;
  ties1       the same with one point per voxel (at its centre): no in-voxel order exists, so even a kernel that fills voxels with
              atomics (the reference's) visits candidates in one order;
  duplicates  a random cloud with about 10 % of its points copied to new indices, some below their source and some above;
  faces       coordinates whose (p - lo) / svs is an integer and their float neighbours on either side, on every axis; p = lo, the upper
              face lo + dim * svs (outside) and one ulp inside it; coordinates where the IEEE divide and a multiply by 1 / svs floor to
              different voxels.  Frustum: the truncation band -1 < q < 0 (and q = -1, q = 0) and columns whose only dilated voxel is depth 0;
  crowded     voxels with exactly P, P + 1 and 3 P points, and a centre voxel with more than K points;
  slot0       (world) the lowest in-range index sits next to the samples, and the first indices lie outside the grid;
  empty       N = 1 and all points outside the grid: every ray misses;
  radius      lattice points at exactly d^2 == r^2 (frustum: z^2 == depth^2 as well).

Every function is deterministic in its arguments.  Hand-built tie cases (world_hand_cases, frustum_hand_cases) carry the slots derived by
hand from the reference's replace-farthest rule (query_worldcoords.cu:276-293, query_point_indices.py:574-591).
"""
import numpy as np

f32 = np.float32

WORLD_FAMILIES = ("ties", "ties1", "duplicates", "faces", "crowded", "slot0", "empty", "radius")
FRUSTUM_FAMILIES = ("ties", "ties1", "duplicates", "faces", "crowded", "empty", "radius")
# (kernel_size, query_size) pairs pnb_frustum_build accepts (the query_size box covers the layered search): cubic, anisotropic, a
# one-voxel kernel, even query sizes, and query_size[2] <= 2 where a point in depth 0 dilates to depth 0 only (ray_mask 0, F4)
FRUSTUM_SIZES = (((3, 3, 3), (3, 3, 3)), ((5, 5, 5), (5, 5, 5)), ((3, 3, 1), (3, 3, 3)), ((5, 5, 3), (5, 5, 5)), ((1, 1, 1), (3, 3, 3)),
                 ((3, 3, 3), (4, 4, 4)), ((3, 3, 1), (4, 4, 2)), ((3, 3, 1), (3, 3, 1)), ((2, 2, 2), (2, 2, 2)))


def ulps(v, n):
    """v moved n float32 ulps (n < 0: down), through the ordered integer image of the fp32 bits."""
    i = int(np.array(v, f32).view(np.int32))
    o = (i if i >= 0 else -(i & 0x7fffffff)) + int(n)
    b = o if o >= 0 else (-o) | 0x80000000
    return np.array(b & 0xffffffff, np.uint32).view(f32)[()]


def vox_div(p, lo, svs):
    """(int)floorf((p - lo) / svs) with the IEEE fp32 subtract and divide of the kernels."""
    return np.floor((np.asarray(p, f32) - np.asarray(lo, f32)).astype(f32) / np.asarray(svs, f32)).astype(np.int64)


def vox_mul(p, lo, svs):
    """The same with a multiply by the fp32 reciprocal: what a fast-math build would compute instead."""
    r = (f32(1) / np.asarray(svs, f32)).astype(f32)
    return np.floor(((np.asarray(p, f32) - np.asarray(lo, f32)).astype(f32) * r).astype(f32)).astype(np.int64)


def face_values(lo, svs, dim, spread=2):
    """Per axis: lo + k * svs for k = 0..dim, each with its float neighbours up to `spread` ulps either side, plus every coordinate of
    the axis range where the IEEE divide and the reciprocal multiply give different voxels."""
    out = []
    for a in range(3):
        vals = set()
        for k in range(int(dim[a]) + 1):
            v = f32(f32(lo[a]) + f32(k) * f32(svs[a]))
            for u in range(-spread, spread + 1):
                vals.add(float(ulps(v, u)))
            for u in range(-40, 41):             # the reciprocal multiply drifts by a few ulps: search wider for discriminators
                w = ulps(v, u)
                if vox_div(w, lo[a], svs[a]) != vox_mul(w, lo[a], svs[a]):
                    vals.add(float(w))
        out.append(np.array(sorted(vals), f32))
    return out


# ---------------------------------------------------------------------------------------------------------------- world query
def world_grid(lo, vsize, vscale, extent):
    """scaled voxel size (vsize * vscale in float64, then fp32, point_query.py:36) and the voxel count covering `extent`."""
    v = np.asarray(vsize, np.float64) * np.asarray(vscale, np.int32)
    return np.asarray(lo, f32), v.astype(f32), np.ceil(np.asarray(extent, np.float64) / v).astype(np.int32)


def _lattice(g, lo, h, n, p):
    idx = np.stack(np.meshgrid(*[np.arange(k) for k in n], indexing="ij"), -1).reshape(-1, 3)
    idx = idx[g.random_sample(len(idx)) < p]
    return (np.asarray(lo, f32) + idx.astype(f32) * np.asarray(h, f32)).astype(f32)


def world_scene(family, vsize=(0.5, 0.5, 0.5), vscale=(1, 1, 1), P=4, K=8, seed=0):
    """dict(name, xyz [N,3], lo, svs, dim, campos [3], raydir [R,3], t [D], radius, max_o).  The grid spans 8 x 8 x 37 voxels of vsize
    (vscale 1: dim[2] = 37 is not a multiple of 32, so a column's cells straddle bit words)."""
    g = np.random.RandomState(seed + 17 * WORLD_FAMILIES.index(family))
    v = np.asarray(vsize, f32)
    h = (v / 2).astype(f32)
    lo = np.array([-2.0, -2.0, -1.0], f32)
    extent = v.astype(np.float64) * np.array([8, 8, 37])
    lo, svs, dim = world_grid(lo, v, vscale, extent)
    hi = (lo + extent).astype(f32)
    # rays: one shared camera below the grid; directions (i/8, j/8, 1) have exact zero components on the axes, plus two that miss
    campos = np.array([lo[0] + 8 * h[0] + h[0] / 2, lo[1] + 8 * h[1], lo[2] - v[2]], f32)
    ij = [(i, j) for i in range(-3, 5) for j in range(-3, 5)]
    raydir = np.array([(i / 8.0, j / 8.0, 1.0) for i, j in ij] + [(0, 0, -1), (1, 0, 0)], f32)
    t = (np.arange(1, 321, dtype=np.float64) / 16.0 * h[2] / 0.25).astype(f32)      # dyadic: samples on lattice planes
    radius = 0.0
    if family in ("ties", "radius"):
        xyz = _lattice(g, lo, h, (16, 16, 74), 0.12)
        if family == "radius":
            campos[0] = lo[0] + 8 * h[0]                 # samples of the axis ray on lattice nodes
            radius = float(2 * h[0]) if h[0] == h[1] == h[2] else float(2 * min(h))
            # and, for the first three in-grid samples of every ray (formed as the kernels form them), points at exactly the radius
            # along each axis: p - s = +-r is exact for these dyadic values, so d^2 == r^2 in fp32
            r = f32(radius)
            extra = []
            for d in raydir:
                s = (campos + (d[None] * t[:, None]).astype(f32)).astype(f32)
                c = vox_div(s, lo, svs)
                for si in s[np.all((c >= 0) & (c < dim), 1)][:3]:
                    for a in range(3):
                        for sg in (-1, 1):
                            q = si.copy()
                            q[a] = f32(q[a] + sg * r)
                            extra.append(q)
            xyz = np.concatenate([xyz, np.array(extra, f32).reshape(-1, 3)])
            xyz = xyz[g.permutation(len(xyz))]
    elif family == "ties1":
        xyz = _lattice(g, lo + svs / 2, svs, dim, 0.5)
    elif family == "duplicates":
        # around the bundle of rays, so that most samples have candidates and copies meet at the K-th distance
        axis = np.array([campos[0], campos[1], lo[2]], np.float64)
        span = np.array([3 * v[0], 3 * v[1], hi[2] - lo[2]], np.float64)
        base = (axis + (g.random_sample((600, 3)) - [0.5, 0.5, 0.0]) * span).astype(f32)
        src = g.choice(len(base), len(base) // 10, replace=False)
        xyz = np.concatenate([base, base[src]])
        xyz = xyz[g.permutation(len(xyz))]
        campos = (campos + f32(0.013)).astype(f32)
        raydir = (raydir + (g.random_sample(raydir.shape) - 0.5) * 0.01).astype(f32)
        t = (t + f32(0.0021)).astype(f32)
    elif family == "faces":
        fv = face_values(lo, svs, dim)
        pts = []
        for a in range(3):
            for val in fv[a]:
                q = lo + g.random_sample(3) * (hi - lo)
                q[a] = val
                pts.append(q)
        pts += [lo.copy(), (lo + dim * svs).astype(f32),
                np.array([ulps(lo[0] + dim[0] * svs[0], -1), ulps(lo[1] + dim[1] * svs[1], -1), ulps(lo[2] + dim[2] * svs[2], -1)], f32)]
        xyz = np.array(pts, f32)
        # samples on faces: the ray through campos along z sits on an x face; the t table puts samples on z faces and one ulp either side
        campos = np.array([lo[0] + 4 * svs[0], lo[1] + 3 * svs[1], lo[2] - svs[2]], f32)
        zf = fv[2] - campos[2]
        t = np.unique(np.concatenate([zf[zf > 0], (g.random_sample(40) * (hi[2] - campos[2])).astype(f32)])).astype(f32)
    elif family == "crowded":
        cx, cy = int(dim[0]) // 2, int(dim[1]) // 2
        zs = [int(dim[2] * f) for f in (0.1, 0.25, 0.4, 0.55, 0.7, 0.85)]
        cells = [(cx, cy, zs[0], P), (cx, cy, zs[1], P + 1), (cx, cy, zs[2], 3 * P), (cx, cy, zs[3], K + 3), (cx - 1, cy, zs[4], 3 * P),
                 (cx, cy, zs[5], 1)]
        pts = [(lo + g.random_sample((60, 3)) * (hi - lo)).astype(f32)]
        for x, y, z, n in cells:
            pts.append((lo + (np.array([x, y, z]) + g.random_sample((n, 3))) * svs).astype(f32))
        xyz = np.concatenate(pts)[g.permutation(60 + sum(c[3] for c in cells))]
        campos = np.array([lo[0] + (cx + 0.5) * svs[0], lo[1] + (cy + 0.5) * svs[1], lo[2] - v[2]], f32)
    elif family == "slot0":
        out = np.array([lo - 1.0, hi + 2.0 * svs, [lo[0], hi[1] + 2.0 * svs[1], lo[2]]], f32)        # indices 0..2 outside the grid
        first = (campos + np.array([h[0] / 3, 0, 4 * v[2]], f32)).astype(f32)        # index 3: the dead voxel, on the axis ray
        rest = (campos + (g.random_sample((400, 3)) - [0.5, 0.5, 0.0]) * [4 * v[0], 4 * v[1], 14 * v[2]]).astype(f32)
        xyz = np.concatenate([out, first[None], rest]).astype(f32)
    elif family == "empty":
        xyz = np.concatenate([(hi + 1.0)[None], (lo - g.random_sample((40, 3)) - 0.5)]).astype(f32)
    else:
        raise ValueError(family)
    xyz = np.ascontiguousarray(xyz, f32)
    return dict(name="world_%s" % family, xyz=xyz, lo=lo, svs=svs, dim=dim, campos=campos, raydir=np.ascontiguousarray(raydir, f32),
                t=np.ascontiguousarray(t, f32), radius=radius, max_o=max(len(xyz), 1))


def world_hand_cases():
    """Eviction among tied distances, derived by hand from query_worldcoords.cu:276-293 (replace-farthest, strict '<', rescan keeping
    the FIRST maximum with a strict '>').  8^3 grid of voxel 1 at lo 0, one sample at (4.5, 4.5, 4.5) (ray along +z), kernel 3 (layers 0
    and 1, x-major then y then z), no radius limit.  Point 0 sits in a far voxel: it wins occupancy slot 0, which holds no points."""
    park = (0.5, 0.5, 0.5)
    cases = [
        # the fill keeps the first maximum (strict '>'): B and D tie at 1, E (0.81) evicts B, slot 0
        dict(name="evict_first_of_tied_fill", K=2, pts=[park, (3.5, 4.5, 4.5), (4.5, 3.5, 4.5), (4.5, 4.5, 5.4)], want=[3, 2]),
        # a later candidate equal to the farthest does not replace it (strict '<')
        dict(name="equal_does_not_replace", K=2, pts=[park, (4.5, 4.5, 4.75), (3.5, 4.5, 4.5), (4.5, 4.5, 5.5)], want=[1, 2]),
        # after a replacement the rescan keeps the FIRST of two tied maxima (slot 1, not slot 2), so E evicts A
        dict(name="rescan_keeps_first_max", K=3,
             pts=[park, (3.5, 3.5, 4.5), (3.5, 4.5, 4.5), (4.5, 3.5, 4.5), (4.5, 4.5, 5.0), (5.2, 4.5, 4.5)], want=[4, 5, 3]),
        # a 4-way tie in one voxel shell, K = 1: the first visited of the four stays
        dict(name="four_way_tie_k1", K=1, pts=[park, (4.5, 5.5, 4.5), (3.5, 4.5, 4.5), (5.5, 4.5, 4.5), (4.5, 3.5, 4.5)], want=[2]),
    ]
    for c in cases:
        c.update(xyz=np.array(c.pop("pts"), f32), lo=np.zeros(3, f32), svs=np.ones(3, f32), dim=np.array([8, 8, 8], np.int32),
                 campos=np.array([4.5, 4.5, -10.0], f32), raydir=np.array([[0, 0, 1]], f32), t=np.array([14.5], f32), ks=(3, 3, 3))
    return cases


# ---------------------------------------------------------------------------------------------------------------- frustum query
def frustum_camera(W=32, H=16, z_depth_dim=40, dz=1 / 16):
    """A camera whose frustum grid is dyadic: x, y in [-1, 1], depth [1, 1 + z_depth_dim * dz]; vsize (2/W, 2/H, dz)."""
    intrinsic = np.array([[W / 2, 0, W / 2], [0, H / 2, H / 2], [0, 0, 1]], f32)
    return dict(W=W, H=H, intrinsic=intrinsic, near=f32(1.0), far=f32(1.0 + z_depth_dim * dz), z_depth_dim=z_depth_dim)


def frustum_opt(vscale=(2, 2, 1), ks=(3, 3, 3), qs=(3, 3, 3), SR=24, K=8, P=8, radius_limit_scale=0.0, depth_limit_scale=0.0,
                z_depth_dim=40, max_o=None):
    from types import SimpleNamespace
    return SimpleNamespace(inverse=0, NN=2, K=K, SR=SR, P=P, max_o=max_o, z_depth_dim=z_depth_dim, vscale=list(vscale),
                           kernel_size=list(ks), query_size=list(qs), radius_limit_scale=radius_limit_scale,
                           depth_limit_scale=depth_limit_scale, gpu_maxthr=1024, is_train=False, shpnt_jitter="uniform", wcoord_query=0)


def frustum_grid(cam, opt):
    from pointnerf_b200 import query_point_indices as qpi
    return qpi.hyperparameters(opt, np.int64(cam["H"]), np.int64(cam["W"]), cam["intrinsic"], cam["near"], cam["far"])


def frustum_pixels(cam, vscale):
    """Every pixel (y outer), so every column of the grid has a ray, plus three outside the grid."""
    px, py = np.meshgrid(np.arange(cam["W"]), np.arange(cam["H"]))
    pix = np.stack((px, py), -1).reshape(-1, 2)
    sx = -(-cam["W"] // vscale[0]) * vscale[0]
    return np.concatenate([pix, [[-1, 3], [sx, 2], [3, cam["H"] + 7]]]).astype(np.int32)


def frustum_scene(family, opt, seed=0):
    """dict(name, pers [N,3], cam, pixel_idx [R,2]) for the options `opt` (vscale, P, K, depth limit shape the family)."""
    g = np.random.RandomState(seed + 31 * FRUSTUM_FAMILIES.index(family))
    cam = frustum_camera(z_depth_dim=opt.z_depth_dim)
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = frustum_grid(cam, opt)
    lo, hi = ranges[:3].astype(f32), ranges[3:].astype(f32)
    h = (vsize / 2).astype(f32)
    if family in ("ties", "radius"):
        # a dense lattice slab through the middle depths: every search box holds equidistant pairs
        n = np.round((hi - lo) / h).astype(int)
        z0 = int(n[2]) // 3
        pers = _lattice(g, lo + np.array([0, 0, z0], f32) * h, h, (n[0], n[1], int(n[2]) // 3), 0.08)
        if family == "radius":
            # z exactly depth_limit from sample depths: samples sit at lo + (fz + 0.5) * svs
            m = max(len(pers) // 8, 1)
            cols = g.randint(0, sdim[0], m), g.randint(0, sdim[1], m), g.randint(0, sdim[2], m)
            cz = (lo[2] + (cols[2] + 0.5) * svs[2]).astype(f32)
            cx = (lo[0] + (cols[0] + 0.5) * svs[0]).astype(f32)
            cy = (lo[1] + (cols[1] + 0.5) * svs[1]).astype(f32)
            sgn = np.where(g.random_sample(m) < 0.5, -1.0, 1.0)
            extra = np.stack([cx, cy, (cz + sgn * f32(dl)).astype(f32)], -1).astype(f32)
            pers = np.concatenate([pers, extra])[g.permutation(len(pers) + m)]
    elif family == "ties1":
        pers = _lattice(g, lo + svs / 2, svs, sdim, 0.3)
    elif family == "duplicates":
        base = (lo + g.random_sample((2500, 3)) * (hi - lo)).astype(f32)
        src = g.choice(len(base), len(base) // 10, replace=False)
        pers = np.concatenate([base, base[src]])
        pers = pers[g.permutation(len(pers))]
    elif family == "faces":
        fv = face_values(lo, svs, sdim)
        pts = []
        for a in range(3):
            band = [lo[a] - 0.5 * svs[a], lo[a] - svs[a], ulps(lo[a] - svs[a], 1), ulps(lo[a], -1), ulps(lo[a] + sdim[a] * svs[a], -1)]
            for val in list(fv[a]) + band:
                q = lo + g.random_sample(3) * (hi - lo)
                if vox_div(val, lo[a], svs[a]) != vox_mul(val, lo[a], svs[a]):
                    # where the divide and the reciprocal multiply disagree, the other two coordinates sit mid-voxel, on a sample's
                    # column and depth: which voxel the point falls in decides whether that sample's search box holds it
                    q = lo + (np.floor(g.random_sample(3) * sdim) + 0.5) * svs
                q[a] = val
                pts.append(q)
        # isolated points in depth 0 (z = near and just above): with query_size[2] <= 2 their columns dilate to depth 0 only
        for x, y in ((1, 1), (sdim[0] - 2, 1), (1, sdim[1] - 2)):
            pts.append([lo[0] + (x + 0.5) * svs[0], lo[1] + (y + 0.5) * svs[1], lo[2]])
            pts.append([lo[0] + (x + 0.25) * svs[0], lo[1] + (y + 0.75) * svs[1], ulps(lo[2], 3)])
        pers = np.array(pts, f32)
        keep = np.ones(len(pers), bool)
        for x, y in ((1, 1), (sdim[0] - 2, 1), (1, sdim[1] - 2)):        # keep those columns' neighbourhoods free of other points
            c = vox_div(pers[:, :2], lo[:2], svs[:2])
            near_col = (np.abs(c[:, 0] - x) <= 3) & (np.abs(c[:, 1] - y) <= 3) & (pers[:, 2] > lo[2] + 0.5 * svs[2])
            keep &= ~near_col
        pers = pers[keep]
    elif family == "crowded":
        P, K = opt.P, opt.K
        cells = [(3, 3, 5, P), (3, 3, 9, P + 1), (3, 3, 13, 3 * P), (4, 3, 17, K + 3), (3, 4, 21, 3 * P), (3, 3, 25, 1)]
        pts = [(lo + g.random_sample((80, 3)) * (hi - lo)).astype(f32)]
        for x, y, z, n in cells:
            pts.append((lo + (np.array([x, y, z]) + g.random_sample((n, 3))) * svs).astype(f32))
        pers = np.concatenate(pts)
        pers = pers[g.permutation(len(pers))]
    elif family == "empty":
        pers = np.concatenate([(hi + 1.0)[None], (lo - 1.5 * svs - g.random_sample((40, 3)) * svs)]).astype(f32)
    else:
        raise ValueError(family)
    return dict(name="frustum_%s" % family, pers=np.ascontiguousarray(pers, f32), cam=cam, pixel_idx=frustum_pixels(cam, vscale))


def frustum_hand_cases():
    """The world cases' tie rule in the frustum kernel (query_point_indices.py:574-591), derived by hand.  Grid 8^3 of 0.25 at lo
    (-1, -1, 1) (frustum_camera(8, 8, 8), vscale 1); pixel (4, 4); its column dilates to depths 3..6 so sample 1 sits at depth 4:
    (cx, cy, cz) = (0.125, 0.125, 2.125).  Same-depth neighbours one voxel away in x or y have xy^2 = (0.25 * 2.125)^2 = 0.2822265625
    exactly; the point one voxel deeper on the axis has 0.001953125 + 0.0625."""
    cz = 2.125
    B, D, E = (-0.125, 0.125, cz), (0.125, -0.125, cz), (0.125, 0.125, cz + 0.25)
    cases = [dict(name="frustum_evict_first_of_tied_fill", K=2, pts=[B, D, E], want=[2, 1]),
             dict(name="frustum_equal_does_not_replace", K=2, pts=[(0.125, 0.125, cz + 0.0625), B, (0.375, 0.125, cz)], want=[0, 1]),
             # the diagonal neighbour (2 x 0.2822265625) fills slot 0, two tied ones slots 1 and 2; E evicts slot 0; the rescan keeps the
             # FIRST tied maximum (slot 1), so the next nearer one (one voxel in +x, 0.15875244140625) evicts slot 1
             dict(name="frustum_rescan_keeps_first_max", K=3,
                  pts=[(-0.125, -0.125, cz), (-0.125, 0.125, cz), D, E, (0.3125, 0.125, cz)], want=[3, 4, 2])]
    for c in cases:
        c.update(pers=np.array(c.pop("pts"), f32), cam=frustum_camera(8, 8, 8, 0.25), pixel_idx=np.array([[4, 4]], np.int32), sample=1,
                 opt=frustum_opt(vscale=(1, 1, 1), SR=4, K=c["K"], P=8, z_depth_dim=8))
    return cases
