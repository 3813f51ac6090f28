"""TEST INFRASTRUCTURE: the plane background of bgmodel plane (pointnerf_b200/csrc/plane_bg.cu) restated twice.

* fp32, in the kernels' exact operation order (numpy float32: every operation rounds once, no contraction).  The GPU tests hold
  pnb_plane_cross, pnb_plane_fg_masks and pnb_plane_bg to it bit for bit.
* float64, with a per-sample bound on the error of ANY fp32 evaluation of the same expressions (the reference's matmuls sum in an order
  of their own), used to tell decisions that sit near a boundary from real disagreements (`compare_reference`).

Views are a dict: w2c [G,4,4], K [G,3,3] (float32), hdwd [G,2] (HD, WD).  Images: one [3,H,W] float32 array per view.

Error bounds (u = 2^-24, first order; tests/test_plane_bg_oracle.py states where they are used):
  camera   c_i = sum of 4 products: any order, with or without fused multiply-adds, errs by at most g4 S_i, S_i = sum_j |W_ij x_j| + |W_i3|
  divide   px = c0 / c2:  |d px| <= (|d c0| + |px| |d c2|) / |c2| + u |px|  (pz = c2 / c2 is exactly 1)
  pixel    u = K00 px + K01 py + K02:  |d u| <= |K00| |d px| + |K01| |d py| + g3 (|K00 px| + |K01 py| + |K02|)
  EPS_U    2 |d u| (g_n = n u, doubled again for safety): a decision on u (bounds, ceil) can flip only within EPS_U of its boundary
  sample   x = (u / ((WD-1)/2) - 1 + 1) (W-1)/2 adds the scaled EPS_U and 4 roundings of x:  EPS_X = ratio EPS_U + 8 u (|x| + W)
  colour   the bilinear interpolant moves by at most 2 M per unit of x or y (M = max |image|), and its 7 operations err by 8 u M:
           EPS_C = 2 M (EPS_X + EPS_Y) + 16 u M
  plane    dot = n . d (3 products) errs by g3 sum |n_k d_k|; the intersection by 8 u (|c_k| + |d_k fac| (1 + S_nw / |nw| + S_dot / |dot|))
"""
import numpy as np

F = np.float32
U = 2.0 ** -24
THRESH = F(0.03)
EPS_DOT = F(1e-3)


# ------------------------------------------------------------------------------------------------ fp32, the kernels' order
def _dot3(a0, a1, a2, b0, b1, b2):
    return (a0 * b0 + a1 * b1) + a2 * b2


def cross(campos, raydir, plane_pnt, plane_normal):
    """get_rayplane_cross on R rays (raydir [R,3]): [R,3] float32."""
    c, n, p = (np.asarray(a, F).reshape(3) for a in (campos, plane_normal, plane_pnt))
    d = np.asarray(raydir, F).reshape(-1, 3)
    with np.errstate(all="ignore"):
        dot = _dot3(n[0], n[1], n[2], d[:, 0], d[:, 1], d[:, 2])
        w = c - p
        nw = _dot3(n[0], n[1], n[2], w[0], w[1], w[2])
        fac = -nw / dot
        out = c[None, :] + d * fac[:, None]
    out[~(dot >= EPS_DOT)] = 0
    return out.astype(F)


def project(xyz, w2c, K, HD, WD):
    """(u, v, in_bounds) of world points xyz [N,3] in one view."""
    x, y, z = (np.asarray(xyz, F)[:, i] for i in range(3))
    w, k = np.asarray(w2c, F), np.asarray(K, F)
    with np.errstate(all="ignore"):
        c = [_dot3(w[i, 0], w[i, 1], w[i, 2], x, y, z) + w[i, 3] for i in range(3)]
        px, py, pz = c[0] / c[2], c[1] / c[2], c[2] / c[2]
        u = _dot3(px, py, pz, k[0, 0], k[0, 1], k[0, 2])
        v = _dot3(px, py, pz, k[1, 0], k[1, 1], k[1, 2])
        inb = (np.isfinite(x) & np.isfinite(y) & np.isfinite(z) & (u >= 0) & (u <= F(WD - 1)) & (v >= 0) & (v <= F(HD - 1)))
    return u, v, inb


def cells(u, v):
    return np.ceil(v).astype(np.int64), np.ceil(u).astype(np.int64)


def fg_masks(xyz, views):
    """id2mask(homo_warp_fg_mask(...)) of every view: a list of int8 [HD,WD]."""
    out = []
    for g in range(len(views["hdwd"])):
        HD, WD = (int(a) for a in views["hdwd"][g])
        u, v, inb = project(xyz, views["w2c"][g], views["K"][g], HD, WD)
        m = np.zeros((HD, WD), np.int8)
        cv, cu = cells(u[inb], v[inb])
        m[cv, cu] = 1
        out.append(m)
    return out


def sample(u, v, HD, WD, img):
    """grid_sample(bilinear, zeros, align_corners=True) of img [3,H,W] at the coordinate set_bg forms from (u, v): [n,3]."""
    H, W = img.shape[1:]
    gx = u / F((WD - 1) * 0.5) - F(1)
    gy = v / F((HD - 1) * 0.5) - F(1)
    sx = (gx + F(1)) * F((W - 1) * 0.5)
    sy = (gy + F(1)) * F((H - 1) * 0.5)
    x0, y0 = np.floor(sx), np.floor(sy)
    a, b = sx - x0, sy - y0
    e, s = F(1) - a, F(1) - b
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)

    def tex(jx, jy):
        ok = (jx >= 0) & (jx < W) & (jy >= 0) & (jy < H)
        t = np.zeros((3, len(jx)), F)
        t[:, ok] = img[:, jy[ok], jx[ok]]
        return t

    with np.errstate(all="ignore"):
        val = ((tex(ix, iy) * (s * e) + tex(ix + 1, iy) * (s * a)) + tex(ix, iy + 1) * (b * e)) + tex(ix + 1, iy + 1) * (b * a)
    return val.T.astype(F)


def bg(xyz, views, masks, imgs, plane_color, detail=False):
    """bg_ray [R,3] of the plane points xyz [R,3] (set_bg's first return value without its batch axis).  masks: one array per view
    (the kernel's int8 masks, or a caller's fg_masks[:, g]); a cell counts where its mask is < 1.  detail=True also returns every
    view's (u, v, in_bounds, selected, value, fit)."""
    pc = np.asarray(plane_color, F).reshape(3)
    lo, hi = pc - THRESH, pc + THRESH
    R = xyz.shape[0]
    best, per = None, []
    for g in range(len(views["hdwd"])):
        HD, WD = (int(a) for a in views["hdwd"][g])
        u, v, inb = project(xyz, views["w2c"][g], views["K"][g], HD, WD)
        sel = inb.copy()
        cv, cu = cells(u[inb], v[inb])
        sel[inb] = masks[g][cv, cu] < 1
        val = sample(u[sel], v[sel], HD, WD, imgs[g])
        fit = np.all((val >= lo) & (val <= hi), axis=1)
        s = np.zeros((R, 3), F)
        s[sel] = np.where(fit[:, None], val, F(0))
        best = s if best is None else np.where(s > best, s, best)
        if detail:
            per.append(dict(u=u, v=v, inb=inb, sel=sel, val=val, fit=fit))
    return (best, per) if detail else best


# ------------------------------------------------------------------------------------------------ float64 and the bounds
def project64(xyz, w2c, K):
    """(u, v, EPS_U, EPS_V) in float64 of the float32 points xyz [N,3]."""
    p = np.asarray(xyz, np.float64)
    w, k = np.asarray(w2c, np.float64), np.asarray(K, np.float64)
    h = np.concatenate([p, np.ones((p.shape[0], 1))], 1)
    with np.errstate(all="ignore"):
        c = h @ w[:3].T
        dc = 5 * U * (np.abs(h) @ np.abs(w[:3]).T)
        px, py = c[:, 0] / c[:, 2], c[:, 1] / c[:, 2]
        dpx = (dc[:, 0] + np.abs(px) * dc[:, 2]) / np.abs(c[:, 2]) + U * np.abs(px)
        dpy = (dc[:, 1] + np.abs(py) * dc[:, 2]) / np.abs(c[:, 2]) + U * np.abs(py)
        out = []
        for r in range(2):
            uu = k[r, 0] * px + k[r, 1] * py + k[r, 2]
            du = abs(k[r, 0]) * dpx + abs(k[r, 1]) * dpy + 4 * U * (np.abs(k[r, 0] * px) + np.abs(k[r, 1] * py) + abs(k[r, 2]))
            out += [uu, 2 * du]
    bad = ~np.all(np.isfinite(p), 1)
    for a in out:
        a[bad] = np.nan
    return out[0], out[2], out[1], out[3]


def _near_int(x, eps):
    return np.abs(x - np.round(x)) <= eps


def near_projection(u, v, eu, ev, HD, WD):
    """True where an fp32 evaluation may decide the bounds test or the cell differently."""
    with np.errstate(invalid="ignore"):
        near = ~np.isfinite(u) | ~np.isfinite(v) | ~np.isfinite(eu) | ~np.isfinite(ev)
        near |= (np.abs(u) <= eu) | (np.abs(u - (WD - 1)) <= eu) | (np.abs(v) <= ev) | (np.abs(v - (HD - 1)) <= ev)
        near |= _near_int(u, eu) | _near_int(v, ev)
    return near & ~(bad_far(u, v, eu, ev, HD, WD))


def bad_far(u, v, eu, ev, HD, WD):
    """Points that are out of bounds whichever way an fp32 evaluation rounds (their cell does not matter)."""
    with np.errstate(invalid="ignore"):
        return np.isfinite(u) & np.isfinite(v) & ((u < -eu) | (u > WD - 1 + eu) | (v < -ev) | (v > HD - 1 + ev))


def color_eps(u, v, eu, ev, HD, WD, img):
    H, W = img.shape[1:]
    rx, ry = (W - 1) / (WD - 1), (H - 1) / (HD - 1)
    ex = rx * eu + 8 * U * (np.abs(u) * rx + W)
    ey = ry * ev + 8 * U * (np.abs(v) * ry + H)
    M = float(np.max(np.abs(img[np.isfinite(img)]))) if np.isfinite(img).any() else 0.0
    return 2 * M * (ex + ey) + 16 * U * M


def cross_bounds(campos, raydir, plane_pnt, plane_normal):
    """(dot in float64, its EPS, the intersection's per-component EPS [R,3])."""
    c, n, p = (np.asarray(a, np.float64).reshape(3) for a in (campos, plane_normal, plane_pnt))
    d = np.asarray(raydir, np.float64).reshape(-1, 3)
    dot = d @ n
    edot = 2 * 3 * U * (np.abs(d) @ np.abs(n))
    w = c - p
    nw = float(w @ n)
    snw = float(np.abs(w) @ np.abs(n)) + 1e-300
    with np.errstate(all="ignore"):
        fac = -nw / dot
        ep = 8 * U * (np.abs(c)[None] + np.abs(d * fac[:, None]) * (1 + snw / (abs(nw) + 1e-300) +
                                                                    (np.abs(d) @ np.abs(n) / np.abs(dot))[:, None]))
    return dot, edot, ep


def compare_reference(case, ref, ref_views, masks_used=None):
    """Classify the reference's results against the fp32 oracle.

    case: the inputs (xyz, campos, raydir, plane_pnt, plane_normal, plane_color, views, imgs); ref: the reference's gen_bg_points
    output `sect` [R,3], set_bg's `bg` [R,3] and its foreground masks `fg` (list per view).  ref_views: per view the reference's
    homo_warp_nongrid `inb` [R] and the `val` [n,3] extract_from_2d_grid returned for its selected samples `sel` [R].  masks_used:
    the masks set_bg tested (the caller's fg_masks, default the reference's own).
    Raises AssertionError on a disagreement that no bound explains; returns counts of what was compared and what was near."""
    views, imgs = case["views"], case["imgs"]
    G = len(views["hdwd"])
    stats = dict(rays=0, near_dot=0, near_rays=0, samples=0, near_samples=0, mask_cells=0, mask_cells_flipped=0, max_dcolor=0.0)
    # gen_bg_points
    mine = cross(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"])
    dot, edot, ep = cross_bounds(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"])
    near_dot = np.abs(dot - float(EPS_DOT)) <= edot
    ok = ~near_dot
    zr, zm = np.all(ref["sect"] == 0, 1), np.all(mine == 0, 1)
    assert np.array_equal(zr[ok], zm[ok]), "dot >= 1e-3 decided differently away from the boundary"
    live = ok & ~zm
    assert np.all(np.abs(ref["sect"][live].astype(np.float64) - mine[live]) <= ep[live]), "intersections differ beyond the bound"
    stats["rays"], stats["near_dot"] = len(dot), int(near_dot.sum())
    # the foreground masks: every differing cell must be one a near point may land in
    xyz_pts = case["xyz"]
    for g in range(G):
        HD, WD = (int(a) for a in views["hdwd"][g])
        mo = fg_masks(xyz_pts, {k: views[k][g:g + 1] for k in ("w2c", "K", "hdwd")})[0]
        diff = np.argwhere(mo != ref["fg"][g])
        stats["mask_cells"] += int(mo.size)
        if len(diff):
            u, v, eu, ev = project64(xyz_pts, views["w2c"][g], views["K"][g])
            nr = near_projection(u, v, eu, ev, HD, WD)
            cand = set()
            for uu, vv, a, b in zip(u[nr], v[nr], eu[nr], ev[nr]):
                for cv in {int(np.ceil(vv - b)), int(np.ceil(vv + b))}:
                    for cu in {int(np.ceil(uu - a)), int(np.ceil(uu + a))}:
                        cand.add((cv, cu))
            for cv, cu in diff:
                assert (int(cv), int(cu)) in cand, "foreground mask cell (%d, %d) of view %d differs with no near point" % (cv, cu, g)
            stats["mask_cells_flipped"] += len(diff)
    # per view on the reference's own plane points
    masks_used = ref["fg"] if masks_used is None else masks_used
    sect = ref["sect"]
    lo, hi = (np.asarray(case["plane_color"], F).reshape(3) - THRESH).astype(np.float64), \
        (np.asarray(case["plane_color"], F).reshape(3) + THRESH).astype(np.float64)
    _, per = bg(sect, views, masks_used, imgs, case["plane_color"], detail=True)
    near_ray = np.zeros(sect.shape[0], bool)
    ceps = np.zeros(sect.shape[0])
    for g in range(G):
        HD, WD = (int(a) for a in views["hdwd"][g])
        o, rv = per[g], ref_views[g]
        u, v, eu, ev = project64(sect, views["w2c"][g], views["K"][g])
        near = near_projection(u, v, eu, ev, HD, WD)
        inb = o["inb"]
        assert np.array_equal(rv["inb"][~near], inb[~near]), "view %d: bounds decided differently away from the boundary" % g
        assert np.array_equal(rv["sel"][~near], o["sel"][~near]), "view %d: mask decided differently away from the boundary" % g
        ce = color_eps(u, v, eu, ev, HD, WD, imgs[g])
        both = rv["sel"] & o["sel"]
        rval = np.zeros((sect.shape[0], 3))
        rval[rv["sel"]] = rv["val"]
        oval = np.zeros((sect.shape[0], 3))
        oval[o["sel"]] = o["val"]
        dcol = np.abs(rval - oval).max(1)
        assert np.all(dcol[both & ~near] <= ce[both & ~near]), "view %d: colours differ beyond the bound" % g
        stats["max_dcolor"] = max(stats["max_dcolor"], float(dcol[both].max()) if both.any() else 0.0)
        near_fit = np.zeros_like(near)
        near_fit[o["sel"]] = np.any((np.abs(oval[o["sel"]] - lo) <= ce[o["sel"], None]) |
                                    (np.abs(oval[o["sel"]] - hi) <= ce[o["sel"], None]), 1)
        nr = (near & ~bad_far(u, v, eu, ev, HD, WD)) | near_fit
        stats["samples"] += int(sect.shape[0])
        stats["near_samples"] += int(nr.sum())
        near_ray |= nr
        ceps = np.maximum(ceps, np.where(np.isfinite(ce), ce, np.inf))
    near_ray |= near_dot
    best = bg(sect, views, masks_used, imgs, case["plane_color"])
    keep = ~near_ray
    d = np.abs(ref["bg"][keep].astype(np.float64) - best[keep]).max(1) if keep.any() else np.zeros(0)
    assert np.all(d <= ceps[keep]), "bg_ray differs beyond the colour bound on a ray with no near decision"
    stats["near_rays"] = int(near_ray.sum())
    return stats
