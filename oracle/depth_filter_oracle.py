"""TEST INFRASTRUCTURE: the depth filter and visual hull of the initial point cloud (pointnerf_b200/csrc/depth_filter.cu) restated twice.

* fp32, in the kernels' exact operation order (numpy float32: every operation rounds once, no contraction), from the same per-pair
  matrices (pointnerf_b200.depth_filter.view_matrices).  The GPU tests hold pnb_depth_filter_* and pnb_alpha_mask to it bit for bit.
* float64, with a first-order bound on the error of ANY fp32 evaluation of the same expressions, used by `compare_reference` to tell
  decisions that sit within their bound of a boundary from real disagreements: the reference inverts K and E with torch.linalg.inv in
  fp32 and its matmuls sum in an order of their own.

A case: depth [V,H,W], xy [V,H,W,2], conf [V,H,W] (fp32), mask [V,H,W] bool, K [V,3,3], E [V,4,4] (fp32), thresh, geo_n, ranges (6 or
None).  Visual hull: points [N,3], alpha [V,H,W], K [V,3,3], w2c [V,4,4], near_far (2 or None), range_test.

Error bounds (u = 2^-24, g_n = n u, |.| elementwise, first order; every bound is then doubled so that it covers two evaluations):
  inverse   an fp32 LU inverse (n = 3 or 4, small growth) errs componentwise by at most 8 u |M^-1| |M| |M^-1|; the kernels' matrices
            by u |entry|.  pair = E_s inv(E_r) in fp32: |E_s| e_inv + g4 |E_s| |inv(E_r)|.
  affine    y = A b (+ a): g_n (|A| |b| + |a|) + |A| e_b + e_A (sum |b| + 1)
  divide    q = a / b: (e_a + |q| e_b) / |b| + u |q|
  sample    sx = ((x 2) / (W-1) - 1 + 1) (W-1) / 2 moves by e_x + 4 u (|x| + W); the clamp is 1-Lipschitz; the bilinear interpolant is
            continuous, so it moves by at most L (e_sx + e_sy) + 8 u M, L and M the largest adjacent-texel difference and |texel| over
            the 4 x 4 texels around the tap.  A tap whose e_sx or e_sy reaches 1, or a divisor within its bound of 0, is unbounded.
  decisions dist = sqrt(dx^2 + dy^2) moves by e_dx + e_dy + 4 u dist; rel = |dre - d| / d by (e_dre + u |dre - d|) / d + 2 u rel; a
            match is near when a test that could be either way (|value - threshold| <= bound) decides it.  The averaged depth errs by
            (sum of the matched e_dre + g_V sum |dre|) / (geo + 1) + u |avg|; the world point as an affine of (x, y, avg) with the
            inverse's bound; a range face is near within that bound.
  hull      c = w2c [p, 1] (g4), k = K c (g3), u = k0 / k2 as above: a floor cell (and with it the image bounds, at integers) is near
            within e_u of an integer, the near/far test within e_c2 of its bound.  The alpha compare uses exact inputs.
"""
import numpy as np

from pointnerf_b200.depth_filter import view_matrices

F = np.float32
U = 2.0 ** -24
DIST, REL, ALPHA = F(1), F(0.01), F(0.1)
FAULTS = ("avg_xy", "dist_le", "range_cam", "no_clamp", "single_view_geo")


# ------------------------------------------------------------------------------------------------ fp32, the kernels' order
def _dot(A, b0, b1, b2):
    return (A[0] * b0 + A[1] * b1) + A[2] * b2


def _aff(A, b0, b1, b2):
    return _dot(A, b0, b1, b2) + A[3]


def _bilinear(img, sx, sy):
    """The kernel's bilinear tap of img [H,W] at (sx, sy) (already clamped): a corner outside reads 0."""
    H, W = img.shape
    x0, y0 = np.floor(sx), np.floor(sy)
    a, b = sx - x0, sy - y0
    e, t = F(1) - a, F(1) - b
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)

    def tap(jx, jy):
        ok = (jx >= 0) & (jx < W) & (jy >= 0) & (jy < H)
        v = np.zeros(jx.shape, F)
        v[ok] = img[jy[ok], jx[ok]]
        return v

    return ((tap(ix, iy) * (t * e) + tap(ix + 1, iy) * (t * a)) + tap(ix, iy + 1) * (b * e)) + tap(ix + 1, iy + 1) * (b * a)


def geo_pass(case, r, mats, pix, fault=None, detail=False):
    """geo_sum, depth_sum of ref view r's pixels pix (flat indices) over its source views; detail=True also returns every source's
    (s, xs, ys, ds, dre, dist, rel, match)."""
    K, Kinv, _, pair = mats
    depth = np.asarray(case["depth"], F)
    V, H, W = depth.shape
    y, x = np.divmod(pix, W)
    fx, fy = x.astype(F), y.astype(F)
    d = depth[r].reshape(-1)[pix]
    p0, p1 = fx * d, fy * d
    q = [_dot(Kinv[r][i], p0, p1, d) for i in range(3)]
    geo = np.zeros(len(pix), np.int64)
    dsum = np.zeros(len(pix), F)
    per = []
    dW, dH, sfW, sfH = F(W - 1), F(H - 1), F((W - 1) * 0.5), F((H - 1) * 0.5)
    with np.errstate(all="ignore"):
        for s in range(V):
            if s == r:
                continue
            A, B = pair[r, s].reshape(3, 4), pair[s, r].reshape(3, 4)
            c = [_aff(A[i], *q) for i in range(3)]
            k = [_dot(K[s][i], *c) for i in range(3)]
            xs, ys = k[0] / k[2], k[1] / k[2]
            gx, gy = (xs * F(2)) / dW - F(1), (ys * F(2)) / dH - F(1)
            sx, sy = (gx + F(1)) * sfW, (gy + F(1)) * sfH
            if fault != "no_clamp":
                sx, sy = np.minimum(np.maximum(sx, F(0)), dW), np.minimum(np.maximum(sy, F(0)), dH)
            ds = _bilinear(depth[s], sx, sy)
            m0, m1 = xs * ds, ys * ds
            h = [_dot(Kinv[s][i], m0, m1, ds) for i in range(3)]
            e = [_aff(B[i], *h) for i in range(3)]
            uu = [_dot(K[r][i], *e) for i in range(3)]
            ddx, ddy = uu[0] / uu[2] - fx, uu[1] / uu[2] - fy
            dist = np.sqrt(ddx * ddx + ddy * ddy)
            rel = np.abs(e[2] - d) / d
            match = ((dist <= DIST) if fault == "dist_le" else (dist < DIST)) & (rel < REL)
            geo += match
            dsum = dsum + np.where(match, e[2], F(0))
            if detail:
                per.append(dict(s=s, xs=xs, ys=ys, ds=ds, dre=e[2], dist=dist, rel=rel, match=match))
    return (geo, dsum, per) if detail else (geo, dsum)


def _world(c2w, x, y, z):
    return np.stack([_aff(c2w[i], x, y, z) for i in range(3)], -1)


def filter_view(case, r, mats=None, fault=None):
    """Ref view r: dict(pix (kept flat indices, row-major), cam [n,3], world [n,3], conf [n], live, geo, avg) in fp32."""
    mats = view_matrices(case["K"], case["E"]) if mats is None else mats
    depth, conf = np.asarray(case["depth"], F), np.asarray(case["conf"], F)
    V, H, W = depth.shape
    c2w = mats[2][r].reshape(3, 4)
    live = ((conf[r] > F(case["thresh"])) & np.asarray(case["mask"][r], bool)).reshape(-1)
    pix = np.nonzero(live)[0]
    if V > 1 or fault == "single_view_geo":
        geo, dsum = geo_pass(case, r, mats, pix, fault)
    else:
        geo, dsum = np.zeros(len(pix), np.int64), np.zeros(len(pix), F)
    d = depth[r].reshape(-1)[pix]
    with np.errstate(all="ignore"):
        avg = (dsum + d) / (geo + 1).astype(F)
    keep = (geo >= case["geo_n"]) if (V > 1 or fault == "single_view_geo") else np.ones(len(pix), bool)
    xy = np.asarray(case["xy"][r], F).reshape(-1, 2)[pix]
    x, y = xy[:, 0], xy[:, 1]
    if fault == "avg_xy":
        with np.errstate(all="ignore"):
            x, y = x / d * avg, y / d * avg
    with np.errstate(all="ignore"):
        world = _world(c2w, x, y, avg)
    if case.get("ranges") is not None:
        rg = np.asarray(case["ranges"], F)
        tst = np.stack([x, y, avg], -1) if fault == "range_cam" else world
        keep &= np.all((tst >= rg[:3]) & (tst <= rg[3:]), 1)
    sel = np.nonzero(keep)[0]
    return dict(pix=pix[sel], cam=np.stack([x, y, avg], -1)[sel].astype(F), world=world[sel].astype(F),
                conf=conf[r].reshape(-1)[pix[sel]], live=live, pix_live=pix, geo=geo, avg=avg)


def alpha_mask(points, alpha, K, w2c, near_far=None, range_test=False, detail=False):
    """The visual-hull mask bool [N]; detail=True also returns per view (ix, iy, z, ok)."""
    p = np.asarray(points, F)[:, :3]
    alpha = np.asarray(alpha, F)
    V, H, W = alpha.shape
    keep = np.ones(len(p), bool)
    per = []
    lo = hi = None
    if near_far is not None:
        lo, hi = F(float(near_far[0]) - 1.0), F(float(near_far[1]))
    with np.errstate(all="ignore"):
        for v in range(V):
            A = np.asarray(w2c[v], F).reshape(4, 4)
            k33 = np.asarray(K[v], F).reshape(3, 3)
            c = [_aff(A[i], p[:, 0], p[:, 1], p[:, 2]) for i in range(3)]
            k = [_dot(k33[i], *c) for i in range(3)]
            # (int64) of a float saturates on the GPU
            ix = np.clip(np.floor(k[0] / k[2]).astype(np.float64), -2.0 ** 63, 2.0 ** 63 - 1024).astype(np.int64)
            iy = np.clip(np.floor(k[1] / k[2]).astype(np.float64), -2.0 ** 63, 2.0 ** 63 - 1024).astype(np.int64)
            inb = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
            a = alpha[v][np.clip(iy, 0, H - 1), np.clip(ix, 0, W - 1)]
            if range_test:
                a = a + np.where(inb, F(0), F(1))
            ok = a > ALPHA
            if lo is not None:
                ok &= (c[2] >= lo) & (c[2] <= hi)
            keep &= ok
            if detail:
                per.append(dict(ix=ix, iy=iy, z=c[2], ok=ok))
    return (keep, per) if detail else keep


# ------------------------------------------------------------------------------------------------ float64 and the bounds
G = lambda n: n * U  # noqa: E731


def _inv_err(M):
    Mi = np.linalg.inv(M)
    return Mi, 8 * U * np.abs(Mi) @ np.abs(M) @ np.abs(Mi) + U * np.abs(Mi)


def _affine(A, eA, b, eb, const=None, econst=None):
    """y_i = sum_j A_ij b_j (+ const_i) with its bound; b, eb: lists of arrays."""
    n = len(b) + (const is not None)
    ys, es = [], []
    for i in range(A.shape[0]):
        v = sum(A[i, j] * b[j] for j in range(len(b)))
        mag = sum(abs(A[i, j]) * np.abs(b[j]) for j in range(len(b)))
        e = G(n) * mag + sum(abs(A[i, j]) * eb[j] + eA[i, j] * np.abs(b[j]) for j in range(len(b)))
        if const is not None:
            v = v + const[i]
            e = e + G(n) * abs(const[i]) + econst[i]
        ys.append(v)
        es.append(e)
    return ys, es


def _div(a, ea, b, eb):
    with np.errstate(all="ignore"):
        q = a / b
        e = (ea + np.abs(q) * eb) / np.abs(b) + U * np.abs(q)
        e = np.where(np.abs(b) > 2 * eb, e, np.inf)
    return q, e


def _local(img, sx, sy):
    """The largest adjacent-texel difference and |texel| over the 4 x 4 texels around (sx, sy) (zeros outside)."""
    H, W = img.shape
    pad = np.zeros((H + 4, W + 4))
    pad[2:-2, 2:-2] = img
    ix = np.clip(np.floor(np.nan_to_num(sx, nan=0.0, posinf=W, neginf=-2)), -2, W).astype(np.int64) + 2
    iy = np.clip(np.floor(np.nan_to_num(sy, nan=0.0, posinf=H, neginf=-2)), -2, H).astype(np.int64) + 2
    L = np.zeros(len(ix))
    M = np.zeros(len(ix))
    for dy in range(-1, 3):
        for dx in range(-1, 3):
            v = pad[np.clip(iy + dy, 0, H + 3), np.clip(ix + dx, 0, W + 3)]
            M = np.maximum(M, np.abs(v))
            if dx < 2:
                L = np.maximum(L, np.abs(pad[np.clip(iy + dy, 0, H + 3), np.clip(ix + dx + 1, 0, W + 3)] - v))
            if dy < 2:
                L = np.maximum(L, np.abs(pad[np.clip(iy + dy + 1, 0, H + 3), np.clip(ix + dx, 0, W + 3)] - v))
    return L, M


def _bilinear64(img, sx, sy):
    H, W = img.shape
    x0, y0 = np.floor(sx), np.floor(sy)
    a, b = sx - x0, sy - y0
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)

    def tap(jx, jy):
        ok = (jx >= 0) & (jx < W) & (jy >= 0) & (jy < H)
        v = np.zeros(jx.shape)
        v[ok] = img[jy[ok], jx[ok]]
        return v

    return (tap(ix, iy) * (1 - b) * (1 - a) + tap(ix + 1, iy) * (1 - b) * a + tap(ix, iy + 1) * b * (1 - a) +
            tap(ix + 1, iy + 1) * b * a)


def bounds_view(case, r, pix):
    """float64 per pixel of pix: geo_min, geo_max (matches certain / possible), avg and its bound (where geo_min == geo_max)."""
    depth = np.asarray(case["depth"], np.float64)
    V, H, W = depth.shape
    K = np.asarray(case["K"], F).astype(np.float64)
    E = np.asarray(case["E"], F).astype(np.float64)
    inv = [_inv_err(E[v]) for v in range(V)]
    kin = [_inv_err(K[v]) for v in range(V)]
    y, x = np.divmod(pix, W)
    d = depth[r].reshape(-1)[pix]
    p = [x * d, y * d, d]
    ep = [U * np.abs(p[0]), U * np.abs(p[1]), np.zeros_like(d)]
    q, eq = _affine(kin[r][0], kin[r][1], p, ep)
    sure = np.zeros(len(pix), np.int64)
    maybe = np.zeros(len(pix), np.int64)
    dsum = np.zeros(len(pix))
    edsum = np.zeros(len(pix))
    mag = np.zeros(len(pix))
    zero3 = np.zeros(3)
    with np.errstate(all="ignore"):
        for s in range(V):
            if s == r:
                continue
            A = E[s] @ inv[r][0]
            eA = np.abs(E[s]) @ inv[r][1] + G(4) * np.abs(E[s]) @ np.abs(inv[r][0])
            B = E[r] @ inv[s][0]
            eB = np.abs(E[r]) @ inv[s][1] + G(4) * np.abs(E[r]) @ np.abs(inv[s][0])
            c, ec = _affine(A[:3, :3], eA[:3, :3], q, eq, A[:3, 3], eA[:3, 3])
            k, ek = _affine(K[s], np.zeros((3, 3)), c, ec)
            xs, exs = _div(k[0], ek[0], k[2], ek[2])
            ys, eys = _div(k[1], ek[1], k[2], ek[2])
            esx, esy = exs + 4 * U * (np.abs(xs) + W), eys + 4 * U * (np.abs(ys) + H)
            sx, sy = np.clip(xs, 0, W - 1), np.clip(ys, 0, H - 1)
            ds = _bilinear64(depth[s], np.nan_to_num(sx), np.nan_to_num(sy))
            L, M = _local(depth[s], sx, sy)
            eds = L * (esx + esy) + 8 * U * M
            eds = np.where((esx < 1) & (esy < 1) & np.isfinite(xs) & np.isfinite(ys), eds, np.inf)
            m = [xs * ds, ys * ds, ds]
            em = [np.abs(xs) * eds + np.abs(ds) * exs + U * np.abs(m[0]), np.abs(ys) * eds + np.abs(ds) * eys + U * np.abs(m[1]), eds]
            h, eh = _affine(kin[s][0], kin[s][1], m, em)
            e, ee = _affine(B[:3, :3], eB[:3, :3], h, eh, B[:3, 3], eB[:3, 3])
            uu, eu = _affine(K[r], np.zeros((3, 3)), e, ee)
            xr, exr = _div(uu[0], eu[0], uu[2], eu[2])
            yr, eyr = _div(uu[1], eu[1], uu[2], eu[2])
            dx, dy = xr - x, yr - y
            edx, edy = exr + U * np.abs(dx), eyr + U * np.abs(dy)
            dist = np.sqrt(dx * dx + dy * dy)
            edist = edx + edy + 4 * U * dist
            rel = np.abs(e[2] - d) / d
            erel = (ee[2] + U * np.abs(e[2] - d)) / d + 2 * U * rel
            edist, erel = 2 * edist, 2 * erel
            dist_yes, dist_no = dist < 1 - edist, dist > 1 + edist
            rel_yes, rel_no = rel < float(REL) - erel, rel > float(REL) + erel
            yes = dist_yes & rel_yes
            no = dist_no | rel_no | (d == 0)           # a zero depth: |dre| / 0 is inf or nan, never < 0.01
            sure += yes
            maybe += ~yes & ~no
            dsum += np.where(yes, e[2], 0.0)
            edsum += np.where(yes, 2 * ee[2], 0.0)
            mag += np.where(yes, np.abs(e[2]), 0.0)
    avg = (dsum + d) / (sure + 1)
    eavg = (edsum + G(V + 1) * (mag + np.abs(d))) / (sure + 1) + 2 * U * np.abs(avg)
    return dict(geo_min=sure, geo_max=sure + maybe, avg=avg, eavg=eavg, c2w=inv[r][0][:3], ec2w=inv[r][1][:3])


def world_bounds(b, sel, x, y):
    """float64 world points and their bounds of the pixels sel of bounds_view's result b (x, y: their raw camera x, y)."""
    z, ez = b["avg"][sel], b["eavg"][sel]
    w, ew = _affine(b["c2w"][:, :3], b["ec2w"][:, :3], [x, y, z], [np.zeros_like(x), np.zeros_like(y), ez], b["c2w"][:, 3],
                    b["ec2w"][:, 3])
    return np.stack(w, -1), 2 * np.stack(ew, -1)


def alpha_bounds(points, K, w2c, near_far=None):
    """float64 per view: (u, v, e_u, e_v, z, e_z) of the points."""
    p = np.asarray(points, F)[:, :3].astype(np.float64)
    out = []
    with np.errstate(all="ignore"):
        for v in range(len(K)):
            A = np.asarray(w2c[v], F).astype(np.float64).reshape(4, 4)
            k33 = np.asarray(K[v], F).astype(np.float64).reshape(3, 3)
            c, ec = _affine(A[:3, :3], np.zeros((3, 3)), [p[:, 0], p[:, 1], p[:, 2]], [0 * p[:, 0]] * 3, A[:3, 3], np.zeros(3))
            k, ek = _affine(k33, np.zeros((3, 3)), c, ec)
            u, eu = _div(k[0], ek[0], k[2], ek[2])
            vv, ev = _div(k[1], ek[1], k[2], ek[2])
            out.append((u, vv, 2 * eu, 2 * ev, c[2], 2 * ec[2]))
    return out


def compare_alpha(case, ref_mask, mine=None):
    """The reference's visual-hull mask against the oracle: they agree on every point with no near decision.  Returns counts."""
    mine = alpha_mask(case["points"], case["alpha"], case["K"], case["w2c"], case.get("near_far"), case["range_test"]) if mine is None \
        else mine
    near = np.zeros(len(mine), bool)
    lo = hi = None
    if case.get("near_far") is not None:
        lo, hi = float(case["near_far"][0]) - 1.0, float(case["near_far"][1])
    for u, v, eu, ev, z, ez in alpha_bounds(case["points"], case["K"], case["w2c"]):
        with np.errstate(invalid="ignore"):
            n = ~np.isfinite(u) | ~np.isfinite(v) | (np.abs(u - np.round(u)) <= eu) | (np.abs(v - np.round(v)) <= ev)
            n |= (np.abs(u) > 2.0 ** 62) | (np.abs(v) > 2.0 ** 62)
            if lo is not None:
                n |= (np.abs(z - lo) <= ez + U * abs(lo)) | (np.abs(z - hi) <= ez + U * abs(hi))
        near |= n
    bad = (np.asarray(ref_mask, bool) != mine) & ~near
    assert not bad.any(), "visual-hull mask differs away from a boundary at %d points (first %s)" % (bad.sum(), np.nonzero(bad)[0][:5])
    return dict(points=len(mine), near=int(near.sum()), flipped=int((np.asarray(ref_mask, bool) != mine).sum()))


def compare_reference(case, ref, fault=None):
    """Classify the reference's filter_by_masks_gpu results against the oracle, view by view.

    ref: per view the reference's geo_sum [H,W] (its check_geometric_consistency_gpu masks summed), its outputs without the range mask
    (`cam0`, `world0`, `conf0`: aligned with its final mask) and with the case's ranges (`cam`, `world`, `conf`).  fault: a planted
    fault of the fp32 oracle (FAULTS), for the test that shows the comparison catches it.  Raises AssertionError on a disagreement no
    bound explains; returns counts."""
    mats = view_matrices(case["K"], case["E"])
    V = len(case["depth"])
    st = dict(pixels=0, kept=0, near_geo=0, near_range=0, max_davg=0.0)
    for r in range(V):
        o = filter_view(case, r, mats, fault)
        rf = ref[r]
        live, pix = o["live"], o["pix_live"]
        single = V == 1 and fault != "single_view_geo"
        geo_r = np.asarray(rf["geo"]).reshape(-1)[pix] if V > 1 else np.zeros(len(pix), np.int64)
        fin_r = np.ones(len(pix), bool) if V == 1 else geo_r >= case["geo_n"]
        assert len(rf["cam0"]) == fin_r.sum(), "view %d: the reference's outputs do not follow its own geo_sum" % r
        if V > 1:
            b = bounds_view(case, r, pix)
            near = b["geo_min"] != b["geo_max"]
            assert np.all((geo_r >= b["geo_min"]) & (geo_r <= b["geo_max"])), "view %d: geo_sum outside its bound" % r
            assert np.all(o["geo"][~near] == geo_r[~near]), "view %d: a geometric decision differs away from its boundary" % r
            st["near_geo"] += int(near.sum())
        else:
            b = bounds_view(case, r, pix)
            near = np.zeros(len(pix), bool)
        fin_o = (o["geo"] >= case["geo_n"]) if not single else np.ones(len(pix), bool)
        both = fin_o & fin_r
        # values of the pixels both keep before the range mask, in the reference's order
        ref_idx = np.cumsum(fin_r) - 1
        ok = both & ~near
        x, y = (np.asarray(case["xy"][r], F).reshape(-1, 2)[pix][:, i] for i in range(2))
        if fault == "avg_xy":
            with np.errstate(all="ignore"):
                d = np.asarray(case["depth"][r], F).reshape(-1)[pix]
                x, y = x / d * o["avg"], y / d * o["avg"]
        rc = np.asarray(rf["cam0"])[ref_idx[ok]]
        assert np.array_equal(rc[:, :2], np.stack([x, y], -1)[ok]), "view %d: raw camera x, y differ" % r
        assert np.array_equal(np.asarray(rf["conf0"])[ref_idx[ok]], np.asarray(case["conf"][r], F).reshape(-1)[pix][ok])
        davg = np.abs(rc[:, 2].astype(np.float64) - o["avg"][ok])
        assert np.all(davg <= 2 * b["eavg"][ok]), "view %d: averaged depths differ beyond the bound (%.3g)" % (r, davg.max())
        st["max_davg"] = max(st["max_davg"], float(davg.max()) if len(davg) else 0.0)
        w64, ew = world_bounds(b, np.nonzero(ok)[0], x[ok], y[ok])
        rw = np.asarray(rf["world0"])[ref_idx[ok]].astype(np.float64)
        assert np.all(np.abs(rw - w64) <= 2 * ew + 1e-30), "view %d: world points differ beyond the bound" % r
        # the range mask on the world point, and with it the final list and its order
        if case.get("ranges") is not None:
            rg = np.asarray(case["ranges"], F).astype(np.float64)
            wr = np.asarray(rf["world0"]).astype(np.float64)
            in_r = np.all((wr >= rg[:3]) & (wr <= rg[3:]), 1)
            assert np.array_equal(np.asarray(rf["world"]), np.asarray(rf["world0"])[in_r]), "view %d: reference range self-check" % r
            w_all, ew_all = world_bounds(b, np.arange(len(pix)), x, y)
            rnear = np.any((np.abs(w_all - rg[:3]) <= 2 * ew_all) | (np.abs(w_all - rg[3:]) <= 2 * ew_all), 1) | near
            kept_r = np.zeros(len(pix), bool)
            kept_r[np.nonzero(fin_r)[0][in_r]] = True
            st["near_range"] += int(rnear.sum())
        else:
            kept_r, rnear = fin_r, near
        kept_o = np.zeros(len(pix), bool)
        kept_o[np.searchsorted(pix, o["pix"])] = True
        diff = kept_o != kept_r
        assert not (diff & ~rnear).any(), "view %d: %d pixels kept differently away from a boundary" % (r, (diff & ~rnear).sum())
        # order: both lists are row-major over the kept pixels, so equal kept sets give equal orders
        st["pixels"] += int(live.size)
        st["kept"] += int(kept_o.sum())
    return st
