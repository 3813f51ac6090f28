"""TEST INFRASTRUCTURE ONLY -- CPU restatement of pnb_vox_build / pnb_vox_outputs (pointnerf_b200/csrc/voxelize.cu), the voxel
down-sampling of models/mvs/mvs_utils.py:484-561.  numpy, serial semantics, bit for bit what the kernels compute:

  * voxel index floor((p - space_min) / vox_sz) per axis in fp32 (subtract, true divide), converted as CUDA's saturating
    float -> int32 (NaN -> 0, as torch's CUDA `.to(torch.int32)` does);
  * voxels in lexicographic (x, y, z) order (torch.unique(dim=0)), points inside a voxel by ascending index (the stable sort);
  * centroid: the fp64 tree of voxelize.cu's header comment (256 lanes, lane t adds x_t, x_{t+256}, ... in order, then a halving
    tree over the lanes present), divided by the count in fp64 and rounded once to fp32;
  * closest point: residual sqrt((dx*dx + dy*dy) + dz*dz) in fp32 against the fp32 centroid, no fused multiply-add; the lowest point
    index among equal residuals.
"""
import numpy as np

LANES = 256
U = 2.0 ** -24


def voxel_index(xyz, space_min, vox_sz):
    """int32 [N,3]: the kernels' voxel index of every point (space_min, vox_sz: float32 [3])."""
    with np.errstate(invalid="ignore", divide="ignore"):             # a zero voxel size (a one-point cloud) gives NaN / inf
        q = np.floor((np.asarray(xyz, np.float32) - np.asarray(space_min, np.float32)) / np.asarray(vox_sz, np.float32))
    q = q.astype(np.float64)
    q = np.where(np.isnan(q), 0.0, np.clip(q, -2147483648.0, 2147483647.0))
    return q.astype(np.int32)


def centroid_tree(val_sorted, seg, start, count):
    """fp64 lane sums and halving tree per voxel; val_sorted [N,3] fp32 in voxel-major, ascending-index order."""
    M = count.shape[0]
    pos = np.arange(val_sorted.shape[0]) - start[seg]
    lane, rnd = pos % LANES, pos // LANES
    P = np.zeros((M, LANES, 3), np.float64)
    x = val_sorted.astype(np.float64)
    for r in range(int(rnd.max()) + 1 if rnd.size else 0):
        sel = rnd == r
        if r == 0:
            P[seg[sel], lane[sel]] = x[sel]
        else:
            P[seg[sel], lane[sel]] = P[seg[sel], lane[sel]] + x[sel]
    width = np.minimum(count, LANES)
    off = LANES // 2
    while off >= 1:
        t = np.arange(off)
        take = (t[None, :] + off) < width[:, None]                    # [M, off]
        summed = P[:, :off] + P[:, off:2 * off]
        P[:, :off] = np.where(take[:, :, None], summed, P[:, :off])
        off //= 2
    return (P[:, 0] / count[:, None].astype(np.float64)).astype(np.float32)


def residual(val, cen):
    d = (val.astype(np.float32) - cen.astype(np.float32)).astype(np.float32)
    s = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(np.float32) + d[:, 2] * d[:, 2]
    return np.sqrt(s.astype(np.float32))


def voxelize(xyz, space_min, vox_sz, val=None, closest=False):
    """xyz [N,3] keys, val [N,3] values (default xyz).  Returns grid_idx int32 [M,3], inv_idx int64 [N], first int64 [M] (lowest point
    index of each voxel) and, with values, centroid float32 [M,3] and, with closest, closest int64 [M]."""
    xyz = np.asarray(xyz, np.float32).reshape(-1, 3)
    val = xyz if val is None else np.asarray(val, np.float32).reshape(-1, 3)
    idx = voxel_index(xyz, space_min, vox_sz)
    grid_idx, inv = np.unique(idx, axis=0, return_inverse=True)
    inv = inv.reshape(-1).astype(np.int64)
    order = np.argsort(inv, kind="stable")
    seg = inv[order]
    count = np.bincount(inv, minlength=grid_idx.shape[0]).astype(np.int64)
    start = np.concatenate([[0], np.cumsum(count)[:-1]]).astype(np.int64)
    out = dict(grid_idx=grid_idx.astype(np.int32).reshape(-1, 3), inv_idx=inv, first=order[start].astype(np.int64) if count.size
               else np.zeros(0, np.int64))
    cen = centroid_tree(val[order], seg, start, count)
    out["centroid"] = cen.reshape(-1, 3)
    if closest:
        r = residual(val, cen[inv]) if inv.size else np.zeros(0, np.float32)
        pick = np.lexsort((np.arange(inv.size), r, inv))               # by voxel, then residual, then point index
        out["closest"] = pick[start].astype(np.int64) if count.size else np.zeros(0, np.int64)
        out["residual"] = r
    return out


def centroid_bound(val, inv, m):
    """Per voxel: the bound (c + 2) u X on |centroid - an fp32 mean summed in any order| (c points of magnitude <= X), and X."""
    x = np.abs(val).max(1)
    xmax = np.zeros(m, np.float64)
    np.maximum.at(xmax, inv, x)
    cnt = np.bincount(inv, minlength=m)
    return (cnt + 2) * U * xmax, xmax


def check_closest(ref_idx, ours, ref_res, inv, bound, xmax):
    """Equal where the reference's two smallest residuals are further apart than the tolerance; else ours is near-tied."""
    tol = 2 * bound + 8 * U * xmax
    order = np.lexsort((ref_res, inv))
    seg_first = np.r_[0, np.flatnonzero(np.diff(inv[order])) + 1]
    best = ref_res[order[seg_first]]
    nxt = np.full_like(best, np.inf)
    has2 = np.r_[np.diff(seg_first) > 1, len(order) - seg_first[-1] > 1]
    nxt[has2] = ref_res[order[seg_first[has2] + 1]]
    clear = (nxt - best) > tol
    assert np.array_equal(ours[clear], ref_idx[clear])
    assert np.all(ref_res[ours[~clear]] <= best[~clear] + tol[~clear])
    return clear
