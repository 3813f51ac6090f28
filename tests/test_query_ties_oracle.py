"""CPU: both neighbour queries' C oracles (oracle/query_oracle.c, oracle/frustum_oracle.c) where one integer or IEEE choice decides the
result: equal distances, coordinates on voxel faces, crowded voxels, the slot-0 voxel, empty grids and candidates on the radius
(oracle/hard_clouds.py).

  * hand-built cases pin the tie rule itself: the expected slots are derived by hand from the reference's replace-farthest loop
    (query_worldcoords.cu:276-293, query_point_indices.py:574-591), not computed by a second implementation;
  * the brute forces of test_oracle_query.py / test_oracle_frustum.py check everything the tie rule does not decide, on every family,
    and count the samples whose K-th distance ties, so each ties / duplicates scene is known to exercise the rule;
  * a face point's voxel is the IEEE divide's, not a multiply by the reciprocal.
"""
import numpy as np
import pytest

from oracle import frustum_oracle, hard_clouds as hc, query_oracle
from test_oracle_frustum import brute_force as frustum_brute_force
from test_oracle_query import brute_force as world_brute_force, check_sets


def _world(sc, ks, qs, K, SR, P, parity_slot0=1):
    return query_oracle.query(sc["xyz"], sc["lo"], sc["svs"], sc["dim"], np.array(ks, np.int32), np.array(qs, np.int32), sc["max_o"], P,
                              sc["radius"], campos=sc["campos"], raydir=sc["raydir"], t=sc["t"], SR=SR, K=K, parity_slot0=parity_slot0)


def _frustum(sc, opt, pixels=None):
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = hc.frustum_grid(sc["cam"], opt)
    grid = (ranges, svs, sdim, vscale, np.float32(rl ** 2), np.float32(dl ** 2))
    pix = sc["pixel_idx"] if pixels is None else pixels
    out = frustum_oracle.query(sc["pers"], ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P, pix,
                               grid[4], grid[5], max_o=opt.max_o)
    return grid, out


# ------------------------------------------------------------------------------------------------------------ hand-built tie cases
@pytest.mark.parametrize("case", hc.world_hand_cases(), ids=lambda c: c["name"])
def test_world_hand_tie_case(case):
    o = query_oracle.query(case["xyz"], case["lo"], case["svs"], case["dim"], case["ks"], case["ks"], 1000, 8, 0.0, campos=case["campos"],
                           raydir=case["raydir"], t=case["t"], SR=1, K=case["K"])
    assert o["counters"]["R2"] == 1 and o["sample_loc_w"][0, 0].tolist() == [4.5, 4.5, 4.5]
    assert o["sample_pidx"][0, 0].tolist() == case["want"]
    m, loc, found = world_brute_force(case["xyz"], case["lo"], case["svs"], case["dim"], case["ks"], case["ks"], 8, 0.0, case["campos"],
                                      case["raydir"], case["t"], 1, case["K"])
    assert check_sets(o["sample_pidx"], found, case["K"]) == 1     # a tie at the K-th distance: the rule decides these cases


def test_earliest_wins_is_not_the_tie_rule():
    """Keeping the K smallest by (distance, visit order) -- the rule the brute force once assumed -- keeps B and E in the first hand
    case; the reference keeps E and D."""
    case = hc.world_hand_cases()[0]
    _, _, found = world_brute_force(case["xyz"], case["lo"], case["svs"], case["dim"], case["ks"], case["ks"], 8, 0.0, case["campos"],
                                    case["raydir"], case["t"], 1, case["K"])
    earliest = sorted(i for _, i in found[0][0][:case["K"]])
    assert earliest == [1, 3] and sorted(case["want"]) == [2, 3]


@pytest.mark.parametrize("case", hc.frustum_hand_cases(), ids=lambda c: c["name"])
def test_frustum_hand_tie_case(case):
    opt = case["opt"]
    grid, o = _frustum(case, opt)
    ranges, svs, sdim = grid[0], grid[1], grid[2]
    assert ranges[:3].tolist() == [-1.0, -1.0, 1.0] and svs.tolist() == [0.25] * 3 and sdim.tolist() == [8, 8, 8]
    s = case["sample"]
    assert o["ray_mask"].tolist() == [1] and o["sample_loc"][0, s].tolist() == [0.125, 0.125, 2.125]
    assert o["sample_pidx"][0, s].tolist() == case["want"]


# ------------------------------------------------------------------------------------------------------------ faces: the IEEE divide
def test_world_face_voxel_is_the_ieee_divide():
    """Coordinates where (p - lo) / svs and (p - lo) * (1 / svs) floor to different voxels: the oracle's voxel (seen through the
    slot-0 cell, which is the voxel of point 0) is the divide's.  Also the upper face: lo + dim * svs is outside, and so is a coordinate
    a few ulps below it whose subtract rounds onto the face; the first one that does not is inside."""
    n_disc = 0
    for vsize, vscale in (((0.5, 0.25, 0.75), (1, 1, 1)), ((0.5, 0.5, 0.5), (3, 3, 3)), ((0.5, 0.25, 0.75), (3, 3, 3))):
        sc = hc.world_scene("faces", vsize, vscale)
        lo, svs, dim = sc["lo"], sc["svs"], sc["dim"]
        fv = hc.face_values(lo, svs, dim)
        centre = (lo + 0.5 * dim * svs).astype(np.float32)
        for a in range(3):
            for w in fv[a]:
                p = centre.copy()
                p[a] = w
                c = hc.vox_div(p, lo, svs)
                inside = bool(np.all((c >= 0) & (c < dim)))
                o = _world(dict(sc, xyz=p[None]), (3, 3, 3), (3, 3, 3), 1, 1, 4)
                assert o["counters"]["n_occ"] == int(inside)
                if inside:
                    assert o["counters"]["slot0_cell"] == int((c[0] * dim[1] + c[1]) * dim[2] + c[2])
                n_disc += int(hc.vox_div(w, lo[a], svs[a]) != hc.vox_mul(w, lo[a], svs[a]))
        for a in range(3):
            # p - lo rounds: a few ulps below the upper face can still land on it (outside); lo itself is voxel 0
            up = np.float32(lo[a] + np.float32(dim[a]) * svs[a])
            seen = set()
            for val in [up] + [hc.ulps(up, -u) for u in range(1, 5)] + [lo[a]]:
                p = centre.copy()
                p[a] = val
                n = int(0 <= hc.vox_div(val, lo[a], svs[a]) < dim[a])
                seen.add((val < up, n))
                assert _world(dict(sc, xyz=p[None]), (3, 3, 3), (3, 3, 3), 1, 1, 4)["counters"]["n_occ"] == n, (a, val)
            assert (True, 1) in seen and (False, 0) in seen
    assert n_disc > 0


# ------------------------------------------------------------------------------------------------------------ world families
WORLD_CELLS = [
    # family, vsize, vscale, (ks, qs), K, SR, P
    *[(f, (0.5, 0.5, 0.5), (1, 1, 1), ((3, 3, 3), (3, 3, 3)), 8, 33, 4) for f in hc.WORLD_FAMILIES],
    *[(f, (0.5, 0.25, 0.75), (3, 3, 3), ((5, 5, 5), (5, 5, 5)), 3, 31, 32) for f in hc.WORLD_FAMILIES],
    *[(f, (0.5, 0.5, 0.5), (1, 1, 1), ((3, 3, 3), (5, 5, 5)), 1, 32, 1) for f in hc.WORLD_FAMILIES],
    *[(f, (0.5, 0.25, 0.75), (1, 1, 1), ((5, 5, 5), (3, 3, 3)), 8, 1, 4) for f in hc.WORLD_FAMILIES],
]


@pytest.mark.parametrize("family,vsize,vscale,sizes,K,SR,P", WORLD_CELLS)
def test_world_oracle_vs_brute_force_on_hard_clouds(family, vsize, vscale, sizes, K, SR, P):
    sc = hc.world_scene(family, vsize, vscale, P=P, K=K)
    ks, qs = sizes
    o = _world(sc, ks, qs, K, SR, P)
    m, loc, found = world_brute_force(sc["xyz"], sc["lo"], sc["svs"], sc["dim"], ks, qs, P, sc["radius"], sc["campos"], sc["raydir"],
                                      sc["t"], SR, K)
    assert np.array_equal(m, o["ray_mask"])
    assert np.array_equal(o["sample_loc_w"], loc)
    tied = check_sets(o["sample_pidx"], found, K)
    n_samples = sum(len(r) for r in found)
    print("[world %s vsize %s vscale %s ks %s qs %s K %d SR %d P %d] rays kept %d, samples %d, tied at the K-th distance %d"
          % (family, vsize, vscale, ks, qs, K, SR, P, int(m.sum()), n_samples, tied))
    c = o["counters"]
    if family in ("ties", "ties1") or (family == "duplicates" and P > 1):         # P = 1 keeps one of two equal points: no tie left
        assert tied > 0, "the scene must exercise the tie rule"
    elif family == "empty":
        assert c["n_occ"] == 0 and c["R1"] == 0 and c["R2"] == 0 and not o["ray_mask"].any()
    elif family == "crowded":
        assert c["max_pts"] >= max(3 * P, K + 3) and c["overflow_p"] == 1
    elif family == "radius":
        r2 = np.float32(sc["radius"]) * np.float32(sc["radius"])
        assert sum(d == r2 for ray in found for cand in ray for d, _ in cand) > 0, "no candidate at exactly the radius"
    elif family == "faces":
        q = (loc[loc.any(-1)] - sc["lo"]) / sc["svs"]
        assert (q == np.floor(q)).any(), "no sample on a voxel face"
    if family != "empty":
        assert c["R2"] > 0


def test_world_slot0_and_parity_switch():
    """The first in-range index (3: indices 0..2 lie outside the grid) owns the dead voxel: with parity_slot0 1 it is never a neighbour,
    with 0 it is, and the two runs differ only by that voxel's points."""
    sc = hc.world_scene("slot0")
    lo, svs, dim = sc["lo"], sc["svs"], sc["dim"]
    c3 = hc.vox_div(sc["xyz"][3], lo, svs)
    on = _world(sc, (3, 3, 3), (3, 3, 3), 8, 24, 8, parity_slot0=1)
    off = _world(sc, (3, 3, 3), (3, 3, 3), 8, 24, 8, parity_slot0=0)
    assert on["counters"]["slot0_cell"] == off["counters"]["slot0_cell"] == int((c3[0] * dim[1] + c3[1]) * dim[2] + c3[2])
    assert not (on["sample_pidx"] == 3).any() and (off["sample_pidx"] == 3).any()
    for parity, o in ((1, on), (0, off)):
        m, loc, found = world_brute_force(sc["xyz"], lo, svs, dim, (3, 3, 3), (3, 3, 3), 8, 0.0, sc["campos"], sc["raydir"], sc["t"], 24, 8,
                                          parity_slot0=parity)
        assert np.array_equal(m, o["ray_mask"]) and np.array_equal(loc, o["sample_loc_w"])
        check_sets(o["sample_pidx"], found, 8)


# ------------------------------------------------------------------------------------------------------------ frustum families
FRUSTUM_CELLS = [
    *[("ties", ks, qs, (2, 2, 1), 8 if ks[0] > 2 else 1, 33) for ks, qs in hc.FRUSTUM_SIZES],   # one-voxel searches: K 1
    *[(f, (3, 3, 3), (3, 3, 3), (3, 3, 1), 3, 31) for f in hc.FRUSTUM_FAMILIES],
    *[(f, (3, 3, 1), (4, 4, 2), (3, 3, 1), 1, 32) for f in hc.FRUSTUM_FAMILIES],
    *[(f, (5, 5, 3), (5, 5, 5), (2, 2, 1), 8, 1) for f in ("duplicates", "faces", "crowded")],
    ("faces", (3, 3, 1), (3, 3, 1), (2, 2, 1), 8, 33),
]


@pytest.mark.parametrize("family,ks,qs,vscale,K,SR", FRUSTUM_CELLS)
def test_frustum_oracle_vs_brute_force_on_hard_clouds(family, ks, qs, vscale, K, SR):
    rl, dl = (2.0, 0.25) if family == "radius" else (0.0, 0.0)      # depth limit a quarter voxel: inside the sample's own voxel
    opt = hc.frustum_opt(vscale=vscale, ks=ks, qs=qs, SR=SR, K=K, P=4, radius_limit_scale=rl, depth_limit_scale=dl)
    sc = hc.frustum_scene(family, opt)
    pix = sc["pixel_idx"]
    if family in ("ties", "radius", "duplicates"):                        # every third pixel, and the three outside the grid
        pix = np.concatenate([pix[:-3][::3], pix[-3:]])
    grid, o = _frustum(sc, opt, pix)
    mask, rows = frustum_brute_force(sc, opt, grid, pix)
    assert np.array_equal(o["ray_mask"], mask)
    assert o["counters"]["n_bad_pixel"] == 3
    assert o["sample_loc"].shape[0] == len(rows)
    for r, ray in enumerate(rows):
        assert np.array_equal(o["sample_loc"][r], np.stack([e[0] for e in ray]))
    tied = check_sets(o["sample_pidx"], [[e[3] for e in ray] for ray in rows], K)
    print("[frustum %s ks %s qs %s vscale %s K %d SR %d] rays kept %d of %d, tied at the K-th distance %d"
          % (family, ks, qs, vscale, K, SR, int(mask.sum()), len(pix), tied))
    if family in ("ties", "ties1", "duplicates"):
        assert tied > 0, "the scene must exercise the tie rule"
    if family == "empty":
        assert o["counters"]["R2"] == 0 and not o["ray_mask"].any()
    else:
        assert o["counters"]["R2"] > 0
    if family == "crowded" and SR > 1:                                   # SR 1 marks the first listed depth only
        assert o["counters"]["max_pts"] >= 3 * opt.P and o["counters"]["overflow_p"] == 1
    if family == "radius":
        d2 = grid[5]
        assert d2 > 0 and any(np.any(fp_z2 == d2) for fp_z2 in _z2_of_candidates(sc, rows)), "no candidate at exactly the depth limit"
    if family == "faces" and qs[2] <= 2:
        # columns whose only dilated voxel is depth 0: far_id 0, so the ray misses although the column holds a point (F4)
        sdim, vs = grid[2], grid[3]
        q = (sc["pers"] - grid[0][:3]) / grid[1]
        deep = {(int(a), int(b)) for a, b, c in np.floor(q[np.all((q >= 0) & (q < sdim), 1)]).astype(int) if c > 0}
        zero = {(int(a), int(b)) for a, b, c in np.floor(q[np.all((q >= 0) & (q < sdim), 1)]).astype(int) if c == 0}
        only0 = [c for c in zero if all((c[0] + dx, c[1] + dy) not in deep for dx in range(-2, 3) for dy in range(-2, 3))]
        assert only0
        for cx, cy in only0:
            sel = [i for i, (px, py) in enumerate(pix) if px >= 0 and py >= 0 and px // vs[0] == cx and py // vs[1] == cy]
            assert sel and not o["ray_mask"][sel].any()


def _z2_of_candidates(sc, rows):
    from test_oracle_frustum import fp32_distances
    for ray in rows:
        for loc, _, _, c32 in ray:
            if c32:
                yield fp32_distances(sc["pers"][[i for _, i in c32]], loc)[1]
