"""GPU: both neighbour queries of libpnb200, through their drop-ins, against the C oracles bit for bit on the adversarial clouds of
oracle/hard_clouds.py (distance ties, voxel faces, crowded voxels, the slot-0 voxel, empty grids, candidates on the radius), over the
options where the kernels branch: K 1 / 3 / 8, SR 1 / 31 / 32 / 33 / 128 (k_march fills 32 steps per ballot), world kernel / query
sizes (3,3) (5,5) (3,5) (5,3) with cubic and anisotropic voxels and vscale 1 / 3, every frustum size class pnb_frustum_build accepts,
pnb_parity_slot0 0 and 1, rotated cameras.

Compared: ray mask, compacted pixels, neighbour indices IN K-SLOT ORDER, sample positions, and every counter both sides define the same
way.  Where oracle/_ref/ was built, the reference's own kernels run on the one-point-per-voxel tie scenes too.
"""
import ctypes as C
import os
import time

import numpy as np
import pytest
import torch

from oracle import frustum_oracle, hard_clouds as hc, query_oracle, shade_oracle
from pointnerf_b200 import point_query as pq
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200 import scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")

WORLD_SIZES = (((3, 3, 3), (3, 3, 3)), ((5, 5, 5), (5, 5, 5)), ((3, 3, 3), (5, 5, 5)), ((5, 5, 5), (3, 3, 3)))
GRIDS = (((0.5, 0.5, 0.5), (1, 1, 1)), ((0.5, 0.25, 0.75), (3, 3, 3)), ((0.5, 0.25, 0.75), (1, 1, 1)), ((0.5, 0.5, 0.5), (3, 3, 3)))
KSR = [(K, SR) for K in (1, 3, 8) for SR in (1, 31, 32, 33, 128)]
_scenes = {}


def _scene(family, vsize, vscale, P, K):
    key = (family, vsize, vscale, P, K)
    if key not in _scenes:
        _scenes[key] = hc.world_scene(family, vsize, vscale, P=P, K=K)
    return _scenes[key]


def world_oracle(sc, ks, qs, K, SR, P, parity_slot0=1):
    return query_oracle.query(sc["xyz"], sc["lo"], sc["svs"], sc["dim"], np.array(ks, np.int32), np.array(qs, np.int32), sc["max_o"], P,
                              sc["radius"], campos=sc["campos"], raydir=sc["raydir"], t=sc["t"], SR=SR, K=K, parity_slot0=parity_slot0)


def world_gpu(sc, ks, qs, K, SR, P, parity_slot0=1, camrot=None):
    """The drop-in's grid and query objects (what lighting_fast_querier.run_query builds), on an explicit grid."""
    xyz = torch.from_numpy(sc["xyz"]).to(DEV).contiguous()
    grid = pq.VoxelGrid(xyz, sc["lo"], sc["svs"], sc["dim"], np.array(qs, np.int32), sc["max_o"], P, parity_slot0=bool(parity_slot0))
    raydir = torch.from_numpy(sc["raydir"]).to(DEV).contiguous()
    t = torch.from_numpy(sc["t"]).to(DEV).contiguous()
    q = pq.QueryResult(grid, [float(v) for v in sc["campos"]], raydir, t, int(t.shape[-1]), SR, K, sc["radius"], np.array(ks, np.int32),
                       want_counters=True)
    rot = torch.eye(3) if camrot is None else torch.as_tensor(camrot)
    ex = q.export(pq.make_cam_opts(torch.from_numpy(sc["campos"]), rot))
    return grid.counters, q.counters, {k: (v.cpu().numpy() if isinstance(v, torch.Tensor) else v) for k, v in ex.items()}


def assert_world_same(sc, ks, qs, K, SR, P, parity_slot0=1, camrot=None, what=""):
    o = world_oracle(sc, ks, qs, K, SR, P, parity_slot0)
    gc, qc, ex = world_gpu(sc, ks, qs, K, SR, P, parity_slot0, camrot)
    tag = "%s ks %s qs %s K %d SR %d P %d parity %d %s" % (sc["name"], ks, qs, K, SR, P, parity_slot0, what)
    assert np.array_equal(ex["ray_mask"], o["ray_mask"]), tag
    assert ex["sample_pidx"].shape == o["sample_pidx"].shape, tag
    assert np.array_equal(ex["sample_pidx"], o["sample_pidx"]), tag + ": neighbours or their K-slot order differ"
    assert np.array_equal(ex["sample_loc_w"], o["sample_loc_w"]), tag
    oc = o["counters"]
    for k in ("n_occ", "max_pts", "overflow_o", "overflow_p", "slot0_cell"):
        assert gc[k] == oc[k], (tag, k, gc[k], oc[k])
    assert (qc["R1"], qc["R2"], qc["n_pairs"], qc["n_valid"]) == (oc["R1"], oc["R2"], oc["n_valid_pairs"], oc["n_valid_samples"]), tag
    return o, ex


# ------------------------------------------------------------------------------------------------------------ world query
@pytest.mark.parametrize("family", hc.WORLD_FAMILIES)
def test_world_query_matches_oracle_on_hard_clouds(family):
    """Every (K, SR) pair against the four kernel / query sizes and the four grids in turn, both slot-0 settings alternating."""
    t0 = time.time()
    n = 0
    for i, (K, SR) in enumerate(KSR):
        for j, (ks, qs) in enumerate(WORLD_SIZES):
            vsize, vscale = GRIDS[(i + j) % len(GRIDS)]
            P = (1, 4, 32)[(i + 2 * j) % 3]
            sc = _scene(family, vsize, vscale, P, K)
            assert_world_same(sc, ks, qs, K, SR, P, parity_slot0=(i + j) % 2)
            n += 1
    print("[gpu world %s] %d cells bit-exact in %.1f s" % (family, n, time.time() - t0))


@pytest.mark.parametrize("family", ["slot0", "ties", "crowded"])
def test_world_parity_slot0_both_settings(family):
    """pnb_parity_slot0 0 keeps the points of the slot-0 voxel; the oracle's switch does the same, and the settings differ on these
    scenes (the first in-range point sits next to the samples)."""
    sc = _scene(family, (0.5, 0.5, 0.5), (1, 1, 1), 8, 8)
    a, _ = assert_world_same(sc, (3, 3, 3), (3, 3, 3), 8, 33, 8, parity_slot0=1)
    b, _ = assert_world_same(sc, (3, 3, 3), (3, 3, 3), 8, 33, 8, parity_slot0=0)
    if family == "slot0":
        assert not np.array_equal(a["sample_pidx"], b["sample_pidx"]) and (b["sample_pidx"] == 3).any() and not (a["sample_pidx"] == 3).any()


def test_world_single_point_and_all_outside():
    sc = _scene("empty", (0.5, 0.5, 0.5), (1, 1, 1), 4, 8)
    for xyz in (sc["xyz"][:1], sc["xyz"]):
        s = dict(sc, xyz=np.ascontiguousarray(xyz), max_o=len(xyz))
        o, ex = assert_world_same(s, (3, 3, 3), (3, 3, 3), 8, 24, 4)
        assert o["counters"]["R2"] == 0 and not ex["ray_mask"].any()


@pytest.mark.parametrize("yaw,pitch", [(0.7, 0.3), (-1.1, 0.45)])
def test_world_rotated_camera(yaw, pitch):
    """Rays from a rotated camera (raydir = R d) on the tie and face clouds: bit-exact against the oracle, and the export's perspective
    coordinates within 1e-6 of shade_oracle.w2pers."""
    rot = scene.orbit_rotation(yaw, pitch)
    for family in ("ties", "faces", "duplicates"):
        sc = dict(_scene(family, (0.5, 0.5, 0.5), (1, 1, 1), 8, 8))
        cam_dirs = np.array([(i / 8.0, j / 8.0, 1.0) for i in range(-3, 5) for j in range(-3, 5)], np.float32)
        centre = (sc["lo"] + 0.5 * sc["dim"] * sc["svs"]).astype(np.float32)
        sc["raydir"] = np.ascontiguousarray(cam_dirs @ rot.T, np.float32)
        sc["campos"] = (centre - 6.0 * rot[:, 2]).astype(np.float32)            # looks at the grid centre along R[:, 2]
        sc["t"] = np.ascontiguousarray(sc["t"][sc["t"] >= 3.0])               # samples at depth >= 3: x/z keeps fp32 accuracy
        o, ex = assert_world_same(sc, (3, 3, 3), (3, 3, 3), 8, 32, 8, camrot=rot, what="rot %s %s" % (yaw, pitch))
        assert o["counters"]["R2"] > 10
        want = shade_oracle.w2pers(torch.from_numpy(o["sample_loc_w"]), torch.from_numpy(rot), torch.from_numpy(sc["campos"])).numpy()
        filled = (o["sample_loc_w"] != 0).any(-1)
        d = np.abs(ex["sample_loc"][filled] - want[filled]).max()
        assert d <= 1e-6, d


# ------------------------------------------------------------------------------------------------------------ frustum query
def frustum_oracle_run(sc, opt, pixels=None):
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = hc.frustum_grid(sc["cam"], opt)
    pix = sc["pixel_idx"] if pixels is None else pixels
    return frustum_oracle.query(sc["pers"], ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P, pix,
                                np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)


def frustum_gpu(sc, opt, pixels=None):
    """The drop-in querier's query_points on the scene's camera (the grid comes from the intrinsic, as in the reference)."""
    cam = sc["cam"]
    q = qpi.lighting_fast_querier(DEV, opt)
    pers = torch.from_numpy(sc["pers"]).to(DEV)[None].contiguous()
    pix = torch.from_numpy(sc["pixel_idx"] if pixels is None else pixels).to(DEV)[None]
    npts = torch.tensor([pers.shape[1]], dtype=torch.int32, device=DEV)
    rot, pos = torch.eye(3, device=DEV)[None], torch.zeros(1, 3, device=DEV)
    out = q.query_points(pix, pers, pers, npts, np.int64(cam["H"]), np.int64(cam["W"]), cam["intrinsic"], cam["near"], cam["far"], None,
                         pos, rot)
    return q, out


def assert_frustum_same(sc, opt, pixels=None, what=""):
    o = frustum_oracle_run(sc, opt, pixels)
    q, out = frustum_gpu(sc, opt, pixels)
    pidx, loc, mask = out[0][0].cpu().numpy(), out[1][0].cpu().numpy(), out[4][0].cpu().numpy()
    tag = "%s ks %s qs %s vscale %s K %d SR %d P %d %s" % (sc["name"], opt.kernel_size, opt.query_size, opt.vscale, opt.K, opt.SR, opt.P,
                                                         what)
    assert np.array_equal(mask, o["ray_mask"]), tag
    assert np.array_equal(q.last_pixel_idx_cur[0].cpu().numpy(), o["pixel_idx_cur"]), tag
    assert np.array_equal(loc, o["sample_loc"]), tag
    assert np.array_equal(pidx, o["sample_pidx"]), tag + ": neighbours or their K-slot order differ"
    bc, qc, oc = q.last_build_counters, q.last_query_counters, o["counters"]
    assert qc["R2"] == oc["R2"] and qc["n_bad_pixel"] == oc["n_bad_pixel"], tag
    assert bc["overflow_o"] == oc["overflow_o"], tag
    # every column has a ray here, so the columns listing more than SR depths are the same set on both sides
    assert bc["n_col_capped"] == oc["n_col_capped"], (tag, bc["n_col_capped"], oc["n_col_capped"])
    # the oracle counts voxel fills in the voxels the rays marked, the build in every voxel: a subset
    assert oc["max_pts"] <= bc["max_pts"] and (oc["overflow_p"] == 0 or bc["overflow_p"] > 0), tag
    return o, out


@pytest.mark.parametrize("family", hc.FRUSTUM_FAMILIES)
def test_frustum_query_matches_oracle_on_hard_clouds(family):
    """Every accepted size class against every (K, SR) pair, vscale 2 and 3 alternating; z extent 40 (not a multiple of 32)."""
    t0 = time.time()
    n = 0
    for j, (ks, qs) in enumerate(hc.FRUSTUM_SIZES):
        for i, (K, SR) in enumerate(KSR):
            vscale = ((2, 2, 1), (3, 3, 1))[(i + j) % 2]
            lim = (2.0, 0.25) if family == "radius" else (0.0, 0.0)
            opt = hc.frustum_opt(vscale=vscale, ks=ks, qs=qs, SR=SR, K=K, P=(1, 4, 8)[(i + j) % 3], radius_limit_scale=lim[0],
                                 depth_limit_scale=lim[1])
            key = (family, vscale, opt.P, K, lim)
            if key not in _scenes:
                _scenes[key] = hc.frustum_scene(family, opt)
            assert_frustum_same(_scenes[key], opt)
            n += 1
    print("[gpu frustum %s] %d cells bit-exact in %.1f s" % (family, n, time.time() - t0))


@pytest.mark.parametrize("case", hc.frustum_hand_cases(), ids=lambda c: c["name"])
def test_frustum_hand_tie_case(case):
    o, out = assert_frustum_same(case, case["opt"])
    assert out[0][0, 0, case["sample"]].tolist() == case["want"]


def test_world_hand_tie_cases():
    for c in hc.world_hand_cases():
        sc = dict(c, name=c["name"], radius=0.0, max_o=len(c["xyz"]))
        o, ex = assert_world_same(sc, c["ks"], c["ks"], c["K"], 1, 8)
        assert ex["sample_pidx"][0, 0].tolist() == c["want"], c["name"]


# ------------------------------------------------------------------------------------------------------------ the reference's kernels
def _ref_world_ext():
    from oracle import build_ref
    ext = build_ref.load_prebuilt()
    if ext is None:
        pytest.skip("oracle/_ref/%s.so was not built (build() makes it where the reference tree exists)" % build_ref.NAME)
    return ext


def _ref_world(ext, sc, ks, qs, K, SR, P):
    """woord_query_grid_point_index with the 18 arguments of the reference's point_query.py:85-93 (as
    oracle/record_ref_kernel.reference_query forms them), on the scene's explicit grid."""
    xyz = torch.from_numpy(sc["xyz"]).to(DEV)[None].contiguous()
    raydir = torch.from_numpy(sc["raydir"]).to(DEV)[None].contiguous()
    t = torch.from_numpy(sc["t"]).to(DEV)
    campos = torch.from_numpy(sc["campos"]).to(DEV)[None]
    raypos = (campos[:, None, None, :] + raydir[:, :, None, :] * t[None, None, :, None]).contiguous()
    R, D = raydir.shape[1], t.shape[0]
    pix = torch.zeros(1, R, 2, dtype=torch.int32, device=DEV)
    ranges = torch.from_numpy(np.concatenate([sc["lo"], sc["lo"] + sc["dim"] * sc["svs"]]).astype(np.float32)).to(DEV)
    i3 = lambda v: torch.tensor(list(v), dtype=torch.int32, device=DEV)  # noqa: E731
    out = ext.woord_query_grid_point_index(pix, raypos, xyz, torch.tensor([xyz.shape[1]], dtype=torch.int32, device=DEV), i3(ks), i3(qs),
                                           SR, K, R, D, i3(sc["dim"]), int(sc["max_o"]), P, float(sc["radius"]), ranges,
                                           torch.from_numpy(sc["svs"]).to(DEV), 1024, 2)
    torch.cuda.synchronize()
    return [v[0].cpu().numpy() for v in out[:3]]


def _coords(idx, pts):
    """[..., K] neighbour indices -> their coordinates, sorted as (x, y, z) records along K (empty slots last): a multiset that does
    not depend on which of two equal points a kernel stored first."""
    c = np.where(idx[..., None] >= 0, pts[np.maximum(idx, 0)], np.float32(np.inf)).astype(np.float32)
    return np.sort(np.ascontiguousarray(c).view([("x", "f4"), ("y", "f4"), ("z", "f4")])[..., 0], axis=-1)


def _shell_near(loc, cell, lo, svs, layers):
    c = hc.vox_div(loc, lo, svs)
    return np.abs(c - np.asarray(cell)).max(-1) < layers


@pytest.mark.parametrize("family,ks,K,SR", [("ties1", (3, 3, 3), 8, 32), ("ties1", (5, 5, 5), 3, 33), ("ties1", (3, 3, 3), 1, 31),
                                            ("duplicates", (3, 3, 3), 8, 24)])
def test_reference_world_kernel_on_tie_scenes(family, ks, K, SR):
    """The reference's own query kernel against the oracle.  One point per voxel: its atomics cannot reorder candidates, so the K-slot
    order must match bit for bit, except in the shells around the voxel that won ITS occupancy slot 0 (an atomic race), recovered from
    the run as the one voxel whose points it never returns.  Duplicates: the multiset of neighbour coordinates."""
    ext = _ref_world_ext()
    sc = _scene(family, (0.5, 0.5, 0.5), (1, 1, 1), 64, K)
    P = 64
    r_pidx, r_loc, r_mask = _ref_world(ext, sc, ks, ks, K, SR, P)
    o = world_oracle(sc, ks, ks, K, SR, P, parity_slot0=0)                       # nothing dead on our side
    assert o["counters"]["max_pts"] <= P and o["counters"]["overflow_o"] == 0
    r_mask = r_mask.reshape(-1) > 0
    both = r_mask & (o["ray_mask"] > 0)
    assert int((r_mask != (o["ray_mask"] > 0)).sum()) <= 2
    ro, rr = (np.cumsum(o["ray_mask"] > 0) - 1)[both], (np.cumsum(r_mask) - 1)[both]
    a, b = o["sample_pidx"][ro], r_pidx[rr]
    la, lb = o["sample_loc_w"][ro], r_loc[rr]
    assert np.array_equal(la, lb)
    missing = np.setdiff1d(np.unique(a[a >= 0]), np.unique(b[b >= 0]))
    cells = np.unique(hc.vox_div(sc["xyz"][missing], sc["lo"], sc["svs"]), axis=0) if len(missing) else np.zeros((0, 3), np.int64)
    assert len(cells) <= 1, "points the reference never returns span %d voxels (expected its slot-0 voxel only)" % len(cells)
    near = np.zeros(a.shape[:2], bool)
    if len(cells):
        near = _shell_near(la, cells[0], sc["lo"], sc["svs"], (ks[0] + 1) // 2) & (la != 0).any(-1)
    keep = ~near
    if family == "ties1":
        bad = (a != b).any(-1) & keep
        assert not bad.any(), "%d samples differ in their K-slot order from the reference kernel" % int(bad.sum())
    else:
        bad = (_coords(a, sc["xyz"]) != _coords(b, sc["xyz"])).any(-1) & keep
        assert not bad.any(), "%d samples differ in their neighbour coordinates from the reference kernel" % int(bad.sum())
    n_cmp = int((keep & ((a >= 0).any(-1) | (b >= 0).any(-1))).sum())
    print("[reference world %s ks %s K %d SR %d] samples compared %d, excluded near its slot-0 voxel %d" % (family, ks, K, SR, n_cmp,
                                                                                                         int(near.sum())))
    assert n_cmp > 200


def _ref_frustum_lib():
    path = os.path.join(REF_DIR, "libref_frustum.so")
    if not os.path.isfile(path):
        pytest.skip("oracle/_ref/libref_frustum.so was not built (build() makes it where the reference tree exists)")
    return C.CDLL(path)


@pytest.mark.parametrize("family,sizes,K,SR", [("ties1", ((3, 3, 3), (3, 3, 3)), 8, 32), ("ties1", ((5, 5, 3), (5, 5, 5)), 3, 33),
                                               ("ties1", ((3, 3, 1), (4, 4, 2)), 1, 31), ("duplicates", ((3, 3, 3), (3, 3, 3)), 8, 24)])
def test_reference_frustum_kernels_on_tie_scenes(family, sizes, K, SR):
    """The reference's frustum kernels against the oracle: one point per voxel, so the K-slot order must match bit for bit;
    duplicates: the multiset of neighbour coordinates."""
    from oracle import record_ref_frustum
    lib = _ref_frustum_lib()
    ks, qs = sizes
    opt = hc.frustum_opt(vscale=(3, 3, 1), ks=ks, qs=qs, SR=SR, K=K, P=64)   # vscale 3: a pixel's sample sits mid-voxel, neighbours tie
    sc = hc.frustum_scene(family, opt)
    hyper = hc.frustum_grid(sc["cam"], opt)
    ref = record_ref_frustum.reference_query(lib, None, dict(pers=sc["pers"], pixel_idx=sc["pixel_idx"][:-3]), opt, hyper, DEV)
    assert ref["max_fill"] <= opt.P
    o = frustum_oracle_run(sc, opt, sc["pixel_idx"][:-3])
    assert np.array_equal(ref["ray_mask"], o["ray_mask"])
    assert np.array_equal(ref["pixel_idx_cur"], o["pixel_idx_cur"])
    assert np.array_equal(ref["sample_loc"], o["sample_loc"])
    a, b = o["sample_pidx"], ref["sample_pidx"]
    if family == "ties1":
        assert np.array_equal(a, b), "%d samples differ in their K-slot order" % int((a != b).any(-1).sum())
    else:
        assert np.array_equal(_coords(a, sc["pers"]), _coords(b, sc["pers"]))
    print("[reference frustum %s ks %s qs %s K %d SR %d] rays kept %d, filled slots %d" % (family, ks, qs, K, SR, int(o["ray_mask"].sum()),
                                                                                        int((a >= 0).sum())))
    assert (a >= 0).sum() > 200
