"""GPU: pointnerf_b200.voxelize (csrc/voxelize.cu) bit for bit against oracle/voxelize_oracle.py on every output, and against the
reference's own results recorded in tests/golden/vox_ref.npz (tests/test_voxelize_oracle.py writes and re-checks that fixture)."""
import os

import numpy as np
import pytest
import torch

from oracle import voxelize_oracle as vo
from pointnerf_b200 import voxelize as V

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vox_ref.npz")


def _np(t):
    return t.cpu().numpy()


def surface(n, seed=0):
    """A COLMAP-like cloud: a wavy ground sheet, a box's faces and sparse outliers."""
    g = np.random.default_rng(seed)
    n1, n2 = n // 2, n // 3
    uv = g.uniform(0, 1, (n1, 2))
    ground = np.stack([uv[:, 0] * 8 - 4, uv[:, 1] * 8 - 4, 0.2 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1])], 1)
    f = g.integers(0, 6, n2)
    w = g.uniform(-1, 1, (n2, 3))
    w[np.arange(n2), f // 2] = np.where(f % 2, 1.0, -1.0)
    box = w * np.array([1.0, 0.7, 0.5]) + np.array([0.5, -0.3, 0.6])
    box += g.normal(0, 2e-3, box.shape)
    out = g.uniform(-6, 6, (n - n1 - n2, 3))
    return np.concatenate([ground, box, out]).astype(np.float32)


def space_np(xyz, vox_res, space_min=None, space_max=None):
    smin, smax, vsz = V._space(xyz, vox_res, space_min, space_max)
    return _np(smin), _np(vsz.reshape(-1).expand(3))


def check_all(xyz_np, vox_res, space_min=None, space_max=None):
    """Every output of the four functions against the oracle, bit for bit.  Returns the oracle's result."""
    xyz = torch.from_numpy(xyz_np).to(DEV)
    smin, vsz = space_np(xyz, vox_res, space_min, space_max)
    o = vo.voxelize(xyz_np, smin, vsz, closest=True)
    kw = dict(space_min=space_min, space_max=space_max)
    cen, grid, first = V.construct_vox_points(xyz, vox_res, **kw)
    cen_x = V.construct_vox_points_xyz(xyz, vox_res, **kw)
    grid_i, inv, smin_r, smax_r = V.construct_vox_points_ind(xyz, vox_res, **kw)
    assert cen.dtype == torch.float32 and grid.dtype == torch.int32 and first.dtype == torch.int64 and inv.dtype == torch.int64
    for g in (grid, grid_i):
        assert np.array_equal(_np(g), o["grid_idx"])
    assert np.array_equal(_np(inv), o["inv_idx"])
    assert np.array_equal(_np(first), o["first"])
    for c in (cen, cen_x):
        assert np.array_equal(_np(c).view(np.uint32), o["centroid"].view(np.uint32))
    assert np.array_equal(_np(smin_r), smin)
    inside = space_min is None or bool(((xyz - space_min) * (space_max - xyz)).prod(-1).gt(0).all())
    if inside:
        cen_c, grid_c, closest = V.construct_vox_points_closest(xyz, vox_res, **kw)
        assert np.array_equal(_np(grid_c), o["grid_idx"])
        assert np.array_equal(_np(cen_c).view(np.uint32), o["centroid"].view(np.uint32))
        assert closest.dtype == torch.int64 and np.array_equal(_np(closest), o["closest"])
    return o


@pytest.mark.parametrize("vox_res", [320, 533.0, 900, 2000])
def test_random_cloud(vox_res):
    g = np.random.default_rng(1)
    check_all(g.uniform(-2.0, 3.0, (300000, 3)).astype(np.float32), vox_res)


@pytest.mark.parametrize("vox_res", [320, 800])
def test_colmap_like_surface(vox_res):
    check_all(surface(1_000_000), vox_res)


def test_points_on_voxel_faces_and_ulps_either_side():
    """Caller space [0, 1]^3 at vox_res 128 (voxel 1/128, exact): points on faces and 1-3 ulps below and above."""
    g = np.random.default_rng(2)
    faces = g.integers(1, 127, (4000, 3)).astype(np.float32) / np.float32(128)
    pts = [faces]
    for k in (1, 2, 3):
        up, dn = faces.copy(), faces.copy()
        for _ in range(k):
            up, dn = np.nextafter(up, np.float32(2)), np.nextafter(dn, np.float32(-1))
        pts += [up, dn]
    mixed = faces.copy()
    ax = g.integers(0, 3, faces.shape[0])
    mixed[np.arange(faces.shape[0]), ax] = g.uniform(0.01, 0.99, faces.shape[0]).astype(np.float32)
    xyz = np.concatenate(pts + [mixed]).astype(np.float32)
    smin = torch.zeros(3, device=DEV)
    smax = torch.ones(3, device=DEV)
    o = check_all(xyz, 128, smin, smax)
    below = vo.voxel_index(pts[2], np.zeros(3, np.float32), np.full(3, 1 / 128, np.float32))
    assert np.array_equal(below, vo.voxel_index(faces, np.zeros(3, np.float32), np.full(3, 1 / 128, np.float32)) - 1)
    assert o["grid_idx"].shape[0] > 10000


def test_one_voxel_holds_a_large_segment():
    g = np.random.default_rng(4)
    spread = g.uniform(0, 1, (20000, 3)).astype(np.float32)
    cluster = (np.float32(0.5) + g.uniform(0, 1e-3, (150000, 3))).astype(np.float32)
    xyz = np.concatenate([spread[:10000], cluster, spread[10000:]])
    o = check_all(xyz, 320)
    big = np.bincount(o["inv_idx"]).max()
    assert big >= 150000 // 8                             # the cluster may straddle a voxel face on each axis
    t = torch.from_numpy(xyz).to(DEV)
    r = V.voxelize(t, *[torch.from_numpy(a).to(DEV) for a in space_np(t, 320)], centroid=True)
    assert r["counters"]["n_big"] >= 1 and r["counters"]["max_pts"] == big


def test_a_cloud_of_one_voxel_only():
    """Every point in one voxel of the caller's space: a single segment of 200k points."""
    g = np.random.default_rng(9)
    xyz = (np.float32(0.25) + g.uniform(0, 0.1, (200000, 3))).astype(np.float32)
    o = check_all(xyz, 4, torch.zeros(3, device=DEV), torch.ones(3, device=DEV))
    assert o["grid_idx"].shape[0] == 1


def test_single_point():
    """N = 1: the extent is 0 and the voxel size 0, so (p - space_min) / 0 is NaN, which converts to voxel 0 (as on the reference)."""
    o = check_all(np.array([[0.3, -1.2, 7.5]], np.float32), 320)
    assert o["grid_idx"].tolist() == [[0, 0, 0]]


def test_empty_cloud():
    xyz = torch.zeros((0, 3), device=DEV)
    smin, smax = torch.zeros(3, device=DEV), torch.ones(3, device=DEV)
    grid, inv, _, _ = V.construct_vox_points_ind(xyz, 64, space_min=smin, space_max=smax)
    cen, grid_c, idx = V.construct_vox_points_closest(xyz, 64, space_min=smin, space_max=smax)
    assert grid.shape == (0, 3) and inv.shape == (0,) and cen.shape == (0, 3) and idx.shape == (0,)
    with pytest.raises(ValueError, match="no extent"):
        V.construct_vox_points(xyz, 64)


def test_duplicate_points_tie_to_the_lowest_index():
    g = np.random.default_rng(5)
    base = g.uniform(0, 1, (20000, 3)).astype(np.float32)
    xyz = np.concatenate([base, base[::-1], base[:5000]])
    o = check_all(xyz, 320)
    # a voxel holding one distinct position (repeated): every residual is equal and the lowest index wins
    cnt_u = np.array([len(np.unique(xyz[o["inv_idx"] == s], axis=0)) for s in range(50)])
    for s in np.flatnonzero(cnt_u == 1):
        assert o["closest"][s] == o["first"][s]


def test_negative_indices_through_a_callers_space():
    """construct_vox_points_ind with another cloud's space (train_ft.py:658-659)."""
    g = np.random.default_rng(6)
    pc = torch.from_numpy(g.uniform(0, 1, (50000, 3)).astype(np.float32)).to(DEV)
    _, _, smin, smax = V.construct_vox_points_ind(pc, 400)
    depth = g.uniform(-0.7, 1.8, (200000, 3)).astype(np.float32)
    o = check_all(depth, 400, smin, smax)
    assert (o["grid_idx"] < 0).any() and (o["grid_idx"] >= 400).any()


def test_key_widths():
    """32-bit keys when the space is the cloud's own and vox_res < 1000, 64-bit otherwise; an index beyond the key fails."""
    xyz = torch.rand((1000, 3), device=DEV)
    assert V._prepare(xyz, 900, None, None, None)[4] == 32
    assert V._prepare(xyz, 2000, None, None, None)[4] == 64
    assert V._prepare(xyz, 64, None, torch.zeros(3, device=DEV), torch.ones(3, device=DEV))[4] == 64
    from pointnerf_b200 import lib
    far = torch.full((1, 3), 5e6, device=DEV)
    with pytest.raises(lib.PnbError, match="outside the 64-bit key"):
        V.construct_vox_points_ind(far, 1, space_min=torch.zeros(3, device=DEV), space_max=torch.ones(3, device=DEV))
    with pytest.raises(lib.PnbError, match="outside the 32-bit key"):
        V.voxelize(far, torch.zeros(3, device=DEV), torch.ones(3, device=DEV), key_bits=32)


def test_closest_with_a_callers_space_that_drops_points():
    xyz = torch.rand((1000, 3), device=DEV)
    xyz[0] = 2.0
    smin, smax = torch.zeros(3, device=DEV), torch.ones(3, device=DEV)
    with pytest.raises(ValueError, match="partition_xyz"):
        V.construct_vox_points_closest(xyz, 64, space_min=smin, space_max=smax)
    kept = xyz[1:]
    cen, grid, idx = V.construct_vox_points_closest(xyz, 64, partition_xyz=kept, space_min=smin, space_max=smax)
    o = vo.voxelize(_np(kept), np.zeros(3, np.float32), np.full(3, 1 / 64, np.float32), closest=True)
    assert np.array_equal(_np(grid), o["grid_idx"]) and np.array_equal(_np(idx), o["closest"])
    assert np.array_equal(_np(cen).view(np.uint32), o["centroid"].view(np.uint32))


def test_golden_reference_fixture():
    """The reference's own results (torch_scatter stand-ins, CPU): equal indices, centroids within the fp32-summation bound, the
    closest point equal wherever the reference's residuals decide it."""
    z = np.load(GOLDEN)
    xyz = torch.from_numpy(z["xyz"]).to(DEV)
    for res in (64, 256):
        k = "r%d_" % res
        cen, grid, first = V.construct_vox_points(xyz, float(res))
        grid_i, inv, smin, smax = V.construct_vox_points_ind(xyz, res)
        cen_c, _, closest = V.construct_vox_points_closest(xyz, res)
        cen_x = V.construct_vox_points_xyz(xyz, res)
        assert np.array_equal(_np(smin), z[k + "space_min"]) and np.array_equal(_np(smax), z[k + "space_max"])
        for g in (grid, grid_i):
            assert np.array_equal(_np(g), z[k + "grid_idx"])
        assert np.array_equal(_np(inv), z[k + "inv_idx"]) and np.array_equal(_np(first), z[k + "first"])
        m = z[k + "grid_idx"].shape[0]
        bound, xmax = vo.centroid_bound(z["xyz"], z[k + "inv_idx"], m)
        for c, want in ((cen, z[k + "centroid"]), (cen_c, z[k + "centroid"]), (cen_x, z[k + "xyz_centroid"])):
            assert np.all(np.abs(_np(c).astype(np.float64) - want).max(1) <= bound)
        vo.check_closest(z[k + "closest"], _np(closest), z[k + "residual"], z[k + "inv_idx"], bound, xmax)


def test_two_runs_give_identical_bits():
    xyz = torch.from_numpy(surface(2_000_000, seed=3)).to(DEV)
    a = V.construct_vox_points_closest(xyz, 800)
    b = V.construct_vox_points_closest(xyz, 800)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x, y.view(torch.int32) if y.dtype == torch.float32 else y)
    c = V.construct_vox_points_ind(xyz, 800)
    d = V.construct_vox_points_ind(xyz, 800)
    assert torch.equal(c[0], d[0]) and torch.equal(c[1], d[1])
