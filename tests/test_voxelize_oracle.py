"""CPU: oracle/voxelize_oracle.py against the reference's own construct_vox_points{,_xyz,_ind,_closest} (models/mvs/mvs_utils.py:484-561),
executed as written with torch_scatter's scatter_mean / scatter_min replaced by stand-ins on torch.Tensor.scatter_reduce_.  Needs the
reference tree; skipped elsewhere.  `python tests/test_voxelize_oracle.py` rewrites tests/golden/vox_ref.npz from the same functions.

sparse_grid_idx and inv_idx must be equal.  The stand-in sums in fp32 and the oracle in fp64, so the centroids differ by the fp32
accumulation error: over c points of magnitude at most X, recursive summation in any order errs by at most (c - 1) u X per point
averaged, plus the roundings of the divide and of the oracle's result, so |d| <= (c + 2) u X with u = 2^-24.  For a voxel of edge v
that is (c + 2) u X / v of the voxel.  The closest point must be the reference's wherever the reference's two smallest residuals in the
voxel are further apart than twice that bound plus the residuals' own rounding; elsewhere it must be one of the near-tied points.
"""
import ast
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, voxelize_oracle as vo  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree (/root/reference): build container only")

NAMES = ("construct_vox_points", "construct_vox_points_xyz", "construct_vox_points_ind", "construct_vox_points_closest")
GOLDEN = os.path.join(ROOT, "tests", "golden", "vox_ref.npz")


def scatter_mean(src, index, dim=0):
    m = int(index.max()) + 1 if index.numel() else 0
    out = torch.zeros((m,) + tuple(src.shape[1:]), dtype=src.dtype)
    return out.scatter_reduce_(0, index[:, None].expand_as(src), src, reduce="mean", include_self=False)


def scatter_min(src, index, dim=0):
    m = int(index.max()) + 1 if index.numel() else 0
    val = torch.zeros(m, dtype=src.dtype).scatter_reduce_(0, index, src, reduce="amin", include_self=False)
    pos = torch.arange(src.shape[0])
    hit = src == val[index]
    arg = torch.full((m,), src.shape[0], dtype=torch.int64).scatter_reduce_(0, index[hit], pos[hit], reduce="amin")
    return val, arg


def load_reference():
    """The four functions, compiled from the reference file's own source into a module whose scatter_* are the stand-ins."""
    path = os.path.join(ref_shim.REF, "models", "mvs", "mvs_utils.py")
    tree = ast.parse(open(path).read(), path)
    mod = types.ModuleType("mvs_utils_vox")
    mod.torch, mod.scatter_mean, mod.scatter_min, mod.print = torch, scatter_mean, scatter_min, lambda *a, **k: None
    body = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in NAMES]
    assert sorted(n.name for n in body) == sorted(NAMES)
    exec(compile(ast.Module(body=body, type_ignores=[]), path, "exec"), mod.__dict__)
    return mod


def space_of(xyz, vox_res, space_min=None, space_max=None):
    """The reference's space and voxel size (mvs_utils.py:487-495) on the CPU, as float32 [3]."""
    from pointnerf_b200.voxelize import _space
    smin, smax, vsz = _space(torch.as_tensor(xyz), vox_res, space_min, space_max)
    return smin.numpy(), smax.numpy(), vsz.expand(3).numpy() if vsz.dim() == 0 else vsz.numpy()


def clouds():
    g = np.random.default_rng(7)
    out = {"uniform": g.uniform(-1.3, 2.1, (20000, 3)).astype(np.float32)}
    uv = g.uniform(0, 1, (30000, 2))
    out["surface"] = np.stack([uv[:, 0] * 4 - 2, uv[:, 1] * 3 + 5, 0.4 * np.sin(5 * uv[:, 0]) * np.cos(3 * uv[:, 1]) + 1.5],
                              1).astype(np.float32)
    out["dup"] = np.repeat(g.uniform(0, 1, (500, 3)).astype(np.float32), 4, axis=0)
    return out


@pytest.fixture(scope="module")
def ref():
    return load_reference()


@pytest.mark.parametrize("name", ["uniform", "surface", "dup"])
@pytest.mark.parametrize("vox_res", [64, 320, 900.0, 2000, 800 // 1.5])
def test_oracle_matches_reference(ref, name, vox_res):
    xyz = clouds()[name]
    t = torch.from_numpy(xyz)
    smin, _, vsz = space_of(xyz, vox_res)
    o = vo.voxelize(xyz, smin, vsz, closest=True)
    cen_r, grid_r, min_r = ref.construct_vox_points(t, vox_res)
    grid_i, inv_i, _, _ = ref.construct_vox_points_ind(t, vox_res)
    cen_c, grid_c, arg_c = ref.construct_vox_points_closest(t, vox_res)
    cen_x = ref.construct_vox_points_xyz(t, vox_res)
    for g in (grid_r, grid_i, grid_c):
        assert g.dtype == torch.int32 and np.array_equal(g.numpy(), o["grid_idx"])
    assert inv_i.dtype == torch.int64 and np.array_equal(inv_i.numpy(), o["inv_idx"])
    assert np.array_equal(min_r.numpy(), o["first"])
    m = o["grid_idx"].shape[0]
    bound, xmax = vo.centroid_bound(xyz, o["inv_idx"], m)
    for c in (cen_r, cen_c, cen_x):
        assert c.dtype == torch.float32
        assert np.all(np.abs(c.numpy().astype(np.float64) - o["centroid"]).max(1) <= bound)
    ref_res = torch.norm(t - cen_c[inv_i], dim=-1).numpy()
    clear = vo.check_closest(arg_c.numpy(), o["closest"], ref_res, o["inv_idx"], bound, xmax)
    many = np.bincount(o["inv_idx"], minlength=m) >= 3    # two points are equidistant from their mean: a tie up to rounding
    if name != "dup":
        assert many.sum() < 100 or clear[many].mean() > 0.9    # most voxels are decided by the residuals alone
    else:
        assert not clear.all()                                  # duplicated points: ties exist, the oracle takes the lowest index
        inv = o["inv_idx"]
        tie = o["residual"] == o["residual"][o["closest"]][inv]
        lowest = np.full(m, len(inv))
        np.minimum.at(lowest, inv[tie], np.flatnonzero(tie))
        assert np.array_equal(lowest, o["closest"])


def test_caller_space_gives_negative_indices(ref):
    """construct_vox_points_ind with the space of another cloud (train_ft.py:658-659): indices below 0 and past vox_res."""
    g = np.random.default_rng(3)
    pc = torch.from_numpy(g.uniform(0, 1, (5000, 3)).astype(np.float32))
    depth = torch.from_numpy(g.uniform(-0.6, 1.7, (8000, 3)).astype(np.float32))
    _, _, smin, smax = ref.construct_vox_points_ind(pc, 128)
    grid, inv, _, _ = ref.construct_vox_points_ind(depth, 128, space_min=smin, space_max=smax)
    _, _, vsz = space_of(depth.numpy(), 128, smin, smax)
    o = vo.voxelize(depth.numpy(), smin.numpy(), vsz)
    assert (o["grid_idx"] < 0).any() and (o["grid_idx"] >= 128).any()
    assert np.array_equal(grid.numpy(), o["grid_idx"]) and np.array_equal(inv.numpy(), o["inv_idx"])


def test_centroid_tree_is_the_documented_one():
    """The vectorised tree against a direct serial restatement, for voxels below, at and above 256 points."""
    g = np.random.default_rng(5)
    for c in (1, 2, 3, 31, 33, 200, 256, 257, 1000, 3001):
        x = (g.standard_normal((c, 3)) * 10).astype(np.float32)
        lanes = [x[t::256].astype(np.float64) for t in range(min(c, 256))]
        p = []
        for col in lanes:
            s = col[0].copy()
            for r in col[1:]:
                s = s + r
            p.append(s)
        w, off = len(p), 128
        while off >= 1:
            for t in range(off):
                if t + off < w:
                    p[t] = p[t] + p[t + off]
            off //= 2
        want = (p[0] / c).astype(np.float32)
        got = vo.centroid_tree(x, np.zeros(c, np.int64), np.zeros(1, np.int64), np.array([c]))[0]
        assert np.array_equal(got, want), c


def test_voxel_index_follows_cuda_conversion():
    assert vo.voxel_index(np.zeros((1, 3), np.float32), np.zeros(3, np.float32), np.zeros(3, np.float32)).tolist() == [[0, 0, 0]]
    big = vo.voxel_index(np.full((1, 3), 3e9, np.float32), np.zeros(3, np.float32), np.ones(3, np.float32))
    assert big.tolist() == [[2147483647] * 3]


def golden_cases(ref):
    """Inputs and reference outputs of the fixture (vox_res powers of two: the space is the same bits on the CPU and the GPU)."""
    g = np.random.default_rng(11)
    uv = g.uniform(0, 1, (6000, 2))
    xyz = np.stack([uv[:, 0] * 2 - 1, uv[:, 1] * 2, 0.3 * np.sin(4 * uv[:, 0]) + 0.5], 1).astype(np.float32)
    xyz = np.concatenate([xyz, xyz[:200]])                # duplicates: tied residuals
    t = torch.from_numpy(xyz)
    out = dict(xyz=xyz)
    for res in (64, 256):
        cen, grid, first = ref.construct_vox_points(t, float(res))
        _, inv, smin, smax = ref.construct_vox_points_ind(t, res)
        cen_c, _, closest = ref.construct_vox_points_closest(t, res)
        out.update({"r%d_centroid" % res: cen.numpy(), "r%d_grid_idx" % res: grid.numpy(), "r%d_first" % res: first.numpy(),
                    "r%d_inv_idx" % res: inv.numpy(), "r%d_closest" % res: closest.numpy(),
                    "r%d_xyz_centroid" % res: ref.construct_vox_points_xyz(t, res).numpy(),
                    "r%d_residual" % res: torch.norm(t - cen_c[inv], dim=-1).numpy(),
                    "r%d_space_min" % res: smin.numpy(), "r%d_space_max" % res: smax.numpy()})
    return out


def test_golden_fixture_is_what_the_reference_returns(ref):
    got = golden_cases(ref)
    want = np.load(GOLDEN)
    assert sorted(want.files) == sorted(got)
    for k in got:
        assert np.array_equal(want[k], got[k]), k


if __name__ == "__main__":
    np.savez_compressed(GOLDEN, **golden_cases(load_reference()))
    print("wrote", GOLDEN)
