"""CPU checks of the perspective-frustum query (wcoord_query 0, NN 2): the serial C oracle against an independent brute-force numpy
formulation and against the reference kernels' recorded run (tests/golden/ref_frustum_*.npz); the drop-in's interface against the
reference class; the fused module's refusal of wcoord_query 0."""
import ast
import inspect
import os

import numpy as np
import pytest

import torch

from oracle import frustum_oracle, ref_shim, shade_oracle, shade_oracle_frustum
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200 import scene

CASES = list(scene.FRUSTUM_CONFIGS)


def run_oracle(name, pixels=None, **over):
    cfg = scene.FRUSTUM_CONFIGS[name]
    s = scene.make_frustum_scene(cfg)
    opt = scene.frustum_opt(cfg, **over)
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    pix = s["pixel_idx"] if pixels is None else pixels
    out = frustum_oracle.query(s["pers"], ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P, pix,
                               np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)
    return cfg, s, opt, (ranges, svs, sdim, vscale, np.float32(rl ** 2), np.float32(dl ** 2)), out


def brute_force(s, opt, grid, pixel_idx):
    """Dilated occupancy as a set, candidates by explicit voxel membership, K nearest by float64 distance."""
    ranges, svs, sdim, vscale, r2, d2 = grid
    lo = ranges[:3]
    q = (s["pers"] - lo) / svs                                    # float32, as the kernels form it
    gx, gy, gz = (int(v) for v in sdim)
    fl = np.all((q >= 0) & (q < sdim), 1)
    tr = np.all((q > -1) & (q < sdim), 1)
    occ = {tuple(v) for v in np.floor(q[fl]).astype(int)}
    cols = {}
    for (x, y, z) in occ:
        for dx in range(-(opt.query_size[0] // 2), (opt.query_size[0] + 1) // 2):
            for dy in range(-(opt.query_size[1] // 2), (opt.query_size[1] + 1) // 2):
                for dz in range(-(opt.query_size[2] // 2), (opt.query_size[2] + 1) // 2):
                    X, Y, Z = x + dx, y + dy, z + dz
                    if 0 <= X < gx and 0 <= Y < gy and 0 <= Z < gz:
                        cols.setdefault((X, Y), set()).add(Z)
    vox = {}
    for i in np.nonzero(tr)[0]:
        vox.setdefault(tuple(q[i].astype(int)), []).append(i)    # astype(int) truncates toward zero
    rvs = (svs[:2].astype(np.float64) / vscale[:2]).astype(np.float32)
    mask, rows = [], []
    for px, py in pixel_idx:
        c = cols.get((px // vscale[0], py // vscale[1]), set())
        m = bool(c) and max(c) > 0
        mask.append(m)
        if not m:
            continue
        listed = sorted(c)[:opt.SR] + [-1] * max(0, opt.SR - len(c))
        fx, fy = px // vscale[0], py // vscale[1]
        ray = []
        for fz in listed:
            # the fp32 fma of fx*svs + lo is exact in float64 before its one rounding; so is the float64 product (px%vs + 0.5)*rvs
            cx = (np.float64(px % vscale[0]) + 0.5) * np.float64(rvs[0]) + np.float64(np.float32(np.float64(fx) * svs[0] + lo[0]))
            cy = (np.float64(py % vscale[1]) + 0.5) * np.float64(rvs[1]) + np.float64(np.float32(np.float64(fy) * svs[1] + lo[1]))
            cz = (fz + 0.5) * np.float64(svs[2]) + np.float64(lo[2])
            loc = np.array([cx, cy, cz], np.float32)
            cand = []
            if fz >= 0:
                for dx in (-1, 0, 1):
                    for dy in (-1, 0, 1):
                        for dz in (-1, 0, 1):
                            v = (fx + dx, fy + dy, fz + dz)
                            if v in occ:
                                cand += sorted(vox.get(v, []))[:opt.P]
            pts = s["pers"][cand].astype(np.float64)
            L = loc.astype(np.float64)
            xy2 = (pts[:, 0] * pts[:, 2] - L[0] * L[2]) ** 2 + (pts[:, 1] * pts[:, 2] - L[1] * L[2]) ** 2
            z2 = (pts[:, 2] - L[2]) ** 2
            ok = ((r2 == 0) | (xy2 <= r2)) & ((d2 == 0) | (z2 <= d2))
            cand, dist = np.asarray(cand, int)[ok], (xy2 + z2)[ok]
            order = np.argsort(dist, kind="stable")
            ray.append((loc, cand[order], dist[order]))
        rows.append(ray)
    return np.asarray(mask, np.int8), rows


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_brute_force(name):
    cfg = scene.FRUSTUM_CONFIGS[name]
    sel = scene.make_frustum_scene(cfg)["pixel_idx"][::7]          # 2,743 rays spread over the frame
    _, s, opt, grid, out = run_oracle(name, pixels=sel)
    mask, rows = brute_force(s, opt, grid, sel)
    assert np.array_equal(out["ray_mask"], mask)
    assert out["counters"]["overflow_p"] == 0 and out["counters"]["overflow_o"] == 0
    near_ties = 0
    for r, ray in enumerate(rows):
        for j, (loc, cand, dist) in enumerate(ray):
            np.testing.assert_array_equal(out["sample_loc"][r, j], loc)
            got = set(int(v) for v in out["sample_pidx"][r, j] if v >= 0)
            want = set(int(v) for v in cand[:opt.K])
            if got != want:
                # a set may only differ where the K-th and (K+1)-th float64 distances tie within fp32 rounding
                assert len(cand) > opt.K and abs(dist[opt.K] - dist[opt.K - 1]) <= 1e-6 * max(dist[opt.K], 1e-12), (r, j)
                near_ties += 1
    assert near_ties <= 5


def _golden(name):
    path = os.path.join(os.path.dirname(__file__), "golden", "ref_frustum_%s.npz" % name)
    return np.load(path)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_recorded_reference(name):
    g = _golden(name)
    assert int(g["max_fill"]) <= scene.FRUSTUM_CONFIGS[name].P and int(g["marked_per_col"]) <= 127   # no reservoir, no int8 wrap
    _, s, opt, grid, out = run_oracle(name)
    R = int(g["R"])
    assert np.array_equal(out["ray_mask"] > 0, np.unpackbits(g["mask_bits"])[:R] > 0)
    assert np.array_equal(out["pixel_idx_cur"], g["pixel_idx_cur"])
    rows = g["rows"]
    np.testing.assert_array_equal(out["sample_loc"][rows], g["sample_loc"])
    ours, ref = out["sample_pidx"][rows], g["sample_pidx"]
    diff = [(r, j) for r in range(len(rows)) for j in range(opt.SR)
            if set(ours[r, j][ours[r, j] >= 0].tolist()) != set(ref[r, j][ref[r, j] >= 0].tolist())]
    # with no overflow the canonical order changes nothing but the order in which equal distances meet the farthest-first rule
    assert len(diff) <= 5, diff[:10]


def test_overflow_flagged_not_hidden():
    _, _, _, _, out = run_oracle("dtu_surface", P=1)
    assert out["counters"]["overflow_p"] == 1
    _, _, _, _, out = run_oracle("dtu_surface", max_o=1)
    assert out["counters"]["overflow_o"] == 1


def _ref_methods():
    path = os.path.join(ref_shim.REF, "models", "neural_points", "query_point_indices.py")
    tree = ast.parse(open(path).read())
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "lighting_fast_querier")
    return {f.name: [a.arg for a in f.args.args] for f in cls.body if isinstance(f, ast.FunctionDef)}


@pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")
def test_drop_in_interface_matches_reference():
    ref = _ref_methods()
    for name in ("__init__", "get_hyperparameters", "query_points", "pers2w", "uniform", "gaussian", "clean_up"):
        ours = list(inspect.signature(getattr(qpi.lighting_fast_querier, name)).parameters)
        assert ours == ref[name], name
    assert len(ref["query_points"]) == 13   # self + 12


def test_hyperparameters_match_reference_expressions():
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface_limits"]
    s = scene.make_frustum_scene(cfg)
    opt = scene.frustum_opt(cfg)
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    assert ranges.dtype == np.float32 and vsize.dtype == np.float32 and sdim.dtype == np.int32
    assert list(sdim) == [cfg.W // 2, cfg.H // 2, cfg.z_depth_dim]
    assert rl == np.float32(cfg.radius_limit_scale * max(vsize[0], vsize[1])) and dl == np.float32(cfg.depth_limit_scale * vsize[2])


@pytest.mark.parametrize("wq,refused", [(0, True), (-1, False), (1, False)])
def test_check_opt_refuses_frustum_query(wq, refused):
    from pointnerf_b200 import harness
    from pointnerf_b200.ray_marching import check_opt
    opt = harness.make_opt(scene.CONFIGS["tiny"], wcoord_query=wq)
    if refused:
        with pytest.raises(NotImplementedError, match="wcoord_query=0"):
            check_opt(opt)
    else:
        check_opt(opt)


def test_drop_in_refuses_unsupported_options():
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    for over in (dict(NN=1), dict(inverse=1), dict(K=9), dict(SR=129)):
        with pytest.raises(NotImplementedError):
            qpi.lighting_fast_querier("cuda:0", scene.frustum_opt(cfg, **over))


def test_frustum_shading_restatement_matches_shade_oracle():
    """Given the world query's per-sample inputs (sample_loc = w2pers(sample_loc_w), one direction per ray), the frustum shading
    restatement computes exactly what oracle/shade_oracle.py computes."""
    from pointnerf_b200 import harness
    from pointnerf_b200.ray_marching import PointAggregator
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    _, s, opt, grid, out = run_oracle("dtu_surface", pixels=scene.make_frustum_scene(cfg)["pixel_idx"][::40])
    pts = scene.make_frustum_points(cfg, s)
    mlp = {k: v.detach() for k, v in PointAggregator(harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63), seed=3).state_dict().items()}
    rot, pos = torch.from_numpy(s["camrotc2w"]), torch.from_numpy(s["campos"])
    loc_w, dirs = qpi.lighting_fast_querier.pers2w(None, torch.from_numpy(out["sample_loc"])[None], rot[None], pos[None])
    loc_w, ray_dir = loc_w[0], dirs[0, :, 0]
    pidx = torch.from_numpy(out["sample_pidx"])
    vsize = (0.005, 0.005, 0.0068125)
    a = shade_oracle.shade(pts, mlp, pidx, loc_w, ray_dir, pos, rot, vsize, torch.ones(3))
    b = shade_oracle_frustum.shade(pts, mlp, pidx, shade_oracle.w2pers(loc_w, rot, pos), loc_w,
                                   ray_dir[:, None, :].expand(-1, opt.SR, -1), pos, rot, vsize, torch.ones(3))
    assert pidx.shape[0] > 100 and (a["opacity"] > 0).any()
    for k in ("ray_color", "opacity", "bg_T"):
        assert torch.equal(a[k], b[k]), k
