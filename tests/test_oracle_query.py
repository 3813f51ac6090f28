"""CPU: pins oracle/query_oracle.c (serial C restatement of query_worldcoords.cu) against an independent
brute-force numpy formulation of the canonical semantics (SURVEY.md 8a) and against the committed fixtures
that were produced through the reference's own lighting_fast_querier class (oracle/make_golden.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import pipeline, query_oracle
from pointnerf_b200 import scene
from oracle import golden  # noqa: E402


def brute_force(xyz, lo, svs, dim, ks, qs, P, r, campos, raydir, t, SR, K):
    """Independent formulation: dict-of-lists voxel map, numpy distance sort (stable), shell by shell."""
    f32 = np.float32
    vox = np.floor(((xyz - lo.astype(f32)).astype(f32) / svs.astype(f32)).astype(f32)).astype(np.int64)
    inside = np.all((vox >= 0) & (vox < dim), axis=1)
    cells, first_cell = {}, None
    for i in np.nonzero(inside)[0]:
        key = tuple(vox[i])
        if first_cell is None:
            first_cell = key
        cells.setdefault(key, []).append(i)
    occ = set()
    for (x, y, z) in cells:
        for a in range(max(0, x - qs[0] // 2), min(dim[0], x + (qs[0] + 1) // 2)):
            for b in range(max(0, y - qs[1] // 2), min(dim[1], y + (qs[1] + 1) // 2)):
                for c in range(max(0, z - qs[2] // 2), min(dim[2], z + (qs[2] + 1) // 2)):
                    occ.add((a, b, c))
    stored = {k: v[:P] for k, v in cells.items() if k != first_cell}   # Q1: slot 0 holds nothing
    r2 = f32(r) * f32(r)
    res_mask = np.zeros(len(raydir), np.int8)
    res_pidx, res_loc = [], []
    for ri in range(len(raydir)):
        pos = (campos.astype(f32)[None] + (raydir[ri].astype(f32)[None] * t.astype(f32)[:, None]).astype(f32)).astype(f32)
        v = np.floor(((pos - lo.astype(f32)).astype(f32) / svs.astype(f32)).astype(f32)).astype(np.int64)
        hits = [d for d in range(len(t)) if np.all(v[d] >= 0) and np.all(v[d] < dim) and tuple(v[d]) in occ]
        if not hits:
            continue
        hits = hits[:SR]
        pidx = -np.ones((SR, K), np.int32)
        loc = np.zeros((SR, 3), f32)
        for s, d in enumerate(hits):
            loc[s] = pos[d]
            f = v[d]
            found = []  # (d2, traversal order, idx)
            order = 0
            for layer in range((ks[0] + 1) // 2):
                for x in range(max(-f[0], -layer), min(dim[0] - f[0], layer + 1)):
                    for y in range(max(-f[1], -layer), min(dim[1] - f[1], layer + 1)):
                        for z in range(max(-f[2], -layer), min(dim[2] - f[2], layer + 1)):
                            if max(abs(x), abs(y), abs(z)) != layer:
                                continue
                            for i in stored.get((f[0] + x, f[1] + y, f[2] + z), []):
                                dv = (xyz[i] - pos[d]).astype(f32)
                                yy = f32(dv[1] * dv[1])
                                d2 = f32(np.float64(dv[2]) * np.float64(dv[2]) + np.float64(
                                    f32(np.float64(dv[0]) * np.float64(dv[0]) + np.float64(yy))))
                                if r2 == 0 or d2 <= r2:
                                    found.append((d2, order, i))
                                    order += 1
                if len(found) >= K:
                    break
            # replace-farthest with strict '<' keeps the K smallest, earliest wins ties
            found.sort(key=lambda e: (e[0], e[1]))
            keep = found[:K]
            pidx[s, :len(keep)] = sorted(e[2] for e in keep)
        if np.any(pidx >= 0):
            res_mask[ri] = 1
            res_pidx.append(pidx)
            res_loc.append(loc)
    return res_mask, np.array(res_pidx), np.array(res_loc)


def _setup(cfg, pixels, SR=24, K=8, P=None):
    pts = scene.make_points(cfg)
    rays = scene.make_rays(cfg, pixels)
    rng6, svs, dim = pipeline.hyperparameters(pts["xyz"], [cfg.vsize] * 3, [cfg.vscale] * 3, [cfg.kernel_size] * 3,
                                              scene.ranges_for(cfg))
    t = pipeline.t_table(cfg.near, cfg.far, cfg.D)
    return pts, rays, rng6, svs, dim, t


@pytest.mark.parametrize("K,SR,P", [(8, 24, 32), (3, 5, 32), (8, 24, 2)])
def test_oracle_vs_bruteforce(K, SR, P):
    cfg = scene.CONFIGS["tiny"]
    pix = scene.centre_patch(cfg, 14)
    pts, rays, rng6, svs, dim, t = _setup(cfg, pix)
    ks = qs = np.array([3, 3, 3], np.int32)
    r = float(pipeline.radius_limit(4.0, [cfg.vsize] * 3))
    o = query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, qs, 100000, P, r, campos=np.array(cfg.campos),
                           raydir=rays["raydir"][0].numpy(), t=t, SR=SR, K=K)
    m, pidx, loc = brute_force(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, qs, P, r, np.array(cfg.campos, np.float32),
                               rays["raydir"][0].numpy(), t, SR, K)
    assert np.array_equal(m, o["ray_mask"])
    assert o["sample_pidx"].shape == pidx.shape
    assert np.array_equal(np.sort(o["sample_pidx"], axis=-1), np.sort(pidx, axis=-1))
    assert np.array_equal(o["sample_loc_w"], loc)
    if P == 2:
        assert o["counters"]["overflow_p"] == 1
    assert o["counters"]["R2"] == int(m.sum()) > 0


def test_oracle_raypos_path_equals_t_path():
    """The pybind-signature entry (raypos given, query_worldcoords.cpp:36) and the campos+raydir*t entry agree bit
    for bit when raypos is formed with the reference's torch ops (diff_ray_marching.py:386)."""
    cfg = scene.CONFIGS["tiny"]
    pix = scene.centre_patch(cfg, 20)
    pts, rays, rng6, svs, dim, t = _setup(cfg, pix)
    raydir = rays["raydir"]
    raypos = rays["campos"][:, None, None, :] + raydir[:, :, None, :] * torch.from_numpy(t)[None, None, :, None]
    ks = np.array([3, 3, 3], np.int32)
    r = float(pipeline.radius_limit(4.0, [cfg.vsize] * 3))
    a = query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, ks, 100000, 32, r, campos=np.array(cfg.campos),
                           raydir=raydir[0].numpy(), t=t)
    b = query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, ks, 100000, 32, r, raypos=raypos[0].numpy())
    for k in ("sample_pidx", "sample_loc_w", "ray_mask"):
        assert np.array_equal(a[k], b[k])


def test_oracle_edge_cases():
    cfg = scene.CONFIGS["tiny"]
    pts, rays, rng6, svs, dim, t = _setup(cfg, scene.centre_patch(cfg, 8))
    ks = np.array([3, 3, 3], np.int32)
    r = float(pipeline.radius_limit(4.0, [cfg.vsize] * 3))
    # rays that look away: nothing hit, empty outputs
    away = -rays["raydir"][0].numpy()
    o = query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, ks, 100000, 32, r, campos=np.array(cfg.campos),
                           raydir=away, t=t)
    assert o["counters"]["R2"] == 0 and o["sample_pidx"].shape[0] == 0 and not o["ray_mask"].any()
    # max_o overflow is flagged
    o = query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, ks, 10, 32, r, campos=np.array(cfg.campos),
                           raydir=rays["raydir"][0].numpy(), t=t)
    assert o["counters"]["overflow_o"] == 1
    # slot-0 quirk (query_worldcoords.cu:147): the lowest-index point is never returned as a neighbour
    o = query_oracle.query(pts["xyz"].numpy(), rng6[:3], svs, dim, ks, ks, 100000, 32, r, campos=np.array(cfg.campos),
                           raydir=scene.make_rays(cfg)["raydir"][0].numpy(), t=t)
    assert not (o["sample_pidx"] == 0).any()
    assert o["counters"]["slot0_cell"] >= 0


@pytest.mark.parametrize("name", ["tiny_opaque", "tiny_thin_sr8"])
def test_oracle_matches_reference_fixture(name, golden_dir):
    """oracle/pipeline.py (restated host logic + C query) == what the reference's own lighting_fast_querier class
    returned when the fixture was generated (oracle/make_golden.py)."""
    fx = golden.load(golden_dir, name)
    cfg = scene.CONFIGS["tiny"]
    pts = scene.make_points(cfg)
    rays = scene.make_rays(cfg, fx["pixels"])
    out = pipeline.render(pts, None, rays["raydir"][0], cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far,
                          [cfg.vsize] * 3, [2, 2, 2], [3, 3, 3], [3, 3, 3], scene.ranges_for(cfg), int(fx["SR"]), 8, cfg.P,
                          100000, want_shade=False)
    assert np.array_equal(out["ranges6"], fx["ranges6"])
    assert np.array_equal(out["scaled_vdim"], fx["scaled_vdim"])
    assert np.array_equal(out["ray_mask"], fx["ray_mask"])
    assert np.array_equal(out["sample_pidx"], fx["sample_pidx"])
    assert np.array_equal(out["sample_loc_w"], fx["sample_loc_w"])
