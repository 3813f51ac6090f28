"""libpnb200's perspective-frustum query (pnb_frustum_*, through the drop-in pointnerf_b200.query_point_indices) against the serial C
oracle and against the reference kernels' recorded run, on the DTU-like scenes of pointnerf_b200.scene.FRUSTUM_CONFIGS."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import frustum_oracle, shade_oracle, shade_oracle_frustum
from pointnerf_b200 import lib as _lib
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200 import scene

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CASES = list(scene.FRUSTUM_CONFIGS)
CHUNK = 2304   # the reference's chunk of 48 x 48 rays (random_sample_size 48)


def inputs(name, **over):
    """Config, numpy scene (plus its device tensors, created once like the model's parameters), querier options."""
    cfg = scene.FRUSTUM_CONFIGS[name]
    s = scene.make_frustum_scene(cfg)
    s["dev"] = {k: torch.from_numpy(s[k]).to(DEV)[None] for k in ("xyz_w", "pers", "camrotc2w", "campos")}
    opt = scene.frustum_opt(cfg, **over)
    return cfg, s, opt


def call(q, cfg, s, pixels, xyz_w=None, camrot=None, campos=None):
    d = s["dev"]
    xyz_w = d["xyz_w"] if xyz_w is None else xyz_w
    pers = d["pers"]
    camrot = d["camrotc2w"] if camrot is None else camrot
    campos = d["campos"] if campos is None else campos
    pix = torch.as_tensor(pixels, device=DEV).reshape(1, -1, 2)
    npts = torch.tensor([pers.shape[1]], dtype=torch.int32, device=DEV)
    return q.query_points(pix, pers, xyz_w, npts, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"], np.float32(cfg.near),
                          np.float32(cfg.far), None, campos, camrot)


def oracle(cfg, s, opt, pixels):
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    return frustum_oracle.query(s["pers"], ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P,
                                pixels, np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)


@pytest.mark.parametrize("name", CASES)
def test_full_frame_matches_oracle(name):
    cfg, s, opt = inputs(name)
    q = qpi.lighting_fast_querier(DEV, opt)
    pidx, loc, loc_w, dirs, mask, vsize, ranges = call(q, cfg, s, s["pixel_idx"])
    ref = oracle(cfg, s, opt, s["pixel_idx"])
    assert np.array_equal(mask[0].cpu().numpy(), ref["ray_mask"])
    assert np.array_equal(q.last_pixel_idx_cur[0].cpu().numpy(), ref["pixel_idx_cur"])
    assert np.array_equal(loc[0].cpu().numpy(), ref["sample_loc"])          # bit-exact, empty slots included
    assert np.array_equal(pidx[0].cpu().numpy(), ref["sample_pidx"])        # same canonical order: same slots
    c = q.last_build_counters
    assert c["overflow_p"] == 0 and c["overflow_o"] == 0 and q.last_query_counters["n_bad_pixel"] == 0
    assert pidx.shape[1] > 1000 and (pidx >= 0).any()
    assert loc_w.shape == loc.shape and dirs.shape == loc.shape and vsize.dtype == np.float32


@pytest.mark.parametrize("name", CASES)
def test_matches_recorded_reference(name):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "ref_frustum_%s.npz" % name))
    cfg, s, opt = inputs(name)
    q = qpi.lighting_fast_querier(DEV, opt)
    pidx, loc, _, _, mask, _, _ = call(q, cfg, s, s["pixel_idx"])
    R = int(g["R"])
    assert np.array_equal(mask[0].cpu().numpy() > 0, np.unpackbits(g["mask_bits"])[:R] > 0)
    assert np.array_equal(q.last_pixel_idx_cur[0].cpu().numpy(), g["pixel_idx_cur"])
    rows = g["rows"]
    assert np.array_equal(loc[0].cpu().numpy()[rows], g["sample_loc"])
    ours, ref = pidx[0].cpu().numpy()[rows], g["sample_pidx"]
    diff = sum(set(ours[r, j][ours[r, j] >= 0].tolist()) != set(ref[r, j][ref[r, j] >= 0].tolist())
               for r in range(len(rows)) for j in range(opt.SR))
    assert diff <= 5


def test_chunk_loop_reuses_build_and_equals_single_call():
    cfg, s, opt = inputs("dtu_surface")
    q = qpi.lighting_fast_querier(DEV, opt)
    full = call(q, cfg, s, s["pixel_idx"])
    assert q.n_builds == 1
    parts = [call(q, cfg, s, s["pixel_idx"][k:k + CHUNK]) for k in range(0, len(s["pixel_idx"]), CHUNK)]
    assert q.n_builds == 1                                              # one build for the whole view
    assert torch.equal(torch.cat([p[4] for p in parts], 1), full[4])
    assert torch.equal(torch.cat([p[0] for p in parts], 1), full[0])
    assert torch.equal(torch.cat([p[1] for p in parts], 1), full[1])
    # a new camera (same values in a new tensor: no rebuild; other values: rebuild), then a point change
    call(q, cfg, s, s["pixel_idx"][:CHUNK], camrot=torch.from_numpy(s["camrotc2w"].copy()).to(DEV)[None])
    assert q.n_builds == 1
    call(q, cfg, s, s["pixel_idx"][:CHUNK], campos=torch.from_numpy(s["campos"] + 0.01).to(DEV)[None])
    assert q.n_builds == 2
    xyz_w = torch.from_numpy(s["xyz_w"]).to(DEV)[None]
    call(q, cfg, s, s["pixel_idx"][:CHUNK], xyz_w=xyz_w)
    n = q.n_builds
    with torch.no_grad():
        xyz_w[0, 0, 0] += 0.001                                         # in-place edit: new version of the same storage
    call(q, cfg, s, s["pixel_idx"][:CHUNK], xyz_w=xyz_w)
    assert q.n_builds == n + 1


def test_overflow_reported():
    cfg, s, opt = inputs("dtu_surface", P=1)
    q = qpi.lighting_fast_querier(DEV, opt)
    pidx = call(q, cfg, s, s["pixel_idx"])[0]
    ref = oracle(cfg, s, opt, s["pixel_idx"])
    assert q.last_build_counters["overflow_p"] > 0 and q.last_build_counters["max_pts"] > 1
    assert np.array_equal(pidx[0].cpu().numpy(), ref["sample_pidx"])     # first P by index, as the oracle
    cfg, s, opt = inputs("dtu_surface", max_o=1)
    q = qpi.lighting_fast_querier(DEV, opt)
    call(q, cfg, s, s["pixel_idx"][:CHUNK])
    assert q.last_build_counters["overflow_o"] == 1


def test_pixels_outside_the_grid_are_counted_misses():
    cfg, s, opt = inputs("dtu_surface")
    q = qpi.lighting_fast_querier(DEV, opt)
    pix = np.array([[-1, 5], [cfg.W, 5], [5, cfg.H + 1], [cfg.W // 2, cfg.H // 2]], np.int32)
    mask = call(q, cfg, s, pix)[4]
    assert mask[0, :3].tolist() == [0, 0, 0]
    assert q.last_query_counters["n_bad_pixel"] == 3


def test_abi_refuses_unsupported():
    cfg, s, opt = inputs("dtu_surface")
    lib = _lib.load()
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    pts = torch.from_numpy(s["pers"]).to(DEV)
    dim = _lib.i3(sdim)
    nbytes = lib.pnb_frustum_bytes(pts.shape[0], dim, opt.SR)
    buf = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    base = dict(B=1, K=8, SR=opt.SR, NN=2, inverse=0, ks=(3, 3, 3), qs=(3, 3, 3))
    for over in (dict(NN=1), dict(inverse=1), dict(K=9), dict(B=2), dict(SR=129), dict(ks=(5, 5, 5))):
        a = dict(base, **over)
        fr = _lib.Frustum()
        rc = lib.pnb_frustum_build(C.byref(fr), buf.data_ptr(), nbytes, pts.data_ptr(), pts.shape[0], a["B"], _lib.f3(ranges[:3]),
                                   _lib.f3(svs), dim, _lib.i3(vscale), _lib.i3(a["ks"]), _lib.i3(a["qs"]), a["SR"], a["K"], opt.P, 0,
                                   a["NN"], a["inverse"], None, None)
        assert rc == -4, over   # PNB_ERR_UNSUPPORTED


def test_sr_cap_matches_oracle():
    """SR 4: most columns hold more dilated voxels than SR, so only the first SR are listed (F5) and the rest of a slot list is -1."""
    cfg, s, opt = inputs("dtu_surface", SR=4)
    q = qpi.lighting_fast_querier(DEV, opt)
    pidx, loc, _, _, mask, _, _ = call(q, cfg, s, s["pixel_idx"])
    ref = oracle(cfg, s, opt, s["pixel_idx"])
    assert q.last_build_counters["n_col_capped"] > 0 and ref["counters"]["n_col_capped"] > 0
    assert q.last_build_counters["max_col_samples"] > opt.SR
    assert np.array_equal(mask[0].cpu().numpy(), ref["ray_mask"])
    assert np.array_equal(loc[0].cpu().numpy(), ref["sample_loc"])
    assert np.array_equal(pidx[0].cpu().numpy(), ref["sample_pidx"])


def test_tuple_shaded_by_reference_eager_path_matches_oracle():
    """The drop-in's 7-tuple, fed to the reference's eager gather + PointAggregator + ray march (oracle/shade_oracle_frustum.py, fp32),
    gives the radiance of the oracle path (C oracle query, the reference's pers2w, the same shading in float64) within 1e-4."""
    from pointnerf_b200 import harness
    from pointnerf_b200.ray_marching import PointAggregator
    cfg, s, opt = inputs("dtu_surface")
    pts = scene.make_frustum_points(cfg, s)
    agg = PointAggregator(harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63), seed=5)
    with torch.no_grad():
        agg.alpha_branch[0].bias += 300.0                               # depth voxels are 0.0068 long: density ~300 makes the surface opaque
    mlp = {k: v.detach() for k, v in agg.state_dict().items()}
    xyz_w = pts["xyz"].to(DEV)[None]
    rot, pos = s["dev"]["camrotc2w"], s["dev"]["campos"]
    pers = shade_oracle.w2pers(xyz_w, rot, pos).contiguous()            # NeuralPoints.w2pers (neural_points.py:604-610), on the device
    q = qpi.lighting_fast_querier(DEV, opt)
    sel = s["pixel_idx"][::16]                                          # 1,200 rays: the float64 shading stays within a few GB
    pix = torch.from_numpy(sel).to(DEV)[None]
    npts = torch.tensor([cfg.N], dtype=torch.int32, device=DEV)
    out = q.query_points(pix, pers, xyz_w, npts, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"], np.float32(cfg.near),
                         np.float32(cfg.far), None, pos, rot)
    pidx, loc, loc_w, dirs, mask, vsize, ranges = out
    # the return types of query_point_indices.py:100
    assert pidx.dtype == torch.int32 and mask.dtype == torch.int8 and mask.shape == (1, len(sel))
    assert loc.dtype == loc_w.dtype == dirs.dtype == torch.float32 and pidx.shape[:3] == loc.shape[:3] == loc_w.shape[:3]
    assert isinstance(vsize, np.ndarray) and vsize.dtype == np.float32 and vsize.shape == (3,)
    assert isinstance(ranges, np.ndarray) and ranges.dtype == np.float32 and ranges.shape == (6,)
    ours = shade_oracle_frustum.shade(pts, mlp, pidx[0].cpu(), loc[0].cpu(), loc_w[0].cpu(), dirs[0].cpu(), pos.cpu(), rot.cpu(), vsize,
                                      torch.ones(3))

    pers_h = pers[0].cpu().numpy()
    rl, dl, rng, vs, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                   np.float32(cfg.near), np.float32(cfg.far))
    ref = frustum_oracle.query(pers_h, rng[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P, sel)
    assert np.array_equal(mask[0].cpu().numpy(), ref["ray_mask"])
    assert np.array_equal(pidx[0].cpu().numpy(), ref["sample_pidx"]) and np.array_equal(loc[0].cpu().numpy(), ref["sample_loc"])
    ref_loc = torch.from_numpy(ref["sample_loc"])
    ref_loc_w, ref_dirs = qpi.lighting_fast_querier.pers2w(None, ref_loc[None], rot.cpu(), pos.cpu())
    assert (loc_w[0].cpu() - ref_loc_w[0]).abs().max().item() <= 1e-5
    assert (dirs[0].cpu() - ref_dirs[0]).abs().max().item() <= 1e-6
    want = shade_oracle_frustum.shade(pts, mlp, torch.from_numpy(ref["sample_pidx"]), ref_loc, ref_loc_w[0], ref_dirs[0], pos.cpu(),
                                      rot.cpu(), vs, torch.ones(3), dtype=torch.float64)
    assert want["opacity"].max().item() > 0.5                           # an opaque surface: the comparison is not all background
    d = (ours["ray_color"].double() - want["ray_color"]).abs().max().item()
    assert d <= 1e-4, d
