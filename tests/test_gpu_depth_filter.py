"""GPU: the depth filter and visual-hull drop-ins (pointnerf_b200.depth_filter: filter_by_masks_gpu, alpha_masking) through
pnb_depth_filter_build / _outputs and pnb_alpha_mask.

  oracle      every case of tests/golden/depth_filter_ref.npz equals oracle/depth_filter_oracle.py's fp32 restatement bit for bit
              (outputs, order, counts) and meets the reference's recorded outputs under compare_reference; a DTU-sized (V 49, 512 x 640)
              and an n360-sized (V 100, 800 x 800) seeded surface with at least 1000 pixel-pairs near each of dist 1 and rel 0.01:
              every DTU view and every tenth n360 view (and the last) equal the oracle bit for bit, counts and order included
  cpu2gpu     301 small views on the host equal the device-input call bit for bit and come back as host tensors; the n360 chain
              (host filter outputs into alpha_masking, chunked) gives a host mask equal to the device-input chain's
  hull        alpha_masking on 20M points x 100 views equals the oracle bit for bit on 1M sampled points, and every fixture case
  chain       filter, points_vid, alpha mask, voxelize.construct_vox_points_closest: the same bits as the chain fed the oracle's outputs
  refusals    manual_depth_view > 1, default_conf > 1, far_plane_shift, B != 1 and views of different sizes raise
Peak device memory is printed.
"""
import types

import numpy as np
import pytest
import torch

from oracle import depth_filter_oracle as do
from pointnerf_b200 import depth_filter, voxelize

import test_depth_filter_oracle as tdo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32 = np.float32


def _inputs(case, dev=DEV):
    cam, K, E, conf, mask = tdo.ref_inputs(case)
    return [t.to(dev) for t in cam], [t.to(dev) for t in K], [t.to(dev) for t in E], [t.to(dev) for t in conf], [t.to(dev) for t in mask]


def _run(case, cpu2gpu=False):
    args = _inputs(case, torch.device("cpu") if cpu2gpu else DEV)
    return depth_filter.filter_by_masks_gpu(*args, tdo._opt(case), cpu2gpu=cpu2gpu)


def _check_views(case, out, views):
    cam, world, conf = out
    mats = do.view_matrices(case["K"], case["E"])
    for r in views:
        o = do.filter_view(case, r, mats)
        assert np.array_equal(cam[r].cpu().numpy(), o["cam"]), "view %d: xyz_cam" % r
        assert np.array_equal(world[r].cpu().numpy(), o["world"]), "view %d: xyz_world" % r
        assert np.array_equal(conf[r].cpu().numpy(), o["conf"]), "view %d: confidence" % r


@pytest.mark.parametrize("name", list(tdo.CASES))
def test_fixture_cases_equal_the_fp32_oracle(name):
    case, ref = tdo.load_case(tdo._load_golden(), name)
    out = _run(case)
    _check_views(case, out, range(len(case["depth"])))
    print("\n[depth_filter gpu %s] %s" % (name, tdo.check(name, case, ref)))


@pytest.mark.parametrize("name", list(tdo.ALPHA_CASES))
def test_fixture_alpha_cases_equal_the_fp32_oracle(name):
    case, ref = tdo.load_alpha_case(tdo._load_golden(), name)
    opt = types.SimpleNamespace(alpha_range=1 if case["range_test"] else 0, inall_img=1)
    V = len(case["alpha"])
    m = depth_filter.alpha_masking(torch.from_numpy(case["points"]).to(DEV), [case["alpha"][v][None] for v in range(V)], list(case["K"]),
                                   None, list(case["w2c"]), case["near_far"], opt=opt)
    assert m.dtype == torch.bool and m.shape == (len(case["points"]),)
    mine = m.cpu().numpy()
    assert np.array_equal(mine, do.alpha_mask(case["points"], case["alpha"], case["K"], case["w2c"], case["near_far"], case["range_test"]))
    do.compare_alpha(case, ref, mine)


def _big_case(V, H, W, seed):
    """V cameras on an arc over the plane z = 3 (depths in closed form) with 0.4 % depth noise, so that thousands of pixels sit near
    dist 1 and rel 0.01, zero-depth patches, 90 % of the mask set and uniform confidences."""
    g = np.random.default_rng(seed)
    f = 0.9 * W
    K = np.array([[f, 0, W / 2 - 0.3], [0, f, H / 2 + 0.2], [0, 0, 1]], F32)
    Es = [tdo._look_at(np.array([3 * np.sin(a), 0.3 * np.cos(5 * a), 3 - 3 * np.cos(a)]), [0.05, 0.0, 3.0])
          for a in np.linspace(-0.4, 0.4, V)]
    yy, xx = np.meshgrid(np.arange(H, dtype=F32), np.arange(W, dtype=F32), indexing="ij")
    depth = np.zeros((V, H, W), F32)
    xy = np.zeros((V, H, W, 2), F32)
    for v, E in enumerate(Es):
        R, cpos = E[:3, :3], -E[:3, :3].T @ E[:3, 3]
        dx, dy = (xx - K[0, 2]) / K[0, 0], (yy - K[1, 2]) / K[1, 1]
        dzw = R[0, 2] * dx + R[1, 2] * dy + R[2, 2]                  # world z of the camera ray (x, y, 1)
        t = ((3.0 - cpos[2]) / dzw).astype(F32)
        z = (t * (1 + g.normal(0, 0.004, (H, W)))).astype(F32)
        z[H // 3:H // 3 + 4, W // 4:W // 4 + 6] = 0.0
        depth[v] = z
        xy[v, ..., 0], xy[v, ..., 1] = dx * z, dy * z
    return dict(depth=depth, xy=xy, conf=g.uniform(0, 1, (V, H, W)).astype(F32), mask=g.uniform(size=(V, H, W)) < 0.9,
                K=np.array([K] * V), E=np.array(Es, F32), thresh=0.3, geo_n=3, ranges=np.array([-3, -3, 2.9, 3, 3, 3.1], F32))


def _near_thresholds(case, r, every=4):
    """Pixel-pairs of ref view r (every `every`-th live pixel) whose fp32 dist lies within 0.02 of 1 and whose rel lies within 1e-4 of
    0.01."""
    live = np.nonzero(((case["conf"][r] > F32(case["thresh"])) & case["mask"][r]).reshape(-1))[0][::every]
    _, _, per = do.geo_pass(case, r, do.view_matrices(case["K"], case["E"]), live, detail=True)
    near_dist = sum(int((np.abs(p["dist"] - 1) < 0.02).sum()) for p in per)
    near_rel = sum(int((np.abs(p["rel"] - 0.01) < 1e-4).sum()) for p in per)
    return near_dist, near_rel


# the DTU size is checked on every view; the n360 size, whose oracle costs seconds per view, on every tenth and the last
@pytest.mark.parametrize("V,H,W,views", [(49, 512, 640, list(range(49))), (100, 800, 800, list(range(0, 100, 10)) + [99])])
def test_large_cases_equal_the_fp32_oracle(V, H, W, views):
    case = _big_case(V, H, W, seed=V)
    near_dist, near_rel = _near_thresholds(case, V // 2)
    assert near_dist >= 1000 and near_rel >= 1000, (near_dist, near_rel)
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    args = _inputs(case)
    out = depth_filter.filter_by_masks_gpu(*args, tdo._opt(case))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    counts = [len(c) for c in out[0]]
    assert sum(counts) > 0
    again = depth_filter.filter_by_masks_gpu(*args, tdo._opt(case))
    for a, b in zip(out, again):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    _check_views(case, out, views)                      # each checked view: its count, order and bits
    print("\n[depth_filter %d x %dx%d] %d points kept, %d views checked, pixel-pairs of view %d near dist 1 / rel 0.01 (1 in 4 "
          "pixels): %d / %d, peak %.0f MiB above the inputs" % (V, H, W, sum(counts), len(views), V // 2, near_dist, near_rel,
                                                              peak / 2 ** 20))


def test_cpu2gpu_equals_device_inputs():
    case = tdo.surface_case(V=301, H=24, W=32, seed=7, geo_n=3)
    dev_out = _run(case)
    host_out = _run(case, cpu2gpu=True)
    for a, b in zip(dev_out, host_out):
        for x, y in zip(a, b):
            assert y.device.type == "cpu" and torch.equal(x.cpu(), y)
    _check_views(case, host_out, [0, 300])


def test_alpha_masking_at_size():
    g = np.random.default_rng(11)
    V, H, W, N = 100, 200, 256, 20_000_000
    case = tdo.alpha_case(N=8, V=V, H=H, W=W, seed=11)
    alpha = g.choice(np.array([0.0, 0.1, 0.5, 1.0], F32), size=(V, H, W), p=[0.001, 0.001, 0.002, 0.996])
    pts = torch.empty((N, 3), device=DEV).uniform_(-1.2, 1.2, generator=torch.Generator(DEV).manual_seed(3))
    pts[:, 2] += 3.0
    torch.cuda.reset_peak_memory_stats(DEV)
    opt = types.SimpleNamespace(alpha_range=1, inall_img=1)
    m = depth_filter.alpha_masking(pts, [alpha[v][None] for v in range(V)], list(case["K"]), None, list(case["w2c"]), (0.5, 6.0), opt=opt)
    torch.cuda.synchronize()
    print("\n[alpha %d x %d] %d kept, peak %.0f MiB" % (N, V, int(m.sum()), torch.cuda.max_memory_allocated(DEV) / 2 ** 20))
    idx = torch.randperm(N, device=DEV, generator=torch.Generator(DEV).manual_seed(5))[:1_000_000]
    want = do.alpha_mask(pts[idx].cpu().numpy(), alpha, case["K"], case["w2c"], (0.5, 6.0), True)
    got = m[idx].cpu().numpy()
    assert np.array_equal(got, want) and got.any() and (~got).any()


def test_chain_into_voxelize():
    """gen_points_filter_embeddings' geometric chain through the drop-ins equals the chain fed the oracle's outputs."""
    case = tdo.surface_case(V=5, H=120, W=160, seed=9, geo_n=2)
    _, world, conf = _run(case)
    points_vid = torch.cat([torch.ones_like(w[..., 0:1]) * i for i, w in enumerate(world)])
    xyz = torch.cat(world)
    ac = tdo.alpha_case(N=8, V=4, H=120, W=160, seed=9)
    alpha = np.ones((4, 120, 160), F32)
    alpha[:, 40:60, 50:90] = 0.0
    m = depth_filter.alpha_masking(xyz, [alpha[v][None] for v in range(4)], list(ac["K"]), None, list(ac["w2c"]), None,
                                   opt=types.SimpleNamespace(alpha_range=0, inall_img=1))
    xyz, points_vid, conf_all = xyz[m], points_vid[m], torch.cat(conf)[m]
    vox, _, idx = voxelize.construct_vox_points_closest(xyz, 64)
    # the same chain on the oracle's outputs
    ow = [do.filter_view(case, r)["world"] for r in range(5)]
    oxyz = np.concatenate(ow)
    om = do.alpha_mask(oxyz, alpha, ac["K"], ac["w2c"], None, False)
    assert np.array_equal(m.cpu().numpy(), om) and om.any() and (~om).any()
    ovox, _, oidx = voxelize.construct_vox_points_closest(torch.from_numpy(oxyz[om]).to(DEV), 64)
    assert torch.equal(vox, ovox) and torch.equal(idx, oidx)
    assert torch.equal(points_vid[idx], torch.from_numpy(np.concatenate([np.full((len(w), 1), i, F32) for i, w in enumerate(ow)])[om]).to(DEV)[oidx])


def test_cpu2gpu_chain_equals_device_chain(monkeypatch):
    """The n360 path of gen_points_filter_embeddings: filter_by_masks_gpu with cpu2gpu returns host tensors, the runner concatenates
    them on the host and passes them to alpha_masking, which returns a host mask.  It equals the device-input chain bit for bit, also
    when the host points are staged in several chunks."""
    monkeypatch.setattr(depth_filter, "HOST_CHUNK", 1000)
    case = tdo.surface_case(V=301, H=24, W=32, seed=8, geo_n=3)
    ac = tdo.alpha_case(N=8, V=4, H=24, W=32, seed=8)
    alpha = np.ones((4, 24, 32), F32)
    alpha[:, 8:14, 10:20] = 0.0
    opt = types.SimpleNamespace(alpha_range=0, inall_img=1)
    masks = []
    for cpu2gpu in (False, True):
        _, world, _ = _run(case, cpu2gpu=cpu2gpu)
        xyz = torch.cat(world)
        assert xyz.is_cuda != cpu2gpu
        masks.append(depth_filter.alpha_masking(xyz, [alpha[v][None] for v in range(4)], list(ac["K"]), None, list(ac["w2c"]), None,
                                                opt=opt))
    dev_mask, host_mask = masks
    assert host_mask.device.type == "cpu" and len(host_mask) > 3000
    assert torch.equal(dev_mask.cpu(), host_mask) and host_mask.any() and (~host_mask).any()


def test_refusals():
    case = tdo.surface_case(V=3, H=16, W=20, seed=1)
    args = _inputs(case)
    for key, val, word in (("manual_depth_view", 2, "manual_depth_view"), ("default_conf", 1.5, "default_conf"),
                           ("far_plane_shift", 0.1, "far_plane_shift")):
        opt = types.SimpleNamespace(**dict(vars(tdo._opt(case)), **{key: val}))
        with pytest.raises(NotImplementedError, match=word):
            depth_filter.filter_by_masks_gpu(*args, opt)
    cam = list(args[0])
    cam[0] = torch.cat([cam[0], cam[0]])
    with pytest.raises(ValueError, match="B = N = 1"):
        depth_filter.filter_by_masks_gpu(cam, *args[1:], tdo._opt(case))
    cam = list(args[0])
    cam[1] = cam[1][..., :10, :, :].contiguous()
    with pytest.raises(ValueError, match="every view"):
        depth_filter.filter_by_masks_gpu(cam, *args[1:], tdo._opt(case))
