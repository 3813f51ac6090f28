"""CPU: the method of tests/test_gpu_frustum_session.py, checked with the C frustum oracle (oracle/frustum_oracle.py) and numpy.

  views     every session view but "away" has thousands of hit rays over the frame and no P overflow; "away" has R' = 0
  grid      v3's intrinsic gives other grid hyperparameters than v0's (ranges and voxel sizes) on the same grid dimensions, and the
            views that share v0's intrinsic share its grid (what lets a stale build stay in bounds)
  stale     v0 and v1 give different sample_pidx on the pixels both hit: a build kept across that switch is visible
  loss      the session's loss in float64 and its zero_one straight-through clamp agree with an fp32 evaluation to fp32 rounding,
            values and gradients, with conf_coefficient entries on both sides of the clamps
"""
import functools

import numpy as np
import pytest
import torch

import test_gpu_frustum_session as session
from oracle import frustum_oracle
from pointnerf_b200 import scene
from pointnerf_b200 import query_point_indices as qpi

CFG = session.CFG
U32 = 2.0 ** -24


def _grid(view):
    _, _, K = session.views()[view]
    opt = scene.frustum_opt(CFG)
    return opt, qpi.hyperparameters(opt, np.int64(CFG.H), np.int64(CFG.W), K, np.float32(CFG.near), np.float32(CFG.far))


@functools.lru_cache(None)
def _query(view):
    """The CPU oracle's query of the whole frame of a view, on the points in the view's perspective coordinates (the reference's
    w2pers on the CPU)."""
    R, c, _ = session.views()[view]
    s = scene.make_frustum_scene(CFG)
    pers = qpi.w2pers(torch.from_numpy(s["xyz_w"]), torch.from_numpy(R)[None], torch.from_numpy(c)[None])[0].numpy()
    opt, (rl, dl, ranges, vsize, vdim, svs, sdim, vscale) = _grid(view)
    return frustum_oracle.query(pers, ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size, opt.SR, opt.K, opt.P,
                                session.frame_pixels(), np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)


@pytest.mark.parametrize("view", list(session.views()))
def test_view_hits(view):
    out = _query(view)
    c = out["counters"]
    valid = int((out["sample_pidx"] >= 0).any(-1).sum())
    print("\n[frustum session method] %s: R'=%d of %d, valid samples %d, counters %s" % (view, c["R2"], CFG.H * CFG.W, valid, c))
    if view == "away":
        assert c["R2"] == 0
        return
    assert c["R2"] >= 5000 and valid >= 20000, (c["R2"], valid)
    assert c["overflow_p"] == 0


def test_v3_has_another_grid_of_the_same_dimensions():
    _, g0 = _grid("v0")
    _, g3 = _grid("v3")
    ranges, vsize, vdim, svs, sdim = 2, 3, 4, 5, 6
    assert not np.array_equal(g0[ranges], g3[ranges]) and not np.array_equal(g0[vsize][:2], g3[vsize][:2])
    assert np.array_equal(g0[vdim], g3[vdim]) and np.array_equal(g0[sdim], g3[sdim])
    for v in ("v1", "v2", "away"):
        _, g = _grid(v)
        assert all(np.array_equal(a, b) for a, b in zip(g, g0)), v


def test_v0_and_v1_differ_on_shared_pixels():
    a, b = _query("v0"), _query("v1")
    pix = session.frame_pixels()
    ids = pix[:, 1] * CFG.W + pix[:, 0]
    rows_a = {int(i): r for r, i in enumerate(ids[a["ray_mask"] > 0])}
    rows_b = {int(i): r for r, i in enumerate(ids[b["ray_mask"] > 0])}
    shared = sorted(set(rows_a) & set(rows_b))
    same = sum(np.array_equal(a["sample_pidx"][rows_a[i]], b["sample_pidx"][rows_b[i]]) for i in shared)
    print("\n[frustum session method] v0 / v1: %d shared hit pixels, %d with the same sample_pidx" % (len(shared), same))
    assert len(shared) >= 5000 and same <= 0.05 * len(shared)


def _loss_inputs(dtype, seed=3, R2=300, SR=40, K=8, N=2000):
    """Seeded fp32 inputs of the session's loss (in `dtype`): colours and transmittance, a bg_ray, ground truth, a conf table with entries below 1e-4,
    inside (1e-4, 1e-3), inside the zero_one clamp, inside (1 - 1e-3, 1) and above 1, and slots with empty neighbours (pidx -1)."""
    g = np.random.RandomState(seed)
    conf = g.uniform(0.0, 1.0, (1, N, 1))
    conf[0, :40, 0] = g.choice([5e-5, 5e-4, 0.9995, 1.2, 2e-3, 0.998], 40)
    pidx = g.randint(-1, N, (R2, SR, K)).astype(np.int32)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float32)).to(dtype)  # noqa: E731  (both precisions on the same fp32 values)
    return dict(color=t(g.uniform(0, 1, (R2, 3))), is_bg=t(g.uniform(0, 1, (R2, 1))), bg=t(g.uniform(0, 1, (R2, 3))),
                gt=t(g.uniform(0, 1, (R2, 3))), conf=t(conf), pidx=torch.from_numpy(pidx))


def _evaluate(dtype):
    x = _loss_inputs(dtype)
    for k in ("color", "is_bg", "conf"):
        x[k].requires_grad_(True)
    cc = session.conf_coefficient(x["conf"], x["pidx"])
    L = session.loss(x["color"], x["is_bg"], x["bg"], x["gt"], cc)
    L.backward()
    return L.detach().double(), cc.detach().double(), {k: x[k].grad.double() for k in ("color", "is_bg", "conf")}


def test_float64_loss_and_clamp_agree_with_fp32():
    L64, cc64, g64 = _evaluate(torch.float64)
    L32, cc32, g32 = _evaluate(torch.float32)
    x = _loss_inputs(torch.float64)
    # the straight-through clamp: values clamped to [1e-4, 1], every slot a slope of 1 into its point's conf
    conf = x["conf"][0, :, 0]
    assert torch.equal(cc64, torch.clamp(conf[torch.clamp(x["pidx"], min=0).long()], 1e-4, 1))
    assert float(cc64.min()) == 1e-4 and float(cc64.max()) == 1.0
    assert torch.equal(cc32, cc64.float().double())
    # the value: colour terms (sum of R' * 3 squares) and the zero_one mean, each within a few fp32 roundings of its magnitude
    n = x["pidx"].numel()
    tol = 4 * U32 * (float(((x["is_bg"] * x["bg"] + x["color"] - x["gt"]) ** 2).sum()) * np.log2(x["color"].numel()) + 1e-3 * 8 * np.log2(n))
    assert abs(float(L32 - L64)) <= tol, (float(L32 - L64), tol)
    # the gradients: colour exact to a few roundings of each entry; conf: the zero_one term flows only through slots inside the
    # zero_one clamp, straight through the [1e-4, 1] clamp
    for k in ("color", "is_bg"):
        assert float((g32[k] - g64[k]).abs().max()) <= 8 * U32 * float(g64[k].abs().max()), k
    gc = g64["conf"][0, :, 0]
    assert float(gc.abs().max()) > 0
    inside = (cc64 >= 1e-3) & (cc64 <= 1 - 1e-3)
    idx = torch.clamp(x["pidx"], min=0).long()
    reached = torch.zeros_like(conf, dtype=torch.bool)
    reached[idx[inside]] = True
    assert torch.all(gc[~reached] == 0) and torch.all(gc[reached] != 0)
    want = torch.zeros_like(conf).index_add_(0, idx[inside], (1e-3 / n) * (1 / cc64[inside] - 1 / (1 - cc64[inside])))
    assert float((gc - want).abs().max()) <= 1e-12 * float(want.abs().max())
    assert float((g32["conf"] - g64["conf"]).abs().max()) <= 64 * U32 * float(gc.abs().max())
