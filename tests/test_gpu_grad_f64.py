"""GPU: the fused backward (pnb_shade_backward) against float64 autograd through the oracle run with the kernel's own LeakyReLU masks.

After the drop-in's forward + backward, pnb_backward_tables gives the recompute buffers the backward took its masks from (the
post-activations of the 7 LeakyReLU layers) and the packed pair rows.  Each row is mapped to its (ray, sample slot, K slot) through
valid_list / samp_off / pair_off, the masks are handed to oracle/shade_oracle.py as `slopes=`, and every point gradient and every one
of the 18 MLP tensors must agree with float64 autograd within one bound per backward mode (oracle/grad_check.py), with no allowance
for outliers: a bug that touches a few pair rows only (a partial GEMM tile, one split-K slab, one K slot, a channel edge of the
F = 63 scatter) shows.  Each case reports how many units the kernel's masks flip against float64's own."""
import ctypes as C

import pytest
import torch

from oracle import forward_check, grad_check, shade_oracle, shade_oracle_rw2c
from pointnerf_b200 import harness, lib, scene
from pointnerf_b200.point_query import make_cam_opts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# (points, MLP tensors): the largest error allowed, relative to the tensor's scale, per (pnb_bwd_fp32 mode, pnb_precision), 4-5x the
# largest measured over this file's cases on an H100 80GB HBM3 at a 400 W power limit:
#   mode 0 (BF16x3 recompute, dX, dW)    bf16x3: points 8.9e-6, MLP 2.8e-5    fp32: points 8.3e-6, MLP 2.7e-5
#   mode 4 (fp32 recompute, BF16x3 dX/dW) bf16x3: points 8.8e-6, MLP 2.6e-5
#   mode 1 (fp32 CUDA-core GEMMs)         bf16x3: points 4.7e-6, MLP 1.2e-6    fp32: points 4.9e-7, MLP 6.7e-7
# The tensor-core dX / dW GEMMs carry the ~1e-5 of the BF16x3 split (tests/test_gpu_umma.py); in mode 1 the points see the BF16x3
# forward's (sigma, rgb), from which the composite backward starts.  One flipped or lost pair row moves its points by ~1e-3 of scale.
RTOL = {(0, "bf16x3"): (4e-5, 1.2e-4), (0, "fp32"): (4e-5, 1.2e-4), (4, "bf16x3"): (4e-5, 1.2e-4),
        (1, "bf16x3"): (2e-5, 5e-6), (1, "fp32"): (2e-6, 3e-6)}


def _kernel_masks(net, q, F, camrotc2w):
    """The backward's masks as `slopes=` of the oracle (pair rows in the flattened [R',SR,K] order of sample_pidx >= 0, colour rows per
    sample slot), the dense export of the query, and the pair-row count."""
    l = lib.load()
    S, P = int(q.counters["n_valid"]), int(q.counters["n_pairs"])
    out = (C.c_void_p * 10)()
    ws = net._bwd_ws
    lib.check(l.pnb_backward_tables(ws.data_ptr(), ws.numel(), S, q.desc.cap_samples, F, out), "pnb_backward_tables")
    dev_view = forward_check.dev_view
    H = [dev_view(ws, out[0], torch.float32, (P, 256)), dev_view(ws, out[1], torch.float32, (P, 272))[:, :256],
         dev_view(ws, out[2], torch.float32, (P, 256)), dev_view(ws, out[3], torch.float32, (P, 256))]
    Cc = [dev_view(ws, out[i], torch.float32, (S, 128)) for i in (4, 5, 6)]
    pair_off = dev_view(ws, out[7], torch.int32, (S + 1,)).long()
    row_samp = dev_view(ws, out[8], torch.int32, (P,)).long()
    pidx = dev_view(ws, out[9], torch.int32, (P,)).long()
    ex = q.export(make_cam_opts(list(q.desc.campos), camrotc2w), want_pers=False, want_dirs=False)
    SR = q.SR
    # valid sample -> (ray, sample slot) -> its row of the export; pair row -> (its sample, K slot)
    srow = forward_check.sample_map(q, ex)["srow"]
    flat = forward_check.pair_map(dict(srow=srow), pair_off, row_samp, pidx, ex, q.K)
    order = torch.argsort(flat)
    slopes = [torch.where(h[order] > 0, 1.0, 0.01).double() for h in H]
    for c in Cc:
        s = torch.ones(ex["sample_pidx"].shape[0] * SR, 128, dtype=torch.float64)
        s[srow] = torch.where(c > 0, 1.0, 0.01).double()
        slopes.append(s)
    return slopes, ex, P


def _forward(net, rays):
    r = {k: v.to(DEV) for k, v in rays.items()}
    return net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
               near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


def _loss(ray_color, conf_coefficient, opacity, bg_T, ext):
    """The colour + conf loss of the fixtures; ext: plus terms on opacity [R',SR] and bg_T [R'] (k_composite_bwd<true>)."""
    loss = (ray_color ** 2).sum() + 1e-3 * conf_coefficient.sum()
    if ext:
        w = torch.rand(opacity.shape, generator=torch.Generator().manual_seed(5)).to(opacity)
        loss = loss + 0.5 * (opacity * w).sum() + 2.0 * (bg_T.reshape(-1) ** 2).sum()
    return loss


def _run_case(cfg_name, side, F=32, frames=False, order=2, mode=0, precision="bf16x3", ext=False, rotated=False, monkeypatch=None,
              **over):
    """rotated: the camera orbited about the origin (scene.orbit_rotation), so that camrotc2w is not the identity."""
    cfg = scene.CONFIGS[cfg_name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, seed=2, feat_dim=F, agg_intrp_order=order, pnb_precision=precision,
                                        pnb_bwd_fp32=mode, **over)
    npn = net.neural_points
    R = torch.eye(3)
    if frames:
        R = scene.edit_frames(pts["xyz"])
        npn.Rw2c = torch.nn.Parameter(R.to(DEV), requires_grad=False)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side), camrotc2w=scene.orbit_rotation() if rotated else None)
    cam = rays["camrotc2w"][0]
    out = _forward(net, rays)
    _loss(out["coarse_raycolor"][0], out["conf_coefficient"], out["coarse_point_opacity"][0], out["coarse_is_background"][0], ext).backward()
    net.check_errors()
    q = net.last
    slopes, ex, P = _kernel_masks(net, q, F, cam)
    hit = ex["ray_mask"].cpu() > 0
    # float64 autograd through the oracle with the kernel's masks, on the kernel's own sample geometry
    pts_g = dict(xyz=npn.xyz.detach().cpu().double(), Rw2c=R.double())
    for k, t in (("embedding", npn.points_embeding), ("color", npn.points_color), ("dir", npn.points_dir), ("conf", npn.points_conf)):
        pts_g[k] = t.detach().cpu().double().requires_grad_(True)
    mlp_g = {k: v.double().requires_grad_(True) for k, v in harness.mlp_cpu(net.aggregator).items()}
    args = (ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu(), rays["raydir"][0][hit], rays["campos"][0], cam, opt.vsize, torch.ones(3))
    sh = shade_oracle_rw2c.shade(pts_g, mlp_g, *args, dtype=torch.float64, agg_intrp_order=order, slopes=slopes)
    _loss(sh["ray_color"], sh["conf_coefficient"], sh["opacity"], sh["bg_T"], ext).backward()
    # float64's own masks: the units the kernel's masks flip (forward only)
    rec = grad_check.MaskRecorder(shade_oracle.F)
    with monkeypatch.context() as m, torch.no_grad():
        m.setattr(shade_oracle, "F", rec)
        shade_oracle_rw2c.shade({k: v.detach() for k, v in pts_g.items()}, {k: v.detach() for k, v in mlp_g.items()}, *args,
                                dtype=torch.float64, agg_intrp_order=order)
    flips = [int((a != b).sum()) for a, b in zip(slopes, rec.slopes)]
    # colour rows of slots without neighbours hold no kernel mask
    sv = (ex["sample_pidx"].cpu() >= 0).any(-1).reshape(-1)
    flips[4:] = [int((a[sv] != b[sv]).sum()) for a, b in zip(slopes[4:], rec.slopes[4:])]
    # every comparison first (the report), then the bounds
    n0 = int((ex["sample_pidx"].cpu().clamp(min=0) == 0).sum())
    err = {k: grad_check.rel_point_errors(getattr(npn, "points_" + s).grad.cpu(), pts_g[k].grad).max()
           for k, s in (("embedding", "embeding"), ("color", "color"), ("dir", "dir"))}
    cg, cr = npn.points_conf.grad.cpu().double().reshape(-1), pts_g["conf"].grad.reshape(-1)
    err["conf"] = grad_check.rel_point_errors(cg[1:, None], cr[1:, None]).max()
    err0 = (abs(cg[0] - cr[0]).item(), grad_check.point0_conf_bound(n0, cr[0]))
    for k, p in net.aggregator.named_parameters():
        err[k] = grad_check.rel_error(p.grad.cpu(), mlp_g[k].grad)
    pts_worst = max(err[k] for k in ("embedding", "color", "dir", "conf"))
    mlp_worst = max(v for k, v in err.items() if "." in k)
    max_nsamp = int(forward_check.dev_view(q.ws, q.desc.nsamp, torch.int32, (q.R,)).max())
    print("\n[grad-f64] %s side=%d F=%d frames=%d order=%d mode=%d %s ext=%d rot=%d %s: P=%d max nsamp=%d flips/layer=%s points=%.2e "
          "mlp=%.2e (%s) conf0=%.2e/%.2e" % (cfg_name, side, F, frames, order, mode, precision, ext, rotated, over, P, max_nsamp, flips,
                                             pts_worst, mlp_worst, max((k for k in err if "." in k), key=err.get), err0[0], err0[1]))
    rtol_points, rtol_mlp = RTOL[(mode, precision)]
    for k, v in err.items():
        rtol = rtol_mlp if "." in k else rtol_points
        assert v <= rtol, "%s: %.3e of scale > %.1e" % (k, v, rtol)
    assert err0[0] <= err0[1], "points_conf of point 0: %.3e > %.3e" % err0
    assert npn.xyz.grad is None
    return P, flips


@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("frames", [False, True])
@pytest.mark.parametrize("F", [32, 63])
def test_backward_matches_float64_with_kernel_masks(F, frames, order, mode, monkeypatch):
    _run_case("tiny", 20, F=F, frames=frames, order=order, mode=mode, monkeypatch=monkeypatch)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_fp32_forward_backward_matches_float64(F, mode, monkeypatch):
    _run_case("tiny", 20, F=F, mode=mode, precision="fp32", monkeypatch=monkeypatch)


@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_chair_patch_beyond_four_split_k_slabs(F, mode, monkeypatch):
    """More than 4 split-K slabs of 2048 rows in every dW GEMM of the pair layers, and partial last tiles."""
    P, flips = _run_case("chair_plumbing", 24, F=F, mode=mode, monkeypatch=monkeypatch)
    assert P > 4 * 2048, P
    if mode == 0:
        assert sum(flips) > 0, "no unit flips: the case does not exercise the kernel's own masks"


@pytest.mark.parametrize("over", [dict(K=3), dict(K=1), dict(SR=8), dict(SR=80), dict(SR=128)], ids=["K3", "K1", "SR8", "SR80", "SR128"])
@pytest.mark.parametrize("F", [32, 63])
def test_edges(F, over, monkeypatch):
    _run_case("tiny", 16, F=F, monkeypatch=monkeypatch, **over)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("frames", [False, True])
@pytest.mark.parametrize("F", [32, 63])
def test_backward_with_rotated_camera(F, frames, mode, monkeypatch):
    """camrotc2w not the identity: the perspective coordinates, dists[3:6] and the ray-distance depth of every pair see the rotation
    (rot3 and rot3T differ), and so do the opacity and bg_T terms of the loss."""
    _run_case("tiny", 20, F=F, frames=frames, mode=mode, ext=True, rotated=True, monkeypatch=monkeypatch)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("order", [2, 1])
def test_opacity_and_background_terms(order, mode, monkeypatch):
    """A loss with opacity and bg_T terms (k_composite_bwd<true>), per-point frames, 63 channels."""
    _run_case("tiny", 20, F=63, frames=True, order=order, mode=mode, ext=True, monkeypatch=monkeypatch)
