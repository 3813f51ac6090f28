"""GPU: the fused backward (pnb_shade_backward) against float64 autograd through the oracle run with the kernel's own LeakyReLU masks.

After the drop-in's forward + backward, pnb_backward_tables gives the recompute buffers the backward took its masks from (the
post-activations of the 7 LeakyReLU layers) and the packed pair rows.  Each row is mapped to its (ray, sample slot, K slot) through
valid_list / samp_off / pair_off, the masks are handed to oracle/shade_oracle.py as `slopes=`, and every point gradient and every one
of the 18 MLP tensors must agree with float64 autograd within one bound per backward mode (oracle/grad_check.py), with no allowance
for outliers: a bug that touches a few pair rows only (a partial GEMM tile, one split-K slab, one K slot, a channel edge of the
F = 63 scatter) shows.  Each case reports how many units the kernel's masks flip against float64's own."""
import pytest
import torch

from oracle import forward_check, grad_check, shade_oracle, shade_oracle_rw2c
from pointnerf_b200 import harness, scene
from pointnerf_b200.point_query import make_cam_opts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
RTOL = grad_check.RTOL       # the bound of each backward mode, measured over this file's cases


def _forward(net, rays):
    r = {k: (None if v is None else v.to(DEV)) for k, v in rays.items()}
    return net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
               near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])


CC_TERM = 2e-3       # the largest weight of a conf_coefficient entry under cc_weights


def _loss(ray_color, conf_coefficient, opacity, bg_T, ext, cc_weights=False, colour=True):
    """The colour + conf loss of the fixtures; ext: plus terms on opacity [R',SR] and bg_T [R'] (k_composite_bwd<true>).  cc_weights:
    every entry of conf_coefficient [R',SR,K] weighted by its own seeded factor in [0, 2e-3) instead of the constant 1e-3, so that its
    upstream gradient differs from entry to entry.  colour: False leaves the conf term alone."""
    if cc_weights:
        w = CC_TERM * torch.rand(conf_coefficient.shape[-3:], generator=torch.Generator().manual_seed(9))
        loss = (conf_coefficient * w.to(conf_coefficient)).sum()
    else:
        loss = 1e-3 * conf_coefficient.sum()
    if not colour:
        return loss
    loss = (ray_color ** 2).sum() + loss
    if ext:
        w = torch.rand(opacity.shape, generator=torch.Generator().manual_seed(5)).to(opacity)
        loss = loss + 0.5 * (opacity * w).sum() + 2.0 * (bg_T.reshape(-1) ** 2).sum()
    return loss


POINT_OPTS = dict(embedding="feat_grad", color="color_grad", dir="dir_grad", conf="conf_grad")


def _run_case(cfg_name, side, F=32, frames=False, order=2, mode=0, precision="bf16x3", ext=False, rotated=False, monkeypatch=None,
              alpha_bias=3.0, bg=(1.0, 1.0, 1.0), cc_weights=False, freeze=(), edit=None, pixels=None, **over):
    """rotated: the camera orbited about the origin (scene.orbit_rotation), so that camrotc2w is not the identity.  bg: the background's
    channels.  cc_weights: see _loss.  freeze: parameter groups without gradient, of "embedding", "color", "dir", "conf" (the
    reference's feat_grad / color_grad / dir_grad / conf_grad = 0) and "mlp" (the aggregator's requires_grad_(False)): their .grad
    stays None, and pnb_shade_backward gets NULL for the point tensors among them.  edit(net, rays): point values written before the
    forward.  over: options of harness.make_opt.  Returns the pair-row count, the unit flips per layer and the model."""
    cfg = scene.CONFIGS[cfg_name]
    over.update({POINT_OPTS[k]: 0 for k in freeze if k != "mlp"})
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=alpha_bias, seed=2, feat_dim=F, agg_intrp_order=order, pnb_precision=precision,
                                        pnb_bwd_fp32=mode, **over)
    if "mlp" in freeze:
        net.aggregator.requires_grad_(False)
    npn = net.neural_points
    R = torch.eye(3)
    if frames:
        R = scene.edit_frames(pts["xyz"])
        npn.Rw2c = torch.nn.Parameter(R.to(DEV), requires_grad=False)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side) if pixels is None else pixels,
                           camrotc2w=scene.orbit_rotation() if rotated else None, bg_color=bg)
    cam = rays["camrotc2w"][0]
    if edit is not None:
        edit(net, rays)
    out = _forward(net, rays)
    _loss(out["coarse_raycolor"][0], out["conf_coefficient"], out["coarse_point_opacity"][0], out["coarse_is_background"][0], ext,
          cc_weights).backward()
    net.check_errors()
    q = net.last
    slopes, ex, P = grad_check.kernel_masks(net, q, F, cam)
    hit = ex["ray_mask"].cpu() > 0
    # float64 autograd through the oracle with the kernel's masks, on the kernel's own sample geometry
    pts_g = dict(xyz=npn.xyz.detach().cpu().double(), Rw2c=R.double())
    for k, t in (("embedding", npn.points_embeding), ("color", npn.points_color), ("dir", npn.points_dir), ("conf", npn.points_conf)):
        pts_g[k] = t.detach().cpu().double().requires_grad_(True)
    mlp_g = {k: v.double().requires_grad_(True) for k, v in harness.mlp_cpu(net.aggregator).items()}
    args = (ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu(), rays["raydir"][0][hit], rays["campos"][0], cam, opt.vsize, rays["bg_color"][0])
    mode_unit = opt.raydist_mode_unit
    sh = shade_oracle_rw2c.shade(pts_g, mlp_g, *args, dtype=torch.float64, agg_intrp_order=order, slopes=slopes, raydist_mode_unit=mode_unit)
    _loss(sh["ray_color"], sh["conf_coefficient"], sh["opacity"], sh["bg_T"], ext, cc_weights).backward()
    # float64's own masks: the units the kernel's masks flip (forward only)
    rec = grad_check.MaskRecorder(shade_oracle.F)
    with monkeypatch.context() as m, torch.no_grad():
        m.setattr(shade_oracle, "F", rec)
        shade_oracle_rw2c.shade({k: v.detach() for k, v in pts_g.items()}, {k: v.detach() for k, v in mlp_g.items()}, *args,
                                dtype=torch.float64, agg_intrp_order=order, raydist_mode_unit=mode_unit)
    flips = [int((a != b).sum()) for a, b in zip(slopes, rec.slopes)]
    # colour rows of slots without neighbours hold no kernel mask
    sv = (ex["sample_pidx"].cpu() >= 0).any(-1).reshape(-1)
    flips[4:] = [int((a[sv] != b[sv]).sum()) for a, b in zip(slopes[4:], rec.slopes[4:])]
    # every comparison first (the report), then the bounds
    n0 = int((ex["sample_pidx"].cpu().clamp(min=0) == 0).sum())
    tensors = dict(embedding=npn.points_embeding, color=npn.points_color, dir=npn.points_dir, conf=npn.points_conf)
    frozen = [k for k, t in list(tensors.items()) + list(net.aggregator.named_parameters()) if (k in freeze or ("." in k and "mlp" in freeze))]
    not_none = [k for k, t in list(tensors.items()) + list(net.aggregator.named_parameters()) if k in frozen and t.grad is not None]
    err = {k: grad_check.rel_point_errors(tensors[k].grad.cpu(), pts_g[k].grad).max() for k in ("embedding", "color", "dir") if k not in freeze}
    err0 = (0.0, 0.0)
    if "conf" not in freeze:
        cg, cr = npn.points_conf.grad.cpu().double().reshape(-1), pts_g["conf"].grad.reshape(-1)
        err["conf"] = grad_check.rel_point_errors(cg[1:, None], cr[1:, None]).max()
        err0 = (abs(cg[0] - cr[0]).item(), grad_check.point0_conf_bound(n0, cr[0], CC_TERM if cc_weights else 1e-3))
    if "mlp" not in freeze:
        for k, p in net.aggregator.named_parameters():
            err[k] = grad_check.rel_error(p.grad.cpu(), mlp_g[k].grad)
    got = [t.grad for t in list(tensors.values()) + list(net.aggregator.parameters()) if t.grad is not None]
    finite = all(bool(torch.isfinite(g).all()) for g in got)
    pts_worst = max([err[k] for k in tensors if k in err] or [0.0])
    mlp_keys = [k for k in err if "." in k]
    mlp_worst = max([err[k] for k in mlp_keys] or [0.0])
    max_nsamp = int(forward_check.dev_view(q.ws, q.desc.nsamp, torch.int32, (q.R,)).max())
    # samples whose opacity is 1 in fp32 and the smallest non-zero transmittance in front of a sample, from the float64 run
    valid = sh["ray_valid"]
    n_sat = int(((sh["opacity"].detach().float() == 1) & valid).sum())
    n_long = int((sh["ray_dist"] > 2 * float(opt.vsize[2])).sum())
    T = sh["acc_T"].detach().float()
    print("\n[grad-f64] %s side=%d F=%d frames=%d order=%d mode=%d %s ext=%d rot=%d ab=%g bg=%s ccw=%d freeze=%s edit=%s %s: P=%d max nsamp=%d "
          "long=%d o==1: %d min T>0: %.2e flips/layer=%s points=%.2e mlp=%.2e (%s) conf0=%.2e/%.2e" % (
              cfg_name, side, F, frames, order, mode, precision, ext, rotated, alpha_bias, bg, cc_weights, list(freeze),
              getattr(edit, "__name__", edit), over, P, max_nsamp, n_long, n_sat, float(T[T > 0].min()), flips, pts_worst, mlp_worst,
              max(mlp_keys, key=err.get) if mlp_keys else "-", err0[0], err0[1]))
    assert finite, "a gradient is not finite"
    assert not not_none, "frozen tensors with a gradient: %s" % not_none
    rtol_points, rtol_mlp = RTOL[(mode, precision)]
    for k, v in err.items():
        rtol = rtol_mlp if "." in k else rtol_points
        assert v <= rtol, "%s: %.3e of scale > %.1e" % (k, v, rtol)
    assert err0[0] <= err0[1], "points_conf of point 0: %.3e > %.3e" % err0
    assert npn.xyz.grad is None
    return P, flips, dict(net=net, n_long=n_long, n_sat=n_sat, hit=hit, S=int(q.counters["n_valid"]))


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


# ---- batches of exactly S valid samples or P pair rows on either side of each point where the backward's launch geometry changes
# ---- (grad_check.S_TARGETS / P_TARGETS): the pixels are a subset of the tiny frame's hit rays whose counts add up to the target
def _exact_case(count, target, F, mode, monkeypatch, order=2, precision="bf16x3", **over):
    census = grad_check.frame_census("tiny", device=DEV, **over)
    pixels = grad_check.pixels_for(census, count, target)
    P, _, info = _run_case("tiny", 0, F=F, order=order, mode=mode, precision=precision, pixels=pixels, monkeypatch=monkeypatch, **over)
    S = info["S"]
    if mode == 1:       # the CUDA-core dW tiles: one atomic z-slice per 2048 rows
        splits = "k_gemm<true> slices S %d P %d" % (-(-S // grad_check.SPLITK_ROWS), -(-P // grad_check.SPLITK_ROWS))
    else:               # (asked, run) of the tensor-core split-K
        splits = "split-K S %s P %s" % (grad_check.dw_splits(S), grad_check.dw_splits(P))
    print("[grad-f64 exact] %s = %d: rays=%d S=%d P=%d dW %s" % (count, target, len(pixels), S, P, splits))
    assert (S if count == "S" else P) == target, "the batch is off its boundary: S=%d P=%d" % (S, P)
    return S, P


@pytest.mark.parametrize("target", grad_check.S_TARGETS)
@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("F,order", [(32, 2), (63, 2), (32, 1)])
def test_exact_valid_sample_counts(F, order, mode, target, monkeypatch):
    _exact_case("S", target, F, mode, monkeypatch, order=order)


@pytest.mark.parametrize("target", grad_check.P_TARGETS)
@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_exact_pair_row_counts(F, mode, target, monkeypatch):
    _exact_case("P", target, F, mode, monkeypatch)


@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_one_sample_one_pair(F, mode, monkeypatch):
    """SR 1, K 1: every hit ray holds one valid sample with one neighbour, so one ray is S = P = 1."""
    S, P = _exact_case("S", 1, F, mode, monkeypatch, SR=1, K=1)
    assert P == 1


@pytest.mark.parametrize("count,target", [("S", 1), ("S", 128), ("S", 2049), ("P", 1), ("P", 33), ("P", 129), ("P", 4097)])
@pytest.mark.parametrize("mode", [0, 1])
def test_exact_counts_fp32_forward(mode, count, target, monkeypatch):
    _exact_case(count, target, 32, mode, monkeypatch, precision="fp32")


@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_chair_patch_beyond_four_split_k_slabs(F, mode, monkeypatch):
    """More than 4 split-K slabs of 2048 rows in every dW GEMM of the pair layers, and partial last tiles."""
    P, flips, _ = _run_case("chair_plumbing", 24, F=F, mode=mode, monkeypatch=monkeypatch)
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


# ---- inputs the cases above hold constant: the background, raydist_mode_unit 0, saturated rays, the gradient of conf_coefficient,
# ---- frozen parameter groups, point values of a trained checkpoint
BG = (0.9, 0.1, 0.4)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("ext", [False, True])
@pytest.mark.parametrize("bg", [BG, (0.0, 0.0, 0.0)], ids=["coloured", "black"])
def test_background(bg, ext, mode, monkeypatch):
    """g . bg_color starts the suffix of k_composite_bwd<false> (colour-only loss) and <true> (ext): three different channels, and
    black.  (The centre patch: across the limb of the shell some consecutive samples lie exactly 2 vsize_z apart in depth, where
    float64 and fp32 take the other side of raydist_mode_unit's test and the gradients of that ray differ by a few per cent.)"""
    _run_case("tiny", 20, mode=mode, ext=ext, rotated=True, bg=bg, monkeypatch=monkeypatch)


@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("alpha_bias", [3.0, 8.0])
@pytest.mark.parametrize("F", [32, 63])
def test_raydist_mode_unit_0(F, alpha_bias, mode, monkeypatch):
    """The reference's default ray distances: the step across the inside of the shell stays (~30 voxels; SR 80 reaches the back)."""
    _, _, info = _run_case("tiny", 12, F=F, mode=mode, alpha_bias=alpha_bias, SR=80, raydist_mode_unit=0, bg=BG, ext=True,
                           monkeypatch=monkeypatch)
    assert info["n_long"] > 50, "no step above 2 vsize_z: the case is the unit mode's"


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("mode_unit,alpha_bias", [(1, 8.0), (0, 48.0)])
def test_saturated_rays(mode_unit, alpha_bias, mode, monkeypatch):
    """alpha_bias 8 with unit steps: opaque after a few samples.  48 with raydist_mode_unit 0: sigma times the long step is beyond
    fp32's 1 - exp(-x) < 1, so o == 1 there, k_composite_bwd divides the suffix by the 1e-10 floor and multiplies by 1 - o == 0."""
    _, _, info = _run_case("tiny", 12, mode=mode, alpha_bias=alpha_bias, SR=80, raydist_mode_unit=mode_unit, bg=BG, ext=True,
                           monkeypatch=monkeypatch)
    if mode_unit == 0:
        assert info["n_sat"] > 20, "no sample with opacity 1"


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_conf_coefficient_gradient_varies(F, mode, monkeypatch):
    """Every entry of conf_coefficient [R',SR,K] with its own upstream gradient (pnb_aux_conf_backward's read of g through the hit rays'
    rows), beside the colour term."""
    _run_case("tiny", 16, F=F, mode=mode, cc_weights=True, bg=BG, monkeypatch=monkeypatch)


def test_conf_only_loss_skips_the_shading_backward():
    """A loss on conf_coefficient alone: points_conf against float64, and nothing else gets a gradient (the shading backward does not
    run)."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0, seed=2)
    npn = net.neural_points
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, 16), camrotc2w=scene.orbit_rotation(), bg_color=BG)
    out = _forward(net, rays)
    _loss(None, out["conf_coefficient"], None, None, False, cc_weights=True, colour=False).backward()
    net.check_errors()
    assert npn.points_embeding.grad is None and npn.points_color.grad is None and npn.points_dir.grad is None
    assert all(p.grad is None for p in net.aggregator.parameters())
    assert getattr(net, "_bwd_ws", None) is None, "the shading backward ran"
    q = net.last
    ex = q.export(make_cam_opts(list(q.desc.campos), rays["camrotc2w"][0]), want_pers=False, want_dirs=False)
    pidx = ex["sample_pidx"].cpu()
    conf = npn.points_conf.detach().cpu().double().requires_grad_(True)
    c0 = conf[0, :, 0][pidx.clamp(min=0).long()]
    cc = c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach()
    assert (out["conf_coefficient"][0].detach().cpu().double() - cc).abs().max().item() <= 1e-7
    _loss(None, cc, None, None, False, cc_weights=True, colour=False).backward()
    n0 = int((pidx.clamp(min=0) == 0).sum())
    cg, cr = npn.points_conf.grad.cpu().double().reshape(-1), conf.grad.reshape(-1)
    e = grad_check.rel_point_errors(cg[1:, None], cr[1:, None]).max()
    d0, b0 = abs(cg[0] - cr[0]).item(), grad_check.point0_conf_bound(n0, cr[0], CC_TERM)
    print("\n[grad-f64] conf-only loss, random weights: points_conf=%.2e conf0=%.2e/%.2e" % (e, d0, b0))
    assert e <= RTOL[(1, "fp32")][0] and d0 <= b0


FREEZES = [("embedding",), ("color",), ("dir",), ("conf",), ("embedding", "color", "dir", "conf"), ("mlp",)]


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("freeze", FREEZES, ids=["+".join(f) if len(f) < 4 else "points" for f in FREEZES])
def test_frozen_parameter_groups(freeze, mode, monkeypatch):
    """feat_grad / color_grad / dir_grad / conf_grad = 0 each alone (one NULL output of pnb_shade_backward, one skipped branch of
    k_bwd_scatter), all four with a trainable aggregator, and a frozen aggregator with trainable points.  The frozen tensors get no
    gradient, and every other one meets the all-trainable bound against float64 (the bias and alpha-branch sums are atomic, so two
    runs are not equal bit for bit and the all-trainable run is no sharper a reference)."""
    _run_case("tiny", 16, mode=mode, freeze=freeze, bg=BG, monkeypatch=monkeypatch)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("what", ["conf", "embedding_x4"])
def test_checkpoint_value_ranges(what, mode, monkeypatch):
    """points_conf outside its clamp (the straight-through clamp passes the gradient there), and embeddings of several units."""
    edit = dict(conf=forward_check.edit_conf, embedding_x4=forward_check.edit_embedding(4.0))[what]
    _, _, info = _run_case("tiny", 16, mode=mode, edit=edit, monkeypatch=monkeypatch)
    if what == "conf":
        c = info["net"].neural_points.points_conf
        assert float(c.min()) < 0 and float(c.max()) > 1 and float(c.grad[0, :, 0][(c[0, :, 0] > 1) | (c[0, :, 0] < 0)].abs().max()) > 0
