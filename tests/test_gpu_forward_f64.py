"""GPU: every forward shading kernel, sample by sample, against float64 (oracle/shade_oracle.py, oracle/forward_check.py).

The drop-in's forward runs (net() under no_grad: the frozen pair kernel k_shade_wg<FROZEN> by default, the general one with
pnb_frozen=0, the CUDA-core kernel with pnb_precision="fp32"), then the oracle runs in float64 on the kernel's own query export with the
case's campos and camrotc2w, and each of the kernels' products is compared with no outlier allowance:
  sigma, rgb   the (sigma, rgb) of every valid sample (net._sigma_rgb); sigma relative to the case's largest |sigma|, rgb absolute;
  hbar         the K-reduced feature the pair kernel hands to the colour kernel, all 256 channels (tensor-core paths), relative to
               the case's largest |h-bar|;
  pre          every row of the frozen cloud's hoisted table pre [N][256] against b1 + W1[:, :7F] [f, PE3(f)], relative to its largest entry;
  composite    ray colour, opacity and bg_T against forward_check.march run on the kernel's own sigma_rgb (k_composite alone);
  aux          weight, conf_coefficient (against the oracle) and blend_weight (against march), absolute;
  poison       sigma_rgb and the h-bar / sigma workspace filled with NaN, the same call again: every output equal bit for bit.
The composited outputs are also held to the 1e-4 rule of the parity tests end to end, against the float64 (sigma, rgb) composited by
march (whose raydist_mode_unit choice is the reference's fp32 one: where two samples lie exactly 2 vsize_z apart in depth, float64
decides differently and moves the ray by ~3e-2).  Most cases orbit the camera
(scene.orbit_rotation), so that a transposed or ignored camera rotation shows.

Bounds per (kernel, quantity), 4-5x the largest error measured over this file's cases on an H100 80GB HBM3 at a 700 W power limit
(measured / bound):
  kernel    sigma            rgb              hbar             pre              composite        aux
  frozen    3.9e-6 / 1.8e-5  1.4e-6 / 6e-6    1.3e-5 / 6e-5    9.2e-7 / 4e-6    2.4e-6 / 1e-5    2.4e-6 / 1e-5
  general   4.6e-6 / 2e-5    1.5e-6 / 7e-6    1.3e-5 / 6e-5                     2.4e-6 / 1e-5    2.4e-6 / 1e-5
  fp32      6.7e-7 / 3e-6    1.3e-7 / 6e-7                                      2.4e-6 / 1e-5    2.4e-6 / 1e-5
The BF16x3 paths carry the split's ~1e-5 (h-bar is stored as bf16 hi + lo, ~2^-17 of each value); the largest sigma errors are at
alpha_bias -6 (softplus's exponential tail).  tests/test_forward_f64_oracle.py shows
defects that pass the 1e-4 rule and fail a per-sample check of this kind.
Section E (background, raydist_mode_unit 0, point values of a trained checkpoint; same card) stays inside this table, embeddings x10
included, except composite / aux at alpha_bias 48 in mode 0 (2.5e-5 / 1.2e-5 measured, bounds set in that test).  In mode 0 the one
choice float64 and fp32 can take differently is rd < 1e-8, which march takes in fp32 like the unit mode's.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import forward_check, grad_check, shade_oracle, shade_oracle_rw2c
from pointnerf_b200 import harness, lib, scene
from pointnerf_b200.point_query import make_cam_opts

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-4           # the end-to-end rule of the parity tests
BOUNDS = {
    "frozen": dict(sigma=1.8e-5, rgb=6e-6, hbar=6e-5, pre=4e-6, composite=1e-5, aux=1e-5),
    "general": dict(sigma=2e-5, rgb=7e-6, hbar=6e-5, composite=1e-5, aux=1e-5),
    "fp32": dict(sigma=3e-6, rgb=6e-7, composite=1e-5, aux=1e-5),
}
# point values beyond the table's (test_checkpoint_value_ranges): the entries of a kernel's row that differ there
VALUE_BOUNDS = {}
KERNELS = {"frozen": dict(), "general": dict(pnb_frozen=0), "fp32": dict(pnb_precision="fp32")}


def _forward(net, rays):
    r = {k: (None if v is None else v.to(DEV)) for k, v in rays.items()}
    with torch.no_grad():
        out = net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
                  near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])
    net.check_errors()
    return {k: v.clone() for k, v in out.items()}


def _tc_buffers(net, n_valid):
    """The h-bar operand (uint8, whole colour tiles) and sigma (float [n_valid]) of the tensor-core workspace."""
    hb, sg = C.c_void_p(), C.c_void_p()
    lib.check(lib.load().pnb_shade_tc_buffers(net._tc_ws.data_ptr(), net._tc_ws.numel(), net._max_valid, C.byref(hb), C.byref(sg)),
              "pnb_shade_tc_buffers")
    return hb.value, sg.value


def _hbar_bytes(n):
    return (n + forward_check.HBAR_TILE - 1) // forward_check.HBAR_TILE * 8 * forward_check.HBAR_BLOCK_BYTES


def _poison(net, kernel):
    """NaN in every buffer a valid sample's result passes through before compositing."""
    net._sigma_rgb.fill_(float("nan"))
    if kernel != "fp32":
        hb, sg = _tc_buffers(net, net._max_valid)
        ws = net._tc_ws
        o = hb - ws.data_ptr()
        ws[o:o + _hbar_bytes(net._max_valid)].view(torch.float32).fill_(float("nan"))
        o = sg - ws.data_ptr()
        ws[o:o + 4 * net._max_valid].view(torch.float32).fill_(float("nan"))


def _pre_errors(net, F):
    """Rows of the hoisted table against float64 b1 + W1[:, :7F] [f, PE3(f)], relative to the table's largest entry."""
    npn = net.neural_points
    N = npn.xyz.shape[0]
    pre = net._pre[:N * 256].view(N, 256).cpu().double()
    f = npn.points_embeding.detach()[0].cpu().double()
    x = torch.cat([f, shade_oracle.positional_encoding(f, 3)], dim=-1)
    w1, b1 = net.aggregator.block1[0].weight.detach().cpu().double(), net.aggregator.block1[0].bias.detach().cpu().double()
    ref = b1 + x @ w1[:, :7 * F].T
    return (pre - ref).abs().amax(-1) / ref.abs().max()


def _run(cfg_name, side=20, F=32, kernel="frozen", frames=False, order=2, rotated=True, alpha_bias=3.0, pixels=None, edit=None,
         bg=(1.0, 1.0, 1.0), bounds=None, **over):
    """bg: the background's three channels, or None (forward(bg_color=None): black).  over: options of harness.make_opt, e.g.
    raydist_mode_unit=0.  bounds: entries of the kernel's BOUNDS row replaced for this case."""
    cfg = scene.CONFIGS[cfg_name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=alpha_bias, seed=2, feat_dim=F, agg_intrp_order=order, **KERNELS[kernel],
                                        **over)
    npn = net.neural_points
    Rw = torch.eye(3)
    if frames:
        Rw = scene.edit_frames(pts["xyz"])
        npn.Rw2c = torch.nn.Parameter(Rw.to(DEV), requires_grad=False)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side) if pixels is None else pixels,
                           camrotc2w=scene.orbit_rotation() if rotated else None, bg_color=bg or (0.0, 0.0, 0.0))
    bg64 = rays["bg_color"][0].double()
    if bg is None:
        rays["bg_color"] = None
    mode_unit = opt.raydist_mode_unit
    if edit is not None:
        edit(net, rays)
    out = _forward(net, rays)
    q = net.last
    cam, campos = rays["camrotc2w"][0], rays["campos"][0]
    ex = q.export(make_cam_opts(list(q.desc.campos), cam), want_pers=False, want_dirs=False)
    smap = forward_check.sample_map(q, ex)
    S = smap["cand"].shape[0]
    hit = ex["ray_mask"].cpu() > 0
    # the kernel's products
    sr = net._sigma_rgb[:q.desc.cap_samples].cpu()[smap["cand"]]
    got = dict(sigma=sr[:, 0], rgb=sr[:, 1:])
    if kernel != "fp32":
        hb, sg = _tc_buffers(net, S)
        got["hbar"] = forward_check.decode_hbar(forward_check.dev_view(net._tc_ws, hb, torch.uint8, (_hbar_bytes(S),)), S)
        sig_ws = forward_check.dev_view(net._tc_ws, sg, torch.float32, (S,))
        assert torch.equal(sig_ws, sr[:, 0]), "the colour kernel did not pass the pair kernel's sigma through"
    # float64 oracle on the kernel's own sample geometry
    pts64 = dict(xyz=npn.xyz.detach().cpu().double(), Rw2c=Rw.double(), embedding=npn.points_embeding.detach().cpu().double(),
                 color=npn.points_color.detach().cpu().double(), dir=npn.points_dir.detach().cpu().double(),
                 conf=npn.points_conf.detach().cpu().double())
    mlp64 = {k: v.double() for k, v in harness.mlp_cpu(net.aggregator).items()}
    pidx, loc_w = ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu()
    shade = shade_oracle_rw2c.shade if frames else shade_oracle.shade
    sh = shade(pts64, mlp64, pidx, loc_w, rays["raydir"][0][hit], campos, cam, opt.vsize, bg64, dtype=torch.float64,
               agg_intrp_order=order, raydist_mode_unit=mode_unit)
    errs = forward_check.sample_errors(got, sh, smap["srow"])
    ray_errs = {}
    if kernel == "frozen":
        ray_errs["pre"] = _pre_errors(net, F)
    # the compositing kernel on the shading kernel's own (sigma, rgb)
    Rn, SR = pidx.shape[0], q.SR
    dec = torch.zeros(Rn * SR, 4, dtype=torch.float64)
    dec[smap["srow"]] = sr.double()
    m = forward_check.march(dec.view(Rn, SR, 4), sh["ray_valid"], loc_w, campos, cam, opt.vsize, bg64, raydist_mode_unit=mode_unit)
    col, op, bg = out["coarse_raycolor"][0].cpu(), out["coarse_point_opacity"][0].cpu(), out["coarse_is_background"][0].cpu()
    ray_errs["composite"] = torch.stack([(col - m["ray_color"]).abs().amax(-1), (op - m["opacity"]).abs().amax(-1),
                                         (bg - m["bg_T"]).abs().amax(-1)], -1).amax(-1)
    ray_errs["aux"] = torch.stack([(out["weight"][0].cpu() - sh["weight"]).abs().amax((-1, -2)),
                                   (out["conf_coefficient"][0].cpu() - sh["conf_coefficient"]).abs().amax((-1, -2)),
                                   (out["blend_weight"][0].cpu() - m["blend_weight"]).abs().amax((-1, -2))], -1).amax(-1)
    # end to end: the float64 oracle's (sigma, rgb), composited with the raydist_mode_unit choice taken in fp32, as the reference takes it
    m64 = forward_check.march(sh["decoded"], sh["ray_valid"], loc_w, campos, cam, opt.vsize, bg64, raydist_mode_unit=mode_unit)
    e2e = max((col - m64["ray_color"]).abs().max().item(), (op - m64["opacity"]).abs().max().item(),
              (bg - m64["bg_T"]).abs().max().item())
    # NaN in the buffers, the same call: equal bits
    _poison(net, kernel)
    out2 = _forward(net, rays)
    poisoned = [k for k in out if out[k].is_floating_point() and not torch.equal(out[k], out2[k])]
    # every comparison first (the report), then the bounds
    rep = {k: forward_check.worst(e) for k, e in list(errs.items()) + list(ray_errs.items())}
    n_bg = float(sh["bg_T"].min())
    # steps above 2 vsize_z (raydist_mode_unit 0 keeps them) and samples whose opacity is 1 in fp32
    n_long, n_sat = int((m["ray_dist"] > 2 * float(opt.vsize[2])).sum()), int((op == 1).sum())
    print("\n[fwd-f64] %s side=%d F=%d %s frames=%d order=%d rot=%d ab=%g bg=%s edit=%s %s: R'=%d of %d S=%d tiles=%d min bg_T=%.3g long=%d "
          "o==1: %d %s e2e=%.2e%s" % (
              cfg_name, side, F, kernel, frames, order, rotated, alpha_bias, bg, getattr(edit, "__name__", edit), over, Rn, hit.numel(), S,
              (S + 127) // 128, n_bg, n_long, n_sat, " ".join("%s=%.2e" % (k, v[0]) for k, v in rep.items()), e2e,
              " POISONED=%s" % poisoned if poisoned else ""))
    b = dict(BOUNDS[kernel], **(bounds or {}))
    forward_check.check(errs, {k: b[k] for k in errs}, lambda i: forward_check.describe_sample(smap, i))
    forward_check.check({k: v for k, v in ray_errs.items() if k != "pre"}, b, lambda i: "ray row %d" % i)
    if "pre" in ray_errs:
        NP = 32 if F == 32 else 16
        forward_check.check(dict(pre=ray_errs["pre"]), b, lambda i: "point %d (block %d of %d points)" % (i, i // NP, NP))
    assert e2e <= TOL, "end to end: %.3e > %.0e" % (e2e, TOL)
    assert not poisoned, "outputs differ after NaN in the shading buffers: %s" % poisoned
    smap.update(sample_pidx=pidx, hit=hit, n_long=n_long, n_sat=n_sat, rays=rays, out=out)
    return net, sh, smap


# ---- A. every forward instantiation: 16 k_shade_wg<FROZEN, O1, PP, F>, both k_color_wg<PP>, k_shade_fwd, k_point_pre<32|63>
@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("frames", [False, True])
@pytest.mark.parametrize("F", [32, 63])
@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
def test_every_instantiation(kernel, F, frames, order):
    net, sh, smap = _run("tiny", 20, F=F, kernel=kernel, frames=frames, order=order)
    assert float(sh["bg_T"].min()) < 0.9, "the case is transparent"
    if kernel == "frozen":
        assert net.neural_points.xyz.shape[0] % (32 if F == 32 else 16) != 0    # a partial last block of k_point_pre


# ---- B. edges
def _single_ray(cfg):
    return scene.centre_patch(cfg, 1)


@pytest.mark.parametrize("edge", ["K1", "K3", "SR8", "SR80", "SR128", "one_ray"])
@pytest.mark.parametrize("F", [32, 63])
@pytest.mark.parametrize("kernel", ["frozen", "general"])
def test_edges(kernel, F, edge):
    over = dict(K1=dict(K=1), K3=dict(K=3), SR8=dict(SR=8), SR80=dict(SR=80), SR128=dict(SR=128), one_ray={})[edge]
    pixels = _single_ray(scene.CONFIGS["tiny"]) if edge == "one_ray" else None
    _, sh, smap = _run("tiny", 16, F=F, kernel=kernel, pixels=pixels, **over)
    if edge == "one_ray":
        assert sh["ray_color"].shape[0] == 1 and 0 < smap["cand"].shape[0] < 128, "one hit ray, one partial colour tile"


# ---- C. many tiles
@pytest.mark.parametrize("dbg", [0, 8])
@pytest.mark.parametrize("kernel", ["frozen", "general"])
def test_chair_patch_many_tiles(kernel, dbg):
    """pnb_dbg_flags 8: one CTA per 8 SMs, so that every CTA runs many tiles and the weight ring runs across tile boundaries."""
    net, _, smap = _run("chair_plumbing", 32, kernel=kernel, pnb_dbg_flags=dbg)
    n_cta = (torch.cuda.get_device_properties(0).multi_processor_count + 7) // 8
    assert net.last.counters["n_pairs"] > 4 * 128 * n_cta and smap["cand"].shape[0] > 2 * 128 * n_cta, "too few tiles per CTA"


@pytest.mark.parametrize("rotated", [False, True])
def test_lego_centre_chunk(rotated):
    _run("lego_render", 48, kernel="frozen", rotated=rotated)


# ---- D. values
@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
@pytest.mark.parametrize("alpha_bias", [-6.0, 8.0])
def test_alpha_bias_extremes(kernel, alpha_bias):
    """-6: every sigma in softplus's exponential tail; +8: opaque after a few samples."""
    _run("tiny", 20, kernel=kernel, alpha_bias=alpha_bias)


def _edit_point_on_sample(net, rays):
    """One point moved exactly onto a sample position of a valid sample it neighbours: the 1e-6 clamp of the distance norm."""
    _forward(net, rays)
    q = net.last
    ex = q.export(make_cam_opts(list(q.desc.campos), rays["camrotc2w"][0]), want_pers=False, want_dirs=False)
    pidx, loc = ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu()
    nz = (pidx >= 0).any(-1).nonzero()
    r, s = nz[len(nz) // 2].tolist()
    p = int(pidx[r, s, 0])
    with torch.no_grad():
        net.neural_points.xyz[p] = loc[r, s].to(DEV)


@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
@pytest.mark.parametrize("what", ["conf", "point_on_sample"])
def test_value_edges(kernel, what):
    edit = dict(conf=forward_check.edit_conf, point_on_sample=_edit_point_on_sample)[what]
    net, sh, smap = _run("tiny", 20, kernel=kernel, edit=edit)
    if what == "point_on_sample":
        assert float(sh["weight"].max()) > 0.999, "no pair at distance below the clamp"
    else:
        pidx = smap["sample_pidx"]
        c = net.neural_points.points_conf[0, :, 0].detach().cpu()[pidx[pidx >= 0].long()]
        assert float(c.min()) < 0 and float(c.max()) > 1, "no pair reaches the clamp of conf_coefficient"


# ---- E. the background, raydist_mode_unit 0, and point values of a trained checkpoint
def _limb_patch(cfg, side):
    """A patch across the limb of the shell: rays that hit it and rays that miss it."""
    return scene.centre_patch(cfg, side) + np.float32([side // 2, 0])


@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
@pytest.mark.parametrize("bg", [(0.9, 0.1, 0.4), (0.0, 0.0, 0.0), None], ids=["coloured", "black", "none"])
def test_background(kernel, bg):
    """Three different channels (a channel of bg_color used for another shows), black, and forward(bg_color=None); render_full paints
    the rays that miss the cloud with the background bit for bit."""
    cfg = scene.CONFIGS["tiny"]
    net, sh, smap = _run("tiny", 20, kernel=kernel, pixels=_limb_patch(cfg, 20), bg=bg)
    hit, rays = smap["hit"], smap["rays"]
    assert 0 < int(hit.sum()) < hit.numel(), "the patch needs rays that hit and rays that miss"
    assert 0.05 < float(sh["bg_T"].min()) and float(sh["bg_T"].max()) > 0.5, "the background does not reach the hit rays' colour"
    bgl = list(bg or (0.0, 0.0, 0.0))
    with torch.no_grad():
        full = net.render_full(rays["campos"][0].tolist(), rays["raydir"].to(DEV), rays["camrotc2w"][0], cfg.near, cfg.far, bgl)
    net.check_errors()
    assert torch.equal(full["ray_mask"][0].cpu() > 0, hit)
    miss = ~hit
    assert torch.equal(full["coarse_raycolor"][0].cpu()[miss], torch.tensor(bgl, dtype=torch.float32).expand(int(miss.sum()), 3))
    assert bool((full["coarse_is_background"][0].cpu()[miss] == 1).all()) and bool((full["coarse_point_opacity"][0].cpu()[miss] == 0).all())
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):       # and on the hit rays it is forward()'s result
        assert torch.equal(full[k][0][hit.to(DEV)], smap["out"][k][0]), k


@pytest.mark.parametrize("F,alpha_bias", [(32, 3.0), (63, 3.0), (32, 8.0), (32, 48.0)])
@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
def test_raydist_mode_unit_0(kernel, F, alpha_bias):
    """The reference's default ray distances: the step from the shell's front crossing to its back crossing stays (~30 voxels, SR 80
    reaches the back).  alpha_bias 48: sigma times that step is beyond fp32's 1 - exp(-x) < 1, so those samples have opacity 1 and the
    transmittance behind them starts from the 1e-10 floor."""
    # at alpha_bias 48 sigma reaches ~45, and the fp32 rounding of a step between depths of ~4 (a few 1e-7) times sigma moves an
    # opacity by ~1e-5: composite and blend_weight are held to 4x what that case measured (2.5e-5, 1.2e-5) instead of the table's 1e-5
    bounds = dict(composite=1e-4, aux=5e-5) if alpha_bias == 48.0 else None
    _, sh, smap = _run("tiny", 16, F=F, kernel=kernel, alpha_bias=alpha_bias, SR=80, raydist_mode_unit=0, bg=(0.9, 0.1, 0.4), bounds=bounds)
    assert smap["n_long"] > 100 and float(sh["ray_dist"].max()) > 20 * 0.03, "no step above 2 vsize_z: the case is the unit mode's"
    if alpha_bias == 48.0:
        assert smap["n_sat"] > 50, "no sample with opacity 1"


@pytest.mark.parametrize("kernel", ["frozen", "general", "fp32"])
@pytest.mark.parametrize("what", ["embedding_x4", "embedding_x10", "dir", "color"])
def test_checkpoint_value_ranges(kernel, what):
    """Embeddings of several units (PE arguments 4 f of tens of radians), non-unit and zero points_dir, colours outside [0, 1]."""
    edit = dict(embedding_x4=forward_check.edit_embedding(4.0), embedding_x10=forward_check.edit_embedding(10.0),
                dir=forward_check.edit_dir, color=forward_check.edit_color)[what]
    net, sh, smap = _run("tiny", 20, kernel=kernel, edit=edit, bounds=VALUE_BOUNDS.get((what, kernel)))
    npn = net.neural_points
    if what == "dir":
        n = npn.points_dir[0].norm(dim=-1)
        assert int((n == 0).sum()) > 0 and float(n.max()) > 2.5
    elif what == "color":
        assert float(npn.points_color.min()) < -0.4 and float(npn.points_color.max()) > 1.4
    else:
        assert float(npn.points_embeding.abs().max()) > (6.0 if what == "embedding_x4" else 15.0)


# ---- F. tile boundaries: batches of exactly 127, 128 or 129 pair rows (the 128-row tile of k_shade_wg) or valid samples (the colour
# ---- tile of k_color_wg), a subset of the tiny frame's hit rays whose counts add up to the target (grad_check.pixels_for)
@pytest.mark.parametrize("count,target", [(c, t) for c in ("P", "S") for t in (127, 128, 129)])
@pytest.mark.parametrize("F", [32, 63])
@pytest.mark.parametrize("kernel", ["frozen", "general"])
def test_tile_boundaries(kernel, F, count, target):
    pixels = grad_check.pixels_for(grad_check.frame_census("tiny", rotated=True, device=DEV), count, target)
    net, _, smap = _run("tiny", 0, F=F, kernel=kernel, pixels=pixels)
    S, P = smap["cand"].shape[0], int(net.last.counters["n_pairs"])
    print("[fwd-f64 exact] %s = %d: rays=%d S=%d P=%d" % (count, target, len(pixels), S, P))
    assert (S if count == "S" else P) == target, "the batch is off its boundary: S=%d P=%d" % (S, P)
