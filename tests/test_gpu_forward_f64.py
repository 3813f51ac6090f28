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
"""
import ctypes as C

import pytest
import torch

from oracle import forward_check, shade_oracle, shade_oracle_rw2c
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
KERNELS = {"frozen": dict(), "general": dict(pnb_frozen=0), "fp32": dict(pnb_precision="fp32")}


def _forward(net, rays):
    r = {k: v.to(DEV) for k, v in rays.items()}
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
         **over):
    cfg = scene.CONFIGS[cfg_name]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=alpha_bias, seed=2, feat_dim=F, agg_intrp_order=order, **KERNELS[kernel],
                                        **over)
    npn = net.neural_points
    Rw = torch.eye(3)
    if frames:
        Rw = scene.edit_frames(pts["xyz"])
        npn.Rw2c = torch.nn.Parameter(Rw.to(DEV), requires_grad=False)
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side) if pixels is None else pixels,
                           camrotc2w=scene.orbit_rotation() if rotated else None)
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
    sh = shade(pts64, mlp64, pidx, loc_w, rays["raydir"][0][hit], campos, cam, opt.vsize, torch.ones(3), dtype=torch.float64,
               agg_intrp_order=order)
    errs = forward_check.sample_errors(got, sh, smap["srow"])
    ray_errs = {}
    if kernel == "frozen":
        ray_errs["pre"] = _pre_errors(net, F)
    # the compositing kernel on the shading kernel's own (sigma, rgb)
    Rn, SR = pidx.shape[0], q.SR
    dec = torch.zeros(Rn * SR, 4, dtype=torch.float64)
    dec[smap["srow"]] = sr.double()
    m = forward_check.march(dec.view(Rn, SR, 4), sh["ray_valid"], loc_w, campos, cam, opt.vsize, torch.ones(3))
    col, op, bg = out["coarse_raycolor"][0].cpu(), out["coarse_point_opacity"][0].cpu(), out["coarse_is_background"][0].cpu()
    ray_errs["composite"] = torch.stack([(col - m["ray_color"]).abs().amax(-1), (op - m["opacity"]).abs().amax(-1),
                                         (bg - m["bg_T"]).abs().amax(-1)], -1).amax(-1)
    ray_errs["aux"] = torch.stack([(out["weight"][0].cpu() - sh["weight"]).abs().amax((-1, -2)),
                                   (out["conf_coefficient"][0].cpu() - sh["conf_coefficient"]).abs().amax((-1, -2)),
                                   (out["blend_weight"][0].cpu() - m["blend_weight"]).abs().amax((-1, -2))], -1).amax(-1)
    # end to end: the float64 oracle's (sigma, rgb), composited with the raydist_mode_unit choice taken in fp32, as the reference takes it
    m64 = forward_check.march(sh["decoded"], sh["ray_valid"], loc_w, campos, cam, opt.vsize, torch.ones(3))
    e2e = max((col - m64["ray_color"]).abs().max().item(), (op - m64["opacity"]).abs().max().item(),
              (bg - m64["bg_T"]).abs().max().item())
    # NaN in the buffers, the same call: equal bits
    _poison(net, kernel)
    out2 = _forward(net, rays)
    poisoned = [k for k in out if out[k].is_floating_point() and not torch.equal(out[k], out2[k])]
    # every comparison first (the report), then the bounds
    rep = {k: forward_check.worst(e) for k, e in list(errs.items()) + list(ray_errs.items())}
    n_bg = float(sh["bg_T"].min())
    print("\n[fwd-f64] %s side=%d F=%d %s frames=%d order=%d rot=%d ab=%g %s: R'=%d S=%d tiles=%d min bg_T=%.3f %s e2e=%.2e%s" % (
        cfg_name, side, F, kernel, frames, order, rotated, alpha_bias, over, Rn, S, (S + 127) // 128, n_bg,
        " ".join("%s=%.2e" % (k, v[0]) for k, v in rep.items()), e2e, " POISONED=%s" % poisoned if poisoned else ""))
    b = BOUNDS[kernel]
    forward_check.check(errs, {k: b[k] for k in errs}, lambda i: forward_check.describe_sample(smap, i))
    forward_check.check({k: v for k, v in ray_errs.items() if k != "pre"}, b, lambda i: "ray row %d" % i)
    if "pre" in ray_errs:
        NP = 32 if F == 32 else 16
        forward_check.check(dict(pre=ray_errs["pre"]), b, lambda i: "point %d (block %d of %d points)" % (i, i // NP, NP))
    assert e2e <= TOL, "end to end: %.3e > %.0e" % (e2e, TOL)
    assert not poisoned, "outputs differ after NaN in the shading buffers: %s" % poisoned
    smap["sample_pidx"] = pidx
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


def _edit_conf(net, rays):
    """5 % of points_conf outside the clamp (0.0001, 1): zero, negative, tiny positive, above 1."""
    c = net.neural_points.points_conf
    N = c.shape[1]
    g = torch.Generator().manual_seed(7)
    idx = torch.randperm(N, generator=g)[:N // 20]
    vals = torch.tensor([0.0, -0.3, 5e-5, 1.7, 1.0 + 1e-3, -1e-6, 9.99e-5, 30.0])
    with torch.no_grad():
        c[0, idx.to(c.device), 0] = vals.repeat(len(idx) // len(vals) + 1)[:len(idx)].to(c.device)


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
    edit = dict(conf=_edit_conf, point_on_sample=_edit_point_on_sample)[what]
    net, sh, smap = _run("tiny", 20, kernel=kernel, edit=edit)
    if what == "point_on_sample":
        assert float(sh["weight"].max()) > 0.999, "no pair at distance below the clamp"
    else:
        pidx = smap["sample_pidx"]
        c = net.neural_points.points_conf[0, :, 0].detach().cpu()[pidx[pidx >= 0].long()]
        assert float(c.min()) < 0 and float(c.max()) > 1, "no pair reaches the clamp of conf_coefficient"
