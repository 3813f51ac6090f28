"""GPU: the fused module's shading of the perspective-frustum query (wcoord_query 0, the XSAMP instantiations of k_shade_wg frozen and
general, k_color_wg, k_shade_fwd, k_composite with and without bg_ray, k_aux_outputs, k_bwd_build, k_bwd_scatter, k_composite_bwd)
against float64, with the checks of DESIGN.md §6 items 5 and 6.  Every input comes from the module's own query (FrustumSamples: the
querier's sample_pidx, jittered sample_loc, sample_loc_w, sample_ray_dirs and vsize); the float64 side is tests/frustum_shade_f64.py.

Scenes (tests/frustum_shade_f64.frustum_scene: the rotated camera, 160 x 120 frame and DTU query options of scene.make_frustum_scene;
K 8, SR 40 unless a case says otherwise), and what each reaches over the whole frame, counted with the CPU query oracle
(frustum_shade_f64.oracle_query / reach; hit rays, capped columns, hit rays without any neighbour, valid samples whose step to the next
slot is above 2 vsize_z, valid samples with 1..8 filled K slots):
  layers              16,576 hit, 0 capped, 0 without neighbours, 33,144 gap steps (two per ray, between the three surfaces),
                      K-fill 28408 18436 14332 13116 11924 10520 9864 148560
  fog (SR 40)         16,576 hit, 289 capped, 0 without neighbours, 30,752 gap steps, K-fill 34824 24776 21476 21276 20832 20948 19984 100344
  fog (SR 128)        288 capped columns (the slab holds ~150 dilated voxels per column)
  dtu_surface_limits  18,060 hit, 0 capped, 3,677 without neighbours, 330 gap steps, K-fill 21739 11911 5804 2401 844 231 52 19
  dtu_surface         the opaque surface of tests/test_gpu_frustum_fused.py (0 capped, every hit ray has a neighbour)
Alpha biases (added to alpha_branch.0's bias, seed-5 MLP): translucent +8 (largest opacity 0.046 on layers, every valid sample carries
weight, mean bg_T 0.68), saturated +3000 (opacity exactly 1.0 in fp32 on ~100 slots of layers at pixels [::61]), opaque +300.
tests/test_oracle_frustum_fused.py asserts these counts on the CPU.

  per sample   (sigma, rgb) of every valid sample and h-bar (pnb_shade_tc_buffers, forward_check.decode_hbar), for the frozen, general
               and fp32 kernels and agg_intrp_order 2 and 1, within DESIGN §6 item 6's table (BOUNDS)
  composite    ray colour, per-slot opacity and bg_T of k_composite on the kernel's own sigma_rgb against frustum_shade_f64.march in
               float64 (background coloured, black, None; bg_ray through render_full; a jittered training forward at two seeds)
  aux          weight and conf_coefficient (against the oracle) and blend_weight (against march) per pair
  edges        K 1 / 3 / 8, SR 1 / 8 / 33 / 128, kernel and query size 5 5 5, a point at a sample's exact position, conf outside its
               clamp, embeddings x10, the frozen kernel with one CTA per 8 SMs
  poison       NaN in sigma_rgb and the h-bar / sigma workspace, the same call again: every output equal bit for bit
  gradients    colour with the bg_ray formula + zero_one on conf_coefficient + a seeded weight on coarse_point_opacity, against float64
               autograd with the backward's own LeakyReLU masks, oracle/grad_check.RTOL with no outlier allowance; for alpha_branch.0
               with agg_intrp_order 1 (a sum over samples whose terms cancel) the report adds sum |terms| / max |grad| and the error
               relative to each entry's sum |terms| (grad_check.sum_error)
The end-to-end 1e-4 rule of the parity tests holds too.  The file prints its errors (pytest -s).
"""
import numpy as np
import pytest
import torch

import frustum_shade_f64
from oracle import forward_check, grad_check
from pointnerf_b200 import harness, scene
from pointnerf_b200.ray_marching import NeuralPoints, NeuralPointsRayMarching, PointAggregator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = 1e-4                      # the end-to-end rule of the parity tests
BIAS = dict(translucent=8.0, saturated=3000.0, opaque=300.0)
COLOURED = (0.9, 0.1, 0.4)
KERNELS = {"frozen": dict(), "general": dict(pnb_frozen=0), "fp32": dict(pnb_precision="fp32")}
# DESIGN.md §6 item 6 (tests/test_gpu_forward_f64.py's BOUNDS): sigma and h-bar relative to the case's largest, the rest absolute
BOUNDS = {
    "frozen": dict(sigma=1.8e-5, rgb=6e-6, hbar=6e-5, composite=1e-5, aux=1e-5),
    "general": dict(sigma=2e-5, rgb=7e-6, hbar=6e-5, composite=1e-5, aux=1e-5),
    "fp32": dict(sigma=3e-6, rgb=6e-7, composite=1e-5, aux=1e-5),
}


def _pixels(name):
    s = frustum_shade_f64.frustum_scene(name)[1]
    if name == "fog":
        return np.concatenate([frustum_shade_f64.fog_pixels(3), s["pixel_idx"][::97]])
    return s["pixel_idx"][::61]


def _net(name, bias, order=2, kernel="frozen", is_train=False, qover=None, **over):
    cfg, _, pts = frustum_shade_f64.frustum_scene(name)
    fo = vars(scene.frustum_opt(cfg, is_train=is_train, **(qover or {})))
    opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, agg_intrp_order=order, **fo)
    for k, v in dict(KERNELS[kernel], **over).items():
        setattr(opt, k, v)
    agg = PointAggregator(opt, seed=5)
    with torch.no_grad():
        agg.alpha_branch[0].bias += bias
    npn = NeuralPoints(opt, DEV)
    npn.set_points(pts["xyz"].to(DEV), pts["embedding"].to(DEV), points_color=pts["color"].to(DEV), points_dir=pts["dir"].to(DEV),
                   points_conf=pts["conf"].to(DEV), parameter=True, as_stored=True)
    return NeuralPointsRayMarching(aggregator=agg.to(DEV), neural_points=npn, opt=opt), opt


def _data(name, pixels, bg):
    """The input dict of a reference dataset item for these pixels (directions through the pixel centres); bg None: bg_color=None."""
    cfg, s, _ = frustum_shade_f64.frustum_scene(name)
    pix = np.asarray(pixels).reshape(-1, 2)
    K = s["intrinsic"]
    d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ s["camrotc2w"].T
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    return dict(campos=torch.from_numpy(s["campos"]).to(DEV)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(DEV)[None],
                raydir=torch.from_numpy(d.astype(np.float32)).to(DEV)[None], pixel_idx=torch.from_numpy(pix.astype(np.int32)).to(DEV)[None],
                h=cfg.H, w=cfg.W, intrinsic=s["intrinsic"], near=cfg.near, far=cfg.far,
                bg_color=None if bg is None else torch.tensor(bg, dtype=torch.float32, device=DEV))


def _forward(net, d, **kw):
    return net(d["campos"], d["raydir"], bg_color=d["bg_color"], camrotc2w=d["camrotc2w"], pixel_idx=d["pixel_idx"], near=d["near"],
               far=d["far"], h=d["h"], w=d["w"], intrinsic=d["intrinsic"], **kw)


def _points_cpu(net, grad=False):
    npn = net.neural_points
    pts = dict(xyz=npn.xyz.detach().cpu(), embedding=npn.points_embeding.detach().cpu(), color=npn.points_color.detach().cpu(),
               dir=npn.points_dir.detach().cpu(), conf=npn.points_conf.detach().cpu(), Rw2c=torch.eye(3))
    if grad:
        pts = {k: (v.double().requires_grad_(True) if k in ("embedding", "color", "dir", "conf") else v) for k, v in pts.items()}
    return pts


def _tup(q):
    return [t.detach().cpu() for t in (q.sample_pidx, q.sample_loc, q.sample_loc_w, q.sample_ray_dirs)]


def _shade64(net, q, d, order, bg, pts=None, mlp=None, slopes=None):
    pidx, loc, loc_w, dirs = _tup(q)
    return frustum_shade_f64.shade(_points_cpu(net) if pts is None else pts, harness.mlp_cpu(net.aggregator) if mlp is None else mlp,
                                   pidx, loc, loc_w, dirs, d["campos"].cpu(), d["camrotc2w"].cpu(), q.vsize,
                                   torch.tensor(bg or (0.0, 0.0, 0.0), dtype=torch.float64), dtype=torch.float64,
                                   agg_intrp_order=order, slopes=slopes)


def _valid_list(q):
    S = int(q.counters["n_valid"])
    vlist = forward_check.dev_view(q.ws, q.desc.valid_list, torch.int32, (S,)).long()
    valid = (q.sample_pidx >= 0).any(-1).cpu().reshape(-1)
    assert torch.equal(torch.sort(vlist)[0], valid.nonzero()[:, 0]), "valid_list is not the valid [R',SR] slots"
    return vlist


def _tc_buffers(net):
    import ctypes as C
    from pointnerf_b200 import lib
    hb, sg = C.c_void_p(), C.c_void_p()
    lib.check(lib.load().pnb_shade_tc_buffers(net._tc_ws.data_ptr(), net._tc_ws.numel(), net._max_valid, C.byref(hb), C.byref(sg)),
              "pnb_shade_tc_buffers")
    return hb.value, sg.value


def _hbar_bytes(n):
    return (n + forward_check.HBAR_TILE - 1) // forward_check.HBAR_TILE * 8 * forward_check.HBAR_BLOCK_BYTES


def _poison(net, kernel):
    net._sigma_rgb.fill_(float("nan"))
    if kernel != "fp32":
        hb, sg = _tc_buffers(net)
        ws = net._tc_ws
        o = hb - ws.data_ptr()
        ws[o:o + _hbar_bytes(net._max_valid)].view(torch.float32).fill_(float("nan"))
        o = sg - ws.data_ptr()
        ws[o:o + 4 * net._max_valid].view(torch.float32).fill_(float("nan"))


def _composite_errors(col, op, bg_T, m):
    """Per ray: the largest |difference| of colour, per-slot opacity and bg_T against a march() dict."""
    return torch.stack([(col.cpu() - m["ray_color"]).abs().amax(-1), (op.cpu() - m["opacity"]).abs().amax(-1),
                        (bg_T.cpu().reshape(-1, 1) - m["bg_T"]).abs().amax(-1)], -1).amax(-1)


def _run(name, bias_name, kernel="frozen", order=2, pixels=None, bg=COLOURED, edit=None, train_seed=None, qover=None, **over):
    """One forward and every forward check of this file.  train_seed: a training forward (jittered samples, the general kernel) drawn
    after torch.manual_seed(train_seed).  Returns (net, q, ref, report)."""
    net, opt = _net(name, BIAS[bias_name], order, kernel, is_train=train_seed is not None, qover=qover, **over)
    if edit is not None:
        edit(net, name)
    d = _data(name, _pixels(name) if pixels is None else pixels, bg)
    if train_seed is None:
        with torch.no_grad():
            out = _forward(net, d)
    else:
        torch.manual_seed(train_seed)
        out = _forward(net, d)
    out = {k: v.detach().clone() for k, v in out.items()}
    net.check_errors()
    q = net.last
    R2, SR = q.R2, q.SR
    vlist = _valid_list(q)
    S = vlist.shape[0]
    # the kernels' products
    sr = net._sigma_rgb[:R2 * SR].detach().cpu()
    got = dict(sigma=sr[vlist, 0], rgb=sr[vlist, 1:])
    if kernel != "fp32" and S > 0:
        hb, sg = _tc_buffers(net)
        got["hbar"] = forward_check.decode_hbar(forward_check.dev_view(net._tc_ws, hb, torch.uint8, (_hbar_bytes(S),)), S)
        assert torch.equal(forward_check.dev_view(net._tc_ws, sg, torch.float32, (S,)), got["sigma"]), \
            "the colour kernel did not pass the pair kernel's sigma through"
    ref = _shade64(net, q, d, order, bg)
    errs = forward_check.sample_errors(got, ref, vlist) if S > 0 else {}
    # k_composite on the kernel's own (sigma, rgb), in float64 with the frustum ray distances
    loc = q.sample_loc.detach().cpu()
    bg64 = torch.tensor(bg or (0.0, 0.0, 0.0), dtype=torch.float64)
    dec = torch.zeros(R2 * SR, 4, dtype=torch.float64)
    dec[vlist] = sr[vlist].double()
    m = frustum_shade_f64.march(dec.view(R2, SR, 4), ref["ray_valid"], loc, q.vsize, bg64)
    col, op, bgT = out["coarse_raycolor"][0], out["coarse_point_opacity"][0], out["coarse_is_background"][0]
    ray_errs = dict(composite=_composite_errors(col, op, bgT, m))
    ray_errs["aux"] = torch.stack([(out["weight"][0].cpu() - ref["weight"]).abs().amax((-1, -2)),
                                   (out["conf_coefficient"][0].cpu() - ref["conf_coefficient"]).abs().amax((-1, -2)),
                                   (out["blend_weight"][0].cpu() - m["blend_weight"]).abs().amax((-1, -2))], -1).amax(-1)
    m64 = frustum_shade_f64.march(ref["decoded"], ref["ray_valid"], loc, q.vsize, bg64)
    e2e = float(_composite_errors(col, op, bgT, m64).max())
    poisoned = []
    if train_seed is None:
        _poison(net, kernel)
        with torch.no_grad():
            out2 = _forward(net, d)
        net.check_errors()
        poisoned = [k for k in out if out[k].is_floating_point() and not torch.equal(out[k], out2[k])]
    rep = {k: forward_check.worst(e) for k, e in list(errs.items()) + list(ray_errs.items())}
    valid = ref["ray_valid"]
    info = dict(R2=R2, S=S, n_nonb=int((~valid.any(-1)).sum()), n_sat=int((op == 1).sum()), max_op=float(op.max()),
                mean_bgT=float(bgT.mean()), capped=net.neural_points.querier.last_build_counters.get("n_col_capped"))
    print("\n[frustum f64] %s %s %s order %d bg=%s edit=%s train=%s %s %s: %s | %s e2e=%.2e%s" % (
        name, bias_name, kernel, order, bg, getattr(edit, "__name__", edit), train_seed, qover or "", over,
        " ".join("%s=%s" % kv for kv in info.items()), " ".join("%s=%.2e" % (k, v[0]) for k, v in rep.items()), e2e,
        " POISONED=%s" % poisoned if poisoned else ""))
    b = BOUNDS[kernel if train_seed is None else "general"]
    smap = dict(ray=vlist // SR, slot=vlist % SR, nnb=(q.sample_pidx.cpu().reshape(-1, q.K)[vlist] >= 0).sum(-1))
    forward_check.check(errs, {k: b[k] for k in errs}, lambda i: forward_check.describe_sample(smap, i))
    forward_check.check(ray_errs, b, lambda i: "ray row %d" % i)
    assert e2e <= TOL, "end to end: %.3e > %.0e" % (e2e, TOL)
    assert not poisoned, "outputs differ after NaN in the shading buffers: %s" % poisoned
    return net, q, ref, dict(info, out=out, d=d)


# ------------------------------------------------------------------------------------------------ every kernel on every scene
CASES = [("layers", "translucent"), ("layers", "saturated"), ("dtu_surface_limits", "translucent"), ("fog", "translucent")]


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("name,bias_name", CASES, ids=["%s-%s" % c for c in CASES])
def test_per_sample_composite_aux(name, bias_name, kernel, order):
    _, q, ref, info = _run(name, bias_name, kernel, order)
    if bias_name == "translucent":
        assert info["max_op"] < 0.1 and info["mean_bgT"] > 0.3, "the case is not translucent"
    else:
        assert info["n_sat"] > 20, "no slot with opacity 1 in fp32"
    if name == "dtu_surface_limits":
        assert info["n_nonb"] > 10, "no hit ray without neighbours"
    if name == "fog":
        assert info["capped"] > 0, "no capped column"


# ------------------------------------------------------------------------------------------------ background, bg_ray, jitter
@pytest.mark.parametrize("bg", [COLOURED, (0.0, 0.0, 0.0), None], ids=["coloured", "black", "none"])
@pytest.mark.parametrize("kernel", list(KERNELS))
def test_background(kernel, bg):
    _run("layers", "translucent", kernel, bg=bg)


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_bg_ray_composite(kernel):
    """k_composite with bg_ray (render_full): bg_T * bg_ray + colour on a hit ray within the composite bound of float64 on the kernel's
    own (sigma, rgb), bg_ray bit for bit on a miss."""
    name = "dtu_surface_limits"
    net, _ = _net(name, BIAS["translucent"], 2, kernel)
    d = _data(name, frustum_shade_f64.frustum_scene(name)[1]["pixel_idx"][::37], COLOURED)
    R = d["pixel_idx"].shape[1]
    bg_ray = torch.rand((1, R, 3), generator=torch.Generator().manual_seed(11)).to(DEV)
    with torch.no_grad():
        full = net.render_full(d["campos"], d["raydir"], d["camrotc2w"], d["near"], d["far"], torch.ones(3), bg_ray=bg_ray,
                               view={k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")})
    net.check_errors()
    q = net.last
    vlist = _valid_list(q)
    sr = net._sigma_rgb[:q.R2 * q.SR].cpu()
    dec = torch.zeros(q.R2 * q.SR, 4, dtype=torch.float64)
    dec[vlist] = sr[vlist].double()
    valid = (q.sample_pidx >= 0).any(-1).cpu()
    m = frustum_shade_f64.march(dec.view(q.R2, q.SR, 4), valid, q.sample_loc.cpu(), q.vsize, torch.zeros(3, dtype=torch.float64))
    hit = full["ray_mask"][0].cpu() > 0
    bgr = bg_ray[0].cpu().double()
    m["ray_color"] = m["ray_color"] + m["bg_T"] * bgr[hit]
    e = float(_composite_errors(full["coarse_raycolor"][0].cpu()[hit], full["coarse_point_opacity"][0].cpu()[hit],
                                full["coarse_is_background"][0].cpu()[hit], m).max())
    print("\n[frustum f64] bg_ray %s: R'=%d of %d, mean bg_T %.3f, composite %.2e" % (kernel, q.R2, R, float(m["bg_T"].mean()), e))
    assert 0 < int(hit.sum()) < R
    assert torch.equal(full["coarse_raycolor"][0][~hit.to(DEV)], bg_ray[0][~hit.to(DEV)])
    assert e <= BOUNDS[kernel]["composite"], e


@pytest.mark.parametrize("seed", [123, 7])
def test_jittered_training_forward(seed):
    """is_train with uniform jitter: sample_loc[..., 2] moves by up to vsize_z/2, so the steps between consecutive valid slots range
    over (0, 2) voxels and the > 2 vsize_z choice acts on non-uniform steps (the cumulative maximum never acts on a valid slot: the
    only backward step is into the first empty slot); the general kernel of a training step against float64 on the jittered tuple."""
    _, q, _, _ = _run("layers", "translucent", "general", train_seed=seed)
    z = q.sample_loc[..., 2].cpu()
    both = ((q.sample_pidx[:, 1:] >= 0).any(-1) & (q.sample_pidx[:, :-1] >= 0).any(-1)).cpu()
    step = (z[:, 1:] - z[:, :-1])[both] / float(q.vsize[2])          # between consecutive valid slots: (0, 2) voxels with the jitter
    assert float(step.min()) < 0.25 and 1.75 < float(step[step <= 2].max()) <= 2, "the jitter did not make the steps non-uniform"


# ------------------------------------------------------------------------------------------------ edges
def _edit_point_on_sample(net, name):
    """One point moved exactly onto the world position of a valid sample it neighbours (the 1e-6 clamp of the distance norm)."""
    d = _data(name, _pixels(name), COLOURED)
    with torch.no_grad():
        _forward(net, d)
    q = net.last
    pidx, loc_w = q.sample_pidx.cpu(), q.sample_loc_w.cpu()
    nz = (pidx >= 0).any(-1).nonzero()
    r, s = nz[len(nz) // 2].tolist()
    with torch.no_grad():
        net.neural_points.xyz[int(pidx[r, s, 0])] = loc_w[r, s].to(DEV)


def _edit_conf(net, name):
    forward_check.edit_conf(net)


def _edit_embedding_x10(net, name):
    forward_check.edit_embedding(10.0)(net)


EDGES = dict(K1=dict(qover=dict(K=1)), K3=dict(qover=dict(K=3)), SR1=dict(qover=dict(SR=1)), SR8=dict(qover=dict(SR=8)),
             SR33=dict(name="fog", qover=dict(SR=33)), SR128=dict(name="fog", qover=dict(SR=128), pixels=frustum_shade_f64.fog_pixels(4)),
             ks555=dict(qover=dict(kernel_size=[5, 5, 5], query_size=[5, 5, 5])), point_on_sample=dict(edit=_edit_point_on_sample),
             conf=dict(edit=_edit_conf), embedding_x10=dict(edit=_edit_embedding_x10))


@pytest.mark.parametrize("kernel", list(KERNELS))
@pytest.mark.parametrize("edge", list(EDGES))
def test_edges(edge, kernel):
    e = dict(EDGES[edge])
    name = e.pop("name", "layers")
    net, q, ref, info = _run(name, "translucent", kernel, **e)
    if edge == "point_on_sample":
        pidx, loc_w = q.sample_pidx.cpu(), q.sample_loc_w.cpu().double()
        xyz = net.neural_points.xyz.detach().cpu().double()
        pm = pidx >= 0
        dist = (xyz[pidx[pm].long()] - loc_w[:, :, None, :].expand(-1, -1, pidx.shape[-1], -1)[pm]).norm(dim=-1)
        assert float(dist.min()) < 1e-6, "no pair at distance below the clamp of the distance norm"
    elif edge == "conf":
        pidx = q.sample_pidx.cpu()
        c = net.neural_points.points_conf[0, :, 0].detach().cpu()[pidx[pidx >= 0].long()]
        assert float(c.min()) < 0 and float(c.max()) > 1, "no pair reaches the clamp of conf_coefficient"
    elif edge == "SR128":
        assert info["capped"] > 0 and int((ref["ray_valid"].sum(-1) == 128).sum()) > 0, "no column capped at SR 128"
    elif edge == "SR33":
        assert info["capped"] > 0


def test_frozen_many_tiles():
    """pnb_dbg_flags 8: one CTA per 8 SMs, so that every CTA of the frozen pair kernel runs many tiles."""
    net, q, _, _ = _run("layers", "translucent", "frozen", pixels=frustum_shade_f64.frustum_scene("layers")[1]["pixel_idx"][::11],
                        pnb_dbg_flags=8)
    n_cta = (torch.cuda.get_device_properties(0).multi_processor_count + 7) // 8
    assert q.counters["n_pairs"] > 4 * 128 * n_cta and q.counters["n_valid"] > 2 * 128 * n_cta, "too few tiles per CTA"


# ------------------------------------------------------------------------------------------------ gradients
def _zero_one(cc, eps=1e-3):
    """The zero_one loss on conf_coefficient (models/base_rendering_model.py:629-641)."""
    val = torch.clamp(cc, eps, 1 - eps)
    return torch.mean(torch.log(val) + torch.log(1 - val))


def _loss(col, bg_T, op, cc, bg_ray, gt, w_op):
    """The model shell's fill_invalid with bg_ray on the hit rays, the colour loss, zero_one on conf_coefficient and a seeded weight on
    every slot's opacity."""
    full = bg_T * bg_ray + col
    return ((full - gt) ** 2).sum() + 1e-3 * _zero_one(cc) + (op * w_op).sum()


GRAD_CASES = [("layers", "translucent"), ("dtu_surface_limits", "translucent"), ("dtu_surface", "opaque")]


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("precision,mode", [("bf16x3", 0), ("bf16x3", 4), ("bf16x3", 1), ("fp32", 0), ("fp32", 1)])
@pytest.mark.parametrize("name,bias_name", GRAD_CASES, ids=["%s-%s" % c for c in GRAD_CASES])
def test_gradients_match_float64_autograd(name, bias_name, precision, mode, order):
    _gradient_case(name, bias_name, precision, mode, order)


@pytest.mark.parametrize("precision,mode", [("bf16x3", 0), ("bf16x3", 4), ("bf16x3", 1)])
def test_gradients_one_hit_ray(precision, mode):
    """A batch of one hit ray (the centre pixel of layers: 14 valid samples on three surfaces): k_bwd_build<..., XSAMP> with one warp
    busy, and every backward GEMM and slab on one partial tile or slab, against float64 as above."""
    q = _gradient_case("layers", "translucent", precision, mode, 2, pixels=np.array([[80, 60]], np.int32))
    assert q.R2 == 1 and 8 < int(q.counters["n_valid"]) < 128, (q.R2, int(q.counters["n_valid"]))


def _gradient_case(name, bias_name, precision, mode, order, pixels=None):
    """One training step of the frustum module on the scene's pixels (or `pixels`), its gradients against float64 autograd with the
    backward's own masks.  Returns the query."""
    net, opt = _net(name, BIAS[bias_name], order, "fp32" if precision == "fp32" else "general", is_train=True, pnb_bwd_fp32=mode)
    d = _data(name, _pixels(name) if pixels is None else pixels, None)
    R = d["pixel_idx"].shape[1]
    g = torch.Generator().manual_seed(3)
    bg_ray = torch.rand((1, R, 3), generator=g)
    torch.manual_seed(29)
    out = _forward(net, d, bg_ray=bg_ray.to(DEV))
    q = net.last
    hit = torch.nonzero(out["ray_mask"][0].cpu())[:, 0]
    gt = torch.rand((q.R2, 3), generator=g)
    w_op = torch.rand((q.R2, q.SR), generator=g) - 0.5
    L = _loss(out["coarse_raycolor"][0], out["coarse_is_background"][0], out["coarse_point_opacity"][0], out["conf_coefficient"][0],
              bg_ray[0][hit].to(DEV), gt.to(DEV), w_op.to(DEV))
    L.backward()
    net.check_errors()
    slopes = frustum_shade_f64.kernel_slopes(net, q)
    # float64 autograd with the kernel's masks
    pts = _points_cpu(net, grad=True)
    mlp = {k: v.detach().cpu().double().requires_grad_(True) for k, v in net.aggregator.state_dict().items()}
    with frustum_shade_f64.recording_softplus() as rec:
        ref = _shade64(net, q, d, order, None, pts=pts, mlp=mlp, slopes=slopes)
    _loss(ref["ray_color"], ref["bg_T"], ref["opacity"], ref["conf_coefficient"], bg_ray[0][hit].double(), gt.double(),
          w_op.double()).backward()
    npn = net.neural_points
    rt = grad_check.RTOL[(mode, precision)]
    got = dict(emb=npn.points_embeding.grad.cpu(), color=npn.points_color.grad.cpu(), dir=npn.points_dir.grad.cpu())
    want = dict(emb=pts["embedding"].grad, color=pts["color"].grad, dir=pts["dir"].grad)
    errs = {k: float(grad_check.rel_point_errors(got[k], want[k]).max()) for k in got}
    errs["conf"] = float(grad_check.rel_point_errors(npn.points_conf.grad.cpu()[0, 1:], pts["conf"].grad[0, 1:]).max())
    params = dict(net.aggregator.named_parameters())
    mlp_errs = {k: grad_check.rel_error(p.grad.cpu(), mlp[k].grad) for k, p in params.items()}
    cond, sum_errs = {}, {}
    if order == 1:
        for k, t in frustum_shade_f64.alpha_branch_abs_terms(rec, ref["hbar"]).items():
            cond[k] = float(t.max() / mlp[k].grad.abs().max())
            sum_errs[k] = grad_check.sum_error(params[k].grad.cpu(), mlp[k].grad, t)
    worst = max(mlp_errs, key=mlp_errs.get)
    print("\n[frustum f64 grads] %s %s %s/%d order %d: R'=%d S=%d mean bg_T %.3f points %s | MLP worst %s %.2e, alpha_branch.0 %s%s" % (
        name, bias_name, precision, mode, order, q.R2, int(q.counters["n_valid"]), float(out["coarse_is_background"].mean()),
        " ".join("%s=%.2e" % kv for kv in errs.items()), worst, mlp_errs[worst],
        " ".join("%s=%.2e" % (k[15:], mlp_errs[k]) for k in ("alpha_branch.0.weight", "alpha_branch.0.bias")),
        (" of sum|terms| " + " ".join("%s=%.2e" % (k[15:], v) for k, v in sum_errs.items()) +
         " sum|terms|/max|grad| " + " ".join("%s=%.1f" % (k[15:], v) for k, v in cond.items())) if cond else ""))
    for k in got:
        grad_check.check_points(got[k], want[k], "points_" + k, rt[0])
    grad_check.check_conf(npn.points_conf.grad.cpu(), pts["conf"].grad, int((q.sample_pidx <= 0).sum()), rt[0])
    # the opaque surface is held to grad_check.FRUSTUM_MLP_RTOL, as the other frustum files hold it; the translucent scenes to RTOL
    b_mlp = grad_check.FRUSTUM_MLP_RTOL[(mode, precision)] if bias_name == "opaque" else rt[1]
    for k, e in sum_errs.items():
        b = grad_check.ALPHA1_SUM_RTOL[(mode, precision)]
        assert e <= b, "aggregator.%s: %.3e of sum |terms| > %.1e" % (k, e, b)
    for k, e in mlp_errs.items():
        assert e <= b_mlp, "aggregator.%s: %.3e > %.1e" % (k, e, b_mlp)
    assert npn.xyz.grad is None
    return q
