"""GPU: the fused module in Point-NeRF's feed-forward mode (run/train.py --feedforward 1, the two dev_scripts/ete scripts): a new point
cloud from the network on every call, installed as plain tensors by the reference's NeuralPoints.set_points(parameter=False), whose
embedding and colour are non-leaf outputs of an upstream network that must receive their gradients.

The upstream network is a seeded stand-in U(theta) mapping fixed per-point inputs to (embedding, colour) in each script's
configuration:
  F 32   world query flavour 1 (wcoord_query 1), SR 40, K 8, kernel 5^3, P 20, vsize 0.002, point modes "1"
         (dtu_dgt_d012_img0123_conf_agg2_32_dirclr20): embedding and colour differentiable, dir and conf not
  F 63   the perspective-frustum query (wcoord_query 0), SR 40, kernel 3^3, point modes "01" (..._conf_color_dir_agg2): set_points
         prepends colour, dir and conf to the 56 upstream channels and keeps them as separate tensors, so U's colour reaches the
         module twice and its gradient is the sum of both paths

  gradients     theta's gradient against float64 autograd through the oracle (oracle/shade_oracle_rw2c.py on the world query's export,
                tests/frustum_shade_f64.py on the frustum querier's tuple), fed by U in float64, with the backward's own LeakyReLU
                masks; every backward mode (pnb_bwd_fp32 0 / 4 / 1) and agg_intrp_order 2 and 1.  The MLP tensors meet
                MLP_RTOL (the existing bounds of each query's checks), theta THETA_RTOL (no outlier allowance)
  fresh clouds  five training steps, each on a new cloud installed without clean_up() (as the reference's set_points does), one of them
                with the previous cloud's size at the previous cloud's address: one build per cloud, the forward and render_full bit
                for bit a freshly built module's, and a chunk loop over the cloud builds nothing more
  eval          model.test()-style chunks, each with a new cloud, on the frozen kernel, bit for bit a fresh module's
The file prints the errors it measures (pytest -s).
"""
import ctypes
import functools

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

import frustum_shade_f64
from oracle import forward_check, grad_check, shade_oracle_rw2c
from pointnerf_b200 import harness, lib, scene
from pointnerf_b200.ray_marching import NeuralPoints, NeuralPointsRayMarching, PointAggregator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# theta's bound per backward mode (pnb_bwd_fp32), relative to the largest |d theta| of each tensor: 4-5x the largest error measured
# over this file's cases on an H100 80GB HBM3 at a 700 W power limit: modes 0 and 4 1.76e-5 (F 63), mode 1 2.69e-6 (F 63)
THETA_RTOL = {0: 8e-5, 4: 8e-5, 1: 1.2e-5}
# the MLP tensors: the existing bounds of each query's gradient checks.  World query: oracle/grad_check.RTOL's tensor-core bound in
# every mode (measured here: modes 0 / 4 3.1e-5; mode 1 6.6e-6, above that table's mode-1 bound of 5e-6 measured on the tiny scene).
# Frustum query: oracle/grad_check.FRUSTUM_MLP_RTOL, as tests/test_gpu_frustum_fused.py; alpha_branch.0 with agg_intrp_order 1 is
# held by grad_check.ALPHA1_RTOL and ALPHA1_SUM_RTOL (its per-sample terms cancel on the opaque surface).
MLP_RTOL = {32: {m: grad_check.RTOL[(0, "bf16x3")][1] for m in (0, 4, 1)}, 63: {m: grad_check.FRUSTUM_MLP_RTOL[(m, "bf16x3")] for m in (0, 4, 1)}}
# the F 32 script's query options (vsize 0.002, kernel 5^3, P 20, SR 40, K 8) on a small shell that the 64x64 camera sees whole
CFG32 = scene.SceneConfig("ete_32", N=20_000, R_s=0.1, vsize=0.002, kernel_size=5, P=20, SR=40, H=64, W=64, near=0.3, far=1.1,
                          campos=(0.0, 0.0, -0.5))
N_IN = 8          # per-point inputs of the stand-in network
CHUNK = 2304


# ------------------------------------------------------------------------------------------------ the upstream stand-in U(theta)
def make_theta(n_emb, seed=7):
    g = torch.Generator().manual_seed(seed)
    th = dict(w1=torch.randn(32, N_IN, generator=g) / N_IN ** 0.5, b1=0.1 * torch.randn(32, generator=g),
              we=torch.randn(n_emb, 32, generator=g) * (0.5 / 32 ** 0.5), be=0.1 * torch.randn(n_emb, generator=g),
              wc=torch.randn(3, 32, generator=g) / 32 ** 0.5, bc=0.1 * torch.randn(3, generator=g))
    return {k: v.to(DEV).requires_grad_(True) for k, v in th.items()}


def upstream(th, x):
    """U(theta): per-point inputs x [N, N_IN] -> embedding [1,N,n_emb], colour [1,N,3] (both contiguous non-leaf tensors)."""
    h = torch.tanh(Fn.linear(x, th["w1"], th["b1"]))
    return Fn.linear(h, th["we"], th["be"])[None], torch.sigmoid(Fn.linear(h, th["wc"], th["bc"]))[None]


def ref_set_points(npn, xyz, emb, color, pdir, conf):
    """The reference's NeuralPoints.set_points(..., parameter=False) (neural_points.py:444-467): plain assignments, no clean_up() of
    the querier; a mode with "0" prepends its tensor to the embedding (conf, then dir, then colour), one with "1" keeps it."""
    o = npn.opt
    npn.xyz = xyz
    for name, t, mode in (("points_conf", conf, o.point_conf_mode), ("points_dir", pdir, o.point_dir_mode),
                          ("points_color", color, o.point_color_mode)):
        if "0" in mode:
            emb = torch.cat([t, emb], dim=-1)
        if "1" in mode:
            setattr(npn, name, t)
    npn.points_embeding = emb
    npn.Rw2c = torch.eye(3, device=xyz.device)


# ------------------------------------------------------------------------------------------------ the two configurations
@functools.lru_cache(None)
def _frustum_scene():
    cfg = scene.FRUSTUM_CONFIGS["dtu_surface"]
    s = scene.make_frustum_scene(cfg)
    return cfg, s, scene.make_frustum_points(cfg, s)


class Setup:
    """One script's configuration: the module, its fixed per-point inputs (xyz, dir, conf, U's input x) and the rays."""

    def __init__(self, F, mode=0, order=2, precision="bf16x3"):
        self.F = F
        extra = dict(agg_intrp_order=order, pnb_bwd_fp32=mode, pnb_precision=precision)
        if F == 32:
            self.opt = harness.make_opt(CFG32, wcoord_query=1, **extra)
            pts = scene.make_points(CFG32)
            self.alpha_bias = 3.0
            self.xyz, self.dir, self.conf = pts["xyz"].to(DEV), pts["dir"].to(DEV), pts["conf"].to(DEV)
        else:
            cfg, s, pts = _frustum_scene()
            self.opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, **vars(scene.frustum_opt(cfg)), **extra)
            self.alpha_bias = 300.0          # an opaque surface: the frustum scene's depth voxels are 0.0068 long
            self.xyz, self.dir, self.conf = pts["xyz"].to(DEV), pts["dir"].to(DEV), pts["conf"].to(DEV)
        self.N = self.xyz.shape[0]
        self.x = torch.randn(self.N, N_IN, generator=torch.Generator().manual_seed(3)).to(DEV)
        self.n_emb = 32 if F == 32 else 56
        self.agg = self.aggregator()

    def aggregator(self):
        agg = PointAggregator(self.opt, seed=2)
        with torch.no_grad():
            agg.alpha_branch[0].bias += self.alpha_bias
        return agg.to(DEV)

    def net(self, agg=None):
        npn = NeuralPoints(self.opt, DEV)
        return NeuralPointsRayMarching(aggregator=self.agg if agg is None else agg, neural_points=npn, opt=self.opt)

    def rays(self, sel):
        """The input dict of forward() for the rays `sel` (F 32: a centre patch side, None for the frame; F 63: a pixel stride of the
        frame)."""
        if self.F == 32:
            r = scene.make_rays(CFG32, None if sel is None else scene.centre_patch(CFG32, sel))
            return {k: v.to(DEV) for k, v in r.items()}
        cfg, s, _ = _frustum_scene()
        pix = s["pixel_idx"][::sel]
        K = s["intrinsic"]
        d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ s["camrotc2w"].T
        d = d / np.linalg.norm(d, axis=-1, keepdims=True)
        return dict(campos=torch.from_numpy(s["campos"]).to(DEV)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(DEV)[None],
                    raydir=torch.from_numpy(d.astype(np.float32)).to(DEV)[None], pixel_idx=torch.from_numpy(pix.astype(np.int32)).to(DEV)[None],
                    h=cfg.H, w=cfg.W, intrinsic=s["intrinsic"], near=cfg.near, far=cfg.far,
                    bg_color=torch.ones(1, 3, device=DEV))


def _forward(net, d):
    return net(d["campos"], d["raydir"], bg_color=d["bg_color"], camrotc2w=d["camrotc2w"], pixel_idx=d["pixel_idx"], near=d["near"],
               far=d["far"], h=d["h"], w=d["w"], intrinsic=d["intrinsic"])


def _render_full(net, d):
    view = {k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")} if net.opt.wcoord_query == 0 else None
    near = float(torch.as_tensor(d["near"]).min())
    far = float(torch.as_tensor(d["far"]).max())
    return net.render_full(d["campos"], d["raydir"], d["camrotc2w"], near, far, d["bg_color"][0], view=view)


def _gt(n):
    return torch.rand((n, 3), generator=torch.Generator().manual_seed(5))


# ------------------------------------------------------------------------------------------------ gradients of theta
def _frustum_slopes(net, q):
    """The LeakyReLU masks of the last backward on the frustum query as `slopes=` of tests/frustum_shade_f64.py (pair rows in the
    flattened [R',SR,K] order of sample_pidx >= 0, colour rows per sample slot), as tests/test_gpu_frustum_fused.py maps them."""
    S, P = int(q.counters["n_valid"]), int(q.counters["n_pairs"])
    out = (ctypes.c_void_p * 10)()
    ws = net._bwd_ws
    lib.check(lib.load().pnb_backward_tables(ws.data_ptr(), ws.numel(), S, q.desc.cap_samples, 63, out), "pnb_backward_tables")
    dv = forward_check.dev_view
    H = [dv(ws, out[0], torch.float32, (P, 256)), dv(ws, out[1], torch.float32, (P, 272))[:, :256],
         dv(ws, out[2], torch.float32, (P, 256)), dv(ws, out[3], torch.float32, (P, 256))]
    Cc = [dv(ws, out[i], torch.float32, (S, 128)) for i in (4, 5, 6)]
    pair_off = dv(ws, out[7], torch.int32, (S + 1,)).long()
    row_samp = dv(ws, out[8], torch.int32, (P,)).long()
    vlist = dv(q.ws, q.desc.valid_list, torch.int32, (S,)).long()
    flat = vlist[row_samp] * q.K + (torch.arange(P, device=row_samp.device) - pair_off[row_samp])
    order = torch.argsort(flat)
    slopes = [torch.where(h[order] > 0, 1.0, 0.01).double().cpu() for h in H]
    for c in Cc:
        sl = torch.ones(q.R2 * q.SR, 128, dtype=torch.float64)
        sl[vlist.cpu()] = torch.where(c > 0, 1.0, 0.01).double().cpu()
        slopes.append(sl)
    return slopes


def _points64(su, th64, x64):
    """The cloud in float64 as set_points forms it from U(theta64): for modes "01" the one colour tensor goes both into the embedding
    and to points_color."""
    emb, col = upstream(th64, x64)
    pdir, conf = su.dir.double().cpu(), su.conf.double().cpu()
    if su.F == 63:
        emb = torch.cat([col, pdir, conf, emb], dim=-1)
    return dict(xyz=su.xyz.double().cpu(), embedding=emb, color=col, dir=pdir, conf=conf, Rw2c=torch.eye(3, dtype=torch.float64))


def _theta_case(F, mode, order):
    su = Setup(F, mode=mode, order=order)
    net = su.net()
    th = make_theta(su.n_emb)
    d = su.rays(20 if F == 32 else 61)
    emb, col = upstream(th, su.x)
    ref_set_points(net.neural_points, su.xyz, emb, col, su.dir, su.conf)
    npn = net.neural_points
    assert not npn.points_embeding.is_leaf and npn.points_embeding.requires_grad and npn.points_color is col
    assert not npn.points_dir.requires_grad and not npn.points_conf.requires_grad
    out = _forward(net, d)
    gt = _gt(out["coarse_raycolor"].shape[1])
    ((out["coarse_raycolor"][0] - gt.to(DEV)) ** 2).sum().backward()
    net.check_errors()
    q = net.last
    th64 = {k: v.detach().cpu().double().requires_grad_(True) for k, v in th.items()}
    mlp64 = {k: v.double().requires_grad_(True) for k, v in harness.mlp_cpu(net.aggregator).items()}
    pts = _points64(su, th64, su.x.cpu().double())
    if F == 32:
        cam = d["camrotc2w"][0].cpu()
        slopes, ex, _ = grad_check.kernel_masks(net, q, F, cam)
        hit = ex["ray_mask"].cpu() > 0
        sh = shade_oracle_rw2c.shade(pts, mlp64, ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu(), d["raydir"][0].cpu()[hit],
                                     d["campos"][0].cpu(), cam, su.opt.vsize, d["bg_color"][0].cpu(), dtype=torch.float64,
                                     agg_intrp_order=order, slopes=slopes, raydist_mode_unit=1)
    else:
        slopes = _frustum_slopes(net, q)
        pidx, loc, loc_w, dirs, vsize = q.sample_pidx, q.sample_loc, q.sample_loc_w, q.sample_ray_dirs, q.vsize
        with frustum_shade_f64.recording_softplus() as rec:
            sh = frustum_shade_f64.shade(pts, mlp64, pidx.cpu(), loc.cpu(), loc_w.cpu(), dirs.cpu(), d["campos"].cpu(),
                                         d["camrotc2w"].cpu(), vsize, d["bg_color"][0].cpu(), dtype=torch.float64, agg_intrp_order=order,
                                         slopes=slopes)
    ((sh["ray_color"] - gt.double()) ** 2).sum().backward()
    err = {k: grad_check.rel_error(th[k].grad.cpu(), th64[k].grad) for k in th}
    mlp = {k: grad_check.rel_error(p.grad.cpu(), mlp64[k].grad) for k, p in net.aggregator.named_parameters()}
    alpha1 = {}
    if F == 63 and order == 1:
        for k, t in frustum_shade_f64.alpha_branch_abs_terms(rec, sh["hbar"]).items():
            alpha1[k] = grad_check.sum_error(dict(net.aggregator.named_parameters())[k].grad.cpu(), mlp64[k].grad, t)
    print("\n[feedforward grads] F=%d mode=%d order=%d: R'=%d valid=%d theta %s | mlp worst %.2e (%s)%s"
          % (F, mode, order, out["coarse_raycolor"].shape[1], int(q.counters["n_valid"]), " ".join("%s %.2e" % kv for kv in err.items()),
             max(mlp.values()), max(mlp, key=mlp.get),
             "".join(" | %s %.2e of scale, %.2e of sum|terms|" % (k, mlp[k], v) for k, v in alpha1.items())))
    assert int(q.counters["n_valid"]) > 500, "too few shaded samples for the case to say anything"
    assert all(bool(torch.isfinite(t.grad).all()) and float(t.grad.abs().max()) > 0 for t in th.values())
    assert npn.xyz.grad is None
    for k, v in err.items():
        assert v <= THETA_RTOL[mode], "theta %s: %.3e of scale > %.1e" % (k, v, THETA_RTOL[mode])
    for k, v in mlp.items():
        if k in alpha1:
            b, bs = grad_check.ALPHA1_RTOL["bf16x3"], grad_check.ALPHA1_SUM_RTOL[(mode, "bf16x3")]
            assert v <= b, "%s: %.3e of scale > %.1e" % (k, v, b)
            assert alpha1[k] <= bs, "%s: %.3e of sum |terms| > %.1e" % (k, alpha1[k], bs)
        else:
            assert v <= MLP_RTOL[F][mode], "%s: %.3e of scale > %.1e" % (k, v, MLP_RTOL[F][mode])


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("mode", [0, 4, 1])
@pytest.mark.parametrize("F", [32, 63])
def test_upstream_gradients_match_float64(F, mode, order):
    _theta_case(F, mode, order)


# ------------------------------------------------------------------------------------------------ fresh clouds
OUT_KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "ray_mask")


def _cloud(su, th, step, n):
    """Step `step`'s cloud of n points: positions moved by a per-step offset (an out-of-place op: a new tensor of version 0) and U's
    outputs on them; dir and conf are views of fixed tensors, as the network's no_grad outputs are plain tensors."""
    off = torch.tensor([0.0004 * step, -0.0003 * step, 0.0002 * step], device=DEV)
    with torch.no_grad():
        xyz = su.xyz[:n] + off
    emb, col = upstream(th, su.x[:n])
    return xyz, emb, col, su.dir[:, :n], su.conf[:, :n]


def _fresh_outputs(su, cloud, d, train):
    """forward() (with the training graph when `train`) and render_full of a freshly built module on this cloud."""
    net = su.net()
    xyz, emb, col, pdir, conf = cloud
    net.neural_points.set_points(xyz, emb, points_color=col, points_dir=pdir, points_conf=conf, parameter=False)
    with torch.set_grad_enabled(train):
        fwd = _forward(net, d)
    with torch.no_grad():
        full = _render_full(net, d)
    torch.cuda.synchronize()
    return {k: fwd[k].detach().clone() for k in OUT_KEYS}, {k: full[k].clone() for k in OUT_KEYS}


def _equal(a, b, what):
    bad = [k for k in OUT_KEYS if not torch.equal(a[k], b[k])]
    assert not bad, "%s differs from a fresh module's in %s" % (what, bad)


@pytest.mark.parametrize("F", [32, 63])
def test_fresh_clouds_one_build_each_and_fresh_module_outputs(F):
    su = Setup(F)
    th = make_theta(su.n_emb)
    net = su.net()
    npn = net.neural_points
    d = su.rays(20 if F == 32 else 61)
    dl = su.rays(40 if F == 32 else 23)     # the chunk loop's rays
    sizes = [su.N, su.N - 300, su.N - 300, su.N - 100, su.N - 500]
    # step 2 takes step 1's size, address and version.  The caching allocator does not reliably hand a freed block back to the next
    # request of its size (and a world grid keeps the points it was built on alive), so the two clouds are two tensors of version 0
    # over one buffer (torch.from_dlpack): step 1's tensor is freed and step 2's positions are written into the buffer.
    via = "dlpack"
    buf = None
    for step, n in enumerate(sizes):
        builds = npn.querier.n_builds
        cloud = _cloud(su, th, step, n) if step != 2 else None
        if step == 1 and via == "dlpack":
            buf = cloud[0]
            cloud = (torch.from_dlpack(buf),) + cloud[1:]
        if step == 2:
            prev_ptr, prev_ver = npn.xyz.data_ptr(), npn.xyz._version
            npn.xyz = npn.points_embeding = npn.points_color = None       # the module's references; the test holds none
            cloud = _cloud(su, th, step, n)
            if via == "dlpack":
                buf.copy_(cloud[0])
                cloud = (torch.from_dlpack(buf),) + cloud[1:]
            xyz = cloud[0]
            assert (xyz.data_ptr(), xyz._version, xyz.shape[0]) == (prev_ptr, prev_ver, sizes[1]), \
                "step 2's cloud is not at step 1's address with its version (%#x v%d vs %#x v%d)" % (xyz.data_ptr(), xyz._version,
                                                                                                   prev_ptr, prev_ver)
        ref_set_points(npn, *cloud)
        out = _forward(net, d)
        ((out["coarse_raycolor"][0] - 0.5) ** 2).sum().backward()
        with torch.no_grad():
            full = _render_full(net, d)
            for i in range(0, dl["raydir"].shape[1], CHUNK // 8):          # a chunk loop over the same cloud
                sl = slice(i, i + CHUNK // 8)
                part = dict(dl, raydir=dl["raydir"][:, sl], pixel_idx=dl["pixel_idx"][:, sl])
                _forward(net, part)
        net.check_errors()
        torch.cuda.synchronize()
        print("\n[feedforward fresh] F=%d step %d: N=%d xyz at %#x v%d, builds %d -> %d%s" % (
            F, step, n, cloud[0].data_ptr(), cloud[0]._version, builds, npn.querier.n_builds,
            " (step 1's address and version, via %s)" % via if step == 2 else ""))
        assert npn.querier.n_builds == builds + 1, "step %d: %d builds for one cloud" % (step, npn.querier.n_builds - builds)
        want_fwd, want_full = _fresh_outputs(su, cloud, d, train=True)
        _equal({k: out[k].detach() for k in OUT_KEYS}, want_fwd, "step %d forward" % step)
        _equal(full, want_full, "step %d render_full" % step)
        del out, full, cloud


@pytest.mark.parametrize("F", [32, 63])
def test_eval_chunks_on_fresh_clouds_run_the_frozen_kernel(F):
    """model.test(gen_points=True): every 2304-ray chunk with a new cloud from the network, under no_grad, on the frozen kernel (its
    per-point table rebuilt for each cloud), bit for bit a fresh module's chunk."""
    su = Setup(F)
    th = make_theta(su.n_emb)
    net = su.net()
    npn = net.neural_points
    d = su.rays(None if F == 32 else 1)
    R = d["raydir"].shape[1]
    n_chunks = 0
    for c, i in enumerate(range(0, R, CHUNK)):
        sl = slice(i, i + CHUNK)
        part = dict(d, raydir=d["raydir"][:, sl], pixel_idx=d["pixel_idx"][:, sl])
        with torch.no_grad():
            cloud = _cloud(su, th, c + 1, su.N - 50 * (c % 2))
            ref_set_points(npn, *cloud)
            builds = npn.querier.n_builds
            got = _forward(net, part)
            assert npn.querier.n_builds == builds + 1
            assert net._pre_src[0]() is npn.points_embeding, "chunk %d did not run the frozen kernel on this cloud's table" % c
            ref = su.net()
            ref.neural_points.set_points(*cloud[:2], points_color=cloud[2], points_dir=cloud[3], points_conf=cloud[4], parameter=False)
            want = _forward(ref, part)
        torch.cuda.synchronize()
        bad = [k for k in OUT_KEYS if not torch.equal(got[k], want[k])]
        assert not bad, "chunk %d differs from a fresh module's in %s" % (c, bad)
        n_chunks += 1
    net.check_errors()
    print("\n[feedforward eval] F=%d: %d chunks of %d rays, one cloud each, bit for bit a fresh module's" % (F, n_chunks, CHUNK))
    assert n_chunks >= 2
