"""GPU: a DTU training session on the perspective-frustum query (wcoord_query 0): one long-lived fused module trained step by step on
scene.FRUSTUM_CONFIGS["dtu_surface"] (an opaque surface, alpha bias +300; F 63, point modes 01, SR 40, K 8, uniform jitter) across
views, with the plane background's bg_ray and a prune / probe / grow cycle in between, as the DTU scripts' training loop runs it
(a random training view per step, bg_ray of that view from a list built once per view, pruning and growing between steps).

The module and its helpers keep state from call to call: the querier's per-view build (keyed on the points, the grid and the camera)
and its query workspace, the MLP's operand images and the frozen kernel's per-point table (keyed on the parameters' versions), the
shading and backward workspaces, and plane_bg's images, views and foreground masks.  A key that misses a change serves stale data
while a freshly built module - what every other frustum test runs - stays right.  At every step:

  fresh module   the training forward (coarse_raycolor, coarse_point_opacity, coarse_is_background, ray_mask, conf_coefficient and
                 R') equals, bit for bit, that of a module loaded by checkpoint.load_checkpoint from the state before the step, under
                 the same torch.manual_seed (the jitter)
  query          the step's sample tuple equals, bit for bit, a newly constructed drop-in querier's for the view and seed: the hit
                 rays' pixel ids, sample_pidx, sample_loc, sample_loc_w, sample_ray_dirs and ray_mask
  float64        the gradients of the step's loss (colour L2 over the hit rays through the model shell's bg_ray formula, plus the
                 zero_one term on conf_coefficient) against float64 autograd of tests/frustum_shade_f64.py on the step's own tuple,
                 with the backward's LeakyReLU masks, at the parameters before the step: points within grad_check.RTOL of scale,
                 point 0's conf by check_conf, no outlier allowance; every MLP tensor, a sum over its layer's rows, within
                 grad_check.FRUSTUM_MLP_RTOL (alpha_branch.0 with order 1: ALPHA1_SUM_RTOL) of max(scale, sum |terms|) per entry
                 (grad_check.sum_error; DESIGN.md §6: over a step's thousands of rays these sums cancel by up to ~100x).  A step
                 whose rays all miss (R' = 0) leaves every gradient exactly zero.
  after the step render_full (frozen kernel) on a fixed patch of the step's view with that view's bg_ray equals, bit for bit, that of a
                 module loaded from the state after the step
  accounting     the querier builds on a call exactly when its camera, intrinsic or cloud differs from the previous call's; no error
                 flag after any call; the shading, backward and query workspaces each grow and are reused with valid samples present
The plane background is built per view at the start (gen_bg_points + set_bg, the create_all_bg pattern), each view's equal to a fresh
model's bit for bit; after the grow, set_bg rebuilds the foreground masks once and again equals a fresh model's.  The probe of the
grow cycle equals a fresh module's bit for bit.

Three planted defects show that the checks see what they claim to: a querier that keeps its build across a camera change, the fused
optimiser without torch.autograd.graph.increment_version (INTEGRATION.md §2), and set_bg served the foreground masks of the cloud
before the grow.  None of them changes the point count or the grid dimensions under a cached build.

The file prints the errors it measures (pytest -s).
"""
import contextlib
import copy
import functools
import math
import types

import numpy as np
import pytest
import torch

import frustum_shade_f64
from oracle import grad_check
from pointnerf_b200 import checkpoint, harness, plane_bg, runner, scene
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200.ray_marching import MLP_KEYS, NeuralPoints, NeuralPointsRayMarching, PointAggregator

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
CFG = scene.FRUSTUM_CONFIGS["dtu_surface"]
OUT_KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "ray_mask", "conf_coefficient")
RENDER_KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "ray_mask")
PROBE_KEYS = runner.PROBE_MAP_KEYS
ZERO_EPS = 1e-3          # the zero_one loss's clamp (models/base_rendering_model.py:629-641)
ZERO_ONE_WEIGHT = 1e-3
LR, PLR = 5e-4, 2e-3     # parallel.TrainStep's learning rates of the MLP and of the point features
PRUNE = 0.3              # conf threshold of the grow cycle's prune: frees enough mask cells to change the plane background


# ------------------------------------------------------------------------------------------------ views
def _rot_y(a):
    return np.array([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]])


@functools.lru_cache(None)
def views():
    """name -> (camrotc2w [3,3], campos [3], intrinsic [3,3]), float32; every view but "away" keeps the surface in the grid.
      v0    the scene's camera
      v1    v0 orbited by 4 degrees about the surface centre (2.5 in front of v0), same intrinsic
      v2    v0's rotation, campos moved by (0.06, -0.04, 0.08) in v0's frame
      v3    v0's pose with another intrinsic: focal x 1.05, principal point moved by (+3.5, -2.5) px (a per-view calibration)
      away  v0 turned by 180 degrees about its y axis: every point lies behind it (R' = 0)"""
    s = scene.make_frustum_scene(CFG)
    R0, c0, K0 = s["camrotc2w"].astype(np.float64), s["campos"].astype(np.float64), s["intrinsic"]
    centre = c0 + R0 @ np.array([0.0, 0.0, 2.5])
    R1 = R0 @ _rot_y(math.radians(4.0))
    f = 1.05 * CFG.focal
    K3 = np.array([[f, 0, CFG.W / 2 + 3.5], [0, f, CFG.H / 2 - 2.5], [0, 0, 1]])
    out = dict(v0=(R0, c0, K0), v1=(R1, centre - R1 @ np.array([0.0, 0.0, 2.5]), K0), v2=(R0, c0 + R0 @ np.array([0.06, -0.04, 0.08]), K0),
               v3=(R0, c0, K3), away=(R0 @ _rot_y(math.pi), c0, K0))
    return {k: tuple(np.ascontiguousarray(a, np.float32) for a in v) for k, v in out.items()}


def frame_pixels():
    """Every pixel (x, y) of the frame, y outer."""
    px, py = np.meshgrid(np.arange(CFG.W), np.arange(CFG.H))
    return np.stack((px, py), -1).reshape(-1, 2).astype(np.int32)


def ray_dirs(view, pix):
    """Unit directions through the pixel centres (as tests/test_gpu_frustum_fused.py forms them), float32 [R,3]."""
    R, _, K = views()[view]
    pix = np.asarray(pix).reshape(-1, 2)
    d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ R.T.astype(np.float64)
    return (d / np.linalg.norm(d, axis=-1, keepdims=True)).astype(np.float32)


def _data(view, pix):
    """The input dict of a reference dataset item of `view` for these pixels."""
    R, c, K = views()[view]
    return dict(campos=torch.from_numpy(c).to(DEV)[None], camrotc2w=torch.from_numpy(R).to(DEV)[None],
                raydir=torch.from_numpy(ray_dirs(view, pix)).to(DEV)[None], pixel_idx=torch.from_numpy(pix.astype(np.int32)).to(DEV)[None],
                h=CFG.H, w=CFG.W, intrinsic=K, near=CFG.near, far=CFG.far, bg_color=torch.zeros(3, device=DEV))


# ------------------------------------------------------------------------------------------------ the loss, both precisions
def zero_one(cc):
    """The zero_one loss on conf_coefficient (models/base_rendering_model.py:629-641)."""
    val = torch.clamp(cc, ZERO_EPS, 1 - ZERO_EPS)
    return torch.mean(torch.log(val) + torch.log(1 - val))


def conf_coefficient(conf, sample_pidx):
    """conf_coefficient of the reference's eager shading: each slot's conf, gathered at clamp(pidx, 0) (neural_points.py:706-717),
    through the straight-through clamp to [1e-4, 1] (point_aggregators.py:722-724).  conf [1,N,1], sample_pidx [R',SR,K]."""
    c0 = conf[0][torch.clamp(sample_pidx, min=0).long()][..., 0]
    return c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach()


def loss(color, is_bg, bg_ray_hit, gt_hit, cc):
    """The step's loss: colour L2 over the hit rays through the model shell's fill_invalid with bg_ray (coarse_is_background *
    bg_ray + coarse_raycolor), plus the zero_one term on conf_coefficient (absent when no ray hits).  color [R',3], is_bg [R',1]."""
    col = is_bg * bg_ray_hit + color
    L = ((col - gt_hit) ** 2).sum()
    if cc is not None and cc.numel():
        L = L + ZERO_ONE_WEIGHT * zero_one(cc)
    return L


# ------------------------------------------------------------------------------------------------ module, plane background
def _opt(order, precision, mode):
    """The DTU scripts' options (scene.frustum_opt on the tiny world config's shading options), training with uniform jitter."""
    fo = vars(scene.frustum_opt(CFG, is_train=True))
    return harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, agg_intrp_order=order, pnb_precision=precision, pnb_bwd_fp32=mode, **fo)


def _net(opt, seed=5):
    """The fused module on the frustum scene's points as stored, with an opaque surface (alpha bias +300: the depth voxels are 0.0068
    long), as tests/test_gpu_frustum_fused.py builds it."""
    s = scene.make_frustum_scene(CFG)
    pts = scene.make_frustum_points(CFG, s)
    agg = PointAggregator(opt, seed=seed)
    with torch.no_grad():
        agg.alpha_branch[0].bias += 300.0
    npn = NeuralPoints(opt, DEV)
    npn.set_points(pts["xyz"].to(DEV), pts["embedding"].to(DEV), points_color=pts["color"].to(DEV), points_dir=pts["dir"].to(DEV),
                   points_conf=pts["conf"].to(DEV), parameter=True, as_stored=True)
    assert isinstance(npn.querier, qpi.lighting_fast_querier)
    return NeuralPointsRayMarching(aggregator=agg.to(DEV), neural_points=npn, opt=opt)


def _snapshot(net):
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def _load(sd, opt):
    return checkpoint.load_checkpoint(sd, copy.copy(opt), DEV)


def _differs(a, b, keys):
    """Keys whose tensors are not equal bit for bit (or present in one dict only)."""
    return [k for k in keys if (k in a) != (k in b) or (k in a and not torch.equal(a[k], b[k]))]


@contextlib.contextmanager
def recording_lin(names):
    """Inside the block, frustum_shade_f64.shade keeps the input x and the output z (its gradient retained) of each call of the
    layers `names`: {name: [(x, z)]}."""
    lin, rec = frustum_shade_f64._lin, {}

    def recording(x, mlp, key):
        z = lin(x, mlp, key)
        if key in names and z.requires_grad:
            z.retain_grad()
            rec.setdefault(key, []).append((x.detach(), z))
        return z
    frustum_shade_f64._lin = recording
    try:
        yield rec
    finally:
        frustum_shade_f64._lin = lin


def sum_abs_terms(rec):
    """After backward(): a layer's weight and bias gradients are sums over its rows of dL/dz [x, 1]; their sums of |terms| per entry,
    {parameter name: tensor}, for grad_check.sum_error."""
    out = {}
    for key, calls in rec.items():
        gs = [(x, z.grad.abs()) for x, z in calls if z.grad is not None]
        out[key + ".bias"] = sum(g.sum(0) for _, g in gs)
        out[key + ".weight"] = sum(g.t() @ x.abs() for x, g in gs)
    return out


class Plane:
    """The DTU scripts' plane background for the session's views: a plane 3.3 in front of v0 (0.8 behind the surface), one seeded
    image per view around the plane colour, the set_bg arguments of all views (img_lst, c2ws, w2cs, intrinsics, HDWD)."""

    def __init__(self, seed=2):
        R0, c0, _ = (a.astype(np.float64) for a in views()["v0"])
        n = R0 @ np.array([0.1, -0.35, 0.93])
        self.pnt = torch.from_numpy((c0 + R0 @ np.array([0.0, 0.0, 3.3])).astype(np.float32))[None]
        self.normal = torch.from_numpy((n / np.linalg.norm(n)).astype(np.float32))[None]
        self.color = torch.tensor([0.55, 0.45, 0.35], device=DEV)
        g = np.random.RandomState(seed)
        self.names = list(views())
        self.img_lst, self.w2cs, self.Ks = [], [], []
        for name in self.names:
            R, c, K = (a.astype(np.float64) for a in views()[name])
            w2c = np.eye(4)
            w2c[:3, :3], w2c[:3, 3] = R.T, -R.T @ c
            img = self.color.cpu().numpy()[:, None, None] + g.uniform(-0.05, 0.05, (3, CFG.H, CFG.W))
            self.img_lst.append(torch.from_numpy(img.astype(np.float32))[None])
            self.w2cs.append(torch.from_numpy(w2c.astype(np.float32)).to(DEV)[None, None])
            self.Ks.append(torch.from_numpy(K.astype(np.float32)).to(DEV)[None])
        self.hdwd = [[CFG.H, CFG.W]] * len(self.names)
        self.frame = frame_pixels()
        self.sect = {}
        for name in self.names:
            R, c, _ = views()[name]
            batch = dict(campos=torch.from_numpy(c).to(DEV)[None], raydir=torch.from_numpy(ray_dirs(name, self.frame)).to(DEV)[None],
                         plane_pnt=self.pnt, plane_normal=self.normal)
            self.sect[name] = plane_bg.gen_bg_points(batch)

    def set_bg(self, model, name):
        bg, ret = plane_bg.set_bg(model, self.sect[name], self.img_lst, [None] * len(self.names), self.w2cs, self.Ks, self.hdwd, self.color)
        assert ret is None
        return bg


# ------------------------------------------------------------------------------------------------ the session
class Session:
    """One long-lived module trained by torch.optim.Adam (TrainStep's two groups and learning rates) on seeded random pixels of a
    view per step, every step checked as the module header says."""

    def __init__(self, order=1, precision="bf16x3", mode=0, optimiser="foreach"):
        self.order, self.precision, self.mode, self.optimiser = order, precision, mode, optimiser
        self.opt = _opt(order, precision, mode)
        self.net = _net(self.opt)
        self.querier = self.net.neural_points.querier
        self.rng = np.random.RandomState(0)
        self.gen = torch.Generator().manual_seed(1)
        self.cloud = 0             # bumped by every change of the point cloud (prune, grow)
        self.prev_call = None      # (view, cloud) of the querier's previous call
        self.history = []
        self.new_optimiser()
        self.sd = _snapshot(self.net)
        self.plane = Plane()
        self.bg = {}
        self.set_bg_all()

    def new_optimiser(self):
        """torch.optim.Adam over TrainStep's two groups: the reference's default (foreach) or fused, whose writes do not advance the
        parameters' _version, followed by increment_version as INTEGRATION.md §2 prescribes."""
        net = self.net
        self.params = [p for p in net.aggregator.parameters() if p.requires_grad] + \
                      [p for p in net.neural_points.parameters() if p.requires_grad]
        groups = [dict(params=[p for p in net.aggregator.parameters() if p.requires_grad], lr=LR),
                  dict(params=[p for p in net.neural_points.parameters() if p.requires_grad], lr=PLR)]
        kw = dict(fused=True) if self.optimiser == "fused" else dict(foreach=True)
        self.adam = torch.optim.Adam(groups, betas=(0.9, 0.999), **kw)

    def set_bg_all(self):
        """bg_ray of every view (create_all_bg), each equal to that of a fresh model on the current cloud; the foreground masks are
        built once per cloud."""
        xyz = self.net.neural_points.xyz
        cache = getattr(self.net, "_pnb_plane_bg", None)
        before = None if cache is None else (cache.n_image_builds, cache.n_view_builds, cache.n_mask_builds)
        fresh = types.SimpleNamespace(neural_points=types.SimpleNamespace(xyz=xyz.detach().clone()))
        out, differs = {}, []
        for name in self.plane.names:
            out[name] = self.plane.set_bg(self.net, name)
            if not torch.equal(out[name], self.plane.set_bg(fresh, name)):
                differs.append(name)
        c = self.net._pnb_plane_bg
        after = (c.n_image_builds, c.n_view_builds, c.n_mask_builds)
        print("\n[frustum session] set_bg on %d points: builds (images, views, masks) %s -> %s, differs from a fresh model's in %s"
              % (xyz.shape[0], before, after, differs or "-"))
        assert not differs, "set_bg differs from a fresh model's for %s" % differs
        assert after == ((1, 1, 1) if before is None else (before[0], before[1], before[2] + 1)), (before, after)
        old, self.bg = self.bg, out
        return old

    def pixels(self, n):
        """n seeded random pixels over the whole frame (the scripts' random_sample random)."""
        return np.stack([self.rng.randint(0, CFG.W, n), self.rng.randint(0, CFG.H, n)], -1).astype(np.int32)

    def bg_ray(self, view, pix):
        pid = torch.from_numpy((pix[:, 1] * CFG.W + pix[:, 0]).astype(np.int64)).to(DEV)
        return self.bg[view][0][pid][None]

    def call(self, view, fn):
        """Runs one call of the long-lived querier and checks the build accounting."""
        nb = self.querier.n_builds
        r = fn()
        want = int((view, self.cloud) != self.prev_call)
        got = self.querier.n_builds - nb
        self.prev_call = (view, self.cloud)
        assert got == want, "%s (cloud %d): the querier built %d times, expected %d" % (view, self.cloud, got, want)
        return r

    def render(self, net, view, seed):
        """render_full (frozen kernel) on the 24 x 24 centre patch of the view with its bg_ray, status checked."""
        x0, y0 = CFG.W // 2 - 12, CFG.H // 2 - 12
        px, py = np.meshgrid(np.arange(x0, x0 + 24), np.arange(y0, y0 + 24))
        pix = np.stack((px, py), -1).reshape(-1, 2).astype(np.int32)
        d = _data(view, pix)
        torch.manual_seed(seed)
        with torch.no_grad():
            out = net.render_full(d["campos"], d["raydir"], d["camrotc2w"], CFG.near, CFG.far, d["bg_color"], bg_ray=self.bg_ray(view, pix),
                                  view={k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")})
        net.check_errors()
        return out

    def forward(self, net, d, bg_ray, seed):
        torch.manual_seed(seed)
        return net(d["campos"], d["raydir"], camrotc2w=d["camrotc2w"], pixel_idx=d["pixel_idx"], near=d["near"], far=d["far"], h=d["h"],
                   w=d["w"], intrinsic=d["intrinsic"], bg_ray=bg_ray)

    def dropin(self, d, seed):
        """A newly constructed drop-in querier's tuple for the view and seed (points in perspective coordinates by the reference's
        w2pers), and its hit rays' pixel ids."""
        q = qpi.lighting_fast_querier(DEV, copy.copy(self.opt))
        xyz = self.net.neural_points.xyz.detach()
        pers = qpi.w2pers(xyz, d["camrotc2w"], d["campos"])
        torch.manual_seed(seed)
        tup = q.query_points(d["pixel_idx"], pers, xyz[None], torch.tensor([xyz.shape[0]], dtype=torch.int32), np.int64(CFG.H),
                             np.int64(CFG.W), d["intrinsic"], np.float32(CFG.near), np.float32(CFG.far), None, d["campos"], d["camrotc2w"])
        return tup, q.last_pixel_idx_cur

    def float64(self, q, d, bg_ray, gt, sd, slopes):
        """Errors of the step's gradients against float64 autograd of the oracle at the parameters `sd`, with the backward's masks."""
        net = self.net
        npn = net.neural_points
        names = dict(embedding="points_embeding", color="points_color", dir="points_dir", conf="points_conf")
        pts = dict(xyz=sd["neural_points.xyz"].cpu().double(), Rw2c=torch.eye(3, dtype=torch.float64))
        for k, name in names.items():
            pts[k] = sd["neural_points." + name].cpu().double().requires_grad_(True)
        mlp = {k[len("aggregator."):]: v.cpu().double().requires_grad_(True) for k, v in sd.items() if k.startswith("aggregator.")}
        pidx = q.sample_pidx.cpu()
        # every layer's weight and bias gradients are sums over its rows (pairs or samples): their sums of |terms| (DESIGN.md §6)
        summed = tuple(k for k in MLP_KEYS if not (k == "alpha_branch.0" and self.order == 1))
        with frustum_shade_f64.recording_softplus() as rec, recording_lin(summed) as lin_rec:
            r = frustum_shade_f64.shade(pts, mlp, pidx, q.sample_loc.cpu(), q.sample_loc_w.cpu(), q.sample_ray_dirs.cpu(), d["campos"].cpu(),
                                        d["camrotc2w"].cpu(), q.vsize, torch.zeros(3), dtype=torch.float64, agg_intrp_order=self.order,
                                        slopes=slopes)
        hit = torch.nonzero(q.ray_mask.cpu())[:, 0]
        L = loss(r["ray_color"], r["bg_T"], bg_ray[0].cpu().double()[hit], gt.cpu().double()[hit], conf_coefficient(pts["conf"], pidx))
        L.backward()
        abs_terms = frustum_shade_f64.alpha_branch_abs_terms(rec, r["hbar"]) if self.order == 1 else {}
        summed_terms = sum_abs_terms(lin_rec)
        rt_points = grad_check.RTOL[(self.mode, self.precision)][0]
        err = {}
        for k in ("embedding", "color", "dir"):
            err[k] = float(grad_check.rel_point_errors(getattr(npn, names[k]).grad.cpu(), pts[k].grad).max())
        n0 = int((pidx <= 0).sum())
        try:
            err["conf"] = grad_check.check_conf(npn.points_conf.grad.cpu(), pts["conf"].grad, n0, rt_points)
        except AssertionError as e:
            err["conf"] = str(e)
        alpha1, summed_err = {}, {}
        for k, p in net.aggregator.named_parameters():
            err[k] = grad_check.rel_error(p.grad.cpu(), mlp[k].grad)
            if k in abs_terms:
                alpha1[k] = grad_check.sum_error(p.grad.cpu(), mlp[k].grad, abs_terms[k])
            if k in summed_terms:
                summed_err[k] = grad_check.sum_error(p.grad.cpu(), mlp[k].grad, summed_terms[k])
        return err, alpha1, summed_err

    def check_float64(self, rec):
        rt_points = grad_check.RTOL[(self.mode, self.precision)][0]
        rt_mlp = grad_check.FRUSTUM_MLP_RTOL[(self.mode, self.precision)]
        err, alpha1, summed = rec["err"], rec["alpha1"], rec["summed"]
        assert not isinstance(err["conf"], str), "step %d: %s" % (rec["step"], err["conf"])
        for k, v in err.items():
            if k in summed:
                # DESIGN.md §6: over a step's thousands of rays these sums cancel; the tensor's bound relative to max(scale, sum |terms|)
                assert summed[k] <= rt_mlp, "step %d: aggregator.%s: %.3e of max(scale, sum |terms|) > %.1e" % (rec["step"], k, summed[k],
                                                                                                                 rt_mlp)
            elif k in alpha1:
                bs = grad_check.ALPHA1_SUM_RTOL[(self.mode, self.precision)]
                assert alpha1[k] <= bs, "step %d: aggregator.%s: %.3e of max(scale, sum |terms|) > %.1e" % (rec["step"], k, alpha1[k], bs)
            else:
                assert v <= rt_points, "step %d: %s: %.3e of scale > %.1e" % (rec["step"], k, v, rt_points)

    def step(self, view, n):
        """One training step with every check of the module header; returns its record."""
        net = self.net
        pix = self.pixels(n)
        d = _data(view, pix)
        bg_ray = self.bg_ray(view, pix)
        gt = torch.rand(n, 3, generator=self.gen).to(DEV)
        step = len(self.history) + 1
        seed = 1000 + step
        sd = self.sd

        def train():
            self.adam.zero_grad(set_to_none=True)
            out = self.forward(net, d, bg_ray, seed)
            hit = torch.nonzero(out["ray_mask"][0])[:, 0]
            loss(out["coarse_raycolor"][0], out["coarse_is_background"][0], bg_ray[0][hit], gt[hit],
                 out["conf_coefficient"][0] if "conf_coefficient" in out else None).backward()
            self.adam.step()
            if self.optimiser == "fused":
                torch.autograd.graph.increment_version(self.params)
            net.check_errors()
            return out
        out = self.call(view, train)
        q = net.last
        n_valid = int(q.counters["n_valid"])
        rec = dict(step=step, view=view, rays=n, R2=q.R2, n_valid=n_valid, tc_ws=0 if net._tc_ws is None else net._tc_ws.numel(),
                   bwd_ws=net._bwd_ws.numel(), q_ws=self.querier._ws.numel())
        pixel_ids = self.querier.last_pixel_idx_cur.clone()
        slopes = frustum_shade_f64.kernel_slopes(net, q) if n_valid else None
        # the query: a newly constructed drop-in's tuple for this view and seed
        tup, dpix = self.dropin(d, seed)
        got = (pixel_ids, q.sample_pidx[None], q.sample_loc[None], q.sample_loc_w[None], q.sample_ray_dirs[None], q.ray_mask[None])
        want = (dpix, tup[0], tup[1], tup[2], tup[3], tup[4])
        names = ("pixel ids", "sample_pidx", "sample_loc", "sample_loc_w", "sample_ray_dirs", "ray_mask")
        rec["query_differs"] = [k for k, a, b in zip(names, got, want) if not torch.equal(a, b)]
        # fresh-module identity of the training forward
        fresh = _load(sd, self.opt)
        fo = self.forward(fresh, d, bg_ray, seed)
        fresh.check_errors()
        rec["forward_differs"] = _differs(out, fo, OUT_KEYS) + ([] if fresh.last.R2 == q.R2 else ["R'"])
        assert not rec["query_differs"], "step %d (%s): the sample tuple differs from a new drop-in querier's in %s" % (
            step, view, rec["query_differs"])
        assert not rec["forward_differs"], "step %d (%s): the training forward differs from a fresh module's in %s" % (
            step, view, rec["forward_differs"])
        if n_valid:
            rec["err"], rec["alpha1"], rec["summed"] = self.float64(q, d, bg_ray, gt, sd, slopes)
        else:
            rec["nonzero_grads"] = [k for k, p in net.named_parameters() if p.grad is not None and bool(p.grad.any())]
        # after the step: render_full of a module loaded from the new state
        self.sd = _snapshot(net)
        mine = self.call(view, lambda: self.render(net, view, seed + 500))
        rec["render_differs"] = _differs(mine, self.render(_load(self.sd, self.opt), view, seed + 500), RENDER_KEYS)
        self.history.append(rec)
        self.report(rec)
        if n_valid:
            self.check_float64(rec)
        else:
            assert not rec["nonzero_grads"], "step %d (%s, no valid sample): non-zero gradients of %s" % (step, view, rec["nonzero_grads"])
        assert not rec["render_differs"], "step %d (%s): render_full after the step differs from a fresh module's in %s" % (
            step, view, rec["render_differs"])
        return rec

    def grow(self):
        """The grow cycle between steps (run/train_ft.py:838, :844-873): prune, the probe of v1's whole frame (opt.prob = 1, no jitter),
        grow_points by tests/test_gpu_train_session.py's rule, new optimisers, set_bg again for every view."""
        net, opt = self.net, self.opt
        npn = net.neural_points
        n_before = npn.xyz.shape[0]
        pruned = npn.prune(PRUNE)
        self.cloud += 1
        opt.prob, opt.is_train = 1, False
        try:
            d = _data("v1", frame_pixels())
            fresh = _load(_snapshot(net), opt)
            maps = self.call("v1", lambda: runner.probe_image(net, d, CFG.H, CFG.W))
            fmaps = runner.probe_image(fresh, d, CFG.H, CFG.W)
        finally:
            opt.prob, opt.is_train = 0, True
        differs = _differs(maps, fmaps, PROBE_KEYS)
        o = maps["ray_max_shading_opacity"].reshape(-1)
        keep = (o > 0.5 * o.max()) & (torch.arange(o.shape[0], device=DEV) % 4 == 0)
        add = [maps[k].reshape(o.shape[0], -1)[keep] for k in ("ray_max_sample_loc_w", "shading_avg_embedding", "shading_avg_color",
                                                                "shading_avg_dir", "shading_avg_conf")]
        npn.grow_points(*add)
        self.cloud += 1
        print("\n[frustum session] grow cycle: %d points, %d pruned, %d grown; probe outputs differ from a fresh module's in: %s"
              % (n_before, pruned, int(keep.sum()), differs or "-"))
        assert 0 < pruned < n_before and int(keep.sum()) > 0
        assert not differs, "probe outputs differ from a fresh module's in %s" % differs
        self.new_optimiser()
        self.sd = _snapshot(net)
        old = self.set_bg_all()
        changed = [k for k in old if not torch.equal(old[k], self.bg[k])]
        assert changed, "the grow cycle leaves every view's bg_ray as it was: a stale foreground mask would not show"

    def report(self, rec):
        if "err" in rec:
            e = rec["err"]
            pts = max(e[k] for k in ("embedding", "color", "dir", "conf") if not isinstance(e[k], str))
            sums = dict(rec["summed"], **rec["alpha1"])
            mk = max((k for k in e if "." in k), key=e.get)
            ms = max(sums, key=sums.get)
            a1 = "".join(" | %s %.2e of scale, %.2e of max(scale, sum|terms|)" % (k, e[k], v) for k, v in rec["alpha1"].items())
            f64 = "points=%.2e mlp: of scale %.2e (%s), of max(scale, sum|terms|) %.2e (%s)%s" % (pts, e[mk], mk, sums[ms], ms, a1)
        else:
            f64 = "no valid sample, non-zero gradients: %s" % (rec["nonzero_grads"] or "-")
        print("\n[frustum session] order %d %s mode %d %s step %d %s rays=%d R'=%d n_valid=%d tc_ws=%d bwd_ws=%d q_ws=%d: %s; query differs: "
              "%s, forward differs: %s, render differs: %s" % (
                  self.order, self.precision, self.mode, self.optimiser, rec["step"], rec["view"], rec["rays"], rec["R2"], rec["n_valid"],
                  rec["tc_ws"], rec["bwd_ws"], rec["q_ws"], f64, rec["query_differs"] or "-", rec["forward_differs"] or "-",
                  rec["render_differs"] or "-"))

    def run(self, plan):
        for item in plan:
            if item == "grow":
                self.grow()
            else:
                self.step(*item)


def _grew_and_reused(sizes, n_valid):
    """A workspace grown after the first step, and one step with samples that ran in the one of the step before."""
    grew = any(sizes[i] > sizes[i - 1] for i in range(1, len(sizes)))
    reused = any(sizes[i] == sizes[i - 1] and n_valid[i] > 0 for i in range(1, len(sizes)))
    return grew and reused


# (view, rays) of the steps: two views and back, the same view with more rays, a moved camera, another intrinsic, a view without a
# hit ray, the grow cycle, then the views again on the grown cloud
PLAN = (("v0", 2304), ("v1", 2304), ("v0", 1024), ("v0", 3000), ("v2", 2304), ("v3", 2304), ("away", 1024), "grow", ("v1", 2304),
        ("v0", 2304))
CASES = {"order1-bf16x3-mode0-foreach": dict(order=1, precision="bf16x3", mode=0, optimiser="foreach"),
         "order1-bf16x3-mode0-fused": dict(order=1, precision="bf16x3", mode=0, optimiser="fused"),
         "order1-bf16x3-mode4": dict(order=1, precision="bf16x3", mode=4, optimiser="fused"),
         "order1-fp32-mode1": dict(order=1, precision="fp32", mode=1, optimiser="fused"),
         "order2-bf16x3-mode0": dict(order=2, precision="bf16x3", mode=0, optimiser="fused")}


@pytest.mark.parametrize("case", list(CASES))
def test_frustum_session_matches_fresh_module_and_float64(case):
    s = Session(**CASES[case])
    s.run(PLAN)
    h = s.history
    nv = [r["n_valid"] for r in h]
    assert [r["R2"] == 0 for r in h] == [r["view"] == "away" for r in h], [r["R2"] for r in h]
    for k in ("bwd_ws", "q_ws") + (("tc_ws",) if s.precision == "bf16x3" else ()):
        sizes = [r[k] for r in h]
        assert _grew_and_reused(sizes, nv), (k, sizes)


def _defect_stale_view(monkeypatch, s):
    """The querier keeps its build when only the camera changed (valid only between views with one intrinsic, near and far: the
    same grid and N, so every index stays in bounds), and counts it as a build, so that only the data can show it."""
    q = s.querier
    build = q._build

    def keep_build(pers, n, key, *a):
        if q._fr is not None and q._key[0] == key[0]:
            q._key = key
            q.n_builds += 1
            return
        build(pers, n, key, *a)
    monkeypatch.setattr(q, "_build", keep_build)
    s.run((("v0", 1024), ("v1", 1024)))


def _defect_stale_weights(monkeypatch, s):
    """The fused optimiser without increment_version."""
    monkeypatch.setattr(torch.autograd.graph, "increment_version", lambda *a, **k: None)
    s.run((("v0", 1024), ("v1", 1024)))


def _defect_stale_masks(monkeypatch, s):
    """set_bg served the foreground masks it holds, whatever the cloud (the mask size depends on the views only)."""
    masks = plane_bg._masks
    monkeypatch.setattr(plane_bg, "_masks", lambda cache, xyz, v, dev: cache.masks if cache.masks is not None else masks(cache, xyz, v, dev))
    s.run(("grow",))


# defect -> (plant, optimiser, the check that must see it)
DEFECTS = {"stale_view": (_defect_stale_view, "foreach", "the sample tuple differs from a new drop-in querier's"),
           "stale_weights": (_defect_stale_weights, "fused", "differs from a fresh module's"),
           "stale_masks": (_defect_stale_masks, "foreach", "set_bg differs from a fresh model's")}


@pytest.mark.parametrize("defect", list(DEFECTS))
def test_planted_defect_is_detected(monkeypatch, defect):
    plant, optimiser, check = DEFECTS[defect]
    s = Session(optimiser=optimiser)
    with pytest.raises(AssertionError) as e:
        plant(monkeypatch, s)
    msg = str(e.value).splitlines()[0]
    print("\n[frustum session] planted defect %s detected: %s" % (defect, msg))
    assert check in msg, msg
