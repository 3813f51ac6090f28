"""GPU: a training session on one long-lived module, every step checked at the module's current parameters (teacher-forced) against a
module freshly loaded from the same state dict and against float64.

The module keeps state across calls: the MLP's padded W^T buffers and wgmma operand images (MlpPack), the frozen kernel's per-point
table (_point_pre), the host copy of a uniform Rw2c (rw2c_host_of), the querier's grid and workspace, the shading and backward
workspaces.  Each is keyed by its source tensors.  A key that misses an update (a fused optimiser writes without advancing _version) or
that matches another tensor at a recycled address (the caching allocator) makes the module shade with stale data, while the single
forward / backward of a fresh module - what every other GPU test runs - stays right.  At every step of a session:

  * fresh-module identity: the training forward's outputs (coarse_raycolor, coarse_point_opacity, coarse_is_background, ray_mask,
    conf_coefficient) equal, bit for bit, those of a module built by checkpoint.load_checkpoint from the state dict taken before the
    step, with the step's jittered t table replayed; after the step, render_full (the frozen kernel and its table) on a fixed patch with
    the host t table equals, bit for bit, that of a module loaded from the state after the step;
  * float64: the step's loss, written through TrainStep.loss_terms on the outputs of the float64 oracle (shade_oracle_rw2c on the
    kernel's export, with the backward's own LeakyReLU masks) and differentiated at the parameters before the step: every point
    gradient and all 18 MLP gradients within grad_check.RTOL of the backward mode, points_conf of point 0 within the bound below.
    (Whole Adam trajectories are not compared: Adam's first steps are close to lr * sign(g), which flips with the rounding of every
    gradient entry near zero.)

Point 0's conf bound under the zero-one term.  TrainStep's conf term is w / n_zo * sum(-log(cc + 1e-3)), w = 1e-4, n_zo the number of
conf_coefficient entries.  Every entry of a slot whose clamped neighbour index is 0 gathers point 0's conf, so all n0 such entries hold
the same cc0 = clamp(conf_0, 1e-4, 1) and receive the same upstream gradient t0 = w / (n_zo (cc0 + 1e-3)) (the clamp is straight
through: d cc / d conf = 1).  pnb_aux_conf_backward adds these n0 terms into point 0's fp32 gradient; each addition is off by at most
U32 of the running sum, which stays below |ref0| + n0 t0 (ref0: the float64 gradient, the shading backward's part included).  That is
grad_check.point0_conf_bound(n0, ref0, t0): the bound of the constant weight with its term 1e-3 replaced by t0.  The fp32 rounding of
t0 itself (a few U32, the same in all n0 terms) stays below it for n0 >= 3.
"""
import copy

import numpy as np
import pytest
import torch

from oracle import grad_check, shade_oracle_rw2c
from pointnerf_b200 import checkpoint, harness, parallel, point_query, scene

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
CFG = scene.CONFIGS["tiny"]
OUT_KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "ray_mask", "conf_coefficient")
RENDER_KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background", "ray_mask")
FWD_KEYS = ("campos", "raydir", "bg_color", "camrotc2w", "pixel_idx", "near", "far", "h", "w", "intrinsic")
# (kind, rays) of the steps: the ray count and the hit density rise, fall (with one step whose rays all miss, n_valid == 0 in the
# backward) and rise again, so that the shading and backward workspaces are grown and reused
PLAN = (("hit", 192), ("hit", 640), ("miss", 96), ("hit", 320), ("hit", 800))


def _snapshot(net):
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


def _load(sd, opt):
    return checkpoint.load_checkpoint(sd, copy.copy(opt), DEV)


def _render(net):
    """render_full on the centre patch with the host t table (no jitter), its status checked."""
    rays = scene.make_rays(CFG, scene.centre_patch(CFG, 24))
    t = point_query.host_t_table(CFG.near, CFG.far, CFG.D).to(DEV)
    with torch.no_grad():
        out = net.render_full(list(CFG.campos), rays["raydir"][0].to(DEV), torch.eye(3), CFG.near, CFG.far, [1., 1., 1.], t=t)
    net.check_errors()
    return out


def _differs(a, b, keys):
    """Keys whose tensors are not equal bit for bit (or present in one dict only)."""
    return [k for k in keys if (k in a) != (k in b) or (k in a and not torch.equal(a[k], b[k]))]


class Session:
    """One long-lived module trained by parallel.TrainStep on random pixel batches (bench.py's train_section, is_train=True)."""

    def __init__(self, F=32, frames=False, precision="bf16x3", mode=0, optimiser="fused"):
        self.F, self.frames, self.mode, self.precision, self.optimiser = F, frames, mode, precision, optimiser
        self.net, _, self.opt = harness.build_model(CFG, DEV, alpha_bias=3.0, seed=2, is_train=True, feat_dim=F, pnb_precision=precision,
                                                    pnb_bwd_fp32=mode)
        npn = self.net.neural_points
        if frames:
            npn.Rw2c = torch.nn.Parameter(scene.edit_frames(npn.xyz.detach()), requires_grad=False)
        self.rng = np.random.RandomState(0)
        self.gen = torch.Generator().manual_seed(1)
        # the t table of each query, recorded by wrapping the querier's own (jittered) table
        self.t_seen = []
        t_for = npn.querier._t_for

        def recording_t_for(*a, **k):
            t = t_for(*a, **k)
            self.t_seen.append(t.clone())
            return t
        npn.querier._t_for = recording_t_for
        self.new_train_step()
        self.resync()
        self.history = []

    def new_train_step(self):
        """TrainStep as shipped (fused Adam on CUDA), or the reference's optimiser (torch.optim.Adam with its default foreach step) on
        the same loss."""
        self.ts = parallel.TrainStep(self.net)
        assert self.ts.opt_mlp.defaults["fused"] and self.ts.opt_pts.defaults["fused"]
        if self.optimiser == "foreach":
            ts = self.ts
            ts.opt_mlp = torch.optim.Adam(ts.mlp_params, lr=ts.opt_mlp.defaults["lr"], betas=(0.9, 0.999))
            ts.opt_pts = torch.optim.Adam(ts.pt_params, lr=ts.opt_pts.defaults["lr"], betas=(0.9, 0.999))

    def resync(self):
        """The state dict before the next step, and a module loaded from it."""
        self.sd = _snapshot(self.net)
        self.fresh = _load(self.sd, self.opt)

    def batch(self, kind, n):
        """n random pixels of the central 32 x 32 window (the shell's disc and some background); kind "miss": the rays reversed."""
        c = CFG.W // 2
        pix = self.rng.randint(c - 16, c + 16, size=(n, 2)).astype(np.float32)
        gt = torch.rand(n, 3, generator=self.gen)
        rays = scene.make_rays(CFG, pix)
        if kind == "miss":
            rays["raydir"] = -rays["raydir"]
        kw = {k: (rays[k].to(DEV) if k in ("raydir", "pixel_idx") else rays[k]) for k in FWD_KEYS}
        return kw, gt.to(DEV), rays

    def float64(self, q, rays, gt, sd):
        """Errors of the step's gradients against float64 autograd at the parameters `sd`, with the backward's masks."""
        net, ts = self.net, self.ts
        cam = rays["camrotc2w"][0]
        slopes, ex, _ = grad_check.kernel_masks(net, q, self.F, cam)
        hit = ex["ray_mask"].cpu() > 0
        pts_g = dict(xyz=sd["neural_points.xyz"].cpu().double(),
                     Rw2c=sd["neural_points.Rw2c"].cpu().double() if self.frames else torch.eye(3, dtype=torch.float64))
        names = dict(embedding="points_embeding", color="points_color", dir="points_dir", conf="points_conf")
        for k, name in names.items():
            pts_g[k] = sd["neural_points." + name].cpu().double().requires_grad_(True)
        mlp_g = {k[len("aggregator."):]: v.cpu().double().requires_grad_(True) for k, v in sd.items() if k.startswith("aggregator.")}
        sh = shade_oracle_rw2c.shade(pts_g, mlp_g, ex["sample_pidx"].cpu(), ex["sample_loc_w"].cpu(), rays["raydir"][0][hit],
                                     rays["campos"][0], cam, self.opt.vsize, rays["bg_color"][0], dtype=torch.float64,
                                     agg_intrp_order=int(self.opt.agg_intrp_order), slopes=slopes,
                                     raydist_mode_unit=int(self.opt.raydist_mode_unit))
        # TrainStep's own loss on the oracle's outputs (world 1: the counts are the local ones, at least 1)
        o = dict(ray_mask=ex["ray_mask"].cpu()[None], coarse_raycolor=sh["ray_color"][None], conf_coefficient=sh["conf_coefficient"][None])
        se, n_se, zo, n_zo = ts.loss_terms(o, gt.cpu().double())
        (se / max(float(n_se), 1.0) + ts.zero_one_weight * zo / max(float(n_zo), 1.0)).backward()
        npn = net.neural_points
        err = {k: grad_check.rel_point_errors(getattr(npn, names[k]).grad.cpu(), pts_g[k].grad).max() for k in ("embedding", "color", "dir")}
        cg, cr = npn.points_conf.grad.cpu().double().reshape(-1), pts_g["conf"].grad.reshape(-1)
        err["conf"] = grad_check.rel_point_errors(cg[1:, None], cr[1:, None]).max()
        for k, p in net.aggregator.named_parameters():
            err[k] = grad_check.rel_error(p.grad.cpu(), mlp_g[k].grad)
        n0 = int((ex["sample_pidx"].cpu().clamp(min=0) == 0).sum())
        cc0 = min(max(float(sd["neural_points.points_conf"][0, 0, 0]), 1e-4), 1.0)
        t0 = ts.zero_one_weight / (max(float(n_zo), 1.0) * (cc0 + 1e-3))
        err0 = (abs(cg[0] - cr[0]).item(), grad_check.point0_conf_bound(n0, cr[0], t0))
        return err, err0

    def step(self, kind, n):
        """One TrainStep.step with every check of the module header; returns the step's record."""
        net, ts = self.net, self.ts
        kw, gt, rays = self.batch(kind, n)
        sd, fresh = self.sd, self.fresh
        self.t_seen.clear()
        ts.step(kw, gt)
        net.check_errors()                      # no error flag of the forward or the backward
        out, q = ts.last["out"], net.last
        t = self.t_seen[-1]
        n_valid = int(q.counters["n_valid"])
        rec = dict(step=len(self.history) + 1, kind=kind, rays=n, n_valid=n_valid, hit=int(q.counters["R2"]),
                   tc_ws=0 if net._tc_ws is None else net._tc_ws.numel(), bwd_ws=net._bwd_ws.numel())
        # float64, before anything else runs a query on this module (the export reads the step's query workspace)
        if n_valid:
            rec["err"], rec["err0"] = self.float64(q, rays, gt, sd)
        else:
            rec["nonzero_grads"] = [k for k, p in net.named_parameters() if p.grad is not None and bool(p.grad.any())]
        # fresh-module identity of the training forward, with the step's t table replayed
        fresh.neural_points.querier._t_for = lambda near, far, R, device: t
        fo = fresh(**kw)
        fresh.check_errors()
        rec["forward_differs"] = _differs(out, fo, OUT_KEYS)
        # after the step: render_full of a module loaded from the new state
        self.resync()
        rec["render_differs"] = _differs(_render(net), _render(self.fresh), RENDER_KEYS)
        self.history.append(rec)
        self.report(rec)
        assert not rec["forward_differs"], "step %d: the training forward differs from a fresh module's in %s" % (rec["step"], rec["forward_differs"])
        if n_valid:
            rtol_points, rtol_mlp = grad_check.RTOL[(self.mode, self.precision)]
            for k, v in rec["err"].items():
                rtol = rtol_mlp if "." in k else rtol_points
                assert v <= rtol, "step %d: %s: %.3e of scale > %.1e" % (rec["step"], k, v, rtol)
            assert rec["err0"][0] <= rec["err0"][1], "step %d: points_conf of point 0: %.3e > %.3e" % ((rec["step"],) + rec["err0"])
        else:
            assert not rec["nonzero_grads"], "step %d (every ray misses): non-zero gradients of %s" % (rec["step"], rec["nonzero_grads"])
        assert not rec["render_differs"], "step %d: render_full after the step differs from a fresh module's in %s" % (rec["step"], rec["render_differs"])
        return rec

    def report(self, rec):
        if "err" in rec:
            e = rec["err"]
            pts = max(e[k] for k in ("embedding", "color", "dir", "conf"))
            mk = max((k for k in e if "." in k), key=e.get)
            f64 = "points=%.2e mlp=%.2e (%s) conf0=%.2e/%.2e" % (pts, e[mk], mk, rec["err0"][0], rec["err0"][1])
        else:
            f64 = "no valid sample, non-zero gradients: %s" % rec["nonzero_grads"]
        print("\n[train-session] F=%d frames=%d %s mode=%d %s step %d %s rays=%d hit=%d n_valid=%d tc_ws=%d bwd_ws=%d: %s "
              "forward differs: %s, render differs: %s" % (
                  self.F, self.frames, self.precision, self.mode, self.optimiser, rec["step"], rec["kind"], rec["rays"], rec["hit"],
                  rec["n_valid"], rec["tc_ws"], rec["bwd_ws"], f64, rec["forward_differs"] or "-", rec["render_differs"] or "-"))


def _grew_and_reused(sizes, n_valid):
    """A workspace grown after the first step, and one step with samples that ran in the one of the step before."""
    grew = any(sizes[i] > sizes[i - 1] for i in range(1, len(sizes)))
    reused = any(sizes[i] == sizes[i - 1] and n_valid[i] > 0 for i in range(1, len(sizes)))
    return grew and reused


CASES = {"F32": dict(F=32), "F63-frames": dict(F=63, frames=True), "F32-fp32": dict(F=32, precision="fp32", mode=1)}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("optimiser", ["fused", "foreach"])
def test_training_session_matches_fresh_module_and_float64(optimiser, case):
    s = Session(optimiser=optimiser, **CASES[case])
    for kind, n in PLAN:
        s.step(kind, n)
    nv = [r["n_valid"] for r in s.history]
    assert nv[2] == 0 and any(nv[j] < nv[i] for i in range(len(nv)) for j in range(i + 1, len(nv))) and nv[-1] > max(nv[:-1]), nv
    assert _grew_and_reused([r["bwd_ws"] for r in s.history], nv), [r["bwd_ws"] for r in s.history]
    if s.precision == "bf16x3":
        assert _grew_and_reused([r["tc_ws"] for r in s.history], nv), [r["tc_ws"] for r in s.history]


def test_grow_cycle_mid_session():
    """bench.py's grow cycle between steps: prune -> probe forward (opt.prob = 1, no gradient) -> grow_points -> a new TrainStep -> steps.
    The probe's outputs equal a fresh module's bit for bit, and every check holds on the steps after the grow."""
    s = Session()
    net, opt = s.net, s.opt
    npn = net.neural_points
    for kind, n in PLAN[:2]:
        s.step(kind, n)
    n_before = npn.xyz.shape[0]
    pruned = npn.prune(0.12)
    opt.prob, opt.is_train = 1, False
    kw, _, _ = s.batch("hit", 640)
    fresh = _load(_snapshot(net), opt)
    with torch.no_grad():
        pr = net(**kw)
        fr = fresh(**kw)
    net.check_errors()
    fresh.check_errors()
    opt.prob, opt.is_train = 0, True
    differs = _differs(pr, fr, sorted(set(pr) | set(fr)))
    # bench.py's rule (every 4th ray whose densest sample is opaque enough), at half the largest opacity instead of 0.5, which no sample of
    # the tiny shell reaches
    o = pr["ray_max_shading_opacity"][0, :, 0]
    keep = (o > 0.5 * o.max()) & (torch.arange(o.shape[0], device=DEV) % 4 == 0)
    add = [pr[k][0][keep] for k in ("ray_max_sample_loc_w", "shading_avg_embedding", "shading_avg_color", "shading_avg_dir", "shading_avg_conf")]
    npn.grow_points(*add)
    print("\n[train-session] grow cycle: %d points, %d pruned, %d grown; probe outputs differ from a fresh module's in: %s"
          % (n_before, pruned, int(keep.sum()), differs or "-"))
    assert 0 < pruned < n_before and int(keep.sum()) > 0
    assert not differs, "probe outputs differ from a fresh module's in %s" % differs
    s.new_train_step()                  # new parameters, new optimisers (train_ft.py:834-842)
    s.resync()
    for kind, n in PLAN[3:]:
        s.step(kind, n)


def _recycled_case(what, via):
    """Render with cloud A; install B and then C (same N) with editing_set_points, A freed before C is allocated; render.  `what`: the
    tensor that differs between the clouds (the embedding, or a uniform [3,3] Rw2c).  `via`: "allocator" (C's tensor allocated right
    after A's was freed) or "dlpack" (A and C are two tensor objects over one buffer, each of version 0: the same address and version
    without relying on the allocator's choice).  Returns None when the allocator put C elsewhere, else the differing render keys."""
    net, _, _ = harness.build_model(CFG, DEV, alpha_bias=3.0, seed=2)
    npn = net.neural_points
    base = {k: getattr(npn, k).detach().clone() for k in ("xyz", "points_embeding", "points_color", "points_dir", "points_conf")}
    values = dict(A=(1.0, 0.3), B=(-1.0, 1.1), C=(2.0, 2.0))     # (embedding scale, yaw of the rotation)
    buf = []

    def make(name):
        scale, yaw = values[name]
        x = base["points_embeding"] * scale if what == "embedding" else torch.from_numpy(scene.orbit_rotation(yaw, 0.2)).to(DEV)
        if via == "dlpack" and name != "B":
            if not buf:
                buf.append(torch.empty_like(x))
            buf[0].copy_(x)
            x = torch.from_dlpack(buf[0])
        return x

    def cloud(x):
        emb, R = (x, None) if what == "embedding" else (base["points_embeding"], x)
        return dict(points_xyz=base["xyz"], points_embeding=emb, points_color=base["points_color"], points_dir=base["points_dir"],
                    points_conf=base["points_conf"], Rw2c=R)

    a = make("A")
    npn.editing_set_points(**cloud(a))
    got_a = _render(net)
    a_key = (a.data_ptr(), a._version)
    b = make("B")                       # allocated while A is alive
    npn.editing_set_points(**cloud(b))
    del a                               # A's last reference
    c = make("C")
    c_key = (c.data_ptr(), c._version)
    print("\n[train-session] recycled %s via %s: A at (%#x, v%d), C at (%#x, v%d)" % (what, via, a_key[0], a_key[1], c_key[0], c_key[1]))
    if c_key != a_key:
        assert via == "allocator", "C is not at A's address with A's version"
        return None
    npn.editing_set_points(**cloud(c))
    got = _render(net)
    ref = harness.build_model(CFG, DEV, alpha_bias=3.0, seed=2)[0]
    ref.neural_points.editing_set_points(**cloud(c.clone()))
    want = _render(ref)
    assert _differs(got_a, want, RENDER_KEYS), "clouds A and C render alike: the case cannot tell a stale cache"
    return _differs(got, want, RENDER_KEYS)


@pytest.mark.parametrize("what", ["embedding", "rw2c"])
def test_recycled_address_is_not_taken_for_the_cached_tensor(what):
    """A new tensor at a freed tensor's address, with its version: the frozen table (embedding) and the host Rw2c must not be served
    from the freed tensor.  The case builds that collision through the allocator where it reproduces, else over one buffer."""
    differs = _recycled_case(what, "allocator")
    via = "allocator"
    if differs is None:
        via = "dlpack"
        differs = _recycled_case(what, via)
    print("[train-session] recycled %s (%s): render differs from a fresh module's in %s" % (what, via, differs or "-"))
    assert not differs, "render after a recycled %s differs from a fresh module's in %s" % (what, differs)
