"""Feed-forward steps (run/train.py --feedforward 1, dev_scripts/ete/*.sh) in the fused module: a new point cloud from the network on
every call, in both scripts' configurations, with a seeded stand-in for the upstream network (a small MLP mapping per-point inputs to the
embedding and colour, as MVSNet + FeatureNet + premlp would; its own cost is printed as `cloud` and is not the real network's):
  F 32   world query flavour 1, SR 40, K 8, kernel 5^3, P 20, vsize 0.002, point modes 1; a 70x70-ray training patch
  F 63   perspective-frustum query, SR 40, kernel 3^3, point modes 01 (colour, dir and conf prepended); a 48x48-ray training patch
Both on about 600k points (three 640x512 depth maps' worth).  Each phase is timed alone between CUDA events, median of --steps after
--warmup, one new cloud per step:
  cloud     the stand-in network's forward and set_points (the reference's parameter=False assignments)
  build     the querier's build on the new cloud: its first query minus a second query of the same rays on the cached build
  query     the query of the training patch on the cached build
  table     the frozen kernel's per-point table (pnb_point_pre), rebuilt for every fresh cloud at eval
  shading   the training forward on the cached build minus the query
  backward  the loss's backward into the aggregator and the upstream network
  eval      one 2304-ray model.test() chunk: a new cloud, then the no_grad forward (build, query, table, frozen kernel)
Nothing here was compared with the reference's eager path.  The card's name and power limit are printed with the numbers.

    python bench_feedforward.py [--steps 10] [--warmup 2]
"""
import argparse
import json
import subprocess

import numpy as np
import torch
import torch.nn.functional as Fn

from pointnerf_b200 import harness, scene
from pointnerf_b200.ray_marching import NeuralPoints, NeuralPointsRayMarching, PointAggregator, points_desc_of

DEV = torch.device("cuda:0")
N_IN = 8


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        return [v.strip() for v in out.split(",")]
    except Exception:  # noqa: BLE001
        return [torch.cuda.get_device_name(0), "unknown"]


def upstream(th, x):
    h = torch.tanh(Fn.linear(x, th["w1"], th["b1"]))
    return Fn.linear(h, th["we"], th["be"])[None], torch.sigmoid(Fn.linear(h, th["wc"], th["bc"]))[None]


def set_points(npn, xyz, emb, color, pdir, conf):
    """The reference's NeuralPoints.set_points(parameter=False): plain assignments, the querier's cache left as it is."""
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


def setup(F):
    """(net, opt, per-point inputs, rays of the training patch, rays of one eval chunk: a 48x48 = 2304-ray patch)."""
    if F == 32:
        cfg = scene.SceneConfig("ete_32_600k", N=600_000, R_s=0.44, vsize=0.002, kernel_size=5, P=20, SR=40, H=512, W=512, near=1.0,
                                far=1.8, campos=(0.0, 0.0, -1.5))
        opt = harness.make_opt(cfg, wcoord_query=1, is_train=False)
        pts = scene.make_points(cfg)
        xyz, pdir, conf = pts["xyz"], pts["dir"], pts["conf"]

        def rays(side):
            return {k: v.to(DEV) for k, v in scene.make_rays(cfg, scene.centre_patch(cfg, side)).items()}
        train, ev = rays(70), rays(48)
        bias = 3.0
    else:
        cfg = scene.FrustumConfig("dtu_600k", N=600_000, H=512, W=640, focal=800.0)
        s = scene.make_frustum_scene(cfg)
        pts = scene.make_frustum_points(cfg, s)
        opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, **vars(scene.frustum_opt(cfg)))
        xyz, pdir, conf = pts["xyz"], pts["dir"], pts["conf"]

        def rays(side):
            x0, y0 = cfg.W // 2 - side // 2, cfg.H // 2 - side // 2
            px, py = np.meshgrid(np.arange(x0, x0 + side), np.arange(y0, y0 + side))
            pix = np.stack((px, py), -1).reshape(-1, 2)
            K = s["intrinsic"]
            d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ s["camrotc2w"].T
            d = d / np.linalg.norm(d, axis=-1, keepdims=True)
            return dict(campos=torch.from_numpy(s["campos"]).to(DEV)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(DEV)[None],
                        raydir=torch.from_numpy(d.astype(np.float32)).to(DEV)[None],
                        pixel_idx=torch.from_numpy(pix.astype(np.int32)).to(DEV)[None], h=cfg.H, w=cfg.W, intrinsic=s["intrinsic"],
                        near=cfg.near, far=cfg.far, bg_color=torch.ones(1, 3, device=DEV))
        train, ev = rays(48), rays(48)
        bias = 300.0
    agg = PointAggregator(opt, seed=2)
    with torch.no_grad():
        agg.alpha_branch[0].bias += bias
    net = NeuralPointsRayMarching(aggregator=agg.to(DEV), neural_points=NeuralPoints(opt, DEV), opt=opt)
    fixed = dict(xyz=xyz.to(DEV), dir=pdir.to(DEV), conf=conf.to(DEV),
                 x=torch.randn(xyz.shape[0], N_IN, generator=torch.Generator().manual_seed(3)).to(DEV))
    return net, opt, fixed, train, ev


def forward(net, d):
    return net(d["campos"], d["raydir"], bg_color=d["bg_color"], camrotc2w=d["camrotc2w"], pixel_idx=d["pixel_idx"], near=d["near"],
               far=d["far"], h=d["h"], w=d["w"], intrinsic=d["intrinsic"])


def query(net, d):
    """The module's own query of these rays (what forward() runs before the shading kernels)."""
    npn = net.neural_points
    if net.opt.wcoord_query == 0:
        view = {k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")}
        return net._frustum_query(d["campos"], d["camrotc2w"], d["near"], d["far"], view, DEV)
    return npn.querier.run_query(npn.xyz.detach(), d["raydir"][0].contiguous(), d["campos"][0].tolist(), float(d["near"].min()),
                                 float(d["far"].max()), want_counters=True)


class Timer:
    def __init__(self):
        self.ms = {}

    def __call__(self, name, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        b.synchronize()
        self.ms.setdefault(name, []).append(a.elapsed_time(b))
        return out


def run(F, steps, warmup):
    net, opt, fx, train, ev = setup(F)
    n_emb = 32 if F == 32 else 56
    g = torch.Generator().manual_seed(7)
    th = {k: v.to(DEV).requires_grad_(True) for k, v in dict(
        w1=torch.randn(32, N_IN, generator=g) / N_IN ** 0.5, b1=0.1 * torch.randn(32, generator=g),
        we=torch.randn(n_emb, 32, generator=g) * (0.5 / 32 ** 0.5), be=0.1 * torch.randn(n_emb, generator=g),
        wc=torch.randn(3, 32, generator=g) / 32 ** 0.5, bc=0.1 * torch.randn(3, generator=g)).items()}
    npn = net.neural_points
    t = Timer()
    N = fx["xyz"].shape[0]
    for i in range(warmup + steps):
        tm = t if i >= warmup else Timer()
        off = torch.tensor([1e-5 * i, 0.0, 0.0], device=DEV)

        def cloud(grad=True):
            with torch.no_grad():
                xyz = fx["xyz"] + off
            with torch.set_grad_enabled(grad):
                emb, col = upstream(th, fx["x"])
            set_points(npn, xyz, emb, col, fx["dir"], fx["conf"])
        tm("cloud", cloud)
        b0 = npn.querier.n_builds
        tm("build_and_query", lambda: query(net, train))
        assert npn.querier.n_builds == b0 + 1
        tm("query", lambda: query(net, train))
        out = tm("forward", lambda: forward(net, train))
        loss = (out["coarse_raycolor"] ** 2).sum()
        tm("backward", lambda: loss.backward())
        with torch.no_grad():
            net._pre_key = None
            pts = points_desc_of(npn)
            mlp = net._mlp.get(net.aggregator)
            tm("table", lambda: net._point_pre(mlp, pts, torch.cuda.current_stream().cuda_stream))

            def eval_chunk():
                cloud(grad=False)
                return forward(net, ev)
            tm("eval", eval_chunk)
        net.check_errors()
        th_grad = float(sum(v.grad.abs().sum() for v in th.values()))
        for v in th.values():
            v.grad = None
        net.aggregator.zero_grad(set_to_none=True)
    med = {k: float(np.median(v)) for k, v in t.ms.items()}
    res = dict(cloud=med["cloud"], build=med["build_and_query"] - med["query"], query=med["query"], table=med["table"],
               shading=med["forward"] - med["query"], backward=med["backward"], eval_chunk=med["eval"])
    q = net.last
    return dict(F=F, N=N, train_rays=int(train["raydir"].shape[1]), eval_rays=int(ev["raydir"].shape[1]),
                hit_rays_train=int(out["coarse_raycolor"].shape[1]), ms={k: round(v, 3) for k, v in res.items()},
                ms_min={k: round(min(v), 3) for k, v in t.ms.items()}, grad_into_upstream=th_grad > 0,
                last_eval_R=int(q.R))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_feedforward.py needs a GPU"
    name, power = card()
    for F in (32, 63):
        print(json.dumps(dict(metric="feed-forward step phases (median ms over %d steps, one new cloud each)" % a.steps, gpu=name,
                              power_limit=power, **run(F, a.steps, a.warmup))))


if __name__ == "__main__":
    main()
