"""Launched by torchrun (NCCL, one rank per GPU) from tests/test_gpu_dist.py or by hand:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P tests/dist_train_check.py [config]

Checks of the multi-GPU paths on real GPUs (SURVEY 8e):
  1. optimisation: parallel.TrainStep, each rank on ITS rays of the step -> the exchanged gradient equals - to fp32 summation order - the
     gradient of the un-sharded step on the union of the rays (run by every rank on a second copy of the model), and after k Adam steps the
     replicas are BIT-identical on every rank (identical all-reduced gradients + identical Adam), and each rank's module renders what a
     module loaded from its own state dict renders (its weight packs and frozen table follow the fused Adam's writes);
  2. render: one frame interleave-sharded over the ranks + all-gather == the frame rendered by one rank, bit for bit;
  3. grow: every rank probes its own frames, allgather_new_points, grow_points -> identical clouds, grid rebuilt, render still agrees.
Prints one JSON line on rank 0; exit code != 0 on any failure."""
import copy
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pointnerf_b200 import checkpoint, harness, parallel, point_query, scene  # noqa: E402


def fwd_kwargs(cfg, pixels, dev):
    rays = {k: v.to(dev) for k, v in scene.make_rays(cfg, pixels).items()}
    return dict(campos=rays["campos"], raydir=rays["raydir"], bg_color=rays["bg_color"], camrotc2w=rays["camrotc2w"],
                pixel_idx=rays["pixel_idx"], near=rays["near"], far=rays["far"], h=rays["h"], w=rays["w"], intrinsic=rays["intrinsic"])


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "chair_plumbing"
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    cfg = scene.CONFIGS[name]
    res = {}
    # ---------------- 1. optimisation
    for sparse in (False, True):
        net, _, _ = harness.build_model(cfg, dev, alpha_bias=3.0)
        ref, _, _ = harness.build_model(cfg, dev, alpha_bias=3.0)
        ts = parallel.TrainStep(net, world=world, rank=rank, sparse_points=sparse)
        ts_ref = parallel.TrainStep(ref, world=1, rank=0)
        rng = np.random.RandomState(0)
        g = torch.Generator().manual_seed(1)
        n_rays = 1024

        def batch():
            c = cfg.W // 2
            px = rng.randint(c - 150, c + 150, size=(n_rays,)).astype(np.float32)
            py = rng.randint(c - 150, c + 150, size=(n_rays,)).astype(np.float32)
            return np.stack([px, py], -1), torch.rand(n_rays, 3, generator=g).to(dev)

        sel = np.arange(rank, n_rays, world)
        sel_t = torch.from_numpy(sel).to(dev)
        # (a) the exchanged gradient of the sharded step == the gradient of the un-sharded step on the union of the rays
        #     (compared BEFORE Adam: its sign-like first steps would amplify rounding noise of near-zero gradient entries)
        pix, gt = batch()
        l_sh = ts.gradients(fwd_kwargs(cfg, pix[sel], dev), gt[sel_t]).clone()
        dist.all_reduce(l_sh)
        l_ref = ts_ref.gradients(fwd_kwargs(cfg, pix, dev), gt)
        assert abs(float(l_sh) - float(l_ref)) <= 1e-5 * max(abs(float(l_ref)), 1e-3), (float(l_sh), float(l_ref))
        gerr = 0.0
        for (n1, p1), (n2, p2) in zip(net.named_parameters(), ref.named_parameters()):
            if p2.grad is None:
                assert p1.grad is None, n1
                continue
            sc = float(p2.grad.abs().max().clamp_min(1e-12))
            e = float((p1.grad - p2.grad).abs().max()) / sc
            assert e <= 2e-4, "gradient of %s: sharded vs un-sharded %.3e of scale" % (n1, e)
            gerr = max(gerr, e)
        # (b) k optimisation steps: the replicas stay bit-identical without a broadcast, the loss tracks the un-sharded run
        for it in range(3):
            pix, gt = batch()
            loss = ts.step(fwd_kwargs(cfg, pix[sel], dev), gt[sel_t])
            loss_ref = ts_ref.step(fwd_kwargs(cfg, pix, dev), gt)
            assert abs(float(loss) - float(loss_ref)) <= 2e-3 * max(abs(float(loss_ref)), 1e-3), (it, float(loss), float(loss_ref))
        net.check_errors()
        flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
        alls = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(alls, flat)
        assert all(torch.equal(alls[0], a) for a in alls), "replicas differ across ranks (sparse=%s)" % sparse
        # a TrainStep compared with a TrainStep cannot see weights the module failed to refresh: compare with a module loaded from the state
        loaded = checkpoint.load_checkpoint({k: v.detach().clone() for k, v in net.state_dict().items()}, copy.copy(net.opt), dev)
        rd = scene.make_rays(cfg, scene.centre_patch(cfg, 100))["raydir"][0].to(dev)
        t = point_query.host_t_table(cfg.near, cfg.far, cfg.D).to(dev)
        with torch.no_grad():
            got, want = (m.render_full(list(cfg.campos), rd, torch.eye(3), cfg.near, cfg.far, [1., 1., 1.], t=t) for m in (net, loaded))
        net.check_errors()
        loaded.check_errors()
        differs = [k for k in got if not torch.equal(got[k], want[k])]
        assert not differs, "rank %d (sparse=%s): render_full after the steps differs from a module loaded from the state dict in %s" % (
            rank, sparse, differs)
        moved = (flat - torch.cat([p.detach().reshape(-1) for p in harness.build_model(cfg, dev, alpha_bias=3.0)[0].parameters()])).abs().max().item()
        assert moved > 1e-3
        err = gerr
        res["train_sparse" if sparse else "train_dense"] = dict(max_gradient_diff_vs_unsharded_rel=err, parameters_moved_by=moved, loss=float(loss),
                                                                replicas_bit_identical=True)
    # ---------------- 2. render: interleave-sharded frame + all-gather == single-rank frame
    # (a centre patch keeps ~22 valid samples per ray, more than the 10 the render_full() workspace heuristic starts from: size it for SR)
    net, _, _ = harness.build_model(cfg, dev, alpha_bias=3.0, pnb_max_valid_per_ray=cfg.SR)
    full = scene.make_rays(cfg, scene.centre_patch(cfg, 300))
    rd = full["raydir"][0]
    R = rd.shape[0]
    cam = (list(cfg.campos), torch.eye(3), cfg.near, cfg.far, [1., 1., 1.])
    with torch.no_grad():
        whole = net.render_full(cam[0], rd.to(dev), cam[1], cam[2], cam[3], cam[4])["coarse_raycolor"][0].clone()
        ids = parallel.shard_indices(R, rank, world)
        part = net.render_full(cam[0], rd[ids].contiguous().to(dev), cam[1], cam[2], cam[3], cam[4])["coarse_raycolor"][0]
    net.check_errors()
    got = parallel.gather_interleaved(parallel.pad_rows(part, parallel.padded_shard_len(R, world)), R, world)
    assert torch.equal(got, whole), "sharded frame differs from the single-rank frame"
    res["render_sharded_bit_identical"] = True
    # ---------------- 3. grow: rank-local new points, merged in rank order on every rank
    gg = torch.Generator().manual_seed(100 + rank)
    n_new = 5 + 3 * rank
    add = [0.05 * torch.randn(n_new, 3, generator=gg).to(dev) + torch.tensor([0.0, 0.0, -cfg.R_s], device=dev),
           0.5 * torch.randn(n_new, 32, generator=gg).to(dev), torch.rand(n_new, 3, generator=gg).to(dev),
           torch.nn.functional.normalize(torch.randn(n_new, 3, generator=gg), dim=-1).to(dev), torch.rand(n_new, 1, generator=gg).to(dev)]
    merged = parallel.allgather_new_points(*add, world)
    n_before = net.neural_points.xyz.shape[0]
    net.neural_points.grow_points(*merged)
    assert net.neural_points.xyz.shape[0] == n_before + sum(5 + 3 * r for r in range(world))
    h = torch.cat([p.detach().reshape(-1) for p in net.neural_points.parameters()])
    alls = [torch.empty_like(h) for _ in range(world)]
    dist.all_gather(alls, h)
    assert all(torch.equal(alls[0], a) for a in alls), "clouds differ after the grow merge"
    with torch.no_grad():
        part = net.render_full(cam[0], rd[ids].contiguous().to(dev), cam[1], cam[2], cam[3], cam[4])["coarse_raycolor"][0]
        whole2 = net.render_full(cam[0], rd.to(dev), cam[1], cam[2], cam[3], cam[4])["coarse_raycolor"][0]
    net.check_errors()
    got = parallel.gather_interleaved(parallel.pad_rows(part, parallel.padded_shard_len(R, world)), R, world)
    assert torch.equal(got, whole2) and not torch.equal(whole2, whole), "render after the grow merge"
    res["grow_merge_identical"] = True
    if rank == 0:
        print(json.dumps(dict(check="dist_train_check", world=world, config=name, **res)))
    dist.destroy_process_group()


if __name__ == "__main__":
    try:
        main()
    except Exception:
        import traceback
        print("RANK %s FAILED:\n%s" % (os.environ.get("RANK"), traceback.format_exc()), flush=True)
        raise
