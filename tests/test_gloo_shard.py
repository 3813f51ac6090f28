"""CPU, world_size 2 over gloo: the N>1 host logic (interleaved ray sharding, colour all-gather, gradient all-reduce)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from pointnerf_b200 import parallel


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, R, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)
        full = torch.rand(R, 3, generator=g)                      # what a single process would render
        ids = parallel.shard_indices(R, rank, world)
        local = parallel.pad_rows(full[ids], parallel.padded_shard_len(R, world))
        out = parallel.gather_interleaved(local, R, world)
        ok_gather = torch.equal(out, full)
        # gradient all-reduce: each rank holds the gradient of its own rays; the sum must equal the unsharded one
        w = torch.nn.Parameter(torch.ones(5, 3))
        feats = torch.rand(R, 5, generator=g)
        (feats[ids] @ w).sum().backward()
        n = parallel.allreduce_gradients([w], world)
        ref = feats.sum(0)[:, None].expand(5, 3)
        ok_grad = torch.allclose(w.grad, ref, rtol=1e-6, atol=1e-6) and n == 15
        # point growing: each rank probed its own frames and found a different number of new points
        assert parallel.shard_frames(list(range(7)), rank, world) == ([0, 2, 4, 6] if rank == 0 else [1, 3, 5])
        n_new = [3, 0] if R == 10 else [2, 5]
        gg = torch.Generator().manual_seed(100 + rank)
        mine = [torch.rand(n_new[rank], c, generator=gg) for c in (3, 32, 3, 3, 1)]
        got = parallel.allgather_new_points(*mine, world)
        exp = [[], [], [], [], []]
        for g_ in range(world):
            g2 = torch.Generator().manual_seed(100 + g_)
            for i, c in enumerate((3, 32, 3, 3, 1)):
                exp[i].append(torch.rand(n_new[g_], c, generator=g2))
        ok_grow = all(torch.equal(a, torch.cat(e, 0)) for a, e in zip(got, exp)) and got[0].shape[0] == sum(n_new)
        # sparse gradient exchange: each rank touched a few (overlapping) point rows
        N, C = 50, 4
        gs = torch.Generator().manual_seed(7)
        dense = [torch.zeros(N, C) for _ in range(world)]
        for g_ in range(world):
            rows = torch.randperm(N, generator=gs)[:9 + 3 * g_]
            dense[g_][rows] = torch.randn(len(rows), C, generator=gs)
        mine = dense[rank].clone()[None]                              # the [1, N, C] shape of points_embeding.grad
        n_rows = parallel.allreduce_rows_sparse(mine, world)
        expect = dense[0].clone()
        for g_ in range(1, world):
            expect += dense[g_]                                       # same rank order -> bit-identical
        ok_sparse = torch.equal(mine[0], expect) and n_rows == sum(int((d.abs().sum(1) > 0).sum()) for d in dense)
        ret[rank] = (ok_gather, ok_grad and ok_grow and ok_sparse)
    finally:
        dist.destroy_process_group()


def test_world2_gloo_shard_gather_allreduce():
    for R in (10, 11):                                            # even and ragged split
        mgr = mp.Manager()
        ret = mgr.dict()
        port = _free_port()
        mp.spawn(_worker, args=(2, port, R, ret), nprocs=2, join=True)
        assert dict(ret) == {0: (True, True), 1: (True, True)}, (R, dict(ret))


def test_single_process_paths():
    full = torch.arange(21.0).view(7, 3)
    assert torch.equal(parallel.gather_interleaved(full, 7, 1), full)
    assert parallel.shard_indices(7, 1, 3).tolist() == [1, 4]
    assert parallel.padded_shard_len(7, 3) == 3
    t = torch.rand(4, 5)
    assert parallel.allgather_varlen(t, 1) is t


# ---- TrainStep on gloo (world 2) with a small differentiable stand-in for the CUDA network: same output dict
# (coarse_raycolor over the hit rays, ray_mask, conf_coefficient), parameters under .aggregator / .neural_points
class _StubPoints(torch.nn.Module):
    def __init__(self, n):
        super().__init__()
        g = torch.Generator().manual_seed(3)
        self.points_embeding = torch.nn.Parameter(torch.rand(1, n, 4, generator=g))
        self.points_conf = torch.nn.Parameter(0.2 + 0.6 * torch.rand(1, n, 1, generator=g))


class _StubNet(torch.nn.Module):
    def __init__(self, n=40):
        super().__init__()
        torch.manual_seed(5)
        self.aggregator = torch.nn.Linear(4, 3)
        self.neural_points = _StubPoints(n)

    def forward(self, ray_ids=None):
        n = self.neural_points.points_embeding.shape[1]
        hit = (ray_ids % 3) != 0                                   # a ray "hits" unless its id is a multiple of 3
        ids = ray_ids[hit]
        nb = torch.stack([ids % n, (ids * 7 + 1) % n], dim=1)      # two "neighbour points" per hit ray (rows shared between rays)
        feat = self.neural_points.points_embeding[0][nb].sum(1)
        col = torch.sigmoid(self.aggregator(feat))
        return dict(coarse_raycolor=col[None], ray_mask=hit[None].to(torch.int8),
                    conf_coefficient=self.neural_points.points_conf[0][nb][None, :, None, :, 0])


def _train_worker(rank, world, port, sparse, ret):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        R = 31
        g = torch.Generator().manual_seed(11)
        gt = torch.rand(R, 3, generator=g)
        net = _StubNet().double()
        ts = parallel.TrainStep(net, world=world, rank=rank, sparse_points=sparse)
        ref_net = _StubNet().double()
        ref = parallel.TrainStep(ref_net, world=1, rank=0)
        for it in range(3):
            ids_all = (torch.arange(R) * 5 + it) % 97              # the step's rays
            mine = parallel.shard_indices(R, rank, world)
            loss = ts.step(dict(ray_ids=ids_all[mine]), gt[mine])
            loss_ref = ref.step(dict(ray_ids=ids_all), gt)        # every rank also runs the un-sharded step on the union of the rays
            assert torch.allclose(loss, loss_ref, rtol=1e-12, atol=1e-12), (float(loss), float(loss_ref))
        same = all(torch.allclose(a, b, rtol=1e-10, atol=1e-12) for a, b in zip(net.parameters(), ref_net.parameters()))
        flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
        others = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(others, flat)
        ident = all(torch.equal(others[0], o) for o in others)     # replicas bit-identical
        ret[rank] = (same, ident)
    finally:
        dist.destroy_process_group()


def test_fused_adam_step_advances_parameter_versions(monkeypatch):
    """torch's fused Adam (what TrainStep builds on CUDA) writes the parameters without advancing their autograd version, which keys the
    module's weight packs and frozen per-point table: TrainStep.step advances it itself.  CPU fused Adam stands in for the CUDA one."""
    adam = torch.optim.Adam
    monkeypatch.setattr(parallel.torch.optim, "Adam", lambda params, **kw: adam(params, **dict(kw, fused=True)))
    net = _StubNet()
    ts = parallel.TrainStep(net)
    assert ts.opt_mlp.defaults["fused"] and ts.opt_pts.defaults["fused"]
    params = ts.mlp_params + ts.pt_params
    R = 31
    gt = torch.rand(R, 3, generator=torch.Generator().manual_seed(11))
    for it in range(2):
        before = [(p.detach().clone(), p._version) for p in params]
        ts.step(dict(ray_ids=(torch.arange(R) * 5 + it) % 97), gt)
        for p, (b, v) in zip(params, before):
            assert not torch.equal(p.detach(), b), "the step did not move a parameter"
            assert p._version > v, "a parameter moved without advancing its version"


def test_world2_gloo_train_step_matches_unsharded_and_replicas_identical():
    for sparse in (False, True):
        mgr = mp.Manager()
        ret = mgr.dict()
        mp.spawn(_train_worker, args=(2, _free_port(), sparse, ret), nprocs=2, join=True)
        assert dict(ret) == {0: (True, True), 1: (True, True)}, (sparse, dict(ret))
