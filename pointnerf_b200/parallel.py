"""Multi-GPU plumbing of the hot path (SURVEY.md 8e): one process per GPU, neural point cloud / voxel grid / MLP
replicated, rays interleave-sharded (ray i -> rank i % world).  Two collectives only:
  * render:        one all_gather of the [R/world, 3] colours per image (7.7 MB @800x800), re-interleaved;
  * optimisation:  one all_reduce(sum) over the point-feature and MLP gradients per step -- every rank then takes
                   the same dense Adam step (the reference's optimisers, mvs_points_volumetric_model.py:87-91), so
                   replicas stay bit-identical without a broadcast.
Backend: NCCL over NVLink on the GPU box; the same code runs on gloo/CPU tensors for the host-logic tests.
"""
import torch
import torch.distributed as dist


def shard_indices(R, rank, world, device="cpu"):
    """Ray ids of this rank: rank, rank+world, ...  (hit density is spatially clustered -> interleave, not blocks)."""
    return torch.arange(rank, R, world, device=device)


def padded_shard_len(R, world):
    return (R + world - 1) // world


def gather_interleaved(local, R, world, group=None):
    """local: [ceil(R/world), C] rows of this rank (rows beyond its share are padding).  Returns the full [R, C]
    tensor in original ray order on every rank (one all_gather)."""
    n = padded_shard_len(R, world)
    assert local.shape[0] == n, "pad the local shard to ceil(R/world) rows"
    out = torch.empty((world, n) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    if world > 1:
        dist.all_gather_into_tensor(out.view(-1, *local.shape[1:]), local.contiguous(), group=group)
    else:
        out[0] = local
    # out[g, j] is ray j*world + g
    full = out.transpose(0, 1).reshape(n * world, *local.shape[1:])
    return full[:R]


def pad_rows(t, n):
    if t.shape[0] == n:
        return t
    pad = torch.zeros((n - t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    return torch.cat([t, pad], dim=0)


def allreduce_gradients(params, world, group=None, average=False):
    """One flat all_reduce(sum) over the gradients of `params` (point features + MLP), written back in place."""
    grads = [p.grad for p in params if p.grad is not None]
    if world <= 1 or not grads:
        return 0
    flat = torch.cat([g.reshape(-1) for g in grads])
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    if average:
        flat /= world
    off = 0
    for g in grads:
        n = g.numel()
        g.copy_(flat[off:off + n].view_as(g))
        off += n
    return flat.numel()


# ---- point growing across ranks (SURVEY.md 8e, "Grow / prune"): probe_hole (run/train_ft.py:417-530) renders whole
# training frames -> shard FRAMES across ranks, then one variable-length all-gather (counts, then payload) of the new
# points; every rank appends them in rank order, so the replicated point clouds stay identical without a broadcast.
# Prune needs no communication: it is a deterministic function of the replicated points_conf.

def shard_frames(frame_ids, rank, world):
    """Frames this rank probes: round-robin over the (already shuffled / ranked) id list, as rays are."""
    return list(frame_ids)[rank::world]


def allgather_varlen(t, world, group=None):
    """t: [n_rank, C] (n differs per rank).  Returns the [sum n, C] concatenation in rank order on every rank:
    one all_gather of the counts, one of the payload padded to the largest count."""
    if world <= 1:
        return t
    cnt = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    counts = torch.empty(world, dtype=torch.int64, device=t.device)
    dist.all_gather_into_tensor(counts, cnt, group=group)
    counts = counts.tolist()
    m = max(counts)
    if m == 0:
        return t
    buf = torch.empty((world, m) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(buf.view(world * m, *t.shape[1:]), pad_rows(t.contiguous(), m), group=group)
    return torch.cat([buf[g, :counts[g]] for g in range(world)], dim=0)


def allgather_new_points(add_xyz, add_embedding, add_color, add_dir, add_conf, world, group=None):
    """The five tensors probe_hole returns (train_ft.py:530), gathered as ONE payload [n, 3+C+3+3+1] so that a rank
    cannot interleave them differently; returns them split again, identical on every rank."""
    c = add_embedding.shape[1]
    packed = torch.cat([add_xyz, add_embedding, add_color, add_dir, add_conf], dim=1)
    allp = allgather_varlen(packed, world, group=group)
    return allp[:, 0:3], allp[:, 3:3 + c], allp[:, 3 + c:6 + c], allp[:, 6 + c:9 + c], allp[:, 9 + c:10 + c]


# ---- sparse gradient exchange (SURVEY.md 8e, "sparse alternative"): a step touches at most 3600*SR*K point rows, so for large
# clouds (N = 5 M: 780 MB of dense gradients per all-reduce) exchanging only the touched rows is far cheaper.

def allreduce_rows_sparse(grad, world, group=None):
    """grad: [N, C] or [1, N, C] dense gradient of a per-point tensor, non-zero only on the rows this rank touched.  In place:
    grad <- sum over ranks, identical bit for bit on every rank (each rank's rows are unique, and the ranks' contributions are
    added in rank order - no atomics on duplicate indices).  One variable-length all-gather of [index | row] pairs.
    Returns the number of rows exchanged."""
    if world <= 1:
        return 0
    g2 = grad.view(-1, grad.shape[-1])
    idx = torch.nonzero(g2.abs().sum(dim=1) > 0)[:, 0]
    payload = torch.cat([idx.to(g2.dtype)[:, None], g2[idx]], dim=1) if idx.numel() else g2.new_zeros((0, g2.shape[1] + 1))
    assert g2.shape[0] < (1 << 24) or g2.dtype == torch.float64, "row indices travel as fp32: N must stay below 2^24"
    cnt = torch.tensor([payload.shape[0]], dtype=torch.int64, device=g2.device)
    counts = torch.empty(world, dtype=torch.int64, device=g2.device)
    dist.all_gather_into_tensor(counts, cnt, group=group)
    counts = counts.tolist()
    allp = allgather_varlen(payload, world, group=group)
    g2.zero_()
    off = 0
    for n in counts:                                       # rank order; indices are unique within a rank's block
        if n:
            blk = allp[off:off + n]
            g2.index_add_(0, blk[:, 0].to(torch.int64), blk[:, 1:])
        off += n
    return int(sum(counts))


# ---- one optimisation step, data-parallel over rays (SURVEY.md 8e; the reference's single-GPU step is
# models/mvs_points_volumetric_model.py:87-118 + models/base_rendering_model.py:533-662)
class TrainStep:
    """Per-scene optimisation step on `world` ranks: every rank runs forward + backward on ITS rays of the step, the gradients
    are summed across ranks (point rows: dense all-reduce or the sparse touched-rows exchange; MLP: one flat all-reduce) and
    every rank takes the same two Adam steps (MLP lr, point-feature plr - the reference's two optimisers), so the replicas stay
    bit-identical without a broadcast.

    The loss is the reference's (`color_loss_items = coarse_raycolor` MSE over the rays that hit, weight 1, plus the zero-one
    log-barrier on conf_coefficient, weight 1e-4), written in SUM form and divided by the GLOBAL counts (one 2-element
    all-reduce before the backward): the summed gradient is then exactly the gradient of the un-sharded step on the union of
    the ranks' rays, whatever the split of hit rays between the ranks."""

    def __init__(self, net, world=1, rank=0, lr=5e-4, plr=2e-3, zero_one_weight=1e-4, sparse_points=False, group=None):
        self.net, self.world, self.rank, self.group = net, world, rank, group
        self.zero_one_weight = zero_one_weight
        self.sparse_points = sparse_points
        self.mlp_params = [p for p in net.aggregator.parameters() if p.requires_grad]
        self.pt_params = [p for p in net.neural_points.parameters() if p.requires_grad]
        # one fused kernel per optimiser on the GPU (the default multi-tensor path is ~12 launches); same arithmetic on every rank
        fused = all(p.is_cuda for p in self.mlp_params + self.pt_params)
        self.opt_mlp = torch.optim.Adam(self.mlp_params, lr=lr, betas=(0.9, 0.999), fused=fused)
        self.opt_pts = torch.optim.Adam(self.pt_params, lr=plr, betas=(0.9, 0.999), fused=fused)
        self.last = {}

    def loss_terms(self, out, gt):
        """Local SUMS and counts: (sum of squared colour errors over hit rays and channels, #terms), (sum of -log(conf + 1e-3), #terms)."""
        mask = out["ray_mask"][0] > 0
        pred = out["coarse_raycolor"][0]
        # (boolean-mask indexing would synchronise for the count, which is pred.shape[0])
        rows = torch.nonzero_static(mask, size=pred.shape[0])[:, 0]
        se = ((pred - gt.index_select(0, rows)) ** 2).sum()
        n_se = pred.numel()
        cc = out.get("conf_coefficient", None)
        if cc is not None and cc.numel() > 0:
            zo = (-torch.log(cc + 1e-3)).sum()
            n_zo = cc.numel()
        else:
            zo, n_zo = pred.sum() * 0.0, 0
        return se, n_se, zo, n_zo

    def gradients(self, fwd_kwargs, gt, mark=None):
        """Forward + backward on this rank's rays and the gradient exchange, WITHOUT the optimiser step: afterwards every rank holds the
        gradient of the un-sharded step on the union of the ranks' rays in `p.grad`.  Returns the local loss term (its sum over the ranks
        is the global loss)."""
        mark = mark or (lambda name: None)
        mark("start")
        out = self.net(**fwd_kwargs)
        se, n_se, zo, n_zo = self.loss_terms(out, gt)
        if self.world > 1:      # the global counts stay on the device: no host synchronisation between forward and backward
            cnt = torch.tensor([float(n_se), float(n_zo)], dtype=torch.float64, device=se.device)
            dist.all_reduce(cnt, op=dist.ReduceOp.SUM, group=self.group)
            cnt = torch.clamp(cnt, min=1.0).to(se.dtype)
            n_se_g, n_zo_g = cnt[0], cnt[1]
        else:
            n_se_g, n_zo_g = max(float(n_se), 1.0), max(float(n_zo), 1.0)
        loss_local = se / n_se_g + self.zero_one_weight * zo / n_zo_g
        self.opt_mlp.zero_grad(set_to_none=True)      # the backward hands over fresh gradient tensors: no zero-fill + accumulate per step
        self.opt_pts.zero_grad(set_to_none=True)
        mark("forward")
        loss_local.backward()
        mark("backward")
        if self.world > 1:
            if self.sparse_points:
                for p in self.pt_params:
                    if p.grad is not None:
                        allreduce_rows_sparse(p.grad, self.world, group=self.group)
                allreduce_gradients(self.mlp_params, self.world, group=self.group)
            else:
                allreduce_gradients(self.pt_params + self.mlp_params, self.world, group=self.group)
        mark("exchange")
        self.last = dict(out=out, n_hit_terms=n_se_g, n_conf_terms=n_zo_g)
        return loss_local.detach()

    def step(self, fwd_kwargs, gt, mark=None):
        """fwd_kwargs: the arguments of NeuralPointsRayMarching.forward for THIS rank's rays; gt: [R_local, 3] colours of those rays.
        mark: optional callable(name) invoked between the phases (forward / backward / exchange / adam) - bench.py records CUDA
        events there.  Returns the global loss (a 0-d tensor, identical on every rank)."""
        loss = self.gradients(fwd_kwargs, gt, mark=mark).clone()
        self.opt_mlp.step()
        self.opt_pts.step()
        # the fused Adam kernels write the parameters without advancing their autograd version, which is what the module's weight
        # packs and its frozen per-point table are keyed on: advance it here, or the next call would shade with the old weights
        torch.autograd.graph.increment_version(self.mlp_params + self.pt_params)
        (mark or (lambda name: None))("adam")
        if self.world > 1:
            dist.all_reduce(loss, op=dist.ReduceOp.SUM, group=self.group)
        return loss
