"""TEST INFRASTRUCTURE ONLY -- CPU restatement (torch, eager, fp32 or fp64) of the reference's probe outputs for point growing
(opt.prob == 1, models/neural_points_volumetric_model.py:331-351) on a dense query export and the [R', SR] opacity of the same rays:

  weights           point_aggregators.py:421-429, :801-802 (linear, normalised over K), conf_coefficient neural_points.py:706-724
  arg-max slot      torch.max(coarse_point_opacity, -1): the first maximal slot wins a tie
  gather            torch.gather along SR of sample_loc_w, weight * conf_coefficient and the neighbours' attributes (the index of an
                    empty slot clamped to 0, neural_points.py:707: it reads point 0)
  far_dist          min over the K slots of |xyz - loc| (point 0 included for empty slots)
  averages          sum over K of attr * (weight * conf_coefficient)

fp32 is the reference's own op sequence (tests/test_probe_oracle.py pins it to tests/golden/tiny_probe.npz, the reference's run);
fp64 is the yardstick of the CUDA kernel (tests/test_gpu_probe.py).  `mutate` injects one defect (tests show the comparison
catches it): "no_conf" (weights without conf_coefficient), "last_max" (the last maximal slot wins a tie), "far_skip_empty" (empty
slots left out of far_dist).
"""
import torch

KEYS = ("ray_max_shading_opacity", "ray_max_sample_loc_w", "ray_max_far_dist", "shading_avg_color", "shading_avg_dir",
        "shading_avg_conf", "shading_avg_embedding")
MUTATIONS = ("no_conf", "last_max", "far_skip_empty")


def probe(points, sample_pidx, sample_loc_w, opacity, dtype=torch.float32, mutate=None):
    """points: dict(xyz [N,3], embedding [1,N,F], color [1,N,3], dir [1,N,3], conf [1,N,1]); sample_pidx [R',SR,K] (-1 pad);
    sample_loc_w [R',SR,3]; opacity [R',SR].  Returns dict KEYS -> [R',C] tensors of `dtype`, plus "slot" (int64 [R']) and
    "weight" ([R',K], weight * conf_coefficient at that slot)."""
    assert mutate in (None,) + MUTATIONS
    cv = lambda t: torch.as_tensor(t).to(dtype)
    xyz = cv(points["xyz"])
    attrs = [cv(points[k][0]) for k in ("color", "dir", "conf", "embedding")]
    pidx = torch.as_tensor(sample_pidx).long()
    loc_w = cv(sample_loc_w)
    op = cv(opacity)
    Rn, SR, K = pidx.shape
    pnt_mask = pidx >= 0
    idx = torch.clamp(pidx, min=0)
    s_xyz = xyz[idx]                                                                      # [R',SR,K,3]
    weight = pnt_mask * (1.0 / torch.clamp(torch.norm(s_xyz - loc_w[..., None, :], dim=-1), min=1e-6))
    weight = weight / torch.clamp(torch.sum(weight, dim=-1, keepdim=True), min=1e-8)
    c0 = attrs[2][idx][..., 0]
    conf_coefficient = c0 - (c0 - torch.clamp(c0, min=0.0001, max=1))                  # gradiant_clamp's value (:722-724)
    omax, oind = torch.max(op, dim=-1, keepdim=True)                                     # [R',1]
    if mutate == "last_max":
        oind = SR - 1 - torch.max(torch.flip(op, dims=[-1]), dim=-1, keepdim=True)[1]
    loc = torch.gather(loc_w, 1, oind[..., None].expand(-1, -1, 3)).squeeze(1)          # [R',3]
    wc = weight if mutate == "no_conf" else weight * conf_coefficient
    wsel = torch.gather(wc, 1, oind[..., None].expand(-1, -1, K)).squeeze(1)            # [R',K]
    sel = torch.gather(idx, 1, oind[..., None].expand(-1, -1, K)).squeeze(1)            # [R',K] clamped indices
    dist = torch.norm(xyz[sel] - loc[:, None, :], dim=-1)                                # [R',K]
    if mutate == "far_skip_empty":
        valid = torch.gather(pnt_mask, 1, oind[..., None].expand(-1, -1, K)).squeeze(1)
        dist = torch.where(valid, dist, torch.full_like(dist, float("inf")))
    out = dict(ray_max_shading_opacity=omax, ray_max_sample_loc_w=loc,
               ray_max_far_dist=torch.min(dist, dim=-1, keepdim=True)[0])
    for name, a in zip(("shading_avg_color", "shading_avg_dir", "shading_avg_conf", "shading_avg_embedding"), attrs):
        out[name] = torch.sum(a[sel] * wsel[..., None], dim=-2)
    out["slot"] = oind[:, 0]
    out["weight"] = wsel
    return out
