"""CPU: per-point world->canonical rotations (neural_points.Rw2c [N,3,3], the frames of edited / composed scenes, run/editing.py).
The oracle (oracle/shade_oracle_rw2c.py) against the reference-generated fixture tests/golden/tiny_rw2c (two objects split by sign(x), each in its own frame), the
host container's bookkeeping of the per-point rows, and the checkpoint validation."""
import numpy as np
import pytest
import torch

from oracle import golden, shade_oracle_rw2c
from pointnerf_b200 import checkpoint, harness, scene
from pointnerf_b200.ray_marching import NeuralPoints


def _mlp_from(fx):
    return {k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")}


def _oracle_fixture_run(fx, Rw2c, dtype=torch.float32):
    cfg = scene.CONFIGS["tiny"]
    pts = scene.make_points(cfg)
    pts["Rw2c"] = Rw2c
    rays = scene.make_rays(cfg, fx["pixels"])
    mask = torch.from_numpy(fx["ray_mask"]) > 0
    pts_g = {k: v.clone().to(dtype).requires_grad_(k in ("embedding", "color", "dir", "conf")) for k, v in pts.items()}
    mlp = {k: v.clone().to(dtype).requires_grad_(True) for k, v in _mlp_from(fx).items()}
    sh = shade_oracle_rw2c.shade(pts_g, mlp, torch.from_numpy(fx["sample_pidx"]), torch.from_numpy(fx["sample_loc_w"]),
                                 rays["raydir"][0][mask], torch.tensor(cfg.campos), torch.eye(3), [cfg.vsize] * 3, torch.ones(3), dtype=dtype)
    return sh, pts_g, mlp


def test_fixture_is_an_edit_with_mixed_frames(golden_dir):
    """The fixture exercises what it is for: two frames, samples whose neighbours come from both objects (the slot-0 view frame rule
    decides their view direction), and colours far from the identity-frame render of the same scene and weights."""
    fx = golden.load(golden_dir, "tiny_rw2c")
    R = torch.from_numpy(fx["Rw2c"])
    xyz = scene.make_points(scene.CONFIGS["tiny"])["xyz"]
    assert torch.equal(R, scene.edit_frames(xyz))
    left = xyz[:, 0] < 0
    assert torch.all(R[left] == R[left][0]) and torch.all(R[~left] == R[~left][0]) and not torch.equal(R[left][0], R[~left][0])
    eye = torch.eye(3)
    for M in (R[left][0], R[~left][0]):
        assert torch.allclose(M @ M.T, eye, atol=1e-6) and not torch.allclose(M, eye, atol=0.1)
    pidx = torch.from_numpy(fx["sample_pidx"]).long()
    side = torch.where(pidx >= 0, left[pidx.clamp(min=0)].long(), torch.full_like(pidx, -1))
    mixed = ((side == 0).any(-1) & (side == 1).any(-1)).sum().item()
    assert mixed >= 50, mixed
    plain = golden.load(golden_dir, "tiny_opaque")
    assert np.array_equal(plain["ray_mask"], fx["ray_mask"])
    assert np.abs(plain["coarse_raycolor"] - fx["coarse_raycolor"]).max() > 1e-2


def test_oracle_matches_reference_fixture(golden_dir):
    """Forward bit for bit (the oracle restates the reference's own batched ops), gradients to fp32 rounding (autograd)."""
    fx = golden.load(golden_dir, "tiny_rw2c")
    sh, pts_g, mlp = _oracle_fixture_run(fx, torch.from_numpy(fx["Rw2c"]))
    for a, b in (("ray_color", "coarse_raycolor"), ("opacity", "coarse_point_opacity"), ("bg_T", "coarse_is_background"),
                 ("weight", "weight"), ("conf_coefficient", "conf_coefficient"), ("blend_weight", "blend_weight")):
        assert np.array_equal(sh[a].detach().numpy(), fx[b]), a
    loss = (sh["ray_color"] ** 2).sum() + 1e-3 * sh["conf_coefficient"].sum()      # the loss of oracle/make_golden_rw2c.py
    loss.backward()
    for k, g in (("embedding", "grad_embedding"), ("color", "grad_color"), ("dir", "grad_dir"), ("conf", "grad_conf")):
        ref = fx[g]
        assert np.abs(pts_g[k].grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    for k in mlp:
        ref = fx["gradmlp." + k]
        assert np.abs(mlp[k].grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k


def test_oracle_equal_rows_give_the_uniform_result(golden_dir):
    """A per-point tensor whose rows all equal M renders what the uniform Rw2c = M renders.  fp32: the batched per-pair products
    round like the single matrix product up to an ulp; the gradients are compared in fp64, where such an ulp cannot flip a
    LeakyReLU mask."""
    fx = golden.load(golden_dir, "tiny_rw2c")
    M = torch.from_numpy(fx["Rw2c"])[0]
    N = fx["Rw2c"].shape[0]
    for dtype, tol in ((torch.float32, 1e-6), (torch.float64, 1e-12)):
        uni, pu, mu = _oracle_fixture_run(fx, M, dtype)
        per, pp, mp = _oracle_fixture_run(fx, M.expand(N, 3, 3).contiguous(), dtype)
        for a in ("ray_color", "opacity", "bg_T", "weight"):
            assert (uni[a] - per[a]).abs().max().item() <= tol, a
    for sh in (uni, per):
        ((sh["ray_color"] ** 2).sum() + 1e-3 * sh["conf_coefficient"].sum()).backward()
    for k in ("embedding", "color", "dir", "conf"):
        ref = pu[k].grad
        assert (pp[k].grad - ref).abs().max().item() <= 1e-10 * max(1.0, ref.abs().max().item()), k
    for k in mu:
        ref = mu[k].grad
        assert (mp[k].grad - ref).abs().max().item() <= 1e-10 * max(1.0, ref.abs().max().item()), k


# ------------------------------------------------------------------------------------------------ host container
def _points(n=10, seed=0):
    g = torch.Generator().manual_seed(seed)
    return dict(xyz=torch.rand(n, 3, generator=g), emb=torch.rand(1, n, 32, generator=g), color=torch.rand(1, n, 3, generator=g),
                dir=torch.rand(1, n, 3, generator=g), conf=torch.rand(1, n, 1, generator=g),
                R=torch.rand(n, 3, 3, generator=g))


def _npts(**over):
    return NeuralPoints(harness.make_opt(scene.CONFIGS["tiny"], **over), torch.device("cpu"))


def _rows_aligned(npn, p):
    """Every surviving point still carries its own frame: match the rows through the (unique) xyz."""
    for i in range(npn.xyz.shape[0]):
        j = int(torch.nonzero((p["xyz"] == npn.xyz[i]).all(-1))[0, 0])
        assert torch.equal(npn.Rw2c[i], p["R"][j]) and torch.equal(npn.points_embeding[0, i], p["emb"][0, j])


def test_set_points_and_prune_keep_rows_aligned():
    p = _points()
    npn = _npts()
    npn.set_points(p["xyz"], p["emb"], points_color=p["color"], points_dir=p["dir"], points_conf=p["conf"], Rw2c=p["R"])
    assert isinstance(npn.Rw2c, torch.nn.Parameter) and not npn.Rw2c.requires_grad and npn.Rw2c.shape == (10, 3, 3)
    assert "Rw2c" in dict(npn.named_parameters())
    thresh = float(p["conf"][0, :, 0].median())
    removed = npn.prune(thresh)
    assert removed > 0 and npn.Rw2c.shape == (10 - removed, 3, 3) and not npn.Rw2c.requires_grad
    _rows_aligned(npn, p)


def test_grow_points_appends_frames():
    p, q = _points(10, seed=0), _points(4, seed=1)
    npn = _npts()
    npn.set_points(p["xyz"], p["emb"], points_color=p["color"], points_dir=p["dir"], points_conf=p["conf"], Rw2c=p["R"])
    npn.grow_points(q["xyz"], q["emb"][0], q["color"][0], q["dir"][0], q["conf"][0], add_Rw2c=q["R"])
    assert npn.Rw2c.shape == (14, 3, 3) and npn.xyz.shape == (14, 3) and not npn.Rw2c.requires_grad
    assert torch.equal(npn.Rw2c[:10], p["R"]) and torch.equal(npn.Rw2c[10:], q["R"])
    with pytest.raises(ValueError, match="add_Rw2c"):
        npn.grow_points(q["xyz"], q["emb"][0], q["color"][0], q["dir"][0], q["conf"][0])
    with pytest.raises(ValueError, match="add_Rw2c"):
        npn.grow_points(q["xyz"], q["emb"][0], q["color"][0], q["dir"][0], q["conf"][0], add_Rw2c=q["R"][:3])
    assert npn.xyz.shape == (14, 3)                        # a refused growth changes nothing
    # a uniform cloud grows as before: add_Rw2c is not needed and the single frame stays
    uni = _npts()
    uni.set_points(p["xyz"], p["emb"], points_color=p["color"], points_dir=p["dir"], points_conf=p["conf"])
    uni.grow_points(q["xyz"], q["emb"][0], q["color"][0], q["dir"][0], q["conf"][0])
    assert torch.equal(uni.Rw2c, torch.eye(3)) and uni.xyz.shape == (14, 3)


def test_editing_set_points_has_the_reference_semantics():
    """neural_points.py:470-484: plain tensors (no parameters), opt.default_conf in (0, 1] overrides every conf, Rw2c as given."""
    p = _points()
    npn = _npts(default_conf=0.25)
    npn.set_points(p["xyz"], p["emb"], points_color=p["color"], points_dir=p["dir"], points_conf=p["conf"], Rw2c=p["R"])
    npn.editing_set_points(p["xyz"], p["emb"], points_color=p["color"], points_dir=p["dir"], points_conf=p["conf"], Rw2c=p["R"])
    assert dict(npn.named_parameters()) == {}
    assert torch.equal(npn.points_conf, torch.full_like(p["conf"], 0.25))
    assert npn.Rw2c is p["R"] and npn.xyz is p["xyz"] and npn.points_embeding is p["emb"]
    keep = _npts()                                          # default_conf -1: the confs are kept
    keep.editing_set_points(p["xyz"], p["emb"], points_color=p["color"], points_dir=p["dir"], points_conf=p["conf"])
    assert keep.points_conf is p["conf"] and torch.equal(keep.Rw2c, torch.eye(3))


# ------------------------------------------------------------------------------------------------ checkpoints
def _net():
    net, pts, opt = harness.build_model(scene.CONFIGS["tiny"], "cpu", seed=3)
    return net, opt


def test_checkpoint_validation_of_per_point_frames():
    net, opt = _net()
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    n = sd["neural_points.xyz"].shape[0]
    sd["neural_points.Rw2c"] = torch.eye(3).expand(n, 3, 3).contiguous()
    assert checkpoint.validate(sd, opt) == n
    for bad in (torch.zeros(n, 3), torch.zeros(n + 1, 3, 3), torch.eye(3, dtype=torch.float64).expand(n, 3, 3).contiguous()):
        sd["neural_points.Rw2c"] = bad
        with pytest.raises(checkpoint.CheckpointError, match="Rw2c"):
            checkpoint.validate(sd, opt)


def test_checkpoint_round_trip_keeps_per_point_frames(tmp_path, golden_dir):
    net, opt = _net()
    R = torch.from_numpy(golden.load(golden_dir, "tiny_rw2c")["Rw2c"])
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    assert R.shape[0] == sd["neural_points.xyz"].shape[0]
    sd["neural_points.Rw2c"] = R
    net2 = checkpoint.load_checkpoint(sd, opt, "cpu")
    assert isinstance(net2.neural_points.Rw2c, torch.nn.Parameter) and not net2.neural_points.Rw2c.requires_grad
    net_path, _ = checkpoint.save_checkpoint(net2, str(tmp_path), "latest")
    assert torch.equal(torch.load(net_path)["neural_points.Rw2c"], R)
    net3 = checkpoint.load_checkpoint(net_path, opt, "cpu")
    assert torch.equal(net3.neural_points.Rw2c.detach(), R)
