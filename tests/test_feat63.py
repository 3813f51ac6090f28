"""CPU: the DTU configuration, point_features_dim 63 with point_{conf,dir,color}_mode "01" (colour, dir and conf prepended to 56 image
features, and kept as tensors of their own).  The oracle (oracle/shade_oracle.py, generic in the width) against the reference-generated
fixtures tests/golden/tiny_feat63 and tiny_feat63_order1, the host container's set_points, the option gate and checkpoints."""
import numpy as np
import pytest
import torch

from oracle import golden, shade_oracle
from pointnerf_b200 import checkpoint, harness, scene
from pointnerf_b200.ray_marching import NeuralPoints, PointAggregator, check_opt, mlp_kpad, mlp_shapes

CASES = ["tiny_feat63", "tiny_feat63_order1"]


def _mlp_from(fx):
    return {k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")}


def _points63(cfg):
    """The points as the reference's set_points leaves them: embedding [color, dir, conf, 56 features], the three kept as well."""
    pts = scene.make_points(cfg, emb_dim=56)
    pts["embedding"] = torch.cat([pts["color"], pts["dir"], pts["conf"], pts["embedding"]], dim=-1)
    return pts


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_fixture(golden_dir, name):
    """Forward bit for bit, gradients to fp32 rounding (autograd through the oracle, as tests/test_rw2c.py)."""
    fx = golden.load(golden_dir, name)
    cfg = scene.CONFIGS["tiny"]
    pts = _points63(cfg)
    assert np.array_equal(pts["embedding"].numpy(), fx["embedding63"])
    assert fx["mlp.block1.0.weight"].shape == (256, 501)
    rays = scene.make_rays(cfg, fx["pixels"])
    mask = torch.from_numpy(fx["ray_mask"]) > 0
    pts_g = {k: v.clone().requires_grad_(k in ("embedding", "color", "dir", "conf")) for k, v in pts.items()}
    mlp = {k: v.clone().requires_grad_(True) for k, v in _mlp_from(fx).items()}
    sh = shade_oracle.shade(pts_g, mlp, torch.from_numpy(fx["sample_pidx"]), torch.from_numpy(fx["sample_loc_w"]), rays["raydir"][0][mask],
                            torch.tensor(cfg.campos), torch.eye(3), [cfg.vsize] * 3, torch.ones(3), agg_intrp_order=int(fx["agg_intrp_order"]))
    for a, b in (("ray_color", "coarse_raycolor"), ("opacity", "coarse_point_opacity"), ("bg_T", "coarse_is_background"),
                 ("weight", "weight"), ("conf_coefficient", "conf_coefficient"), ("blend_weight", "blend_weight")):
        assert np.array_equal(sh[a].detach().numpy(), fx[b]), a
    ((sh["ray_color"] ** 2).sum() + 1e-3 * sh["conf_coefficient"].sum()).backward()   # the loss of oracle/make_golden_feat63.py
    for k, g in (("embedding", "grad_embedding"), ("color", "grad_color"), ("dir", "grad_dir"), ("conf", "grad_conf")):
        ref = fx[g]
        assert pts_g[k].grad.shape == ref.shape, k
        assert np.abs(pts_g[k].grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    for k in mlp:
        ref = fx["gradmlp." + k]
        assert np.abs(mlp[k].grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    # the prepended copies of colour, dir and conf are independent of the kept tensors: both receive gradients
    assert np.abs(fx["grad_embedding"][0, :, :7]).max() > 0 and np.abs(fx["grad_color"]).max() > 0


def test_set_points_builds_the_reference_embedding(golden_dir):
    """Mode "01": [color, dir, conf, emb] (prepended conf, then dir, then colour), the three kept as parameters of their own."""
    fx = golden.load(golden_dir, "tiny_feat63")
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, "cpu", feat_dim=63)
    npn = net.neural_points
    assert opt.point_features_dim == 63 and opt.point_color_mode == "01"
    assert np.array_equal(npn.points_embeding.detach().numpy(), fx["embedding63"])
    assert torch.equal(npn.points_color.detach(), pts["color"]) and torch.equal(npn.points_conf.detach(), pts["conf"])
    names = dict(npn.named_parameters())
    assert {"points_embeding", "points_color", "points_dir", "points_conf"} <= set(names)
    assert npn.points_embeding.requires_grad and npn.points_color.requires_grad
    # mode "1" keeps the 32-channel behaviour; a longer embedding is cut to point_features_dim before anything is prepended
    plain = NeuralPoints(harness.make_opt(cfg), torch.device("cpu"))
    p32 = scene.make_points(cfg)
    plain.set_points(p32["xyz"], torch.cat([p32["embedding"], p32["embedding"]], -1), points_color=p32["color"],
                     points_dir=p32["dir"], points_conf=p32["conf"])
    assert torch.equal(plain.points_embeding.detach(), p32["embedding"])


def test_aggregator_and_mlp_sizes_follow_the_width():
    cfg = scene.CONFIGS["tiny"]
    agg = PointAggregator(harness.make_opt(cfg, feat_dim=63))
    assert tuple(agg.block1[0].weight.shape) == (256, 501) == mlp_shapes(63)[0]
    assert tuple(PointAggregator(harness.make_opt(cfg)).block1[0].weight.shape) == (256, 284) == mlp_shapes(32)[0]
    assert mlp_kpad(63)[0] == 512 and mlp_kpad(32)[0] == 288 and mlp_shapes(63)[1:] == mlp_shapes(32)[1:]


def test_option_gate_accepts_the_dtu_configuration():
    cfg = scene.CONFIGS["tiny"]
    check_opt(harness.make_opt(cfg, feat_dim=63))
    check_opt(harness.make_opt(cfg, feat_dim=63, agg_intrp_order=1))
    check_opt(harness.make_opt(cfg, point_color_mode="01"))
    for over in (dict(point_features_dim=48), dict(point_features_dim=64), dict(point_features_dim=16),
                 dict(point_conf_mode="0"), dict(point_dir_mode="10"), dict(point_color_mode="2"), dict(feat_dim=63, agg_intrp_order=0)):
        with pytest.raises(NotImplementedError):
            check_opt(harness.make_opt(cfg, **over))


def test_checkpoint_round_trip_63_channels(tmp_path):
    """A DTU checkpoint: points_embeding [1,N,63] beside colour / dir / conf, block1.0 [256, 501]; loading installs the stored
    embedding as it is (nothing prepended a second time)."""
    cfg = scene.CONFIGS["tiny"]
    net, pts, opt = harness.build_model(cfg, "cpu", seed=3, feat_dim=63)
    sd = {k: v.detach().clone() for k, v in net.state_dict().items()}
    assert sd["neural_points.points_embeding"].shape[-1] == 63 and sd["aggregator.block1.0.weight"].shape == (256, 501)
    assert checkpoint.validate(sd, opt) == cfg.N
    net_path, _ = checkpoint.save_checkpoint(net, str(tmp_path), "latest")
    net2 = checkpoint.load_checkpoint(net_path, opt, "cpu")
    for k, v in net2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    with pytest.raises(checkpoint.CheckpointError, match="point_features_dim"):
        checkpoint.validate(sd, harness.make_opt(cfg))
