"""GPU: the pieces either side of the seam (SURVEY 8(f) ranks 2-3): whole-image entry point vs the reference's chunk loop,
and a reference-format checkpoint loaded from disk vs the fixture the reference module produced with those weights."""
import os

import numpy as np
import pytest
import torch

from pointnerf_b200 import checkpoint, harness, runner, scene
from oracle import golden  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def test_whole_image_equals_reference_chunk_loop():
    """render_vid.py:45-71 renders `random_sample_size**2`-ray chunks and assembles them on the host; one whole-image call
    must give the same pixels bit for bit (48x48 = 2304 rays, the shipped chunk; a 640x96 strip through the lego view's centre:
    hits and misses)."""
    cfg = scene.CONFIGS["lego_render"]
    net, pts, opt = harness.build_model(cfg, DEV, alpha_bias=3.0)
    W, H = 640, 96
    x0, y0 = cfg.W // 2 - W // 2, cfg.H // 2 - H // 2
    px, py = np.meshgrid(np.arange(x0, x0 + W), np.arange(y0, y0 + H))
    rays = scene.make_rays(cfg, np.stack((px, py), -1).reshape(-1, 2).astype(np.float32))
    data = {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in rays.items()}
    whole = runner.render_image(net, data, H, W)
    chunked = runner.render_image_chunked(net, data, H, W, 48 * 48)
    assert whole["coarse_raycolor"].shape == (H, W, 3) and whole["ray_mask"].shape == (H, W)
    assert np.array_equal(whole["coarse_raycolor"].cpu().numpy(), chunked["coarse_raycolor"])
    hit = whole["ray_mask"] > 0
    frac = hit.float().mean().item()
    assert 0.2 < frac < 0.98, frac
    assert torch.all(whole["coarse_raycolor"][~hit] == 1.0) and torch.all(whole["coarse_point_opacity"][~hit] == 0)
    net.check_errors()


def test_reference_format_checkpoint_from_disk(golden_dir, tmp_path):
    """A `*_net_ray_marching.pth` file in the reference's layout (weights = the ones the reference module used for the
    tiny_opaque fixture) -> load_checkpoint -> drop-in forward() reproduces what the reference returned."""
    fx = golden.load(golden_dir, "tiny_opaque")
    cfg = scene.CONFIGS["tiny"]
    pts = scene.make_points(cfg)
    sd = {"aggregator." + k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")}
    sd.update({"neural_points.xyz": pts["xyz"], "neural_points.points_embeding": pts["embedding"],
               "neural_points.points_conf": pts["conf"], "neural_points.points_dir": pts["dir"],
               "neural_points.points_color": pts["color"]})
    path = os.path.join(str(tmp_path), "200000_net_ray_marching.pth")
    torch.save(sd, path)
    opt = harness.make_opt(cfg, SR=int(fx["SR"]), max_o=100000)
    net = checkpoint.load_checkpoint(path, opt, DEV)
    rays = scene.make_rays(cfg, fx["pixels"])
    r = {k: v.to(DEV) for k, v in rays.items()}
    with torch.no_grad():
        out = net(r["campos"], r["raydir"], bg_color=r["bg_color"], camrotc2w=r["camrotc2w"], pixel_idx=r["pixel_idx"],
                  near=r["near"], far=r["far"], h=r["h"], w=r["w"], intrinsic=r["intrinsic"])
    assert np.array_equal(out["ray_mask"][0].cpu().numpy(), fx["ray_mask"])
    for k in ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background"):
        d = np.abs(out[k][0].cpu().numpy() - fx[k]).max()
        assert d <= 1e-4, "%s max abs diff %.3e" % (k, d)
    # and back to disk in the same format
    p2, _ = checkpoint.save_checkpoint(net, str(tmp_path), "latest")
    sd2 = torch.load(p2)
    assert sd2.keys() == sd.keys() and all(torch.equal(sd2[k], sd[k].float()) for k in sd)
