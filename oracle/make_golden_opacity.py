"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/tiny_opacity_loss by running the reference's OWN, unmodified Python hot path on
CPU (the build of oracle/make_golden.py) with a loss that also reads coarse_is_background and coarse_point_opacity, the two outputs the
reference keeps in the autograd graph besides the colour (neural_points_volumetric_model.py:312-324; ray_march,
diff_ray_marching.py:508-554):

    python -m oracle.make_golden_opacity

The cases are tiny_opaque's and tiny_thin_sr8's (same seed-0 MLP, alpha bias, SR and pixels; the thin scene has a non-trivial bg_T),
so the fixture stores no weights: they come from those fixtures.  The loss (opacity_loss) is the golden loss of make_golden.py plus
the reference's own loss terms on the outputs of the model shell's fill_invalid (neural_points_volumetric_model.py:87-123):
  bg_loss   base_rendering_model.py:620-627, on coarse_is_background with a fixed seeded per-ray mask (gt_mask)
  zero_one  base_rendering_model.py:630-641, on coarse_point_opacity with the default zero_epsilon = 1e-3
Stored per case (key prefix "<case>."): gt_mask, the loss value and the gradients of the 4 point tensors and the 18 MLP tensors.
It pins autograd through oracle/shade_oracle.py (tests/test_opacity_grads.py) and the CUDA path (tests/test_gpu_opacity_grads.py).
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CASES = (("tiny_opaque", 4.0, 24), ("tiny_thin_sr8", 0.0, 8))   # (name of the fixture with the MLP, alpha bias, SR)
BG_WEIGHT = 1.0e3
ZERO_ONE_WEIGHT = 1.0e2
ZERO_EPSILON = 1e-3     # base_rendering_model.py:119-123 default


def gt_mask_of(R, seed=0):
    """The fixed per-ray foreground mask [R,1] of the bg_loss term (the dataset's gt_mask)."""
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(R, 1, generator=g) < 0.5).float()


def fill_rays(ray_mask, x, fill):
    """fill_invalid (neural_points_volumetric_model.py:87-123): the [R',C] values of the hit rays scattered into [R,C] filled with
    `fill` (1 for coarse_is_background, 0 for coarse_point_opacity).  Out of place, so autograd carries the gradients back to x."""
    inds = torch.nonzero(ray_mask.reshape(-1))[:, 0]
    full = torch.full((ray_mask.numel(), x.shape[-1]), fill, dtype=x.dtype, device=x.device)
    return full.index_put((inds,), x.reshape(inds.shape[0], -1))


def opacity_loss(ray_color, conf_coefficient, is_background, point_opacity, gt_mask, bg_weight=BG_WEIGHT,
                 zero_one_weight=ZERO_ONE_WEIGHT):
    """ray_color [R',3] and conf_coefficient of the hit rays; is_background [R,1], point_opacity [R,SR] and gt_mask [R,1] over every ray
    (after fill_invalid).  The golden loss plus bg_loss and zero_one, in the reference's formulas."""
    loss = (ray_color ** 2).sum() + 1e-3 * conf_coefficient.sum()
    bg = F.mse_loss(is_background * (1 - gt_mask), 1 - gt_mask)                                  # l2loss = MSELoss, :274
    val = torch.clamp(point_opacity, ZERO_EPSILON, 1 - ZERO_EPSILON)
    zero_one = torch.mean(torch.log(val) + torch.log(1 - val))
    return loss + bg_weight * bg + zero_one_weight * zero_one


def _case(name, alpha_bias, SR, cfg, pixels):
    from types import SimpleNamespace
    from oracle.make_golden import build_reference_net
    from pointnerf_b200 import scene

    net, agg, npts, pts, opt = build_reference_net(cfg, alpha_bias, SR=SR)        # installs the reference's import shim
    from models.neural_points_volumetric_model import NeuralPointsVolumetricModel
    from models.rendering.diff_render_func import find_tone_map
    rays = scene.make_rays(cfg, pixels)

    def run(extra):
        net.zero_grad(set_to_none=True)
        out = net(rays["campos"], rays["raydir"], bg_color=rays["bg_color"], camrotc2w=rays["camrotc2w"],
                  pixel_idx=rays["pixel_idx"], near=rays["near"], far=rays["far"], h=rays["h"], w=rays["w"],
                  intrinsic=rays["intrinsic"])
        col, cc = out["coarse_raycolor"][0], out["conf_coefficient"]
        hit = out["ray_mask"][0]
        compact = (out["coarse_is_background"][0], out["coarse_point_opacity"][0])
        # the model shell's own fill_invalid (no bg_ray input, tone map off), run on a stand-in for the shell
        shell = SimpleNamespace(tonemap_func=find_tone_map("off"), opt=opt, input={})
        full = NeuralPointsVolumetricModel.fill_invalid(shell, out, rays)
        is_bg, op = full["coarse_is_background"][0], full["coarse_point_opacity"][0]
        assert torch.equal(is_bg, fill_rays(hit, compact[0], 1.0)) and torch.equal(op, fill_rays(hit, compact[1], 0.0))
        gt_mask = gt_mask_of(hit.numel())
        if extra:
            loss = opacity_loss(col, cc, is_bg, op, gt_mask)
        else:
            loss = (col ** 2).sum() + 1e-3 * cc.sum()
        loss.backward()
        return loss.detach(), gt_mask, {n: p.grad.clone() for n, p in net.named_parameters() if p.grad is not None}

    _, _, g0 = run(False)
    loss, gt_mask, g = run(True)
    fx = {"gt_mask": gt_mask.numpy(), "loss": np.float32(loss)}
    names = dict(embedding="points_embeding", color="points_color", dir="points_dir", conf="points_conf")
    for short, full in names.items():
        fx["grad_" + short] = g["neural_points." + full].numpy()
    for k in agg.state_dict():
        fx["gradmlp." + k] = g["aggregator." + k].numpy()
    moved = {short: float((g["neural_points." + full] - g0["neural_points." + full]).abs().max() /
                          g0["neural_points." + full].abs().max()) for short, full in names.items()}
    moved_mlp = max(float((g["aggregator." + k] - g0["aggregator." + k]).abs().max() / g0["aggregator." + k].abs().max().clamp(min=1e-12))
                    for k in agg.state_dict())
    print(name, "loss %.4f" % float(loss), "foreground rays %d of %d" % (int(gt_mask.sum()), gt_mask.shape[0]),
          "change of the gradients by the new terms, relative to the colour-loss gradient's max:",
          ", ".join("%s %.3f" % kv for kv in moved.items()), ", MLP (largest) %.3f" % moved_mlp)
    return fx


if __name__ == "__main__":
    from oracle import golden, ref_shim
    from oracle.make_golden import OUT
    from pointnerf_b200 import scene
    assert ref_shim.available(), "needs the reference tree"
    tiny = scene.CONFIGS["tiny"]
    arrays = dict(bg_weight=np.float32(BG_WEIGHT), zero_one_weight=np.float32(ZERO_ONE_WEIGHT), zero_epsilon=np.float32(ZERO_EPSILON))
    for name, alpha_bias, SR in CASES:
        for k, v in _case(name, alpha_bias, SR, tiny, scene.centre_patch(tiny, 40)).items():
            arrays[name + "." + k] = v
    golden.save(OUT, "tiny_opacity_loss", arrays)                 # split into files < 1 MB (oracle/golden.py)
