"""CPU: gradients of a loss on coarse_is_background and coarse_point_opacity (bg_loss and zero_one in the reference's formulas, on top of
the golden colour + conf loss) through autograd of oracle/shade_oracle.py, against the gradients the reference's own autograd produced
(tests/golden/tiny_opacity_loss, oracle/make_golden_opacity.py)."""
import numpy as np
import pytest
import torch

from oracle import golden, shade_oracle
from oracle.make_golden_opacity import CASES, fill_rays, gt_mask_of, opacity_loss
from pointnerf_b200 import scene


def _mlp_from(fx):
    return {k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")}


@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_oracle_gradients_match_reference_fixture(name, golden_dir):
    fx = golden.load(golden_dir, name)                       # weights, pixels, SR and the query of the case
    gx = golden.load(golden_dir, "tiny_opacity_loss")
    cfg = scene.CONFIGS["tiny"]
    pts = scene.make_points(cfg)
    rays = scene.make_rays(cfg, fx["pixels"])
    hit = torch.from_numpy(fx["ray_mask"])
    mask = hit > 0
    gt_mask = torch.from_numpy(gx[name + ".gt_mask"])
    assert torch.equal(gt_mask, gt_mask_of(hit.shape[0]))
    pts_g = {k: v.clone().requires_grad_(k in ("embedding", "color", "dir", "conf")) for k, v in pts.items()}
    mlp = {k: v.clone().requires_grad_(True) for k, v in _mlp_from(fx).items()}
    sh = shade_oracle.shade(pts_g, mlp, torch.from_numpy(fx["sample_pidx"]), torch.from_numpy(fx["sample_loc_w"]),
                            rays["raydir"][0][mask], torch.tensor(cfg.campos), torch.eye(3), [cfg.vsize] * 3, torch.ones(3))
    loss = opacity_loss(sh["ray_color"], sh["conf_coefficient"], fill_rays(hit, sh["bg_T"], 1.0), fill_rays(hit, sh["opacity"], 0.0),
                        gt_mask, float(gx["bg_weight"]), float(gx["zero_one_weight"]))
    assert abs(loss.item() - float(gx[name + ".loss"])) <= 1e-5 * abs(float(gx[name + ".loss"]))
    loss.backward()
    # the tolerances of tests/test_oracle_shade.py
    for k in ("embedding", "color", "dir", "conf"):
        ref = gx[name + ".grad_" + k]
        assert np.abs(pts_g[k].grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k
    for k in mlp:
        ref = gx[name + ".gradmlp." + k]
        assert np.abs(mlp[k].grad.numpy() - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max()), k


def test_render_backward_without_upstream_gradients_returns_none():
    """The shading backward reached with no gradient for any of its outputs (a consumer returned None for them) passes nothing back
    and launches nothing (the fake context carries no query, module or buffers)."""
    from types import SimpleNamespace
    from pointnerf_b200.ray_marching import MLP_KEYS, _RenderFn
    ctx = SimpleNamespace(mlp_shapes=[()] * (2 * len(MLP_KEYS)))
    grads = _RenderFn.backward(ctx, None, None, None, None)
    assert len(grads) == 6 + 2 * len(MLP_KEYS) and all(g is None for g in grads)


def test_fixture_terms_move_the_gradients(golden_dir):
    """The new terms are not negligible: without them the gradients (those of the colour + conf loss, the case's own fixture) differ
    by a sizeable fraction of their scale, in both scenes, and the thin scene's rays are far from opaque."""
    gx = golden.load(golden_dir, "tiny_opacity_loss")
    for name, _, _ in CASES:
        fx = golden.load(golden_dir, name)
        ref = fx["grad_embedding"]
        assert np.abs(gx[name + ".grad_embedding"] - ref).max() > 0.1 * np.abs(ref).max(), name
    assert golden.load(golden_dir, "tiny_thin_sr8")["coarse_is_background"].min() > 0.5
