"""CPU: pins oracle/probe_oracle.py (the probe outputs of point growing, opt.prob == 1, neural_points_volumetric_model.py:331-351).

  fixture   fed by the query oracle's export and the shading oracle's opacity, the fp32 oracle reproduces tests/golden/tiny_probe.npz
            (the reference module's own run) bit for bit, all seven keys
  rules     on a transparent frame (alpha_bias -100: every opacity is 0, so every slot ties and torch.max picks slot 0, whose K slots
            are all empty on about half the rays) the oracle agrees with a per-ray float64 loop over the stated rules: first maximal
            slot, position of that slot, weight * conf_coefficient, point 0 for an empty slot in far_dist and in the averages
  defects   dropping the conf factor, the last maximum winning ties and empty slots skipped in far_dist each fail one of the two
"""
import numpy as np
import pytest
import torch

from oracle import golden, pipeline, probe_oracle
from pointnerf_b200 import harness, scene


def _case(golden_dir, alpha_bias):
    """Query export + opacity of the tiny_probe rays, MLP of tiny_opaque with alpha_branch.0.bias moved to `alpha_bias`."""
    w = golden.load(golden_dir, "tiny_opaque")
    fx = np.load(golden_dir + "/tiny_probe.npz")
    cfg = scene.CONFIGS["tiny"]
    opt = harness.make_opt(cfg)
    pts = scene.make_points(cfg)
    mlp = {k[4:]: torch.from_numpy(w[k]).clone() for k in w.files if k.startswith("mlp.")}
    mlp["alpha_branch.0.bias"] += alpha_bias - float(w["alpha_bias"])
    rays = scene.make_rays(cfg, fx["pixels"])
    ref = pipeline.render(pts, mlp, rays["raydir"][0], cfg.campos, np.eye(3, dtype=np.float32), cfg.near, cfg.far, opt.vsize, opt.vscale,
                          opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P, 100000, D=cfg.D)
    return fx, pts, ref


@pytest.fixture(scope="module")
def cases(golden_dir):
    return dict(fixture=_case(golden_dir, 4.0), transparent=_case(golden_dir, -100.0))


def _fixture_mismatch(cases, mutate=None):
    fx, pts, ref = cases["fixture"]
    assert float(fx["alpha_bias"]) == 4.0
    out = probe_oracle.probe(pts, ref["sample_pidx"], ref["sample_loc_w"], ref["opacity"], mutate=mutate)
    return [k for k in probe_oracle.KEYS if not np.array_equal(out[k].numpy(), fx[k])]


def _rules(pts, pidx, loc_w, op):
    """The stated rules, one ray at a time in float64."""
    xyz = pts["xyz"].double().numpy()
    attrs = [pts[k][0].double().numpy() for k in ("color", "dir", "conf", "embedding")]
    conf = attrs[2][:, 0]
    res = {k: [] for k in probe_oracle.KEYS}
    for r in range(pidx.shape[0]):
        o = op[r].astype(np.float64)
        j = int(np.flatnonzero(o == o.max())[0])                         # first maximal slot
        loc = loc_w[r, j].astype(np.float64)
        p = pidx[r, j]
        i = np.maximum(p, 0)                                              # empty slot -> point 0
        d = np.linalg.norm(xyz[i] - loc, axis=-1)
        wgt = np.where(p >= 0, 1.0 / np.maximum(d, 1e-6), 0.0)
        wc = wgt / max(wgt.sum(), 1e-8) * np.clip(conf[i], 1e-4, 1.0)
        res["ray_max_shading_opacity"].append([o[j]])
        res["ray_max_sample_loc_w"].append(loc)
        res["ray_max_far_dist"].append([d.min()])
        for name, a in zip(("shading_avg_color", "shading_avg_dir", "shading_avg_conf", "shading_avg_embedding"), attrs):
            res[name].append((a[i] * wc[:, None]).sum(0))
    return {k: np.asarray(v) for k, v in res.items()}


def _rules_mismatch(cases, mutate=None, tol=1e-6):
    _, pts, ref = cases["transparent"]
    pidx, loc_w, op = ref["sample_pidx"], ref["sample_loc_w"], ref["opacity"].numpy()
    out = probe_oracle.probe(pts, pidx, loc_w, op, mutate=mutate)
    want = _rules(pts, pidx, loc_w, op)
    bad = []
    for k in probe_oracle.KEYS:
        a, b = out[k].double().numpy(), want[k]
        if not (np.isfinite(a).all() and np.abs(a - b).max() <= tol * max(1.0, np.abs(b).max())):
            bad.append(k)
    return bad


def test_fp32_oracle_reproduces_reference_fixture(cases):
    assert _fixture_mismatch(cases) == []


def test_oracle_follows_tie_and_empty_slot_rules(cases):
    _, pts, ref = cases["transparent"]
    op, pidx = ref["opacity"], ref["sample_pidx"]
    # the case exercises the rules: every opacity 0 (all slots tie), slot 0 entirely empty on some rays
    assert float(op.abs().max()) == 0.0
    assert 0 < int((pidx[:, 0, :] < 0).all(-1).sum()) < pidx.shape[0]
    assert _rules_mismatch(cases) == []
    out = probe_oracle.probe(pts, pidx, ref["sample_loc_w"], op, dtype=torch.float64)
    assert torch.all(out["slot"] == 0)


@pytest.mark.parametrize("mutate", probe_oracle.MUTATIONS)
def test_defects_fail_the_comparison(cases, mutate):
    assert _fixture_mismatch(cases, mutate) or _rules_mismatch(cases, mutate)
