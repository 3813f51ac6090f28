"""CPU: the method of tests/test_gpu_forward_f64.py checked on the oracle itself (oracle/forward_check.py).

The fp32 oracle agrees with float64 on every sample without any LeakyReLU masks; forward_check.march reproduces shade()'s compositing bit
for bit; defects that the 1e-4 rule on radiance and opacity lets through (one K slot dropped, every sigma 3e-4 too large, one h-bar
channel of one sample off by 1e-3 of scale) fail the per-sample check; decode_hbar reads the colour kernel's operand layout; the
orbited camera of the GPU tests hits the shell and changes the oracle's outputs; and defects in the use of bg_color that no comparison
sees under a white background fail the per-ray comparison under (0.9, 0.1, 0.4)."""
import numpy as np
import pytest
import torch

from oracle import forward_check, pipeline, shade_oracle, shade_oracle_rw2c
from pointnerf_b200 import harness, scene
from pointnerf_b200.ray_marching import PointAggregator

# the fp32 oracle against float64, per sample: sigma relative to the largest |sigma|, rgb absolute, hbar relative to the largest |hbar|
# 4-5x the largest measured over test_fp32_matches_float64_without_masks' cases: sigma 3.0e-7, rgb 1.2e-7, hbar 8.2e-7
RTOL_FP32 = dict(sigma=1.5e-6, rgb=6e-7, hbar=4e-6)
OLD_TOL = 1e-4


def _case(F=32, order=2, frames=False, rotated=True, alpha_bias=3.0, side=20, pixels=None, **over):
    cfg = scene.CONFIGS["tiny"]
    opt = harness.make_opt(cfg, feat_dim=F, agg_intrp_order=order, **over)
    agg = PointAggregator(opt, seed=2)
    with torch.no_grad():
        agg.alpha_branch[0].bias += alpha_bias
    mlp = harness.mlp_cpu(agg)
    if F == 32:
        pts = scene.make_points(cfg)
    else:                           # set_points in mode "01": colour, dir and conf prepended to 56 features
        pts = scene.make_points(cfg, emb_dim=F - 7)
        pts["embedding"] = torch.cat([pts["color"], pts["dir"], pts["conf"], pts["embedding"]], dim=-1)
    if frames:
        pts["Rw2c"] = scene.edit_frames(pts["xyz"])
    rays = scene.make_rays(cfg, scene.centre_patch(cfg, side) if pixels is None else pixels,
                           camrotc2w=scene.orbit_rotation() if rotated else None)
    cam, campos = rays["camrotc2w"][0], rays["campos"][0]
    q = pipeline.render(pts, mlp, rays["raydir"][0], campos.numpy(), cam.numpy(), cfg.near, cfg.far, opt.vsize, opt.vscale,
                        opt.kernel_size, opt.query_size, opt.ranges, opt.SR, opt.K, opt.P, cfg.N, D=cfg.D, want_shade=False)
    mask = torch.from_numpy(q["ray_mask"]) > 0
    args = (torch.from_numpy(q["sample_pidx"]), torch.from_numpy(q["sample_loc_w"]), rays["raydir"][0][mask], campos, cam, opt.vsize,
            torch.ones(3))
    shade = shade_oracle_rw2c.shade if frames else shade_oracle.shade
    run = lambda dtype, a=args: shade(pts, mlp, *a, dtype=dtype, agg_intrp_order=order)
    return dict(run=run, args=args, pts=pts, mlp=mlp, order=order, mask=mask, sh32=run(torch.float32), sh64=run(torch.float64))


def _rows(sh):
    return sh["ray_valid"].reshape(-1).nonzero()[:, 0]


def _got(sh, rows, decoded=None, hbar=None):
    dec = (sh["decoded"] if decoded is None else decoded).reshape(-1, 4)[rows]
    return dict(sigma=dec[:, 0], rgb=dec[:, 1:], hbar=(sh["hbar"] if hbar is None else hbar)[rows])


def _march(c, decoded, dtype=torch.float32, bg=None):
    _, loc_w, _, campos, cam, vsize, bg0 = c["args"]
    bg = bg0 if bg is None else bg
    return forward_check.march(decoded, c["sh32"]["ray_valid"], loc_w, campos, cam, vsize, bg, dtype=dtype)


def _old_rule(m, sh):
    """The parity tests' rule: radiance, opacity and bg_T within 1e-4 absolute."""
    return max((m[k].double() - sh[k].double()).abs().max().item() for k in ("ray_color", "opacity", "bg_T")) <= OLD_TOL


@pytest.mark.parametrize("order", [2, 1])
@pytest.mark.parametrize("frames", [False, True])
@pytest.mark.parametrize("F", [32, 63])
def test_fp32_matches_float64_without_masks(F, frames, order):
    c = _case(F, order, frames)
    rows = _rows(c["sh64"])
    assert rows.shape[0] > 500
    errs = forward_check.sample_errors(_got(c["sh32"], rows), c["sh64"], rows)
    rep = forward_check.check(errs, RTOL_FP32)
    print("\n[oracle fp32-f64] F=%d frames=%d order=%d S=%d %s" % (F, frames, order, rows.shape[0],
                                                                   " ".join("%s=%.2e" % (k, v[0]) for k, v in rep.items())))


@pytest.mark.parametrize("rotated", [False, True])
@pytest.mark.parametrize("order", [2, 1])
def test_march_matches_shade(order, rotated):
    c = _case(order=order, rotated=rotated)
    sh = c["sh32"]
    m = _march(c, sh["decoded"])
    for k in ("ray_dist", "opacity", "bg_T", "blend_weight", "ray_color"):
        assert torch.equal(m[k], sh[k]), k


def test_dropped_k_slot_is_caught():
    """One neighbour of one sample dropped (the test takes a sample whose ray moves by less than 1e-4)."""
    c = _case()
    sh32, sh64 = c["sh32"], c["sh64"]
    pidx, loc_w, raydir, *rest = c["args"]
    rows = _rows(sh64)
    SR = pidx.shape[1]
    g = torch.Generator().manual_seed(3)
    tried = 0
    for i in torch.randperm(rows.shape[0], generator=g)[:40].tolist():
        r, s = divmod(int(rows[i]), SR)
        k = (pidx[r, s] >= 0).nonzero()[:, 0]
        if k.shape[0] < 2:
            continue
        tried += 1
        p1 = pidx[r:r + 1].clone()
        p1[0, s, k[-1]] = -1
        one = shade_oracle.shade(c["pts"], c["mlp"], p1, loc_w[r:r + 1], raydir[r:r + 1], *rest, dtype=torch.float32)
        dec = sh32["decoded"].clone()
        dec[r] = one["decoded"][0]
        hbar = sh32["hbar"].clone()
        hbar[r * SR:(r + 1) * SR] = one["hbar"]
        if _old_rule(_march(c, dec), sh64):
            with pytest.raises(AssertionError, match="slot %d" % s):
                forward_check.check(forward_check.sample_errors(_got(sh32, rows, dec, hbar), sh64, rows), RTOL_FP32,
                                    lambda j: "slot %d" % (int(rows[j]) % SR))
            return
    pytest.fail("none of %d dropped slots passes the 1e-4 rule" % tried)


def test_sigma_scaled_by_3e4_is_caught():
    c = _case()
    sh32, sh64 = c["sh32"], c["sh64"]
    dec = sh32["decoded"].clone()
    dec[..., 0] *= 1 + 3e-4
    assert _old_rule(_march(c, dec), sh64)
    rows = _rows(sh64)
    with pytest.raises(AssertionError, match="sigma"):
        forward_check.check(forward_check.sample_errors(_got(sh32, rows, dec), sh64, rows), RTOL_FP32)


def test_one_hbar_channel_is_caught(monkeypatch):
    """1e-3 of scale added to one h-bar channel of one sample, as the colour branch consumes it."""
    c = _case()
    sh32, sh64 = c["sh32"], c["sh64"]
    pidx, loc_w, raydir, *rest = c["args"]
    rows = _rows(sh64)
    SR = pidx.shape[1]
    r, s = divmod(int(rows[rows.shape[0] // 2]), SR)
    ch, delta = 77, 1e-3 * float(sh64["hbar"].abs().max())
    lin = shade_oracle._lin

    def bad_lin(x, mlp, key):
        if key == "color_branch.0":
            x = x.clone()
            x[s, ch] += delta
        return lin(x, mlp, key)

    monkeypatch.setattr(shade_oracle, "_lin", bad_lin)
    one = shade_oracle.shade(c["pts"], c["mlp"], pidx[r:r + 1], loc_w[r:r + 1], raydir[r:r + 1], *rest, dtype=torch.float32)
    monkeypatch.undo()
    dec = sh32["decoded"].clone()
    dec[r] = one["decoded"][0]
    hbar = sh32["hbar"].clone()
    hbar[r * SR + s, ch] += delta
    assert _old_rule(_march(c, dec), sh64)
    with pytest.raises(AssertionError, match="hbar"):
        forward_check.check(forward_check.sample_errors(_got(sh32, rows, dec, hbar), sh64, rows), RTOL_FP32)


def test_decode_hbar_offsets():
    """Offsets worked out by hand from the operand layout: per 128 samples 8 blocks of 16 KB (one per 32 channels, lo 8 KB after hi),
    inside a block byte (r, k) = (r/8)*512 + (k/8)*128 + (r%8)*16 + (k%8)*2."""
    n = 300                                       # 3 colour tiles, the last one partial
    buf = np.zeros(3 * 8 * 16384, np.uint8)
    cases = {(0, 0): 0, (1, 0): 16, (0, 1): 2, (0, 8): 128, (8, 0): 512, (9, 9): 512 + 128 + 16 + 2, (0, 32): 16384,
             (128, 0): 8 * 16384, (127, 31): 15 * 512 + 3 * 128 + 7 * 16 + 7 * 2, (200, 255): 15 * 16384 + 9 * 512 + 3 * 128 + 7 * 2,
             (299, 100): 19 * 16384 + 5 * 512 + 0 * 128 + 3 * 16 + 4 * 2}
    want = torch.zeros(n, 256, dtype=torch.float64)
    for j, ((vi, c), off) in enumerate(cases.items()):
        assert forward_check.hbar_offset(vi, c) == off, (vi, c)
        hi = np.float32(1.5 + j)                  # exact in bf16
        lo = np.float32(2.0 ** -10 * (j + 1))     # exact in bf16
        for o, v in ((off, hi), (off + 8192, lo)):
            u = int(np.array(v, np.float32).view(np.uint32)) >> 16
            buf[o], buf[o + 1] = u & 0xff, u >> 8
        want[vi, c] = float(hi) + float(lo)
    assert torch.equal(forward_check.decode_hbar(torch.from_numpy(buf), n), want)


def test_rotated_camera_matters():
    """The orbited camera of the GPU tests hits the shell, and the oracle's outputs with it differ from those with the same rays but
    camrotc2w = I by far more than 1e-4: the camera rotation reaches the shading inputs."""
    cfg = scene.CONFIGS["tiny"]
    R = scene.orbit_rotation()
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-6) and abs(np.linalg.det(R) - 1) < 1e-6
    c = _case(rotated=True)
    hit = c["args"][0].shape[0]
    assert hit > 300, "the orbited camera misses the shell"
    pidx, loc_w, raydir, campos, cam, vsize, bg = c["args"]
    assert np.allclose(campos.numpy(), R @ np.asarray(cfg.campos, np.float32), atol=1e-6)
    ident = shade_oracle.shade(c["pts"], c["mlp"], pidx, loc_w, raydir, campos, torch.eye(3), vsize, bg)
    d = max((ident[k] - c["sh32"][k]).abs().max().item() for k in ("ray_color", "opacity", "bg_T"))
    assert d > 100 * OLD_TOL, d
    assert float(c["sh32"]["bg_T"].min()) < 0.9


@pytest.mark.parametrize("defect", ["channels_0_2_swapped", "white_on_missed_rays"])
def test_background_defects_need_a_coloured_background(defect):
    """bg_color with its channels 0 and 2 swapped in the compositing, and missed rays painted 1 instead of bg_color: under the white
    background every ray agrees bit for bit, under (0.9, 0.1, 0.4) the per-ray comparison fails."""
    cfg = scene.CONFIGS["tiny"]
    side = 20
    c = _case(pixels=scene.centre_patch(cfg, side) + np.float32([side // 2, 0]))       # across the limb of the shell
    mask = c["mask"]
    assert 0 < int(mask.sum()) < mask.numel(), "the patch needs hit and missed rays"
    dec = c["sh32"]["decoded"]

    def full(bg_march, bg_fill):
        m = _march(c, dec, bg=bg_march)
        return shade_oracle.fill_invalid(mask, m["ray_color"], m["opacity"], m["bg_T"], torch.zeros(int(mask.sum()), 3), bg_fill)["coarse_raycolor"]

    for bg in (torch.ones(3), torch.tensor([0.9, 0.1, 0.4])):
        ref = full(bg, bg)
        bad = full(bg.flip(0), bg) if defect == "channels_0_2_swapped" else full(bg, torch.ones(3))
        errs = dict(composite=(bad - ref).abs().amax(-1))
        if bool((bg == 1).all()):
            assert torch.equal(bad, ref)
        else:
            with pytest.raises(AssertionError, match="composite"):
                forward_check.check(errs, dict(composite=1e-5))


def test_raydist_mode_unit_0_keeps_the_long_steps():
    """raydist_mode_unit 0 drops the `> 2 vsize_z` replacement only: the shell's front-to-back step stays (tens of voxels), every other
    step is the unit mode's, march follows shade, and the default is the unit mode.  SR 80: 24 slots end inside the front crossing."""
    c = _case(side=12, SR=80)
    pidx, loc_w, raydir, campos, cam, vsize, bg = c["args"]
    sh0 = shade_oracle.shade(c["pts"], c["mlp"], *c["args"], raydist_mode_unit=0)
    sh1 = c["sh32"]
    assert torch.equal(shade_oracle.shade(c["pts"], c["mlp"], *c["args"], raydist_mode_unit=1)["ray_color"], sh1["ray_color"])
    vz = float(vsize[2])
    long = sh0["ray_dist"] > 2 * vz
    assert int(long.sum()) > 50 and float(sh0["ray_dist"].max()) > 10 * vz
    assert torch.equal(sh0["ray_dist"][~long], sh1["ray_dist"][~long]) and bool((sh1["ray_dist"][long] == vz).all())
    assert (sh0["ray_color"] - sh1["ray_color"]).abs().max().item() > 100 * OLD_TOL
    m = forward_check.march(sh0["decoded"], sh0["ray_valid"], loc_w, campos, cam, vsize, bg, dtype=torch.float32, raydist_mode_unit=0)
    for k in ("ray_dist", "opacity", "bg_T", "blend_weight", "ray_color"):
        assert torch.equal(m[k], sh0[k]), k
