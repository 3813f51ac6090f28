"""GPU: the plane background drop-ins (pointnerf_b200.plane_bg: gen_bg_points, get_rayplane_cross, set_bg) through
pnb_plane_cross, pnb_plane_fg_masks and pnb_plane_bg.

  oracle      intersections, foreground masks and bg_ray equal to oracle/plane_bg_oracle.py's fp32 restatement bit for bit on every
              case of tests/golden/plane_bg_ref.npz and on a seeded DTU-sized case (512 x 640, G = 32, N = 1M)
  reference   set_bg on the reference's own plane points meets the reference's recorded results within the bounds and with the flip
              classification of tests/test_plane_bg_oracle.py (oracle.plane_bg_oracle.compare_reference)
  caching     a second frame reuses the images and the masks (build counters); a replaced xyz, an in-place edit autograd sees and a
              new img_lst each rebuild; a write through .data needs plane_bg.reset; results never change
  refusals    non-fp32 images and a raydir batch other than 1 raise
  end to end  runner.render_image on the dtu_surface frame with the drop-in's bg_ray is bit-identical to the same render given the
              oracle's bg_ray
"""
import types

import numpy as np
import pytest
import torch

from oracle import plane_bg_oracle as po
from pointnerf_b200 import plane_bg, runner, scene

import test_plane_bg_oracle as tpo

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
F32 = np.float32


def _fixture():
    return np.load(tpo.GOLDEN)


def _model(xyz):
    return types.SimpleNamespace(neural_points=types.SimpleNamespace(xyz=xyz))


def _inputs(case):
    """The reference's list arguments of set_bg (img_lst on the host, as gen_points_filter_embeddings keeps them)."""
    v = case["views"]
    G = len(v["hdwd"])
    img_lst = [torch.from_numpy(np.ascontiguousarray(im))[None] for im in case["imgs"]]
    w2cs = [torch.from_numpy(v["w2c"][g]).to(DEV)[None, None] for g in range(G)]
    Ks = [torch.from_numpy(v["K"][g]).to(DEV)[None] for g in range(G)]
    hdwd = [[int(h[0]), int(h[1])] for h in v["hdwd"]]
    return img_lst, [None] * G, w2cs, Ks, hdwd


def _batch(case):
    return dict(campos=torch.from_numpy(case["campos"]).to(DEV)[None], raydir=torch.from_numpy(case["raydir"]).to(DEV)[None],
                plane_pnt=torch.from_numpy(case["plane_pnt"])[None], plane_normal=torch.from_numpy(case["plane_normal"])[None],
                plane_color=torch.from_numpy(case["plane_color"]).to(DEV)[None])


def _oracle_masks(case):
    G = len(case["views"]["hdwd"])
    if "fg_masks" in case:
        return [case["fg_masks"][:, g] for g in range(G)]
    return po.fg_masks(case["xyz"], case["views"])


def _run(case, model=None, sect=None):
    model = model or _model(torch.from_numpy(case["xyz"]).to(DEV))
    b = _batch(case)
    sect = plane_bg.gen_bg_points(b) if sect is None else sect
    fg = torch.from_numpy(case["fg_masks"]) if "fg_masks" in case else None
    bg, ret = plane_bg.set_bg(model, sect, *_inputs(case), b["plane_color"], fg_masks=fg)
    assert ret is fg
    return sect, bg, model


@pytest.mark.parametrize("name", list(tpo.CASES))
def test_fixture_cases_equal_the_fp32_oracle(name):
    case, ref, per = tpo.load_case(_fixture(), name)
    sect, bg, model = _run(case)
    want_sect = po.cross(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"])
    assert sect.shape == (1, len(case["raydir"]), 3)
    assert np.array_equal(sect[0].cpu().numpy(), want_sect)
    masks = _oracle_masks(case)
    if "fg_masks" not in case:
        assert np.array_equal(model._pnb_plane_bg.masks.cpu().numpy(), np.concatenate([m.ravel() for m in masks]))
    assert np.array_equal(bg[0].cpu().numpy(), po.bg(want_sect, case["views"], masks, case["imgs"], case["plane_color"]))
    # on the reference's own plane points: the oracle bit for bit, and the reference within the CPU test's bounds
    _, bg_r, _ = _run(case, sect=torch.from_numpy(ref["sect"]).to(DEV)[None])
    mine = bg_r[0].cpu().numpy()
    assert np.array_equal(mine, po.bg(ref["sect"], case["views"], masks, case["imgs"], case["plane_color"]))
    st = tpo.check_case(case, ref, per)
    print("\n[plane_bg gpu %s] %s" % (name, st))


def _dtu_case(G=32, N=1_000_000, H=512, W=640, seed=3):
    """A seeded DTU-sized case: a bumpy surface of N points, a plane behind it, G views on two rings around the scene, the frame's
    H*W rays from the first ring's middle camera."""
    g = np.random.default_rng(seed)
    f = 1.2 * W
    uv = g.uniform(-0.5, 0.5, (N, 2))
    z = 3.0 + 0.3 * np.sin(4 * uv[:, 0]) * np.cos(3 * uv[:, 1])
    xyz = np.stack([uv[:, 0] * W / f * z, uv[:, 1] * H / f * z, z], -1).astype(F32)
    centre = np.array([0, 0, 3.0])
    views = []
    for k in range(G):
        rot = tpo._rot_y(-0.6 + 1.2 * (k // 2) / max(G // 2 - 1, 1)) @ tpo._rot_x(0.15 if k % 2 else -0.15)
        views.append(tpo._w2c_of(rot, centre - rot @ np.array([0, 0, 3.0])))
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], F32)
    px, py = np.meshgrid(np.arange(W), np.arange(H))
    d = np.stack([(px.ravel() + 0.5 - W / 2) / f, (py.ravel() + 0.5 - H / 2) / f, np.ones(H * W)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    n = np.array([0.05, -0.4, 0.9])
    pc = np.array([0.6, 0.4, 0.3], F32)
    return dict(xyz=xyz, campos=np.zeros(3, F32), raydir=d.astype(F32), plane_pnt=np.array([0, 0, 3.6], F32),
                plane_normal=(n / np.linalg.norm(n)).astype(F32), plane_color=pc,
                views=dict(w2c=np.array(views), K=np.array([K] * G), hdwd=np.array([[H, W]] * G)),
                imgs=list(tpo._images(g, G, H, W, pc)))


def test_dtu_sized_case_equals_the_fp32_oracle():
    case = _dtu_case()
    sect, bg, model = _run(case)
    want_sect = po.cross(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"])
    assert np.array_equal(sect[0].cpu().numpy(), want_sect)
    masks = po.fg_masks(case["xyz"], case["views"])
    assert np.array_equal(model._pnb_plane_bg.masks.cpu().numpy(), np.concatenate([m.ravel() for m in masks]))
    want = po.bg(want_sect, case["views"], masks, case["imgs"], case["plane_color"])
    got = bg[0].cpu().numpy()
    assert np.array_equal(got, want)
    print("\n[plane_bg dtu] %d rays, %.1f %% with a plane colour, %.1f %% foreground cells"
          % (len(got), 100 * float(np.any(got != 0, 1).mean()), 100 * float(np.mean([m.mean() for m in masks]))))


def test_caching_reuses_and_rebuilds():
    case, _, _ = tpo.load_case(_fixture(), "frustum")
    xyz = torch.nn.Parameter(torch.from_numpy(case["xyz"]).to(DEV))
    model = _model(xyz)
    b = _batch(case)
    args = _inputs(case)
    sect = plane_bg.gen_bg_points(b)
    first, _ = plane_bg.set_bg(model, sect, *args, b["plane_color"])
    c = model._pnb_plane_bg
    assert (c.n_image_builds, c.n_view_builds, c.n_mask_builds) == (1, 1, 1)
    half = sect[:, ::2].contiguous()                     # a second frame: other rays, the same views and cloud
    second, _ = plane_bg.set_bg(model, half, *args, b["plane_color"])
    assert torch.equal(second, first[:, ::2])
    assert (c.n_image_builds, c.n_view_builds, c.n_mask_builds) == (1, 1, 1)
    model.neural_points.xyz = torch.nn.Parameter(xyz.detach().clone())          # a replaced cloud
    assert torch.equal(plane_bg.set_bg(model, sect, *args, b["plane_color"])[0], first) and c.n_mask_builds == 2
    with torch.no_grad():
        model.neural_points.xyz.mul_(1.0)                                        # an in-place edit autograd sees
    assert torch.equal(plane_bg.set_bg(model, sect, *args, b["plane_color"])[0], first) and c.n_mask_builds == 3
    new_imgs = [t.clone() for t in args[0]]                                      # a new img_lst
    assert torch.equal(plane_bg.set_bg(model, sect, new_imgs, *args[1:], b["plane_color"])[0], first)
    assert c.n_image_builds == 2 and c.n_mask_builds == 3
    # a write through .data is invisible to the version counter: the masks stay those of the old cloud until reset
    model.neural_points.xyz.data += 100.0
    assert torch.equal(plane_bg.set_bg(model, sect, new_imgs, *args[1:], b["plane_color"])[0], first) and c.n_mask_builds == 3
    plane_bg.reset(model)
    moved, _ = plane_bg.set_bg(model, sect, new_imgs, *args[1:], b["plane_color"])
    assert model._pnb_plane_bg.n_mask_builds == 1
    want = po.bg(sect[0].cpu().numpy(), case["views"], po.fg_masks(case["xyz"] + F32(100), case["views"]), case["imgs"],
                 case["plane_color"])
    assert np.array_equal(moved[0].cpu().numpy(), want)


def test_refusals():
    case, _, _ = tpo.load_case(_fixture(), "frustum")
    model = _model(torch.from_numpy(case["xyz"]).to(DEV))
    b = _batch(case)
    img_lst, c2w, w2c, K, hdwd = _inputs(case)
    sect = plane_bg.gen_bg_points(b)
    with pytest.raises(ValueError, match="float32"):
        plane_bg.set_bg(model, sect, [t.double() for t in img_lst], c2w, w2c, K, hdwd, b["plane_color"])
    b2 = dict(b, raydir=torch.cat([b["raydir"], b["raydir"]]))
    with pytest.raises(ValueError, match="raydir"):
        plane_bg.gen_bg_points(b2)
    with pytest.raises(ValueError, match=r"\[1,R,3\]"):
        plane_bg.set_bg(model, torch.cat([sect, sect]), img_lst, c2w, w2c, K, hdwd, b["plane_color"])


def test_render_image_with_the_dropin_bg_ray():
    """The dtu_surface frame of tests/test_gpu_frustum_fused.py rendered with the drop-in's bg_ray and with the oracle's: the same
    bits (the plane 3.3 behind the camera's surface, 7 views around it)."""
    import test_gpu_frustum_fused as tff
    cfg, s, _ = tff._scene()
    net, _ = tff._net()
    d = tff._data(tff._frame())
    R0, c0 = s["camrotc2w"].astype(np.float64), s["campos"].astype(np.float64)
    centre = c0 + R0 @ np.array([0, 0, 2.5])
    n = R0 @ np.array([0.1, -0.35, 0.93])
    views = []
    for k in range(7):
        Rv = R0 @ tpo._rot_y(-0.3 + 0.1 * k)
        views.append(tpo._w2c_of(Rv, centre - Rv @ np.array([0, 0, 2.5])))
    K = s["intrinsic"].astype(F32)
    pc = np.array([0.55, 0.45, 0.35], F32)
    case = dict(xyz=net.neural_points.xyz.detach().cpu().numpy(), campos=s["campos"], raydir=d["raydir"][0].cpu().numpy(),
                plane_pnt=(c0 + R0 @ np.array([0, 0, 3.3])).astype(F32), plane_normal=(n / np.linalg.norm(n)).astype(F32),
                plane_color=pc, views=dict(w2c=np.array(views), K=np.array([K] * 7), hdwd=np.array([[cfg.H, cfg.W]] * 7)),
                imgs=list(tpo._images(np.random.default_rng(2), 7, cfg.H, cfg.W, pc)))
    b = _batch(case)
    bg_ray, _ = plane_bg.set_bg(types.SimpleNamespace(neural_points=net.neural_points), plane_bg.gen_bg_points(b), *_inputs(case),
                                b["plane_color"])
    sect = po.cross(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"])
    want = po.bg(sect, case["views"], po.fg_masks(case["xyz"], case["views"]), case["imgs"], pc)
    assert np.array_equal(bg_ray[0].cpu().numpy(), want) and np.any(want != 0)
    mine = runner.render_image(net, d, cfg.H, cfg.W, bg_ray=bg_ray)
    theirs = runner.render_image(net, d, cfg.H, cfg.W, bg_ray=torch.from_numpy(want).to(DEV)[None])
    assert torch.equal(mine["coarse_raycolor"], theirs["coarse_raycolor"])
    miss = mine["ray_mask"] == 0
    assert miss.any() and torch.equal(mine["coarse_raycolor"][miss], bg_ray[0].view(cfg.H, cfg.W, 3)[miss])
