"""CPU: oracle/plane_bg_oracle.py against the reference's own gen_bg_points, get_rayplane_cross, homo_warp_nongrid, homo_warp_fg_mask,
id2mask, extract_from_2d_grid (models/mvs/mvs_utils.py:299-421) and MvsPointsVolumetricModel.set_bg
(models/mvs_points_volumetric_model.py:272-310), compiled from the reference source.  Needs the reference tree; skipped elsewhere.
`python tests/test_plane_bg_oracle.py` rewrites tests/golden/plane_bg_ref.npz from the same functions.

Redirection: the reference creates its identity c2w with `device="cuda"` and moves the grid_sample result back with `.cuda()`.  The
compiled functions have every `device="cuda"` keyword replaced by `device="cpu"` and every `.cuda()` call by `.cpu()`; nothing else
changes, and the images are sampled on the CPU exactly as the reference samples them.

Bounds (oracle/plane_bg_oracle.py derives them): the reference's matmuls sum the 4 camera terms and the 3 pixel terms in an order of
their own, so a decision may differ where the float64 value lies within EPS_U = 2 (|K00| |d px| + |K01| |d py| + g3 sum |terms|) of its
boundary (bounds, ceil), with |d px| <= (g4 S_x + |px| g4 S_z) / |z| + u |px| and g_n = n u, u = 2^-24; dot >= 1e-3 within
2 g3 sum |n_k d_k|; the fit within EPS_C = 2 M (EPS_X + EPS_Y) + 16 u M of c +- 0.03 (M = max |image|, EPS_X the scaled EPS_U plus four
roundings of x).  Where every decision of a ray agrees, its bg_ray agrees within the largest EPS_C of its views; a foreground-mask cell
may differ only where a point within EPS_U of a cell boundary may land.  The dyadic case (power-of-two intrinsics, axis-aligned
views, dyadic points and rays, (WD-1)/2 a power of two) is exact in any summation order, so there everything must be equal, including
the samples on integer coordinates, on u = WD-1 and on pixels whose colour is exactly an fp32 fit bound.
"""
import ast
import math
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import plane_bg_oracle as po, ref_shim  # noqa: E402
from pointnerf_b200 import scene  # noqa: E402

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")

GOLDEN = os.path.join(ROOT, "tests", "golden", "plane_bg_ref.npz")
MVS_NAMES = ("gen_bg_points", "get_rayplane_cross", "homo_warp_nongrid", "homo_warp_fg_mask", "id2mask", "extract_from_2d_grid")
F32 = np.float32


class _ToCpu(ast.NodeTransformer):
    def visit_keyword(self, node):
        self.generic_visit(node)
        if node.arg == "device" and isinstance(node.value, ast.Constant) and node.value.value == "cuda":
            node.value = ast.Constant("cpu")
        return node

    def visit_Attribute(self, node):
        self.generic_visit(node)
        if node.attr == "cuda":
            node.attr = "cpu"
        return node


def _compile(path, defs, ns):
    tree = ast.Module(body=[_ToCpu().visit(d) for d in defs], type_ignores=[])
    exec(compile(ast.fix_missing_locations(tree), path, "exec"), ns)


def load_reference():
    """A module with the six mvs_utils functions and set_bg, compiled from the reference's source with the CPU redirection."""
    path = os.path.join(ref_shim.REF, "models", "mvs", "mvs_utils.py")
    tree = ast.parse(open(path).read(), path)
    mod = types.ModuleType("mvs_utils_plane")
    mod.torch, mod.F = torch, Fn
    defs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in MVS_NAMES]
    assert sorted(n.name for n in defs) == sorted(MVS_NAMES)
    _compile(path, defs, mod.__dict__)
    mpath = os.path.join(ref_shim.REF, "models", "mvs_points_volumetric_model.py")
    mtree = ast.parse(open(mpath).read(), mpath)
    cls = [n for n in mtree.body if isinstance(n, ast.ClassDef) and n.name == "MvsPointsVolumetricModel"][0]
    sb = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "set_bg"]
    ns = dict(torch=torch, mvs_utils=mod)
    _compile(mpath, sb, ns)
    mod.set_bg = ns["set_bg"]
    return mod


# ------------------------------------------------------------------------------------------------ cases
def _w2c_of(rot_c2w, campos):
    w = np.eye(4)
    w[:3, :3] = rot_c2w.T
    w[:3, 3] = -rot_c2w.T @ campos
    return w.astype(F32)


def _rot_y(a):
    return np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])


def _rot_x(a):
    return np.array([[1, 0, 0], [0, math.cos(a), -math.sin(a)], [0, math.sin(a), math.cos(a)]])


def _images(g, G, H, W, pc, step=2.0 ** -10):
    """Values around the plane colour on a 2^-10 grid (about 1 in 8 samples fits all three channels), with some pixels exactly on an
    fp32 fit bound and some one ulp outside it."""
    pc = np.asarray(pc, F32)
    lo, hi = pc - po.THRESH, pc + po.THRESH
    img = (pc[None, :, None, None] + np.round(g.uniform(-0.06, 0.06, (G, 3, H, W)) / step) * step).astype(F32)
    for v in (lo, hi, np.nextafter(lo, F32(-1)), np.nextafter(hi, F32(2))):
        sel = g.uniform(size=(G, H, W)) < 0.04
        for c in range(3):
            img[:, c][sel] = v[c]
    return img


def frustum_case():
    """scene.make_frustum_scene (a bumpy surface 2.5 in front of the camera) with a plane behind it, its normal pointing away from the
    camera as DTU's does; 7 views: the render camera, two orbits, a pitch, a grazing orbit, one inside the cloud (points behind it)
    and one whose HDWD differs from its image; rays through every pixel centre plus rays with n . d < 1e-3 and on either side of it."""
    cfg = scene.FrustumConfig("plane_bg", N=6000, H=48, W=64, focal=80.0)
    s = scene.make_frustum_scene(cfg)
    R0, c0 = s["camrotc2w"].astype(np.float64), s["campos"].astype(np.float64)
    centre = c0 + R0 @ np.array([0, 0, 2.5])
    n_cam = np.array([0.1, -0.35, 0.93])
    n = R0 @ (n_cam / np.linalg.norm(n_cam))
    pnt = c0 + R0 @ np.array([0, 0, 3.3])
    views = []
    for rot, dist in ((np.eye(3), 2.5), (_rot_y(0.25), 2.5), (_rot_y(-0.3), 2.6), (_rot_x(0.3), 2.5), (_rot_y(1.4), 2.5),
                      (np.eye(3), 0.0), (_rot_y(0.15), 2.4)):
        Rv = R0 @ rot
        views.append(_w2c_of(Rv, centre - Rv @ np.array([0, 0, dist])))
    G = len(views)
    K = np.array([[cfg.focal, 0, cfg.W / 2], [0, cfg.focal, cfg.H / 2], [0, 0, 1]], F32)
    hdwd = np.array([[cfg.H, cfg.W]] * (G - 1) + [[36, 50]], np.int64)
    Kd = np.array([K] * G)
    pix = s["pixel_idx"].astype(np.float64)
    d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ R0.T
    t = np.cross(n, [0.0, 1.0, 0.0])
    t /= np.linalg.norm(t)
    extra = [t + a * n for a in (0.0, -0.3, -1.0, 5e-4, 9.99e-4, 1e-3, 1.01e-3, 2e-3)] + [-d[0], np.cross(n, t)]
    d = np.concatenate([d, np.array(extra)])
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    g = np.random.default_rng(21)
    pc = np.array([0.55, 0.45, 0.35], F32)
    return dict(xyz=s["xyz_w"], campos=c0.astype(F32), raydir=d.astype(F32), plane_pnt=pnt.astype(F32), plane_normal=n.astype(F32),
                plane_color=pc, views=dict(w2c=np.array(views), K=Kd, hdwd=hdwd), imgs=list(_images(g, G, cfg.H, cfg.W, pc)))


def dyadic_case():
    """Exact in any summation order: plane z = 4 seen from the origin along (a, b, 1), a and b on a 1/8 grid, views with
    power-of-two intrinsics and axis-aligned w2c (one turned round so the plane is behind it, one looking along the plane whose
    every cell the points cover, one with a smaller HDWD than its image), HDWD and image sizes with (WD-1)/2 a power of two.  Samples land on pixel centres and half-pixels
    (bilinear weights 1, 1/2 or 1/4: every product is exact), on u = 0 and u = WD-1 exactly, and on pixels exactly on a fit bound."""
    a, b = np.meshgrid(np.arange(-32, 33) / 8.0, np.arange(-16, 17) / 8.0)
    d = np.stack([a.ravel(), b.ravel(), np.ones(a.size)], -1)
    d = np.concatenate([d, [[1, 0, 0], [0, 1, -1], [1, 1, 2.0 ** -10], [1, 0, 2.0 ** -9], [0.5, 0.25, 1]]])
    eye = np.eye(4)

    def w(rows, t):
        m = eye.copy()
        m[:3, :3] = rows
        m[:3, 3] = t
        return m

    views = [w(np.eye(3), [0, 0, 0]), w(np.eye(3), [1, -0.5, 0]), w(np.eye(3), [0, 0, 4]), w(np.diag([-1, 1, -1]), [0, 0, 2]),
             w(np.array([[0, 1, 0], [0, 0, 1], [1, 0, 0]]), [0, -4, 8]), w(np.eye(3), [0, 0, 0])]
    K = np.array([[8, 0, 32], [0, 8, 16], [0, 0, 1]], F32)
    Ks = np.array([K] * 5 + [np.array([[4, 0, 16], [0, 4, 8], [0, 0, 1]], F32)])
    hdwd = np.array([[33, 65]] * 5 + [[17, 33]], np.int64)
    ga, gb = np.meshgrid(np.arange(-8, 9) / 2.0, np.arange(-4, 5) / 2.0)
    xyz = np.stack([4 * ga.ravel(), 4 * gb.ravel(), np.full(ga.size, 4.0)], -1)
    # (0, y, 4) fill row 16 of the view along the plane, where the plane's points land at non-dyadic u: that view is all foreground
    along = np.stack([np.zeros(65), np.arange(-32, 33), np.full(65, 4.0)], -1)
    xyz = np.concatenate([xyz, along, [[0, 0, 2], [1, 1, 1], [np.inf, 0, 4], [np.nan, 0, 4]]])
    g = np.random.default_rng(5)
    pc = np.array([0.5, 0.25, 0.75], F32)
    return dict(xyz=xyz.astype(F32), campos=np.zeros(3, F32), raydir=d.astype(F32), plane_pnt=np.array([0, 0, 4], F32),
                plane_normal=np.array([0, 0, 1], F32), plane_color=pc, views=dict(w2c=np.array(views, F32), K=Ks, hdwd=hdwd),
                imgs=list(_images(g, 6, 33, 65, pc)))


def given_masks_case():
    """The frustum case's first six views (one HDWD) with a caller's fg_masks [HD, G, WD] holding 0, 0.5, 1 and 2."""
    c = frustum_case()
    G = 6
    c["views"] = {k: v[:G] for k, v in c["views"].items()}
    c["imgs"] = c["imgs"][:G]
    HD, WD = (int(x) for x in c["views"]["hdwd"][0])
    g = np.random.default_rng(8)
    c["fg_masks"] = g.choice(np.array([0, 0.5, 1, 2], F32), size=(HD, G, WD), p=[0.5, 0.2, 0.2, 0.1])
    return c


CASES = dict(frustum=frustum_case, dyadic=dyadic_case, given_masks=given_masks_case)


# ------------------------------------------------------------------------------------------------ the reference on a case
def run_reference(ref, case):
    """gen_bg_points, set_bg and, per view, the reference functions set_bg calls (homo_warp_nongrid, homo_warp_fg_mask + id2mask,
    extract_from_2d_grid) as set_bg's loop calls them.  Returns numpy arrays."""
    views, imgs = case["views"], case["imgs"]
    G = len(views["hdwd"])
    batch = dict(campos=torch.from_numpy(case["campos"])[None], raydir=torch.from_numpy(case["raydir"])[None],
                 plane_pnt=torch.from_numpy(case["plane_pnt"])[None], plane_normal=torch.from_numpy(case["plane_normal"])[None])
    sect = ref.gen_bg_points(batch)
    xyz = torch.from_numpy(case["xyz"])
    model = types.SimpleNamespace(neural_points=types.SimpleNamespace(xyz=xyz))
    img_lst = [torch.from_numpy(im)[None] for im in imgs]
    w2cs_lst = [torch.from_numpy(views["w2c"][g])[None, None] for g in range(G)]
    K_lst = [torch.from_numpy(views["K"][g])[None] for g in range(G)]
    hdwd_lst = [[int(h[0]), int(h[1])] for h in views["hdwd"]]
    given = torch.from_numpy(case["fg_masks"]) if "fg_masks" in case else None
    bg, fg_ret = ref.set_bg(model, sect, img_lst, [None] * G, w2cs_lst, K_lst, hdwd_lst, torch.from_numpy(case["plane_color"]),
                            fg_masks=given)
    assert fg_ret is given
    c2w = torch.eye(4)[None]
    out = dict(sect=sect[0].numpy(), bg=bg[0].numpy(), fg=[], per=[])
    for g in range(G):
        HD, WD = hdwd_lst[g]
        src_grid, mask, hard = ref.homo_warp_nongrid(c2w, w2cs_lst[g][:, 0], K_lst[g], sect, HD, WD, filter=False, tolerate=0.1)
        fg = ref.homo_warp_fg_mask(c2w, w2cs_lst[g][:, 0], K_lst[g], xyz[None], HD, WD, tolerate=0.1)
        out["fg"].append(fg.numpy())
        used = given[:, g] if given is not None else fg
        inb = mask[0, :, 0].clone()
        hv = hard[:, inb, :]
        mask[0, inb, 0] = used[hv[0, :, 1].long(), hv[0, :, 0].long()] < 1
        sel = mask[0, :, 0]
        val = ref.extract_from_2d_grid(img_lst[g][0:1], src_grid[:, sel, :], mask)
        out["per"].append(dict(inb=inb.numpy(), sel=sel.numpy(), val=val[0, sel].numpy()))
    return out


def golden_cases(ref):
    out = {}
    for name, make in CASES.items():
        c = make()
        r = run_reference(ref, c)
        p = name + "_"
        out.update({p + "ref_sect": r["sect"], p + "ref_bg": r["bg"]})
        if name != "given_masks":                        # its inputs are the frustum case's first six views
                out.update({p + "xyz": c["xyz"], p + "campos": c["campos"], p + "raydir": c["raydir"], p + "plane_pnt": c["plane_pnt"],
                        p + "plane_normal": c["plane_normal"], p + "plane_color": c["plane_color"], p + "w2c": c["views"]["w2c"],
                        p + "K": c["views"]["K"], p + "hdwd": c["views"]["hdwd"], p + "imgs": np.stack(c["imgs"])})
        if "fg_masks" in c:
            out[p + "fg_masks"] = c["fg_masks"]
        for g, (fg, pv) in enumerate(zip(r["fg"], r["per"])):
            out.update({p + "ref_fg%d" % g: fg, p + "ref_inb%d" % g: pv["inb"], p + "ref_sel%d" % g: pv["sel"], p + "ref_val%d" % g: pv["val"]})
    return out


def load_case(z, name):
    """A case and the reference's results from the fixture (also used by tests/test_gpu_plane_bg.py)."""
    p = name + "_"
    q = "frustum_" if name == "given_masks" else p
    G = z[p + "fg_masks"].shape[1] if name == "given_masks" else len(z[q + "hdwd"])
    case = dict(xyz=z[q + "xyz"], campos=z[q + "campos"], raydir=z[q + "raydir"], plane_pnt=z[q + "plane_pnt"],
                plane_normal=z[q + "plane_normal"], plane_color=z[q + "plane_color"],
                views=dict(w2c=z[q + "w2c"][:G], K=z[q + "K"][:G], hdwd=z[q + "hdwd"][:G]), imgs=list(z[q + "imgs"][:G]))
    if p + "fg_masks" in z:
        case["fg_masks"] = z[p + "fg_masks"]
    ref = dict(sect=z[p + "ref_sect"], bg=z[p + "ref_bg"], fg=[z[p + "ref_fg%d" % g] for g in range(G)])
    per = [dict(inb=z[p + "ref_inb%d" % g], sel=z[p + "ref_sel%d" % g], val=z[p + "ref_val%d" % g]) for g in range(G)]
    return case, ref, per


def check_case(case, ref, per):
    """compare_reference with the case's masks; returns its counts."""
    used = None
    if "fg_masks" in case:
        used = [case["fg_masks"][:, g] for g in range(len(case["views"]["hdwd"]))]
    return po.compare_reference(case, ref, per, masks_used=used)


@pytest.fixture(scope="module")
def ref():
    return load_reference()


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(ref, name):
    case = CASES[name]()
    r = run_reference(ref, case)
    st = check_case(case, dict(sect=r["sect"], bg=r["bg"], fg=r["fg"]), r["per"])
    print("\n[plane_bg %s] %s" % (name, st))
    mine = po.bg(r["sect"], case["views"], [case["fg_masks"][:, g] for g in range(len(r["fg"]))] if "fg_masks" in case else r["fg"],
                 case["imgs"], case["plane_color"])
    if name != "dyadic":
        assert st["near_rays"] <= 0.1 * st["rays"]      # the bounds leave most rays to be compared
    else:
        # exact arithmetic: no near decision may differ, every result is equal
        assert np.array_equal(r["sect"], po.cross(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"]))
        for a, b in zip(r["fg"], po.fg_masks(case["xyz"], case["views"])):
            assert np.array_equal(a, b)
        assert np.array_equal(r["bg"], mine)


@pytest.mark.parametrize("name", list(CASES))
def test_cases_reach_every_branch(name):
    """Every case has grazing rays, samples out of bounds, on a foreground cell, fitting and not fitting; the dyadic case has samples
    on u = WD-1 and v = HD-1 exactly and pixels exactly on a fit bound that fit."""
    case = CASES[name]()
    sect = po.cross(case["campos"], case["raydir"], case["plane_pnt"], case["plane_normal"])
    assert np.all(sect == 0, 1).any() and (~np.all(sect == 0, 1)).any()
    G = len(case["views"]["hdwd"])
    masks = [case["fg_masks"][:, g] for g in range(G)] if "fg_masks" in case else po.fg_masks(case["xyz"], case["views"])
    _, per = po.bg(sect, case["views"], masks, case["imgs"], case["plane_color"], detail=True)
    inb = np.array([p["inb"] for p in per])
    sel = np.array([p["sel"] for p in per])
    fit = np.concatenate([p["fit"] for p in per])
    assert (~inb).any() and (inb & ~sel).any() and fit.any() and (~fit).any()
    if name == "dyadic":
        edge = any((p["inb"] & (p["u"] == F32(int(h[1]) - 1))).any() for p, h in zip(per, case["views"]["hdwd"]))
        edge_v = any((p["inb"] & (p["v"] == F32(int(h[0]) - 1))).any() for p, h in zip(per, case["views"]["hdwd"]))
        lo = case["plane_color"] - po.THRESH
        on_bound = any((p["fit"] & np.any(p["val"] == lo, 1)).any() for p in per)
        assert edge and edge_v and on_bound
        behind = case["views"]["w2c"][3]
        assert (sect[~np.all(sect == 0, 1)] @ behind[2, :3] + behind[2, 3] < 0).all() and per[3]["inb"].any()


def test_golden_fixture_is_what_the_reference_returns(ref):
    got = golden_cases(ref)
    want = np.load(GOLDEN)
    assert sorted(want.files) == sorted(got)
    for k in got:
        assert np.array_equal(want[k], got[k], equal_nan=True), k


def test_golden_fixture_meets_the_oracle():
    z = np.load(GOLDEN)
    for name in CASES:
        check_case(*load_case(z, name))


if __name__ == "__main__":
    np.savez_compressed(GOLDEN, **golden_cases(load_reference()))
    print("wrote", GOLDEN)
