"""CPU: oracle/depth_filter_oracle.py against the reference's own reproject_with_depth_gpu, check_geometric_consistency_gpu,
filter_by_masks_gpu, range_mask_torch (models/mvs/filter_utils.py:146-291) and alpha_masking (models/mvs/mvs_utils.py:573-607),
compiled from the reference source with the CPU redirection of tests/test_plane_bg_oracle.py.  Needs the reference tree; skipped
elsewhere, except the fixture checks.  `python tests/test_depth_filter_oracle.py` rewrites tests/golden/depth_filter_ref.npz.

Bounds (oracle/depth_filter_oracle.py derives them): a geometric match may differ only where dist < 1 or rel < 0.01 sits within its
bound of the threshold, a kept pixel only where such a match or a range face is near; averaged depths and world points agree within
their bounds; raw x, y and confidences are equal.  The dyadic case (power-of-two intrinsics, axis-permutation rotations, integer
translations and depths) is exact in any summation order: there every output is equal, including a pixel exactly at dist == 1.
"""
import ast
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import depth_filter_oracle as do, ref_shim  # noqa: E402

import test_plane_bg_oracle as tpo  # noqa: E402

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")
GOLDEN = os.path.join(ROOT, "tests", "golden", "depth_filter_ref.npz")
F32 = np.float32
FILTER_NAMES = ("reproject_with_depth_gpu", "check_geometric_consistency_gpu", "filter_by_masks_gpu", "range_mask_torch")


def load_reference():
    """A module with the four filter_utils functions and alpha_masking, compiled from the reference's source (CPU redirection)."""
    mod = types.ModuleType("filter_utils_cpu")
    mod.torch, mod.F, mod.np, mod.tqdm = torch, Fn, np, lambda x: x
    path = os.path.join(ref_shim.REF, "models", "mvs", "filter_utils.py")
    tree = ast.parse(open(path).read(), path)
    defs = [n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name in FILTER_NAMES]
    assert sorted(n.name for n in defs) == sorted(FILTER_NAMES)
    tpo._compile(path, defs, mod.__dict__)
    mpath = os.path.join(ref_shim.REF, "models", "mvs", "mvs_utils.py")
    mtree = ast.parse(open(mpath).read(), mpath)
    # alpha_masking calls torch.cuda.empty_cache(), which the redirection turns into torch.cpu.empty_cache(): give it a no-op one
    tns = types.ModuleType("torch_for_alpha_masking")
    tns.__dict__.update(torch.__dict__)
    tns.cpu = types.SimpleNamespace(empty_cache=lambda: None)
    ns = dict(torch=tns)
    tpo._compile(mpath, [n for n in mtree.body if isinstance(n, ast.FunctionDef) and n.name == "alpha_masking"], ns)
    mod.alpha_masking = ns["alpha_masking"]
    return mod


# ------------------------------------------------------------------------------------------------ cases
def _look_at(campos, target):
    z = np.asarray(target, float) - campos
    z /= np.linalg.norm(z)
    x = np.cross([0.0, 1.0, 0.0], z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    E = np.eye(4)
    E[:3, :3] = np.stack([x, y, z])
    E[:3, 3] = -E[:3, :3] @ campos
    return E


def surface_case(V=5, H=40, W=48, seed=0, geo_n=2, ranges=(-1.2, -1.2, 2.0, 1.2, 1.2, 3.6), thresh=0.5):
    """V cameras on an arc looking at a bumpy surface about 3 away, rendered exactly (ray / height-field by bisection), with
    noise of 0.4 % so that many pixels sit near dist 1 and rel 0.01; a zero-depth patch, one camera behind the surface's
    edge points (points behind a source camera) and taps that leave the image (border clamp)."""
    g = np.random.default_rng(seed)
    f = 0.9 * W
    K = np.array([[f, 0, W / 2 - 0.3], [0, f * 1.02, H / 2 + 0.2], [0, 0, 1]], F32)
    Es = []
    for v in range(V):
        a = -0.35 + 0.7 * v / max(V - 1, 1)
        c = np.array([3 * np.sin(a), 0.25 * np.cos(3 * a), 3 - 3 * np.cos(a)])
        Es.append(_look_at(c, [0.05, 0.0, 3.0]))
    if V >= 4:
        Es[-1] = _look_at(np.array([0.0, 0.0, 3.4]), [0.0, 0.0, 6.0])      # inside the scene, looking away: points behind it

    def height(x, y):
        return 3.0 + 0.25 * np.sin(3 * x) * np.cos(2 * y)

    depth = np.zeros((V, H, W), F32)
    xy = np.zeros((V, H, W, 2), F32)
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    for v in range(V):
        E = Es[v]
        Rc, cpos = E[:3, :3].T, -E[:3, :3].T @ E[:3, 3]
        dcam = np.stack([(xx - K[0, 2]) / K[0, 0], (yy - K[1, 2]) / K[1, 1], np.ones_like(xx, float)], -1)
        dw = dcam @ Rc.T
        lo, hi = np.zeros((H, W)), np.full((H, W), 8.0)
        for _ in range(60):
            mid = (lo + hi) / 2
            pw = cpos + mid[..., None] * dw
            above = pw[..., 2] < height(pw[..., 0], pw[..., 1])
            lo, hi = np.where(above, mid, lo), np.where(above, hi, mid)
        z = lo * (1 + g.normal(0, 0.004, (H, W)))
        z[5:8, 6:10] = 0.0                                              # a zero-depth patch
        depth[v] = z
        xy[v] = np.stack([(xx - K[0, 2]) / K[0, 0] * z, (yy - K[1, 2]) / K[1, 1] * z], -1)
    conf = g.uniform(0, 1, (V, H, W)).astype(F32)
    mask = g.uniform(size=(V, H, W)) < 0.9
    return dict(depth=depth, xy=xy, conf=conf, mask=mask, K=np.array([K] * V), E=np.array(Es, F32), thresh=thresh, geo_n=geo_n,
                ranges=None if ranges is None else np.array(ranges, F32))


def dyadic_case():
    """Exact in any order: K = [[128, 0, 32], [0, 128, 16]], view 0 at the origin, view 1 translated by 129 along x, view 2 an axis
    permutation (x and y swapped, z kept).  Depth 128 everywhere in view 0 and 129 in view 1, so that (x, y) of view 0 reprojects to
    (x + 1, y) exactly: dist == 1 with rel = 1/128 < 0.01 (a `<=` would match).  Some pixels depth 256 (no match), some 0; ranges
    with a face exactly on a world coordinate."""
    H, W = 32, 64
    K = np.array([[128, 0, 32], [0, 128, 16], [0, 0, 1]], F32)
    E0 = np.eye(4)
    E1 = np.eye(4)
    E1[0, 3] = 129.0
    E2 = np.eye(4)
    E2[:3, :3] = [[0, 1, 0], [1, 0, 0], [0, 0, 1]]
    depth = np.full((3, H, W), 128.0, F32)
    depth[1] = 129.0
    depth[0, 5:9, 10:20] = 256.0
    depth[0, 20, 3:7] = 0.0
    depth[2, :, ::3] = 64.0
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    xy = np.stack([np.stack([(xx - 32) * depth[v] / 128, (yy - 16) * depth[v] / 128], -1) for v in range(3)]).astype(F32)
    conf = np.ones((3, H, W), F32)
    conf[:, ::5, ::7] = 0.25
    mask = np.ones((3, H, W), bool)
    return dict(depth=depth, xy=xy, conf=conf, mask=mask, K=np.array([K] * 3), E=np.array([E0, E1, E2], F32), thresh=0.5, geo_n=1,
                ranges=np.array([-30.0, -16.0, 0.0, 24.0, 15.0, 200.0], F32))


def alpha_case(N=20000, V=6, H=30, W=40, seed=1, near_far=(0.5, 6.0), range_test=True):
    g = np.random.default_rng(seed)
    f = 0.9 * W
    K = np.array([[f, 0, W / 2], [0, f, H / 2], [0, 0, 1]], F32)
    Es = [_look_at(np.array([3 * np.sin(a), 0.2, 3 - 3 * np.cos(a)]), [0, 0, 3]) for a in np.linspace(-0.5, 0.5, V)]
    Es[-1] = _look_at(np.array([0.0, 0.0, 3.2]), [0.0, 0.0, 6.0])          # points behind this camera
    pts = np.concatenate([g.uniform([-1.5, -1.5, 1.5], [1.5, 1.5, 4.5], (N, 3)), [[0, 0, 3.2 + 1e-7]]]).astype(F32)
    alpha = g.choice(np.array([0.0, 0.1, 0.5, 1.0], F32), size=(V, H, W), p=[0.02, 0.02, 0.04, 0.92])
    return dict(points=pts, alpha=alpha, K=np.array([K] * V), w2c=np.array(Es, F32), near_far=near_far, range_test=range_test)


def dyadic_alpha_case():
    """Power-of-two intrinsics, axis-permutation w2c, dyadic points: projections land exactly on integers (floor boundaries), on the
    image's right and bottom edges, and z exactly on near - 1 and far."""
    H, W = 16, 32
    K = np.array([[8, 0, 16], [0, 8, 8], [0, 0, 1]], F32)
    w = [np.eye(4), np.eye(4)]
    w[1][:3, :3] = [[0, 1, 0], [1, 0, 0], [0, 0, 1]]
    gx, gy, gz = np.meshgrid(np.arange(-20, 21) / 8.0, np.arange(-12, 13) / 8.0, [1.0, 2.0, 4.0, 5.0], indexing="ij")
    pts = np.stack([gx.ravel() * gz.ravel(), gy.ravel() * gz.ravel(), gz.ravel()], -1).astype(F32)
    g = np.random.default_rng(4)
    alpha = g.choice(np.array([0.0, 0.1, 0.5, 1.0], F32), size=(2, H, W))
    return dict(points=pts, alpha=alpha, K=np.array([K] * 2), w2c=np.array(w, F32), near_far=(2.0, 4.0), range_test=True)


CASES = dict(surface=lambda: surface_case(geo_n=3), surface_geo0=lambda: surface_case(V=4, seed=2, geo_n=0, ranges=None),
             surface_geoV=lambda: surface_case(V=4, seed=3, geo_n=4), single=lambda: surface_case(V=1, seed=4),
             dyadic=dyadic_case)
ALPHA_CASES = dict(range_nf=lambda: alpha_case(), norange_nf=lambda: alpha_case(seed=2, range_test=False),
                   range_nonf=lambda: alpha_case(seed=3, near_far=None), norange_nonf=lambda: alpha_case(seed=4, near_far=None,
                                                                                                       range_test=False),
                   dyadic=dyadic_alpha_case)


def _opt(case):
    return types.SimpleNamespace(manual_depth_view=1, depth_conf_thresh=case["thresh"], geo_cnsst_num=case["geo_n"], default_conf=-1,
                                 far_plane_shift=None, ranges=list(case["ranges"]) if case["ranges"] is not None else [-100.0] * 6)


def ref_inputs(case):
    V = len(case["depth"])
    cam = [torch.from_numpy(np.concatenate([case["xy"][v], case["depth"][v][..., None]], -1))[None, None, None] for v in range(V)]
    K = [torch.from_numpy(case["K"][v])[None] for v in range(V)]
    E = [torch.from_numpy(case["E"][v])[None] for v in range(V)]
    conf = [torch.from_numpy(case["conf"][v])[None, None] for v in range(V)]
    mask = [torch.from_numpy(case["mask"][v])[None, None] for v in range(V)]
    return cam, K, E, conf, mask


def run_reference(ref, case):
    cam, K, E, conf, mask = ref_inputs(case)
    V = len(cam)
    out = []
    opt0 = types.SimpleNamespace(**dict(vars(_opt(case)), ranges=[-100.0] * 6))
    c0, w0, f0 = ref.filter_by_masks_gpu(cam, K, E, conf, mask, opt0)
    c1, w1, f1 = ref.filter_by_masks_gpu(cam, K, E, conf, mask, _opt(case))
    for r in range(V):
        geo = np.zeros(case["depth"].shape[1:], np.int64)
        for s in range(V):
            if s != r:
                m = ref.check_geometric_consistency_gpu(cam[r][0, 0, 0, ..., 2], K[r][0], E[r][0], cam[s][0, 0, 0, ..., 2], K[s][0],
                                                        E[s][0])[0]
                geo += m.numpy()
        out.append(dict(geo=geo, cam0=c0[r].numpy(), world0=w0[r].numpy(), conf0=f0[r].numpy(), cam=c1[r].numpy(), world=w1[r].numpy(),
                        conf=f1[r].numpy()))
    return out


def run_reference_alpha(ref, case):
    V = len(case["alpha"])
    opt = types.SimpleNamespace(alpha_range=1 if case["range_test"] else 0, inall_img=1)
    with torch.no_grad():
        m = ref.alpha_masking(torch.from_numpy(case["points"]), [case["alpha"][v][None] for v in range(V)], list(case["K"]), list(case["w2c"]),
                              list(case["w2c"]), case["near_far"], opt=opt)
    return m.numpy()


# ------------------------------------------------------------------------------------------------ fixture
CASE_KEYS = ("depth", "xy", "conf", "mask", "K", "E")


def golden_cases(ref):
    out = {}
    for name, make in CASES.items():
        c = make()
        p = "f_%s_" % name
        out.update({p + k: c[k] for k in CASE_KEYS})
        out[p + "scalars"] = np.array([c["thresh"], c["geo_n"]], np.float64)
        if c["ranges"] is not None:
            out[p + "ranges"] = c["ranges"]
        for r, rv in enumerate(run_reference(ref, c)):
            for k, v in rv.items():
                out[p + "ref%d_%s" % (r, k)] = v
    for name, make in ALPHA_CASES.items():
        c = make()
        p = "a_%s_" % name
        out.update({p + k: c[k] for k in ("points", "alpha", "K", "w2c")})
        out[p + "opts"] = np.array([-1, -1, int(c["range_test"])] if c["near_far"] is None else list(c["near_far"]) + [int(c["range_test"])],
                                   np.float64)
        out[p + "ref_mask"] = run_reference_alpha(ref, c)
    return out


def load_case(z, name):
    """A filter case and the reference's per-view results from the fixture (also used by tests/test_gpu_depth_filter.py)."""
    p = "f_%s_" % name
    c = {k: z[p + k] for k in CASE_KEYS}
    c["thresh"], c["geo_n"] = float(z[p + "scalars"][0]), int(z[p + "scalars"][1])
    c["ranges"] = z[p + "ranges"] if p + "ranges" in z else None
    keys = ("geo", "cam0", "world0", "conf0", "cam", "world", "conf")
    return c, [{k: z[p + "ref%d_%s" % (r, k)] for k in keys} for r in range(len(c["depth"]))]


def load_alpha_case(z, name):
    p = "a_%s_" % name
    c = {k: z[p + k] for k in ("points", "alpha", "K", "w2c")}
    o = z[p + "opts"]
    c["near_far"] = None if o[0] == -1 and o[1] == -1 else (float(o[0]), float(o[1]))
    c["range_test"] = bool(o[2])
    return c, z[p + "ref_mask"]


def check(name, case, r, fault=None):
    """compare_reference; on the dyadic case, which is exact in any order, every output of every view must also be equal."""
    st = do.compare_reference(case, r, fault=fault)
    if name == "dyadic":
        for v, rv in enumerate(r):
            o = do.filter_view(case, v, fault=fault)
            for k in ("cam", "world", "conf"):
                assert np.array_equal(rv[k], o[k]), "dyadic view %d: %s differs" % (v, k)
    return st


@pytest.fixture(scope="module")
def ref():
    return load_reference()


@needs_ref
@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference(ref, name):
    case = CASES[name]()
    r = run_reference(ref, case)
    st = check(name, case, r)
    print("\n[depth_filter %s] %s" % (name, st))
    assert (st["kept"] > 0) == (name != "surface_geoV")         # geo_cnsst_num V: no pixel has V matches
    if name != "dyadic":
        assert st["near_geo"] <= 0.1 * st["pixels"]                # the bounds leave most pixels to be compared


@needs_ref
@pytest.mark.parametrize("name", list(ALPHA_CASES))
def test_alpha_oracle_matches_reference(ref, name):
    case = ALPHA_CASES[name]()
    m = run_reference_alpha(ref, case)
    st = do.compare_alpha(case, m)
    print("\n[alpha %s] %s" % (name, st))
    mine = do.alpha_mask(case["points"], case["alpha"], case["K"], case["w2c"], case["near_far"], case["range_test"])
    assert mine.any() and (~mine).any()
    if name == "dyadic":
        assert np.array_equal(m, mine)
    else:
        assert st["near"] <= 0.05 * st["points"]


def test_cases_reach_every_branch():
    """The dyadic case has a match at dist == 1 exactly and a world coordinate exactly on a range face; the surface cases have
    zero depths, taps clamped at the border and source points behind a camera; the alpha cases have points in and out of the image."""
    c = dyadic_case()
    mats = do.view_matrices(c["K"], c["E"])
    pix = np.nonzero(c["conf"][0].reshape(-1) > 0.5)[0]
    _, _, per = do.geo_pass(c, 0, mats, pix, detail=True)
    one = per[0]
    assert np.any((one["dist"] == 1) & (one["rel"] < do.REL))
    o = do.filter_view(dict(c, ranges=None), 0, mats)
    assert np.any(o["world"] == c["ranges"][None, :3]) or np.any(o["world"] == c["ranges"][None, 3:])
    s = surface_case()
    mats = do.view_matrices(s["K"], s["E"])
    pix = np.nonzero(s["conf"][0].reshape(-1) > s["thresh"])[0]
    _, _, per = do.geo_pass(s, 0, mats, pix, detail=True)
    H, W = s["depth"].shape[1:]
    assert (s["depth"][0].reshape(-1)[pix] == 0).any()
    assert any(((p["xs"] < 0) | (p["xs"] > W - 1) | (p["ys"] < 0) | (p["ys"] > H - 1)).any() for p in per)
    back = per[-1]
    E = s["E"][-1].astype(np.float64)
    assert (back["match"] == 0).any()
    d = s["depth"][0].reshape(-1)[pix].astype(np.float64)
    y, x = np.divmod(pix, W)
    cam = np.stack([(x - s["K"][0][0, 2]) / s["K"][0][0, 0] * d, (y - s["K"][0][1, 2]) / s["K"][0][1, 1] * d, d, np.ones_like(d)], -1)
    world = cam @ np.linalg.inv(s["E"][0].astype(np.float64)).T
    assert ((world @ E.T)[:, 2] < 0).any()
    for make in ALPHA_CASES.values():
        a = make()
        _, per = do.alpha_mask(a["points"], a["alpha"], a["K"], a["w2c"], a["near_far"], a["range_test"], detail=True)
        H, W = a["alpha"].shape[1:]
        inb = np.concatenate([(p["ix"] >= 0) & (p["ix"] < W) & (p["iy"] >= 0) & (p["iy"] < H) for p in per])
        assert inb.any() and (~inb).any()


@needs_ref
@pytest.mark.parametrize("fault", do.FAULTS)
def test_planted_faults_are_caught(ref, fault):
    """Each planted fault of the fp32 oracle makes the bounded comparison fail on at least one case."""
    names = dict(single_view_geo=["single"], dist_le=["dyadic"]).get(fault, list(CASES))
    caught = False
    for name in names:
        case = CASES[name]()
        try:
            check(name, case, run_reference(ref, case), fault=fault)
        except AssertionError:
            caught = True
            break
    assert caught, "the comparison did not catch the planted fault %s" % fault


@needs_ref
def test_golden_fixture_is_what_the_reference_returns(ref):
    got = golden_cases(ref)
    want = _load_golden()
    assert sorted(want) == sorted(got)
    for k in got:
        assert np.array_equal(want[k], got[k], equal_nan=True), k


def _load_golden():
    z = {}
    for i in range(1, 100):
        p = GOLDEN.replace(".npz", ".part%d.npz" % i) if i > 1 else GOLDEN
        if not os.path.exists(p):
            break
        z.update(dict(np.load(p)))
    return z


def test_golden_fixture_meets_the_oracle():
    z = _load_golden()
    for name in CASES:
        check(name, *load_case(z, name))
    for name in ALPHA_CASES:
        do.compare_alpha(*load_alpha_case(z, name))


if __name__ == "__main__":
    got = golden_cases(load_reference())
    parts, cur, size = [], {}, 0
    for k, v in got.items():
        if size + v.nbytes > 1_500_000 and cur:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    for i, p in enumerate(parts):
        path = GOLDEN if i == 0 else GOLDEN.replace(".npz", ".part%d.npz" % (i + 1))
        np.savez_compressed(path, **p)
        print("wrote", path, os.path.getsize(path))
