"""GPU: the DTU frame bench_frustum.py times, at its size, against the CPU query oracle and float64.

Every other frustum test runs the 160 x 120 frame of 30k points (an 80 x 60 x 400 grid).  bench_frustum.py times the DTU scripts'
configuration (wcoord_query 0, F = 63, SR 40, K 8) on FRAME: 800 x 600 pixels, 400k points, focal 1000, a 400 x 300 x 400 grid.  Counted
with the CPU oracle over the whole frame (tests/test_frustum_bench_scale_method.py asserts these figures on the CPU):
  R' 430,164 of 480,000 rays; 1.5M words per frustum bitmask (the build's block-sum scan runs two passes of 1024); 2,982,660 valid
  samples and 15,187,372 pair rows, so h-bar is 23,303 tiles of 128 KB (3.05 GB: byte offsets above 2^31); 223,952 valid samples take
  the > 2 vsize_z step replacement; point indices up to 399,999; max_pts 11, max_o 5, no overflow, no capped column.  The 2,796 pixels
  of the frame's border (the grid's edge columns) give 923 hit rays.

The network is bench_frustum.fused_net's, built by net() with options overridden (kernel, backward mode, agg_intrp_order, prob);
test_builder_is_the_bench_network holds net() without overrides to fused_net bit for bit.

A. The query: the drop-in querier on all 480,000 pixels, as the bench's first line calls it, equals frustum_oracle.query bit for bit
   (ray_mask, pixel ids, sample_pidx in K-slot order, sample_loc) with the same counters; the bench's chunk loop (209 calls of 2304
   rays, one build), concatenated, equals the full-frame call bit for bit, sample_loc_w and sample_ray_dirs included.
B. The forward, sample by sample: tests/test_gpu_frustum_f64.py's _run and BOUNDS on 4,096 seeded pixels over the frame and every
   border pixel ((sigma, rgb) and h-bar of every valid sample, the composite against frustum_shade_f64.march on the kernel's own
   sigma_rgb, the aux outputs, poison and the same call again), frozen, general and fp32 at agg_intrp_order 2, frozen and general at 1.
   The float64 shading runs one chunk of rays at a time on the rows of the points gathered.
C. The whole frame: runner.render_image of the frame (the bench's call) equals render_full on B's pixels bit for bit, which equals
   forward() on them; runner.probe_image of the frame equals render_full(probe=True) on B's pixels bit for bit, and those meet
   oracle/probe_oracle.py in float64 within tests/test_gpu_frustum_fused.py's PROBE_BOUNDS.
D. The training step: the bench's step() (the 48 x 48 centre patch, colour L2 mean over the hit rays + 1e-3 x the zero_one mean on the
   clamped conf_coefficient), its gradients against float64 autograd of frustum_shade_f64.shade on the step's own tuple with the
   backward's own LeakyReLU masks (frustum_shade_f64.kernel_slopes), one chunk of rays at a time: points within grad_check.RTOL of
   scale and point 0's conf within grad_check.point0_conf_bound, every untouched row of the 400k exactly zero, each MLP tensor within
   grad_check.FRUSTUM_MLP_RTOL of max(scale, sum |terms|) (alpha_branch.0 at order 1: ALPHA1_SUM_RTOL), the loss to float64; no
   outlier allowance.  A 96 x 96 patch (~355k pair rows) runs the dW GEMMs of a whole F = 63 backward at the split-K cap.

Measured on an H100 80GB HBM3 at a 700 W power limit: see DESIGN §6 ("The DTU frame at its size").  The file prints its regimes and
errors (pytest -s).
"""
import functools
import time

import numpy as np
import pytest
import torch

import bench_frustum
import frustum_shade_f64
import test_gpu_bench_scale_f64 as bs
import test_gpu_frustum_f64 as ff64
import test_gpu_frustum_fused as fused
import test_gpu_frustum_session as session
from oracle import frustum_oracle, grad_check, probe_oracle
from pointnerf_b200 import harness, runner, scene
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200.ray_marching import MLP_KEYS, NeuralPoints, NeuralPointsRayMarching, PointAggregator, probe_keys

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FRAME = scene.FrustumConfig("dtu_frame", N=400_000, H=600, W=800, focal=1000.0)    # bench_frustum.main's frame
CHUNK = 2304                 # the bench's chunk loop (random_sample_size 48)
ALPHA_BIAS = 300.0           # bench_frustum.fused_net: an opaque surface
ZERO_ONE_WEIGHT = 1e-3       # the bench's weight of the zero_one term
ZERO_EPS = 1e-3              # its clamp of conf_coefficient
POINT_KEYS = bs.POINT_KEYS
CHUNK_RAYS = 256             # rays per float64 chunk (~10k pair rows)


# ---- the frame, the network, the bench's inputs ----
@functools.lru_cache(None)
def frame():
    """(s, points): scene.make_frustum_scene and make_frustum_points of FRAME, as bench_frustum.main makes them."""
    s = scene.make_frustum_scene(FRAME)
    return s, scene.make_frustum_points(FRAME, s)


def net(is_train=False, **over):
    """bench_frustum.fused_net with the options `over` set before the aggregator is built (pnb_frozen, pnb_precision, pnb_bwd_fp32,
    agg_intrp_order, prob)."""
    s, pts = frame()
    opt = harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, **vars(scene.frustum_opt(FRAME, is_train=is_train)))
    for k, v in over.items():
        setattr(opt, k, v)
    agg = PointAggregator(opt, seed=5)
    with torch.no_grad():
        agg.alpha_branch[0].bias += ALPHA_BIAS
    npn = NeuralPoints(opt, DEV)
    npn.set_points(pts["xyz"].to(DEV), pts["embedding"].to(DEV), points_color=pts["color"].to(DEV), points_dir=pts["dir"].to(DEV),
                   points_conf=pts["conf"].to(DEV), parameter=True, as_stored=True)
    return NeuralPointsRayMarching(aggregator=agg.to(DEV), neural_points=npn, opt=opt)


def bench_data():
    """bench_frustum.fused's data dict: the whole frame's pixel ids, zero ray directions, a white background."""
    s, _ = frame()
    R = FRAME.H * FRAME.W
    return dict(campos=torch.from_numpy(s["campos"]).to(DEV)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(DEV)[None],
                raydir=torch.zeros((1, R, 3), device=DEV), pixel_idx=torch.from_numpy(s["pixel_idx"]).to(DEV)[None], h=FRAME.H,
                w=FRAME.W, intrinsic=s["intrinsic"], near=FRAME.near, far=FRAME.far, bg_color=torch.ones(3, device=DEV))


def pixel_data(pixels, bg=(1.0, 1.0, 1.0)):
    """The input dict of a reference dataset item of the frame for these pixels (directions through the pixel centres), as
    tests/test_gpu_frustum_f64.py forms it."""
    s, _ = frame()
    pix = np.asarray(pixels).reshape(-1, 2)
    K = s["intrinsic"]
    d = np.stack([(pix[:, 0] + 0.5 - K[0, 2]) / K[0, 0], (pix[:, 1] + 0.5 - K[1, 2]) / K[1, 1], np.ones(len(pix))], -1) @ s["camrotc2w"].T
    d = d / np.linalg.norm(d, axis=-1, keepdims=True)
    return dict(campos=torch.from_numpy(s["campos"]).to(DEV)[None], camrotc2w=torch.from_numpy(s["camrotc2w"]).to(DEV)[None],
                raydir=torch.from_numpy(d.astype(np.float32)).to(DEV)[None], pixel_idx=torch.from_numpy(pix.astype(np.int32)).to(DEV)[None],
                h=FRAME.H, w=FRAME.W, intrinsic=K, near=FRAME.near, far=FRAME.far,
                bg_color=None if bg is None else torch.tensor(bg, dtype=torch.float32, device=DEV))


def border_pixels(cfg=FRAME):
    """Every pixel (x, y) of the frame's border: 2 (W + H) - 4 of them."""
    px, py = np.meshgrid(np.arange(cfg.W), np.arange(cfg.H))
    b = (px == 0) | (px == cfg.W - 1) | (py == 0) | (py == cfg.H - 1)
    return np.stack([px[b], py[b]], -1).astype(np.int32)


def check_pixels(cfg=FRAME):
    """B's pixels: 4,096 seeded pixels over the frame and every border pixel, each once, in flat-id order."""
    pix = np.concatenate([bs.frame_pixels(cfg, 4096, seed=0).astype(np.int32), border_pixels(cfg)])
    flat = np.unique(pix[:, 1].astype(np.int64) * cfg.W + pix[:, 0])
    return np.stack([flat % cfg.W, flat // cfg.W], -1).astype(np.int32)


def centre_patch(side, cfg=FRAME):
    """bench_frustum.fused's training patch: side x side pixels around the centre of the frame, [1,side^2,2] int32 (x, y)."""
    y0, x0 = cfg.H // 2 - side // 2, cfg.W // 2 - side // 2
    py, px = np.meshgrid(np.arange(y0, y0 + side), np.arange(x0, x0 + side), indexing="ij")
    return np.stack([px, py], -1).reshape(1, -1, 2).astype(np.int32)


# ---- the method (also run on the CPU by tests/test_frustum_bench_scale_method.py) ----
def oracle_query(s, pixels, opt, cfg=FRAME, pers=None):
    """frustum_oracle.query on the frame's points in perspective coordinates (s["pers"], what the bench hands the querier, or
    `pers`).  Returns (out, vsize, grid dims)."""
    rl, dl, ranges, vsize, vdim, svs, sdim, vscale = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"],
                                                                         np.float32(cfg.near), np.float32(cfg.far))
    out = frustum_oracle.query(s["pers"] if pers is None else pers, ranges[:3], svs, sdim, vscale, opt.kernel_size, opt.query_size,
                               opt.SR, opt.K, opt.P, pixels, np.float32(rl ** 2), np.float32(dl ** 2), max_o=opt.max_o)
    return out, vsize, sdim


def regime(out, vsize, sdim):
    """What a query result of the frame reaches: frustum_shade_f64.reach (R', capped columns, rays without neighbours, gap steps,
    K-fill), valid samples S, pair rows, largest point index, words per bitmask of the grid, bytes of h-bar, the counters."""
    r = frustum_shade_f64.reach(out, vsize)
    pidx = out["sample_pidx"]
    S = int((pidx >= 0).any(-1).sum())
    r.update(S=S, pairs=int((pidx >= 0).sum()), max_idx=int(pidx.max()), words=int(np.prod(np.asarray(sdim, np.int64))) // 32,
             hbar_bytes=ff64._hbar_bytes(S), counters=dict(out["counters"]))
    return r


def chunk_loop_differs(full, parts):
    """Keys of a query result (numpy or torch values, [R',...] rows in ray order) whose chunk-loop concatenation is not the full
    call's bit for bit."""
    bad = []
    for k in full:
        cat = torch.cat([torch.as_tensor(p[k]) for p in parts])
        if not torch.equal(cat, torch.as_tensor(full[k])):
            bad.append(k)
    return bad


def restrict(points, pidx):
    """The rows of the points a set of samples gathers (test_gpu_bench_scale_f64.touched_rows: point 0 included, which every empty
    slot gathers), and sample_pidx renumbered into them: (keep [U], xyz [U,3], {embedding, color, dir, conf: [1,U,C]}, pidx)."""
    keep = bs.touched_rows(pidx)
    cpidx = torch.where(pidx >= 0, torch.searchsorted(keep, pidx.long().clamp(min=0)), -1)
    return keep, points["xyz"][keep], {k: points[k][:, keep] for k in POINT_KEYS}, cpidx


def shade_in_chunks(points, mlp, tup, campos, cam, vsize, bg, order, chunk=CHUNK_RAYS):
    """frustum_shade_f64.shade in float64 one chunk of rays at a time on the rows the samples gather, its outputs concatenated over
    the chunks (every output is per ray, per sample or per pair of a ray)."""
    pidx, loc, loc_w, dirs = tup
    _, xyz, feats, cpidx = restrict(points, pidx)
    pts = dict(xyz=xyz, Rw2c=torch.eye(3), **feats)
    parts = [frustum_shade_f64.shade(pts, mlp, cpidx[r0:r1], loc[r0:r1], loc_w[r0:r1], dirs[r0:r1], campos, cam, vsize, bg,
                                     dtype=torch.float64, agg_intrp_order=order)
             for r0, r1 in bs.ray_chunks(pidx.shape[0], chunk)]
    return {k: torch.cat([p[k] for p in parts]) for k in parts[0]}


def bench_loss(ray_color, gt, conf_coefficient, n_col, n_cc):
    """The bench's loss on one set of rays, as sums over the global counts n_col (colour terms) and n_cc (conf_coefficient entries):
    the colour L2 mean plus ZERO_ONE_WEIGHT x the mean of log(c) + log(1 - c), c = conf_coefficient clamped to [1e-3, 1 - 1e-3]."""
    c = torch.clamp(conf_coefficient, ZERO_EPS, 1 - ZERO_EPS)
    return ((ray_color - gt) ** 2).sum() / n_col + ZERO_ONE_WEIGHT * (torch.log(c) + torch.log(1 - c)).sum() / n_cc


def point0_term(conf, n_cc):
    """|Gradient| of one empty slot's zero_one term into points_conf of point 0 (the slot gathers point 0's conf, clamped straight
    through to [1e-4, 1], then to the zero_one clamp)."""
    c = min(max(float(conf.reshape(-1)[0]), 1e-4), 1.0)
    if not ZERO_EPS < c < 1 - ZERO_EPS:
        return 0.0
    return ZERO_ONE_WEIGHT / n_cc * abs(1 / c - 1 / (1 - c))


def _add(acc, terms):
    for k, v in terms.items():
        acc[k] = acc[k] + v if k in acc else v


def reference_gradients(points, mlp, tup, campos, cam, vsize, bg, gt_hit, slopes, n_col, n_cc, chunks, order=2):
    """float64 autograd of bench_loss through frustum_shade_f64.shade with the given masks, one chunk of rays at a time on the rows
    the samples gather.  tup: (sample_pidx, sample_loc, sample_loc_w, sample_ray_dirs) of the R' hit rays; slopes: the 7 layers of
    shade()'s `slopes=` for the whole step (bool: True = slope 1, or float), each chunk taking its own pair and sample rows.
    Returns (gradients: the four point tensors [1,U,C] on the rows keep and the MLP tensors; keep [U]; the loss; per MLP tensor the
    sum of |terms| of its gradient, for grad_check.sum_error)."""
    pidx, loc, loc_w, dirs = tup
    keep, xyz, feats, cpidx = restrict(points, pidx)
    leaves = {k: v.double().requires_grad_(True) for k, v in feats.items()}
    pts = dict(xyz=xyz.double(), Rw2c=torch.eye(3, dtype=torch.float64), **leaves)
    w = {k: v.double().requires_grad_(True) for k, v in mlp.items()}
    poff, SR = bs.pair_offsets(pidx), pidx.shape[1]
    summed = tuple(k for k in MLP_KEYS if not (k == "alpha_branch.0" and order == 1))
    loss, terms = 0.0, {}
    for r0, r1 in chunks:
        p0, p1 = int(poff[r0]), int(poff[r1])
        sl = [bs._slopes(s[p0:p1]) for s in slopes[:4]] + [bs._slopes(s[r0 * SR:r1 * SR]) for s in slopes[4:]]
        with frustum_shade_f64.recording_softplus() as rec, session.recording_lin(summed) as lin:
            sh = frustum_shade_f64.shade(pts, w, cpidx[r0:r1], loc[r0:r1], loc_w[r0:r1], dirs[r0:r1], campos, cam, vsize, bg,
                                         dtype=torch.float64, agg_intrp_order=order, slopes=sl)
        lc = bench_loss(sh["ray_color"], gt_hit[r0:r1].double(), sh["conf_coefficient"], n_col, n_cc)
        lc.backward()
        _add(terms, session.sum_abs_terms(lin))
        if order == 1:
            _add(terms, frustum_shade_f64.alpha_branch_abs_terms(rec, sh["hbar"]))
        loss += float(lc.detach())
    grads = {k: v.grad for k, v in leaves.items()}
    grads.update({k: v.grad for k, v in w.items()})
    return grads, keep, loss, terms


def mlp_errors(got, ref, terms):
    """{MLP tensor: largest error relative to max(scale, the entry's sum of |terms|)} (grad_check.sum_error)."""
    return {k: grad_check.sum_error(got[k].cpu(), ref[k], terms[k]) for k in terms}


def mlp_bound(k, mode, precision, order):
    if order == 1 and k.startswith("alpha_branch.0"):
        return grad_check.ALPHA1_SUM_RTOL[(mode, precision)]
    return grad_check.FRUSTUM_MLP_RTOL[(mode, precision)]


def check_mlp(errs, mode, precision, order):
    bad = ["aggregator.%s: %.3e of max(scale, sum |terms|) > %.1e" % (k, e, mlp_bound(k, mode, precision, order))
           for k, e in errs.items() if not e <= mlp_bound(k, mode, precision, order)]
    assert not bad, "; ".join(bad)


# ---- the network is the bench's ----
def test_builder_is_the_bench_network():
    s, _ = frame()
    for is_train in (False, True):
        a, b = net(is_train), bench_frustum.fused_net(DEV, FRAME, s, is_train)
        assert vars(a.opt) == vars(b.opt), is_train
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa), is_train
        del a, b, sa, sb
    torch.cuda.empty_cache()


# ---- A. the query over the whole frame ----
def test_query_of_the_frame_is_the_oracle_and_the_chunk_loop():
    with bs._device_released():
        _query_case()


def _query_case():
    s, _ = frame()
    opt = scene.frustum_opt(FRAME)
    q = qpi.lighting_fast_querier(DEV, opt)
    pers = torch.from_numpy(s["pers"]).to(DEV)[None]
    xyz_w = torch.from_numpy(s["xyz_w"]).to(DEV)[None]
    camrot = torch.from_numpy(s["camrotc2w"]).to(DEV)[None]
    campos = torch.from_numpy(s["campos"]).to(DEV)[None]
    npts = torch.tensor([FRAME.N], dtype=torch.int32, device=DEV)
    pix = torch.from_numpy(s["pixel_idx"]).to(DEV)[None]
    R = pix.shape[1]

    def run(p):           # bench_frustum.main's call
        tup = q.query_points(p, pers, xyz_w, npts, np.int64(FRAME.H), np.int64(FRAME.W), s["intrinsic"], np.float32(FRAME.near),
                             np.float32(FRAME.far), None, campos, camrot)
        return dict(ray_mask=tup[4][0], pixel_idx_cur=q.last_pixel_idx_cur[0], sample_pidx=tup[0][0], sample_loc=tup[1][0],
                    sample_loc_w=tup[2][0], sample_ray_dirs=tup[3][0])

    full = run(pix)
    bc, qc = dict(q.last_build_counters), dict(q.last_query_counters)
    n_words = int(q._fr.n_words)
    builds = q.n_builds
    parts = [run(pix[:, k:k + CHUNK]) for k in range(0, R, CHUNK)]
    n_chunks, chunk_builds = len(parts), q.n_builds - builds
    loop_differs = chunk_loop_differs(full, parts)
    del parts
    full = {k: v.cpu() for k, v in full.items()}
    torch.cuda.empty_cache()
    t0 = time.time()
    ref, vsize, sdim = oracle_query(s, s["pixel_idx"], opt)
    t_oracle = time.time() - t0
    oracle_differs = [k for k in ("ray_mask", "pixel_idx_cur", "sample_pidx", "sample_loc")
                      if not np.array_equal(full[k].numpy(), ref[k])]
    rc = ref["counters"]
    # the build keeps the max_o option (0: none given); the oracle counts the max_o it derives, 5 here, as in the regime check
    gpu_counters = dict(R2=qc["R2"], n_bad_pixel=qc["n_bad_pixel"], max_pts=bc["max_pts"], overflow_p=bc["overflow_p"],
                        overflow_o=bc["overflow_o"], n_col_capped=bc["n_col_capped"])
    counters_differ = {k: (v, rc[k]) for k, v in gpu_counters.items() if v != rc[k]}
    reg = regime(ref, vsize, sdim)
    print("\n[frustum bench f64] query of the %dx%d frame, N=%d: R'=%d of %d, words/bitmask %d (GPU %d), S=%d pairs=%d h-bar %.2f GB, "
          "gap steps %d, K-fill %s, max point %d, counters GPU %s oracle %s (%.1f s); oracle differs in %s; %d chunks, %d builds, "
          "chunk loop differs in %s" % (
              FRAME.W, FRAME.H, FRAME.N, reg["R2"], R, reg["words"], n_words, reg["S"], reg["pairs"], reg["hbar_bytes"] / 1e9,
              reg["gap"], reg["kfill"], reg["max_idx"], gpu_counters, rc, t_oracle, oracle_differs or "-", n_chunks, chunk_builds,
              loop_differs or "-"))
    assert not oracle_differs, "the full-frame query differs from the oracle in %s" % oracle_differs
    assert not counters_differ, "counters (GPU, oracle): %s" % counters_differ
    assert n_chunks == 209 and chunk_builds == 0, (n_chunks, chunk_builds)
    assert not loop_differs, "the chunk loop differs from the full-frame call in %s" % loop_differs
    # the regime: the frame's figures, which the small scenes never reach
    assert n_words == reg["words"] > 1 << 20
    assert reg["R2"] == 430_164 and reg["S"] > 1 << 21 and reg["hbar_bytes"] > 1 << 31
    assert reg["gap"] == 223_952 and reg["capped"] == 0
    assert rc["overflow_p"] == 0 and rc["overflow_o"] == 0 and rc["n_bad_pixel"] == 0 and (rc["max_pts"], rc["max_o"]) == (11, 5)


# ---- B. the forward sample by sample; C. the whole frame equals its subsets ----
def _ff64_net(name, bias, order=2, kernel="frozen", is_train=False, qover=None, **over):
    """test_gpu_frustum_f64._net for the frame: net() with the kernel's options."""
    assert name == FRAME.name and bias == ALPHA_BIAS and qover is None
    n = net(is_train, agg_intrp_order=order, **ff64.KERNELS[kernel], **over)
    return n, n.opt


def _ff64_data(name, pixels, bg):
    return pixel_data(pixels, bg)


def _ff64_shade64(n, q, d, order, bg, pts=None, mlp=None, slopes=None):
    """test_gpu_frustum_f64._shade64 in ray chunks."""
    assert pts is None and mlp is None and slopes is None
    return shade_in_chunks(ff64._points_cpu(n), harness.mlp_cpu(n.aggregator), ff64._tup(q), d["campos"].cpu(), d["camrotc2w"].cpu(),
                           q.vsize, torch.tensor(bg or (0.0, 0.0, 0.0), dtype=torch.float64), order)


FWD_CASES = [("frozen", 2), ("general", 2), ("fp32", 2), ("frozen", 1), ("general", 1)]
RENDER_KEYS = ("coarse_raycolor", "coarse_point_opacity", "coarse_is_background")


@pytest.mark.parametrize("kernel,order", FWD_CASES, ids=["%s-order%d" % c for c in FWD_CASES])
def test_forward_over_the_frame(kernel, order, monkeypatch):
    monkeypatch.setattr(ff64, "_net", _ff64_net)
    monkeypatch.setattr(ff64, "_data", _ff64_data)
    monkeypatch.setattr(ff64, "_shade64", _ff64_shade64)
    with bs._device_released():
        _forward_case(kernel, order)


def _forward_case(kernel, order):
    pixels = check_pixels()
    bs._reset_peak_memory()
    t0 = time.time()
    n, q, ref, info = ff64._run(FRAME.name, "opaque", kernel, order, pixels=pixels, bg=(1.0, 1.0, 1.0))
    t_check = time.time() - t0
    d, out = info["d"], info["out"]
    hit = out["ray_mask"][0] > 0
    flat = torch.from_numpy(pixels[:, 1].astype(np.int64) * FRAME.W + pixels[:, 0]).to(DEV)
    border = torch.from_numpy(np.isin(flat.cpu().numpy(), border_pixels()[:, 1].astype(np.int64) * FRAME.W + border_pixels()[:, 0]))
    n_border_hit = int((hit.cpu() & border).sum())
    max_idx, n_pairs = int(q.sample_pidx.max()), int(q.counters["n_pairs"])
    with torch.no_grad():
        sub = n.render_full(d["campos"], d["raydir"], d["camrotc2w"], FRAME.near, FRAME.far, d["bg_color"],
                            view={k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")})
        n.check_errors()
        img = runner.render_image(n, bench_data(), FRAME.H, FRAME.W)
    n.check_errors()
    same_sub = {k: torch.equal(sub[k][0][hit], out[k][0]) for k in RENDER_KEYS}
    same_sub["ray_mask"] = torch.equal(sub["ray_mask"], out["ray_mask"])
    same_frame = {k: torch.equal(img[k].reshape(FRAME.H * FRAME.W, -1)[flat], sub[k][0].reshape(flat.shape[0], -1))
                  for k in RENDER_KEYS + ("ray_mask",)}
    n_frame_hit = int(img["ray_mask"].sum())
    peak = torch.cuda.max_memory_allocated(DEV)
    del n, q, ref, info, d, out, sub, img
    print("[frustum bench f64] frame %s order %d: %d pixels (%d border, %d of them hit), R'=%d pairs=%d, max point %d; frame %d hit; "
          "peak %.2f GB; check %.0f s; subset == forward %s; frame == subset %s" % (
              kernel, order, pixels.shape[0], int(border.sum()), n_border_hit, int(hit.sum()), n_pairs, max_idx, n_frame_hit, peak / 1e9,
              t_check, same_sub, same_frame))
    assert all(same_sub.values()), "render_full on the pixels differs from forward(): %s" % same_sub
    assert all(same_frame.values()), "the whole frame differs from render_full on its pixels: %s" % same_frame
    # the module's own query (points in perspective coordinates by w2pers on the device) reaches the oracle's regime
    assert int(border.sum()) == 2796 and n_border_hit > 800, (int(border.sum()), n_border_hit)
    assert n_frame_hit > 400_000 and max_idx > 1 << 18, (n_frame_hit, max_idx)


def test_probe_image_of_the_frame():
    with bs._device_released():
        _probe_case()


def _probe_case():
    pixels = check_pixels()
    n = net(prob=1)
    bs._reset_peak_memory()
    maps = runner.probe_image(n, bench_data(), FRAME.H, FRAME.W)
    d = pixel_data(pixels)
    with torch.no_grad():
        full = n.render_full(d["campos"], d["raydir"], d["camrotc2w"], FRAME.near, FRAME.far, d["bg_color"], probe=True,
                             view={k: d[k] for k in ("pixel_idx", "h", "w", "intrinsic")})
    n.check_errors()
    peak = torch.cuda.max_memory_allocated(DEV)
    flat = torch.from_numpy(pixels[:, 1].astype(np.int64) * FRAME.W + pixels[:, 0]).to(DEV)
    differs = [k for k in runner.PROBE_MAP_KEYS
               if maps[k].dtype != full[k].dtype or not torch.equal(maps[k].reshape(FRAME.H * FRAME.W, -1)[flat],
                                                                     full[k][0].reshape(flat.shape[0], -1))]
    del maps
    # float64: the probe oracle on a drop-in querier's tuple for the pixels and the fused opacity
    npn = n.neural_points
    xyz = npn.xyz.detach()
    qd = qpi.lighting_fast_querier(DEV, n.opt)
    tup = qd.query_points(d["pixel_idx"], qpi.w2pers(xyz, d["camrotc2w"], d["campos"]), xyz[None],
                          torch.tensor([xyz.shape[0]], dtype=torch.int32), np.int64(FRAME.H), np.int64(FRAME.W), d["intrinsic"],
                          np.float32(FRAME.near), np.float32(FRAME.far), None, d["campos"], d["camrotc2w"])
    mask = full["ray_mask"][0] > 0
    same_mask = torch.equal(full["ray_mask"], tup[4])
    inds = torch.nonzero(mask)[:, 0]
    op = full["coarse_point_opacity"][0][inds]
    pts64 = dict(xyz=xyz.double(), embedding=npn.points_embeding.detach().double(), color=npn.points_color.detach().double(),
                 dir=npn.points_dir.detach().double(), conf=npn.points_conf.detach().double())
    ref = probe_oracle.probe(pts64, tup[0][0], tup[2][0], op, dtype=torch.float64)
    slot = torch.max(op, -1)[1]
    same_slot = torch.equal(ref["slot"], slot)
    rows = torch.arange(inds.shape[0], device=DEV)
    same_loc = torch.equal(full["ray_max_sample_loc_w"][0][inds], tup[2][0][rows, slot])
    errs = {k: float((full[k][0][inds].double() - ref[k]).abs().max() / ref[k].abs().max().clamp(min=1e-30)) for k in fused.PROBE_BOUNDS}
    misses_zero = all(bool(torch.all(full[k][0][~mask] == 0)) for k, _ in probe_keys(63))
    print("\n[frustum bench f64] probe of the %dx%d frame: %d pixels, R'=%d; peak %.2f GB; frame == subset except %s; oracle slot %s "
          "loc_w %s, errors %s" % (FRAME.W, FRAME.H, pixels.shape[0], inds.shape[0], peak / 1e9, differs or "-", same_slot, same_loc,
                                   " ".join("%s %.2e" % kv for kv in errs.items())))
    assert not differs, "probe_image of the frame differs from render_full(probe=True) on its pixels in %s" % differs
    assert same_mask and same_slot and same_loc and misses_zero, (same_mask, same_slot, same_loc, misses_zero)
    for k, b in fused.PROBE_BOUNDS.items():
        assert errs[k] <= b, (k, errs[k], b)


# ---- D. the bench's training step ----
def bench_step(n, data, patch, gt):
    """bench_frustum.fused's step(): forward on the patch with the train jitter, the bench's loss, backward.  Returns (out, loss)."""
    m = patch.shape[1]
    out = n(data["campos"], data["raydir"][:, :m], bg_color=data["bg_color"], camrotc2w=data["camrotc2w"], pixel_idx=patch,
            near=FRAME.near, far=FRAME.far, h=FRAME.H, w=FRAME.W, intrinsic=data["intrinsic"])
    hit = torch.nonzero(out["ray_mask"][0])[:, 0]
    cc = torch.clamp(out["conf_coefficient"], 1e-3, 1 - 1e-3)
    loss = ((out["coarse_raycolor"][0] - gt[0][hit]) ** 2).mean() + 1e-3 * torch.mean(torch.log(cc) + torch.log(1 - cc))
    loss.backward()
    return out, loss


# (patch side, agg_intrp_order, pnb_bwd_fp32 mode, pnb_precision)
STEP_CASES = [(48, 2, 0, "bf16x3"), (48, 2, 4, "bf16x3"), (48, 2, 1, "bf16x3"), (48, 2, 1, "fp32"), (48, 1, 0, "bf16x3"),
              (96, 2, 0, "bf16x3"), (96, 2, 4, "bf16x3")]


@pytest.mark.parametrize("side,order,mode,precision", STEP_CASES, ids=["%dx%d-order%d-mode%d-%s" % ((c[0],) + c) for c in STEP_CASES])
def test_training_step_gradients(side, order, mode, precision):
    with bs._device_released():
        _step_case(side, order, mode, precision)


def _step_case(side, order, mode, precision):
    bs._reset_peak_memory()
    n = net(True, pnb_bwd_fp32=mode, pnb_precision=precision, agg_intrp_order=order)
    data = bench_data()
    patch = torch.from_numpy(centre_patch(side)).to(DEV)
    gt = torch.rand((1, side * side, 3), generator=torch.Generator().manual_seed(1)).to(DEV)
    torch.manual_seed(0)        # the train jitter: a failure replays
    out, loss = bench_step(n, data, patch, gt)
    n.check_errors()
    q = n.last
    peak = torch.cuda.max_memory_allocated(DEV)
    slopes = [s == 1 for s in frustum_shade_f64.kernel_slopes(n, q)]
    tup = ff64._tup(q)
    pidx = tup[0]
    Rn, SR, K = pidx.shape
    hit = torch.nonzero(out["ray_mask"][0])[:, 0].cpu()
    n_col, n_cc = 3 * Rn, int(out["conf_coefficient"].numel())
    P, S = int(q.counters["n_pairs"]), int(q.counters["n_valid"])
    npn = n.neural_points
    got = dict(embedding=npn.points_embeding.grad, color=npn.points_color.grad, dir=npn.points_dir.grad, conf=npn.points_conf.grad)
    got.update({k: p.grad for k, p in n.aggregator.named_parameters()})
    points = ff64._points_cpu(n)
    mlp = harness.mlp_cpu(n.aggregator)
    colour = out["coarse_raycolor"][0].detach().cpu().double()
    loss = float(loss)
    t0 = time.time()
    ref, keep, loss64, terms = reference_gradients(points, mlp, tup, data["campos"][0].cpu(), data["camrotc2w"][0].cpu(), q.vsize,
                                                   torch.ones(3), gt[0][hit.to(DEV)].cpu(), slopes, n_col, n_cc,
                                                   bs.ray_chunks(Rn, CHUNK_RAYS), order)
    t_oracle = time.time() - t0
    n0 = int((pidx.clamp(min=0) == 0).sum())
    err, conf0, untouched = bs.step_errors(got, ref, keep, n0, point0_term(points["conf"], n_cc))
    merr = mlp_errors(got, ref, terms)
    mse = float(((colour - gt[0][hit.to(DEV)].cpu().double()) ** 2).mean())
    d_loss, b_loss = abs(loss - loss64), bs.loss_bound(loss, mse, ff64.BOUNDS["fp32" if precision == "fp32" else "general"]["composite"])
    max_idx, N = int(keep.max()), npn.xyz.shape[0]
    del n, npn, got, q, out, data
    torch.cuda.empty_cache()
    worst_pt = max(POINT_KEYS, key=err.get)
    worst_mlp = max(merr, key=merr.get)
    print("\n[frustum bench f64] step %dx%d order %d mode %d %s: N=%d R'=%d of %d S=%d P=%d (%.1f x 2048, dW splits %s) U=%d max point %d "
          "n0=%d peak %.2f GB oracle %.0f s | points %.2e (%s) conf0 %.2e/%.2e untouched %s | MLP of max(scale, sum|terms|) %.2e (%s), "
          "of scale %.2e | loss %.9f |d| %.2e/%.2e" % (
              side, side, order, mode, precision, N, Rn, side * side, S, P, P / 2048, grad_check.dw_splits(P), keep.numel(), max_idx, n0,
              peak / 1e9, t_oracle, err[worst_pt], worst_pt, conf0[0], conf0[1], untouched, merr[worst_mlp], worst_mlp,
              max(err[k] for k in err if k not in POINT_KEYS), loss, d_loss, b_loss))
    assert n_cc == Rn * SR * K and len(merr) == 18
    bs.check_step({k: err[k] for k in POINT_KEYS}, conf0, untouched, grad_check.RTOL[(mode, precision)])
    check_mlp(merr, mode, precision, order)
    assert d_loss <= b_loss, "loss %.9f vs float64 %.9f: %.3e > %.3e" % (loss, loss64, d_loss, b_loss)
    if side == 96:
        assert P > 64 * 2048, "%d pair rows: the split-K cap is not reached" % P
