"""CPU: the method of tests/test_gpu_frustum_bench_scale_f64.py, checked with the C frustum oracle and the float64 shading oracle.

  frame     the CPU oracle's figures for the bench's DTU frame (800 x 600, 400k points): R', words per bitmask, valid samples, pair rows,
            h-bar bytes, gap steps, K-fill, largest point index, counters, and the 923 hits among the 2,796 border pixels
  gradient  on the dtu_surface scene's 24 x 24 centre patch (the oracle's query, an opaque surface, some confs outside the [1e-4, 1]
            clamp): fp32 autograd through frustum_shade_f64.shade on all rows stands in for the kernel, its LeakyReLU masks for the
            backward's.  The float64 reference in ray chunks equals the unchunked one to 1e-12, and the stand-in meets the fp32 bounds
            against it
  loss      bench_loss in float64 (sums over the global counts) is the bench's fp32 expression (means) to fp32 rounding, values and
            gradients, straight-through clamp included
  defects   each fails its comparison: a dropped ray chunk, a gradient written to the next row, chunk outputs shifted by one pixel
            against the whole frame, a conf clamp that is not straight-through
"""
import functools

import numpy as np
import pytest
import torch

import frustum_shade_f64
import test_gpu_bench_scale_f64 as bs
import test_gpu_frustum_bench_scale_f64 as fb
from oracle import grad_check, shade_oracle
from pointnerf_b200 import harness, scene
from pointnerf_b200 import query_point_indices as qpi
from pointnerf_b200.ray_marching import PointAggregator

# the fp32 stand-in is held to the fp32 forward's mode-0 bounds: on the opaque surface with confs edited beyond the clamp its points_conf
# measures 2.5e-6 of scale against float64, above mode 1's 2e-6 (a CPU fp32 autograd, not the kernel's split backward)
MODE = (0, "fp32")
RTOL = grad_check.RTOL[MODE]
CHUNK = 100          # rays per float64 chunk: 6 chunks, the last one partial
U32 = 2.0 ** -24


# ---- the bench's frame ----
@functools.lru_cache(None)
def _frame_query():
    s, _ = fb.frame()
    return fb.oracle_query(s, s["pixel_idx"], scene.frustum_opt(fb.FRAME))


def test_frame_figures():
    out, vsize, sdim = _frame_query()
    r = fb.regime(out, vsize, sdim)
    c = r["counters"]
    ids = fb.border_pixels()
    n_border_hit = int(out["ray_mask"][ids[:, 1] * fb.FRAME.W + ids[:, 0]].sum())
    print("\n[frustum bench method] frame: %s; border pixels %d, %d hit" % ({k: v for k, v in r.items()}, len(ids), n_border_hit))
    assert (r["R2"], r["S"], r["pairs"], r["gap"]) == (430_164, 2_982_660, 15_187_372, 223_952)
    assert r["kfill"] == [0, 986_800, 119_352, 85_584, 69_556, 61_900, 54_464, 49_424, 1_555_580]
    assert r["words"] == 1_500_000 and r["words"] > 1 << 20            # the build's block-sum scan: two passes of 1024
    assert r["S"] > 1 << 21 and r["hbar_bytes"] == 23_303 * 131_072 and r["hbar_bytes"] > 1 << 31
    assert r["max_idx"] == 399_999 and r["capped"] == 0
    assert (c["max_pts"], c["max_o"], c["overflow_p"], c["overflow_o"], c["n_bad_pixel"]) == (11, 5, 0, 0, 0)
    assert (len(ids), n_border_hit) == (2796, 923)


# ---- the gradient method on a small frustum scene ----
@pytest.fixture(scope="module")
def case():
    cfg, s, pts = frustum_shade_f64.frustum_scene("dtu_surface")
    opt = scene.frustum_opt(cfg)
    pix = fb.centre_patch(24, cfg)[0]
    out, vsize, _ = fb.oracle_query(s, pix, opt, cfg)
    pidx = torch.from_numpy(out["sample_pidx"])
    loc = torch.from_numpy(out["sample_loc"])
    cam, campos = torch.from_numpy(s["camrotc2w"]), torch.from_numpy(s["campos"])
    loc_w, dirs = qpi.lighting_fast_querier.pers2w(None, loc[None], cam[None], campos[None])
    tup = (pidx, loc, loc_w[0], dirs[0])
    Rn, SR, K = pidx.shape
    # confs on both sides of the straight-through clamp [1e-4, 1] on some touched points (the bench's confs lie in [0.1, 1))
    pts = dict(pts, conf=pts["conf"].clone())
    touched = bs.touched_rows(pidx)[1:]
    edited = touched[::7]
    pts["conf"][0, edited, 0] = torch.tensor([5e-5, 1.3]).repeat(len(edited))[:len(edited)]
    agg = PointAggregator(harness.make_opt(scene.CONFIGS["tiny"], feat_dim=63, **vars(opt)), seed=5)
    with torch.no_grad():
        agg.alpha_branch[0].bias += fb.ALPHA_BIAS
    mlp = harness.mlp_cpu(agg)
    gt = torch.rand(Rn, 3, generator=torch.Generator().manual_seed(1))
    bg = torch.ones(3)
    # the stand-in for the kernel: fp32 autograd on every row, the bench's loss as it writes it, and the masks its LeakyReLUs took
    p32 = {k: v.clone().requires_grad_(k in fb.POINT_KEYS) for k, v in pts.items()}
    m32 = {k: v.clone().requires_grad_(True) for k, v in mlp.items()}
    rec = grad_check.MaskRecorder(shade_oracle.F)
    with pytest.MonkeyPatch.context() as m:
        m.setattr(shade_oracle, "F", rec)
        sh = frustum_shade_f64.shade(p32, m32, pidx, loc, tup[2], tup[3], campos, cam, vsize, bg, dtype=torch.float32)
    cc = torch.clamp(sh["conf_coefficient"], 1e-3, 1 - 1e-3)
    loss32 = ((sh["ray_color"] - gt) ** 2).mean() + 1e-3 * torch.mean(torch.log(cc) + torch.log(1 - cc))
    loss32.backward()
    got = {k: p32[k].grad for k in fb.POINT_KEYS}
    got.update({k: v.grad for k, v in m32.items()})
    n_col, n_cc = 3 * Rn, Rn * SR * K

    def reference(chunks=None, points=pts):
        chunks = bs.ray_chunks(Rn, CHUNK) if chunks is None else chunks
        return fb.reference_gradients(points, mlp, tup, campos, cam, vsize, bg, gt, rec.slopes, n_col, n_cc, chunks)

    return dict(got=got, loss=float(loss32.detach()), reference=reference, ref=reference(), Rn=Rn, pidx=pidx, edited=edited,
                n0=int((pidx.clamp(min=0) == 0).sum()), term=fb.point0_term(pts["conf"], n_cc), slopes=rec.slopes, pts=pts)


def _check(c, got, ref):
    g, keep, _, terms = ref
    err, conf0, untouched = bs.step_errors(got, g, keep, c["n0"], c["term"])
    bs.check_step({k: err[k] for k in fb.POINT_KEYS}, conf0, untouched, RTOL)
    fb.check_mlp(fb.mlp_errors(got, g, terms), *MODE, 2)


def test_chunked_equals_unchunked_and_fp32_meets_the_bounds(case):
    c = case
    g, keep, loss, terms = c["ref"]
    g1, keep1, loss1, terms1 = c["reference"](chunks=[(0, c["Rn"])])
    assert torch.equal(keep, keep1) and len(bs.ray_chunks(c["Rn"], CHUNK)) == 6
    worst = max(grad_check.rel_error(g[k], g1[k]) for k in g)
    worst_terms = max(grad_check.rel_error(terms[k], terms1[k]) for k in terms)
    print("\n[frustum bench method] R'=%d, chunked vs unchunked: gradients %.1e, sum |terms| %.1e" % (c["Rn"], worst, worst_terms))
    assert worst <= 1e-12 and worst_terms <= 1e-12, (worst, worst_terms)
    assert abs(loss - loss1) <= 1e-12 * abs(loss1)
    assert len(terms) == 18
    _check(c, c["got"], c["ref"])
    assert abs(c["loss"] - loss) <= 1e-6 * abs(loss)
    assert keep.numel() < c["got"]["embedding"].shape[1], "every point touched: the untouched-row check checks nothing"
    # the edited confs reach the loss through the straight-through clamp
    assert float(c["got"]["conf"][0, c["edited"]].abs().max()) > 0


def test_bench_loss_in_float64_is_the_bench_expression():
    g = np.random.RandomState(3)
    R2, SR, K, N = 300, 40, 8, 2000
    conf = g.uniform(0.0, 1.0, (1, N, 1))
    conf[0, :40, 0] = g.choice([5e-5, 5e-4, 0.9995, 1.2, 2e-3, 0.998], 40)
    pidx = torch.from_numpy(g.randint(-1, N, (R2, SR, K)).astype(np.int32))
    col, gt = g.uniform(0, 1, (R2, 3)), g.uniform(0, 1, (R2, 3))

    def evaluate(dtype, form):
        x = {k: torch.from_numpy(np.asarray(v, np.float32)).to(dtype).requires_grad_(True) for k, v in (("col", col), ("conf", conf))}
        c0 = x["conf"][0][torch.clamp(pidx, min=0).long()][..., 0]
        cc = c0 - (c0 - torch.clamp(c0, min=0.0001, max=1)).detach()           # point_aggregators.py:722-724
        if form == "bench":
            c = torch.clamp(cc, 1e-3, 1 - 1e-3)
            L = ((x["col"] - torch.from_numpy(gt).to(dtype)) ** 2).mean() + 1e-3 * torch.mean(torch.log(c) + torch.log(1 - c))
        else:
            L = fb.bench_loss(x["col"], torch.from_numpy(gt).to(dtype), cc, 3 * R2, cc.numel())
        L.backward()
        return float(L.detach()), x["col"].grad.double(), x["conf"].grad.double()

    L32, gc32, gf32 = evaluate(torch.float32, "bench")
    L64, gc64, gf64 = evaluate(torch.float64, "sums")
    L64b, gc64b, gf64b = evaluate(torch.float64, "bench")
    assert abs(L64 - L64b) <= 1e-14 * abs(L64) and float((gf64 - gf64b).abs().max()) <= 1e-12 * float(gf64.abs().max())
    assert abs(L32 - L64) <= 16 * U32 * abs(L64) + 1e-3 * 16 * U32, (L32, L64)
    assert float((gc32 - gc64).abs().max()) <= 8 * U32 * float(gc64.abs().max())
    assert float((gf32 - gf64).abs().max()) <= 64 * U32 * float(gf64.abs().max())
    assert float(gf64.abs().max()) > 0


# ---- planted defects ----
def test_a_dropped_ray_chunk_fails(case):
    c = case
    chunks = bs.ray_chunks(c["Rn"], CHUNK)
    with pytest.raises(AssertionError, match="of scale"):
        _check(c, c["got"], c["reference"](chunks=chunks[:2] + chunks[3:]))


def test_a_gradient_written_to_the_next_row_fails(case):
    c = case
    ref = c["ref"]
    keep = ref[1]
    nxt = set(keep.tolist())
    for p, msg in ((next(i for i in keep.tolist()[1:] if i + 1 not in nxt), "untouched rows not zero"),
                   (next(i for i in keep.tolist()[1:] if i + 1 in nxt), "embedding: .* of scale")):
        bad = dict(c["got"])
        e = c["got"]["embedding"].clone()
        e[0, p + 1] += e[0, p]
        e[0, p] = 0
        bad["embedding"] = e
        with pytest.raises(AssertionError, match=msg):
            _check(c, bad, ref)


def test_chunk_outputs_shifted_by_one_pixel_fail():
    """The chunk-loop comparison of the whole-frame query, on the dtu_surface frame with the oracle: the true loop equals the full
    call, a loop whose chunks start one pixel late does not."""
    cfg, s, _ = frustum_shade_f64.frustum_scene("dtu_surface")
    opt = scene.frustum_opt(cfg)
    pix = s["pixel_idx"]

    def query(p):
        out = fb.oracle_query(s, p, opt, cfg)[0]
        return {k: out[k] for k in ("ray_mask", "pixel_idx_cur", "sample_pidx", "sample_loc")}

    full = query(pix)
    parts = [query(pix[k:k + fb.CHUNK]) for k in range(0, len(pix), fb.CHUNK)]
    assert fb.chunk_loop_differs(full, parts) == []
    shifted = [query(np.roll(pix, -1, 0)[k:k + fb.CHUNK]) for k in range(0, len(pix), fb.CHUNK)]
    assert "ray_mask" in fb.chunk_loop_differs(full, shifted)


def test_a_clamp_that_is_not_straight_through_fails(case, monkeypatch):
    c = case
    shade = frustum_shade_f64.shade

    def plain_clamp(points, *a, **k):
        return shade(dict(points, conf=torch.clamp(points["conf"], 1e-4, 1)), *a, **k)
    monkeypatch.setattr(frustum_shade_f64, "shade", plain_clamp)
    with pytest.raises(AssertionError, match="conf"):
        _check(c, c["got"], c["reference"]())
