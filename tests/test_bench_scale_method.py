"""CPU: the method of tests/test_gpu_bench_scale_f64.py's training-step check, on the oracle itself.

The tiny_opaque fixture's query (927 hit rays) and MLP; TrainStep's loss on seeded target colours.  The oracle in fp32 stands in for
the kernel: its gradients over all N rows and its LeakyReLU masks.  The float64 reference runs with those masks one chunk of rays at a
time, on the touched rows only.  Chunked, it equals the unchunked run to float64 rounding, and the fp32 run meets mode 1's fp32 bounds
against it (grad_check.RTOL).  Three planted defects each fail the comparison: one ray chunk left out, one point's gradient written to
the next row, and a global count off by one."""
import pytest
import torch

import test_gpu_bench_scale_f64 as bs
from oracle import golden, grad_check, shade_oracle, shade_oracle_rw2c
from pointnerf_b200 import scene

RTOL = grad_check.RTOL[(1, "fp32")]
CHUNK = 200          # rays per chunk: 5 chunks, the last one partial


@pytest.fixture(scope="module")
def case(golden_dir):
    fx = golden.load(golden_dir, "tiny_opaque")
    cfg = scene.CONFIGS["tiny"]
    pts = scene.make_points(cfg)
    rays = scene.make_rays(cfg, fx["pixels"])
    hit = torch.from_numpy(fx["ray_mask"]) > 0
    pidx, loc_w = torch.from_numpy(fx["sample_pidx"]), torch.from_numpy(fx["sample_loc_w"])
    mlp = {k[4:]: torch.from_numpy(fx[k]) for k in fx.files if k.startswith("mlp.")}
    gt = torch.rand(int(hit.sum()), 3, generator=torch.Generator().manual_seed(1))
    Rn, SR, K = pidx.shape
    n_se, n_zo = 3 * Rn, Rn * SR * K
    args = (pidx, loc_w, rays["raydir"][0][hit], gt, rays["campos"][0], rays["camrotc2w"][0], [cfg.vsize] * 3, rays["bg_color"][0])
    # the stand-in for the kernel: fp32 autograd through the oracle on every row, and the masks its LeakyReLUs took
    p32 = {k: v.clone().requires_grad_(k in bs.POINT_KEYS) for k, v in pts.items()}
    m32 = {k: v.clone().requires_grad_(True) for k, v in mlp.items()}
    rec = grad_check.MaskRecorder(shade_oracle.F)
    with pytest.MonkeyPatch.context() as m:
        m.setattr(shade_oracle, "F", rec)
        sh = shade_oracle_rw2c.shade(p32, m32, pidx, loc_w, args[2], *args[4:], dtype=torch.float32)
    loss32 = bs.train_loss(sh["ray_color"], gt, sh["conf_coefficient"], n_se, n_zo)
    loss32.backward()
    got = {k: p32[k].grad for k in bs.POINT_KEYS}
    got.update({k: v.grad for k, v in m32.items()})
    n0 = int((pidx.clamp(min=0) == 0).sum())
    term = bs.point0_term(pts["conf"], n_zo)

    def reference(chunks=None, n_se=n_se, slopes=rec.slopes):
        chunks = bs.ray_chunks(Rn, CHUNK) if chunks is None else chunks
        return bs.reference_gradients(pts, mlp, *args, slopes, n_se, n_zo, chunks)

    return dict(got=got, loss=loss32.item(), reference=reference, ref=reference(), n0=n0, term=term, Rn=Rn, slopes=rec.slopes)


def _check(c, got, ref):
    g, keep, _ = ref
    bs.check_step(*bs.step_errors(got, g, keep, c["n0"], c["term"]), RTOL)


def test_chunked_equals_unchunked_and_fp32_meets_the_bounds(case):
    c = case
    g, keep, loss = c["ref"]
    g1, keep1, loss1 = c["reference"](chunks=[(0, c["Rn"])])
    assert torch.equal(keep, keep1) and len(bs.ray_chunks(c["Rn"], CHUNK)) == 5
    worst = max(grad_check.rel_error(g[k], g1[k]) for k in g)
    assert worst <= 1e-12, worst
    assert abs(loss - loss1) <= 1e-12 * abs(loss1)
    # boolean masks (what the GPU test keeps per unit) give the same slopes, bit for bit
    assert all(torch.equal(bs._slopes(s == 1), s) for s in c["slopes"])
    err, conf0, untouched = bs.step_errors(c["got"], g, keep, c["n0"], c["term"])
    bs.check_step(err, conf0, untouched, RTOL)
    assert abs(c["loss"] - loss) <= 1e-6 * loss
    assert keep.numel() < c["got"]["embedding"].shape[1], "every point touched: the untouched-row check checks nothing"


def test_a_dropped_ray_chunk_fails(case):
    c = case
    chunks = bs.ray_chunks(c["Rn"], CHUNK)
    with pytest.raises(AssertionError, match="of scale"):
        _check(c, c["got"], c["reference"](chunks=chunks[:2] + chunks[3:]))


def test_a_gradient_written_to_the_next_row_fails(case):
    c = case
    ref = c["ref"]
    keep = ref[1]
    # a touched point whose next row is untouched, and one whose next row is touched
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


def test_a_global_count_off_by_one_fails(case):
    c = case
    g, keep, loss = c["reference"](n_se=3 * c["Rn"] + 1)
    with pytest.raises(AssertionError, match="of scale"):
        _check(c, c["got"], (g, keep, loss))
    assert abs(c["loss"] - loss) > 1e-4 * loss
