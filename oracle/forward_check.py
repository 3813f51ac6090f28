"""TEST INFRASTRUCTURE ONLY -- the per-sample check of the fused forward against float64 (tests/test_gpu_forward_f64.py,
tests/test_forward_f64_oracle.py).

The composited outputs average dozens of samples per ray, so a bug confined to a few samples (a partial tile, one quadrant's segmented
scan, a wrong `pre` row, one K slot) hides under a 1e-4 rule on radiance and opacity.  This module compares the kernels' own products
instead:
  sample_map / pair_map  the kernel's sample-compacted buffers (valid_list, samp_off, the backward's pair rows) -> the rows of the query
                         export's dense [R', SR(, K)] layout the oracles work in;
  decode_hbar            h-bar as the pair kernel hands it to the colour kernel (bf16 hi + lo operand blocks);
  march                  the ray-distance + ray_march tail of shade_oracle.shade on a given (sigma, rgb), so that the compositing kernel
                         is checked on the shading kernel's own output;
  edit_*                 point values a trained checkpoint has and the generator does not (conf outside its clamp, embeddings of several
                         units, non-unit and zero directions, colours outside [0, 1]), written into a built model in place;
  sample_errors / check  errors per valid sample relative to the case's scale, with no outlier allowance; a failure names the worst
                         sample's ray, slot, valid index, colour tile and row, and neighbour count.
The forward needs no LeakyReLU masks (unlike the backward, oracle/grad_check.py): LeakyReLU is 1-Lipschitz, so a unit that rounding
puts on the other side of zero moves its output by no more than that rounding.
"""
import numpy as np
import torch

from . import shade_oracle

HBAR_TILE = 128                      # valid samples per colour tile (k_color_wg)
HBAR_BLOCK_BYTES = 2 * 8192          # one [128 x 32] bf16 block: hi, then lo 8 KB further


def dev_view(buf, ptr, dtype, shape):
    """A CPU copy of a device array at address ptr inside the uint8 CUDA tensor buf."""
    off = int(ptr) - buf.data_ptr()
    n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
    assert 0 <= off and off + n <= buf.numel()
    return buf[off:off + n].view(dtype).view(*shape).cpu()


def sample_map(q, ex):
    """Valid-sample index vi (the order of valid_list, of the h-bar / sigma workspace and of the backward's sample rows) -> dict of [S]
    tensors: cand (candidate index, the row of sigma_rgb), ray (query ray), slot (sample slot), srow (row of the export's flattened
    [R'*SR] layout), nnb (neighbours of the sample)."""
    S = int(q.counters["n_valid"])
    valid_list = dev_view(q.ws, q.desc.valid_list, torch.int32, (S,)).long()
    samp_off = dev_view(q.ws, q.desc.samp_off, torch.int32, (q.R + 1,)).long()
    ray_row = ex["ray_row"].cpu().long()
    ray = torch.searchsorted(samp_off, valid_list, right=True) - 1
    slot = valid_list - samp_off[ray]
    assert bool((slot >= 0).all() and (slot < q.SR).all()), "a valid sample outside its ray's slots"
    assert bool((ray_row[ray] >= 0).all()), "a valid sample on a ray the export does not hold"
    srow = ray_row[ray] * q.SR + slot
    nnb = (ex["sample_pidx"].cpu().reshape(-1, q.K)[srow] >= 0).sum(-1)
    assert bool((nnb > 0).all()), "a valid sample without neighbours in the export"
    assert int((ex["sample_pidx"].cpu() >= 0).any(-1).sum()) == S, "the export holds valid samples the kernel's list does not"
    return dict(cand=valid_list, ray=ray, slot=slot, srow=srow, nnb=nnb)


def pair_map(smap, pair_off, row_samp, pidx, ex, K):
    """The backward's packed pair rows (pair_off [S+1], row_samp [P], pidx [P]) -> their rows of the export's flattened [R'*SR*K] layout;
    every packed row is one valid pair of the export, with the export's point."""
    P = row_samp.shape[0]
    assert pair_off[-1].item() == P
    k = torch.arange(P) - pair_off[row_samp]
    assert bool(((k >= 0) & (k < (pair_off[1:] - pair_off[:-1])[row_samp])).all())
    flat = smap["srow"][row_samp] * K + k
    pm = ex["sample_pidx"].cpu().reshape(-1).long()
    assert torch.equal(torch.sort(flat)[0], (pm >= 0).nonzero()[:, 0]), "the packed rows are not the export's valid pairs"
    assert torch.equal(pm[flat], pidx), "a packed row's point differs from the export's"
    return flat


def tile_offset_bytes(r, k):
    """wgmma.cuh tile_offset_bytes<LAYOUT_NONE>: byte of (row r, column k < 32) in a [128 x 32] bf16 block of 8 x 16-byte core matrices."""
    return (r >> 3) * 512 + (k >> 3) * 128 + (r & 7) * 16 + (k & 7) * 2


def hbar_offset(vi, c):
    """Byte offset of the hi half of h-bar (valid sample vi, channel c) in the colour kernel's operand: per 128 samples 8 blocks (one per
    32 channels) of 16 KB, lo 8 KB after hi."""
    return ((vi >> 7) * 8 + (c >> 5)) * HBAR_BLOCK_BYTES + tile_offset_bytes(vi & 127, c & 31)


def _bf16(b, off):
    u = b[off].astype(np.uint32) | (b[off + 1].astype(np.uint32) << 8)
    return (u << 16).view(np.float32)


def decode_hbar(ws, n_valid):
    """h-bar [n_valid, 256] float64 = hi + lo from the operand blocks; ws: uint8 tensor (or array) starting at the h-bar buffer."""
    b = ws.cpu().numpy() if isinstance(ws, torch.Tensor) else np.asarray(ws)
    assert b.dtype == np.uint8 and b.size >= (n_valid + HBAR_TILE - 1) // HBAR_TILE * 8 * HBAR_BLOCK_BYTES
    off = hbar_offset(np.arange(n_valid)[:, None], np.arange(256)[None, :])
    return torch.from_numpy(_bf16(b, off).astype(np.float64) + _bf16(b, off + 8192).astype(np.float64))


def march(decoded, ray_valid, sample_loc_w, campos, camrotc2w, vsize, bg_color, dtype=torch.float64, raydist_mode_unit=1):
    """The ray-distance and ray_march tail of shade_oracle.shade on a given decoded [R',SR,4] (sigma, rgb).  The one discontinuous
    choice, the ray-distance mask (< 1e-8 or, with raydist_mode_unit, > 2 vz), is taken on fp32 distances as the reference takes it; the
    rest runs in `dtype`.  In fp32 this is shade()'s own arithmetic."""
    vz = float(vsize[2])
    Rn = decoded.shape[0]
    cam = camrotc2w.reshape(3, 3)

    def steps(dt):
        loc = shade_oracle.w2pers(sample_loc_w.to(dt), cam.to(dt), campos.to(dt).reshape(3))
        z = torch.cummax(loc[..., 2], dim=-1)[0]
        return torch.cat([z[..., 1:] - z[..., :-1], torch.full((Rn, 1), vz, dtype=dt)], dim=-1)

    d32 = steps(torch.float32)
    m = d32 < 1e-8
    if raydist_mode_unit > 0:
        m = torch.logical_or(m, d32 > 2 * vz)
    m = m.to(dtype)
    ray_dist = d32.to(dtype) if dtype == torch.float32 else steps(dtype)
    ray_dist = ray_dist * (1.0 - m) + m * vz
    ray_dist = ray_dist * ray_valid.to(dtype)
    decoded = decoded.to(dtype)
    sig = decoded[..., 0] * ray_valid.to(dtype)
    opacity = 1 - torch.exp(-sig * ray_dist)
    acc = torch.cumprod(1. - opacity + 1e-10, dim=-1)
    bg_T = acc[:, -1:]
    acc_T = torch.cat([torch.ones(Rn, 1, dtype=dtype), acc[:, :-1]], dim=-1)
    blend_weight = (opacity * acc_T)[..., None]
    ray_color = torch.sum(decoded[..., 1:4] * blend_weight, dim=-2) + bg_color.to(dtype).view(1, 3) * bg_T
    return dict(ray_dist=ray_dist, opacity=opacity, bg_T=bg_T, blend_weight=blend_weight, ray_color=ray_color)


def edit_conf(net, rays=None):
    """5 % of points_conf outside the clamp (0.0001, 1): zero, negative, tiny positive, above 1."""
    c = net.neural_points.points_conf
    N = c.shape[1]
    g = torch.Generator().manual_seed(7)
    idx = torch.randperm(N, generator=g)[:N // 20]
    vals = torch.tensor([0.0, -0.3, 5e-5, 1.7, 1.0 + 1e-3, -1e-6, 9.99e-5, 30.0])
    with torch.no_grad():
        c[0, idx.to(c.device), 0] = vals.repeat(len(idx) // len(vals) + 1)[:len(idx)].to(c.device)


def edit_embedding(scale):
    """points_embeding times `scale` (the generator's is 0.5 randn; the PE of the features takes 4 f)."""
    def edit(net, rays=None):
        with torch.no_grad():
            net.neural_points.points_embeding.mul_(scale)
    return edit


def edit_dir(net, rays=None):
    """points_dir of every point scaled by a seeded factor in [0, 3], 2 % of the points exactly zero."""
    d = net.neural_points.points_dir
    N = d.shape[1]
    g = torch.Generator().manual_seed(8)
    f = 3.0 * torch.rand(N, generator=g)
    f[torch.randperm(N, generator=g)[:N // 50]] = 0.0
    with torch.no_grad():
        d.mul_(f.to(d.device)[None, :, None])


def edit_color(net, rays=None):
    """points_color from [0, 1] to [-0.5, 1.5]."""
    with torch.no_grad():
        net.neural_points.points_color.mul_(2.0).sub_(0.5)


def sample_errors(got, ref, rows):
    """Errors per valid sample.  got: sigma [S], rgb [S,3] and optionally hbar [S,256], in valid-sample order; ref: an oracle dict
    (float64); rows: [S] rows of ref's flattened [R'*SR] layout.  sigma relative to the case's largest |sigma|, rgb absolute, hbar
    relative to the case's largest |hbar| (each over the valid samples)."""
    dec = ref["decoded"].reshape(-1, 4)[rows].double()
    err = dict(sigma=(got["sigma"].double() - dec[:, 0]).abs() / dec[:, 0].abs().max().clamp(min=1e-30),
               rgb=(got["rgb"].double() - dec[:, 1:]).abs().amax(-1))
    if got.get("hbar") is not None:
        h = ref["hbar"][rows].double()
        err["hbar"] = (got["hbar"].double() - h).abs().amax(-1) / h.abs().max().clamp(min=1e-30)
    return err


def describe_sample(smap, vi):
    """Where valid sample vi sits: ray, slot, colour tile and row, neighbours."""
    return "ray %d slot %d vi %d (tile %d row %d) %d neighbours" % (
        int(smap["ray"][vi]), int(smap["slot"][vi]), vi, vi // HBAR_TILE, vi % HBAR_TILE, int(smap["nnb"][vi]))


def worst(err):
    """(largest error, its index) of a per-row error tensor (0, -1 when empty)."""
    if err.numel() == 0:
        return 0.0, -1
    i = int(torch.argmax(err))
    return float(err[i]), i


def check(errs, bounds, where=lambda i: "row %d" % i):
    """errs: {name: per-row error tensor}; bounds: {name: largest allowed}.  Every comparison first, then one AssertionError naming each
    quantity beyond its bound and its worst row (`where` describes a row).  Returns {name: (worst error, row)}."""
    rep = {k: worst(e) for k, e in errs.items()}
    bad = ["%s: %.3e > %.1e at %s" % (k, rep[k][0], bounds[k], where(rep[k][1])) for k in errs if not rep[k][0] <= bounds[k]]
    assert not bad, "; ".join(bad)
    return rep
