"""TEST INFRASTRUCTURE ONLY -- records what the reference's own CUDA query kernel returns, for tests/test_gpu_ref_kernel.py.

Runs the un-modified `query_worldcoords_cuda` extension that oracle/build_ref.py compiled into oracle/_ref/ (needs a GPU and that
build, not the reference tree) on the cases of the test, with the 18 arguments of the reference's
models/neural_points/point_query.py:85-93 formed from the same inputs the product receives, and stores per case:
  * R and the reference's full ray mask (bit-packed),
  * for every ray the reference kept (chair: a fixed, seeded sample of MAX_RAYS["chair_centre"] of its 9,216, so that the file stays
    under 1 MB): their indices, neighbour indices [SR, K] and world sample positions [SR, 3].
The files are committed as tests/golden/ref_kernel_<case>.npz (each < 1 MB).

    python -m oracle.record_ref_kernel OUT_DIR
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pointnerf_b200 import harness, scene  # noqa: E402

MAX_RAYS = {"chair_centre": 2500}      # kept rays stored per case (default: all)
MAX_FILE_BYTES = 1 << 20
# case -> (config, pixels, overrides); pixels: None = full frame, ("centre", side) or ("block", x0, y0, w, h)
CASES = {
    "tiny_full": ("tiny", None, {}),
    "chair_centre": ("chair_plumbing", ("centre", 96), {}),
    "lego_centre_sr24": ("lego_render", ("centre", 48), dict(SR=24)),
    "lego_centre_sr80": ("lego_render", ("centre", 48), dict(SR=80)),
    "lego_silhouette": ("lego_render", ("block", 640, 388, 96, 24), {}),
    "truck_centre": ("truck_8gpu", ("centre", 32), {}),
    "truck_corner": ("truck_8gpu", ("block", 860, 0, 100, 16), {}),
    "scannet_centre": ("scannet_8gpu", ("centre", 24), {}),
}


def case_pixels(cfg, spec):
    if spec is None:
        return None
    if spec[0] == "centre":
        return scene.centre_patch(cfg, spec[1])
    x0, y0, w, h = spec[1:]
    px, py = np.meshgrid(np.arange(x0, x0 + w), np.arange(y0, y0 + h))
    return np.stack((px, py), -1).reshape(-1, 2).astype(np.float32)


def setup(case, dev):
    """The product's model and query inputs of a case (also what the test runs)."""
    name, spec, over = CASES[case]
    cfg = scene.CONFIGS[name]
    net, pts, opt = harness.build_model(cfg, dev, **over)
    rays = scene.make_rays(cfg, case_pixels(cfg, spec))
    r = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in rays.items()}
    return cfg, net, opt, r


def product_query(cfg, net, r):
    querier = net.neural_points.querier
    xyz = net.neural_points.xyz.detach().contiguous()
    npts = torch.tensor([xyz.shape[0]], dtype=torch.int32, device=xyz.device)
    pix = r["pixel_idx"].to(torch.int32)
    return querier.query_points(pix, None, xyz[None], npts, r["h"], r["w"], r["intrinsic"], np.float32(cfg.near),
                                np.float32(cfg.far), r["raydir"].contiguous(), r["campos"], r["camrotc2w"])


def reference_query(ext, cfg, net, opt, r):
    """woord_query_grid_point_index with the arguments of point_query.py:85-93 (after product_query set up the querier)."""
    dev = r["raydir"].device
    querier = net.neural_points.querier
    raydir = r["raydir"].contiguous()
    R = raydir.shape[1]
    xyz = net.neural_points.xyz.detach().contiguous()
    npts = torch.tensor([xyz.shape[0]], dtype=torch.int32, device=dev)
    ranges_tensor, ranges_np, vsize_np, scaled_vdim_np = querier._hyper
    t = querier._t_for(cfg.near, cfg.far, R, dev)
    # ray generation of diff_ray_marching.py:386-388 as torch runs it on the device: one mul kernel, one add kernel
    raypos = (r["campos"][:, None, None, :] + raydir[:, :, None, :] * t[None, None, :, None]).contiguous()
    max_o = int(opt.max_o) if opt.max_o is not None else int(xyz.shape[0])
    out = ext.woord_query_grid_point_index(
        r["pixel_idx"].to(torch.int32), raypos, xyz[None], npts, querier.kernel_size_tensor, querier.query_size_tensor, int(opt.SR),
        int(opt.K), R, raypos.shape[2], torch.as_tensor(scaled_vdim_np, device=dev), max_o, int(opt.P), float(querier.radius_limit_np),
        ranges_tensor.to(dev), querier.scaled_vsize_tensor, 1024, 2)
    torch.cuda.synchronize()
    return out


def record(case, ext, dev, max_rays=None):
    cfg, net, opt, r = setup(case, dev)
    product_query(cfg, net, r)
    pidx, locw, mask = reference_query(ext, cfg, net, opt, r)[:3]
    mask = mask[0].reshape(-1).cpu().numpy() > 0
    hit = np.nonzero(mask)[0]
    rng = np.random.RandomState(0)
    sel = hit if max_rays is None or max_rays >= hit.size else np.sort(rng.choice(hit, size=max_rays, replace=False))
    rows = np.cumsum(mask)[sel] - 1
    return dict(R=np.int64(mask.size), mask_bits=np.packbits(mask), ray_idx=sel.astype(np.int32),
                pidx=pidx[0].cpu().numpy()[rows].astype(np.int32), locw=locw[0].cpu().numpy()[rows].astype(np.float32))


def main(out_dir):
    from oracle import build_ref
    ext = build_ref.load_prebuilt()
    assert ext is not None, "oracle/_ref/query_worldcoords_cuda.so is missing: run `python -m oracle.build_ref`"
    os.makedirs(out_dir, exist_ok=True)
    for case in CASES:
        d = record(case, ext, torch.device("cuda:0"), MAX_RAYS.get(case))
        path = os.path.join(out_dir, "ref_kernel_%s.npz" % case)
        np.savez_compressed(path, **d)
        assert os.path.getsize(path) <= MAX_FILE_BYTES, "%s: %d bytes" % (path, os.path.getsize(path))
        print(case, "rays", int(d["R"]), "kept", int(np.unpackbits(d["mask_bits"])[:int(d["R"])].sum()), "sampled", d["ray_idx"].size)


if __name__ == "__main__":
    main(sys.argv[1])
