"""TEST INFRASTRUCTURE ONLY -- records what the reference's own frustum query kernels return, for tests/test_oracle_frustum.py and
tests/test_gpu_frustum.py.

Runs the kernels oracle/build_ref_frustum.py compiled into oracle/_ref/libref_frustum.so (needs a GPU and that build, not the
reference tree) with the host glue of query_point_indices.py:615-770 restated step for step in torch (same allocations, same int8
cumsum, same block size), on the DTU-like scenes of pointnerf_b200.scene.FRUSTUM_CONFIGS.  Stores per case: the full ray mask
(bit-packed), the compacted pixel_idx, and for a seeded sample of the kept rays their sample_loc [SR,3] and neighbours [SR,K]; plus
max_o, the largest voxel fill and the number of marked voxels per column, asserted below the P and int8 limits (no reservoir, no wrap).

    python -m oracle.record_ref_frustum OUT_DIR
"""
import ctypes as C
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from pointnerf_b200 import query_point_indices as qpi, scene  # noqa: E402

LIB = os.path.join(ROOT, "oracle", "_ref", "libref_frustum.so")
MAX_RAYS = 1500
MAX_FILE_BYTES = 1 << 20
THREADS = 1024   # opt.gpu_maxthr


def case_inputs(name):
    cfg = scene.FRUSTUM_CONFIGS[name]
    s = scene.make_frustum_scene(cfg)
    opt = scene.frustum_opt(cfg)
    hyper = qpi.hyperparameters(opt, np.int64(cfg.H), np.int64(cfg.W), s["intrinsic"], np.float32(cfg.near), np.float32(cfg.far))
    return cfg, s, opt, hyper


def reference_query(lib, cfg, s, opt, hyper, dev):
    radius_limit, depth_limit, ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale = hyper
    P_ = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    pts = torch.from_numpy(s["pers"])[None].to(dev).contiguous()
    B, N = 1, pts.shape[1]
    npts = torch.tensor([N], dtype=torch.int32, device=dev)
    range_gpu = torch.from_numpy(ranges).to(dev)
    svs_gpu = torch.from_numpy(scaled_vsize).to(dev)
    sdim_gpu = torch.from_numpy(scaled_vdim).to(dev)
    vscale_gpu = torch.from_numpy(vscale).to(dev)
    ks_gpu = torch.tensor(opt.kernel_size, dtype=torch.int32, device=dev)
    qs_gpu = torch.tensor(opt.query_size, dtype=torch.int32, device=dev)
    sd = [int(v) for v in scaled_vdim]
    pixel_size, grid_size_vol = sd[0] * sd[1], sd[0] * sd[1] * sd[2]
    pix = torch.from_numpy(s["pixel_idx"]).to(dev).reshape(B, -1, 2).clone()
    R = pix.shape[1]
    SR, K, P = opt.SR, opt.K, opt.P

    coor_occ = torch.zeros([B] + sd, dtype=torch.uint8, device=dev)
    loc = torch.zeros([B] + sd, dtype=torch.int8, device=dev)
    near_id = torch.full([B, sd[0], sd[1]], sd[2], dtype=torch.int32, device=dev)
    far_id = torch.full([B, sd[0], sd[1]], -1, dtype=torch.int32, device=dev)
    g = (B * N + THREADS - 1) // THREADS
    assert lib.ref_get_occ_vox(g, THREADS, P_(pts), P_(npts), B, N, P_(range_gpu), P_(svs_gpu), P_(sdim_gpu), P_(qs_gpu), pixel_size,
                               grid_size_vol, P_(coor_occ), P_(loc), P_(near_id), P_(far_id), 0) == 0
    coorz = torch.full([B, sd[0], sd[1], SR], -1, dtype=torch.int16, device=dev)
    pixel_map = torch.zeros([B, sd[0], sd[1]], dtype=torch.uint8, device=dev)
    ray_mask = torch.zeros([B, R], dtype=torch.int8, device=dev)
    g = (B * R + THREADS - 1) // THREADS
    assert lib.ref_near_vox_full(g, THREADS, B, SR, P_(pix), R, P_(vscale_gpu), P_(sdim_gpu), pixel_size, grid_size_vol, P_(qs_gpu),
                                 P_(pixel_map), P_(ray_mask), P_(coor_occ), P_(loc), P_(near_id), P_(far_id), P_(coorz)) == 0
    pix_cur = torch.masked_select(pix, (ray_mask > 0)[..., None].expand(-1, -1, 2)).reshape(1, -1, 2).contiguous()
    R2 = int(torch.sum(ray_mask, dim=-1).max().item())
    marked = (loc > 0).to(torch.int8)
    marked_per_col = int(marked.to(torch.int32).sum(-1).max().item())
    loc = (marked * torch.cumsum(marked, dtype=torch.int8, dim=-1) - 1).contiguous()
    max_o = int(torch.max(loc).item()) + 1
    vcnt = torch.zeros([B, sd[0], sd[1], max_o], dtype=torch.int16, device=dev)
    vpt = torch.zeros([B, sd[0], sd[1], max_o, P], dtype=torch.int32, device=dev)
    ray_vsize_gpu = (svs_gpu.double() / vscale_gpu.double()).float()
    g = (B * N + THREADS - 1) // THREADS
    assert lib.ref_insert_vox_points(g, THREADS, P_(pts), P_(npts), B, N, P, max_o, pixel_size, grid_size_vol, P_(range_gpu),
                                     P_(sdim_gpu), P_(svs_gpu), P_(loc), P_(vcnt), P_(vpt), C.c_ulong(12345), 0) == 0
    sample_pidx = torch.full([B, R2, SR, K], -1, dtype=torch.int32, device=dev)
    sample_loc = torch.full([B, R2, SR, 3], 0.0, dtype=torch.float32, device=dev)
    if R2 > 0:
        g = (R2 * SR + THREADS - 1) // THREADS
        assert lib.ref_query_layered(g, THREADS, P_(pts), B, SR, R2, max_o, P, K, pixel_size, grid_size_vol,
                                     C.c_float(float(np.float32(radius_limit ** 2))), C.c_float(float(np.float32(depth_limit ** 2))),
                                     P_(range_gpu), P_(sdim_gpu), P_(svs_gpu), P_(ray_vsize_gpu), P_(vscale_gpu), P_(ks_gpu), P_(pix_cur),
                                     P_(loc), P_(coorz), P_(vcnt), P_(vpt), P_(sample_pidx), P_(sample_loc), C.c_ulong(12345), 2, 0) == 0
    return dict(ray_mask=ray_mask[0].cpu().numpy(), pixel_idx_cur=pix_cur[0].cpu().numpy(), sample_pidx=sample_pidx[0].cpu().numpy(),
                sample_loc=sample_loc[0].cpu().numpy(), max_o=max_o, max_fill=int(vcnt.max().item()), marked_per_col=marked_per_col)


def record(name, lib, dev):
    cfg, s, opt, hyper = case_inputs(name)
    out = reference_query(lib, cfg, s, opt, hyper, dev)
    assert out["max_fill"] <= cfg.P, "%s: a voxel holds %d > P points (the reference samples a reservoir)" % (name, out["max_fill"])
    assert out["marked_per_col"] <= 127, "%s: %d marked voxels in one column wrap the int8 numbering" % (name, out["marked_per_col"])
    R2 = out["pixel_idx_cur"].shape[0]
    rng = np.random.RandomState(0)
    rows = np.arange(R2) if R2 <= MAX_RAYS else np.sort(rng.choice(R2, size=MAX_RAYS, replace=False))
    return dict(R=np.int64(out["ray_mask"].size), mask_bits=np.packbits(out["ray_mask"] > 0), pixel_idx_cur=out["pixel_idx_cur"],
                rows=rows.astype(np.int32), sample_loc=out["sample_loc"][rows], sample_pidx=out["sample_pidx"][rows],
                max_o=np.int64(out["max_o"]), max_fill=np.int64(out["max_fill"]), marked_per_col=np.int64(out["marked_per_col"]))


def main(out_dir):
    assert os.path.isfile(LIB), "%s is missing: run `python -m oracle.build_ref_frustum` where the reference tree exists" % LIB
    lib = C.CDLL(LIB)
    os.makedirs(out_dir, exist_ok=True)
    for name in scene.FRUSTUM_CONFIGS:
        d = record(name, lib, torch.device("cuda:0"))
        path = os.path.join(out_dir, "ref_frustum_%s.npz" % name)
        np.savez_compressed(path, **d)
        assert os.path.getsize(path) <= MAX_FILE_BYTES, "%s: %d bytes" % (path, os.path.getsize(path))
        print(name, "rays", int(d["R"]), "kept", d["pixel_idx_cur"].shape[0], "stored", d["rows"].size, "max_o", int(d["max_o"]),
              "max_fill", int(d["max_fill"]), "marked/col", int(d["marked_per_col"]), "bytes", os.path.getsize(path))


if __name__ == "__main__":
    main(sys.argv[1])
