"""Voxel down-sampling of a point cloud on the GPU: drop-ins for construct_vox_points, construct_vox_points_xyz,
construct_vox_points_ind and construct_vox_points_closest of models/mvs/mvs_utils.py:484-561, without torch_scatter.

Same signatures, return values and dtypes as the reference (centroids float32, sparse_grid_idx int32, inv_idx and min_idx int64).  The
space and voxel size come from the reference's own torch expressions, so the kernels start from the reference's bits.  Unlike the
reference, the result is the same on every run: the centroid is summed in fp64 in a fixed order and rounded once to fp32, and among
tied residuals the closest point is the lowest index (DESIGN.md §5 "Voxel down-sampling").

Each call synchronises once, to size the outputs by the number of voxels M.
"""
import torch

from . import lib as _lib

# With the space derived from the cloud, every voxel index lies in [0, ~0.98 * vox_res]: below this, 10 bits per axis hold it.
KEY32_MAX_RES = 1000


def _space(xyz, vox_res, space_min, space_max):
    """space_min, space_max and the voxel size, written as mvs_utils.py:487-495 writes them."""
    if space_min is None:
        xyz_min, xyz_max = torch.min(xyz, dim=-2)[0], torch.max(xyz, dim=-2)[0]
        space_edge = torch.max(xyz_max - xyz_min) * 1.05
        xyz_mid = (xyz_max + xyz_min) / 2
        space_min = xyz_mid - space_edge / 2
        space_max = xyz_mid + space_edge / 2
    else:
        space_edge = space_max - space_min
    construct_vox_sz = space_edge / vox_res
    return space_min, space_max, construct_vox_sz


def _check_points(name, t):
    if not isinstance(t, torch.Tensor) or t.dim() != 2 or t.shape[1] != 3 or t.dtype != torch.float32 or not t.is_cuda:
        raise ValueError("%s must be a float32 CUDA tensor of shape [N, 3] (got %s)" % (
            name, "%s %s %s" % (tuple(t.shape), t.dtype, t.device) if isinstance(t, torch.Tensor) else type(t).__name__))


def voxelize(xyz, space_min, vox_sz, val=None, key_bits=64, inv_idx=False, grid_idx=True, centroid=False, min_idx=None):
    """The kernels on xyz [N,3] (keys) and val [N,3] (values, default xyz); space_min and vox_sz are float32 CUDA tensors of 3 (or 1)
    elements.  min_idx: None, "first" (lowest point index of each voxel) or "closest" (nearest its centroid).  Returns a dict of the
    requested outputs and the counters of the build."""
    _check_points("xyz", xyz)
    val = xyz if val is None else val
    _check_points("xyz_val", val)
    if val.shape[0] != xyz.shape[0]:
        raise ValueError("xyz_val has %d points and partition_xyz %d: the voxel of every value point comes from its key point"
                         % (val.shape[0], xyz.shape[0]))
    N = int(xyz.shape[0])
    if N >= 2 ** 31:
        raise ValueError("at most 2^31 - 1 points (got %d)" % N)
    dev = xyz.device
    smin = space_min.to(device=dev).reshape(-1).expand(3).contiguous()
    vsz = vox_sz.to(device=dev).reshape(-1).expand(3).contiguous()
    if smin.dtype != torch.float32 or vsz.dtype != torch.float32:
        raise ValueError("space_min / space_max must be float32, as the points are")
    xyz, val = xyz.contiguous(), val.contiguous()
    lib = _lib.load()
    ws = torch.empty(lib.pnb_vox_bytes(N, key_bits), dtype=torch.uint8, device=dev)
    inv = torch.empty(N, dtype=torch.int64, device=dev) if inv_idx else None
    v, hc = _lib.Vox(), (_lib.C.c_int32 * 16)()
    stream = torch.cuda.current_stream(dev).cuda_stream
    _lib.check(lib.pnb_vox_build(_lib.C.byref(v), ws.data_ptr(), ws.numel(), xyz.data_ptr(), N, smin.data_ptr(), vsz.data_ptr(),
                                 key_bits, inv.data_ptr() if inv is not None else None, stream, hc), "pnb_vox_build")
    M = v.n_vox
    out = dict(counters={k: int(hc[i]) for k, i in _lib.VC.items()})
    out["grid_idx"] = torch.empty((M, 3), dtype=torch.int32, device=dev) if grid_idx else None
    out["centroid"] = torch.empty((M, 3), dtype=torch.float32, device=dev) if centroid or min_idx == "closest" else None
    out["min_idx"] = torch.empty(M, dtype=torch.int64, device=dev) if min_idx else None
    out["inv_idx"] = inv
    ptr = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    _lib.check(lib.pnb_vox_outputs(_lib.C.byref(v), val.data_ptr(), ptr(out["grid_idx"]), ptr(out["centroid"]), ptr(out["min_idx"]),
                                   int(min_idx == "closest"), stream), "pnb_vox_outputs")
    del ws                                               # the caching allocator reuses it only after the outputs' kernels on stream
    return out


def _prepare(xyz_val, vox_res, partition_xyz, space_min, space_max):
    if not vox_res > 0:
        raise ValueError("vox_res must be > 0 (got %r)" % (vox_res,))
    xyz = xyz_val if partition_xyz is None else partition_xyz
    _check_points("partition_xyz" if partition_xyz is not None else "xyz_val", xyz)
    if space_min is None and xyz.shape[0] == 0:
        raise ValueError("an empty point cloud has no extent: pass space_min and space_max")
    own_space = space_min is None
    space_min, space_max, vox_sz = _space(xyz, vox_res, space_min, space_max)
    key_bits = 32 if own_space and vox_res < KEY32_MAX_RES else 64
    return xyz, space_min, space_max, vox_sz, key_bits


def construct_vox_points(xyz_val, vox_res, partition_xyz=None, space_min=None, space_max=None):
    """(xyz_centroid [M,3], sparse_grid_idx [M,3] int32, min_idx [M] int64: the lowest point index of each voxel)."""
    xyz, space_min, _, vox_sz, bits = _prepare(xyz_val, vox_res, partition_xyz, space_min, space_max)
    o = voxelize(xyz, space_min, vox_sz, val=xyz_val, key_bits=bits, centroid=True, min_idx="first")
    return o["centroid"], o["grid_idx"], o["min_idx"]


def construct_vox_points_xyz(xyz_val, vox_res, partition_xyz=None, space_min=None, space_max=None):
    """xyz_centroid [M,3] (a tensor, as the reference returns it)."""
    xyz, space_min, _, vox_sz, bits = _prepare(xyz_val, vox_res, partition_xyz, space_min, space_max)
    return voxelize(xyz, space_min, vox_sz, val=xyz_val, key_bits=bits, grid_idx=False, centroid=True)["centroid"]


def construct_vox_points_ind(xyz_val, vox_res, partition_xyz=None, space_min=None, space_max=None):
    """(sparse_grid_idx [M,3] int32, inv_idx [N] int64, space_min, space_max)."""
    xyz, space_min, space_max, vox_sz, bits = _prepare(xyz_val, vox_res, partition_xyz, space_min, space_max)
    o = voxelize(xyz, space_min, vox_sz, key_bits=bits, inv_idx=True)
    return o["grid_idx"], o["inv_idx"], space_min, space_max


def construct_vox_points_closest(xyz_val, vox_res, partition_xyz=None, space_min=None, space_max=None):
    """(xyz_centroid [M,3], sparse_grid_idx [M,3] int32, min_idx [M] int64: the point nearest each voxel's centroid).

    With space_min the reference drops the points of xyz_val outside (space_min, space_max) (mvs_utils.py:547-550) but keeps every
    point of the cloud it voxelises, so it can only run when nothing is dropped or partition_xyz holds the kept points; any other
    case raises ValueError here (the reference fails on a shape mismatch)."""
    callers_space = space_min is not None
    xyz, space_min, _, vox_sz, bits = _prepare(xyz_val, vox_res, partition_xyz, space_min, space_max)
    val = xyz_val
    if callers_space:                                    # mvs_utils.py:545-550
        mask = (xyz_val - space_min[None, ...])
        mask *= (space_max[None, ...] - xyz_val)
        mask = torch.prod(mask, dim=-1) > 0
        val = xyz_val[mask, :]
        if val.shape[0] != xyz.shape[0]:
            raise ValueError("construct_vox_points_closest: %d of %d points of xyz_val lie outside (space_min, space_max) and are "
                             "dropped, but %s still has %d; pass the kept points as partition_xyz"
                             % (xyz_val.shape[0] - val.shape[0], xyz_val.shape[0],
                                "partition_xyz" if partition_xyz is not None else "the voxelised cloud", xyz.shape[0]))
    o = voxelize(xyz, space_min, vox_sz, val=val, key_bits=bits, min_idx="closest")
    return o["centroid"], o["grid_idx"], o["min_idx"]
