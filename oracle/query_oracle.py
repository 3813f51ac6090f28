"""TEST INFRASTRUCTURE ONLY -- Python face of oracle/query_oracle.c (the serial C restatement of
/root/reference/models/neural_points/cuda/query_worldcoords.cu).  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import this module.

Two entry points:
  query(...)                        numpy in / numpy out, campos+raydir+t-table form (what the CUDA
                                    path is compared against);
  woord_query_grid_point_index(...) the 18-argument torch-level signature of the reference's pybind op
                                    (query_worldcoords.cpp:34-82) so that the reference's own
                                    lighting_fast_querier (point_query.py) can run on top of it on CPU.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "liboracle_query.so")
_lib = None

COUNTER_NAMES = ("n_occ", "max_pts", "overflow_o", "overflow_p", "R1", "R2",
                 "n_valid_samples", "n_valid_pairs", "n_cand", "slot0_cell")


def build(force=False):
    """gcc the C restatement (building the checker is not using it)."""
    src = os.path.join(_HERE, "query_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return _SO


def _load():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        _lib.pnb_oracle_query.restype = ctypes.c_int
    return _lib


def _p(a, ty):
    return a.ctypes.data_as(ctypes.POINTER(ty)) if a is not None else None


def query(xyz, lo, svs, dim, kernel_size, query_size, max_o, P, radius_limit,
          campos=None, raydir=None, t=None, raypos=None, SR=24, K=8, parity_slot0=1):
    """Returns dict(sample_pidx[R2,SR,K] i32, sample_loc_w[R2,SR,3] f32, ray_mask[R] i8, counters{}).
    t: [D] shared table or [R,D] per-ray table (train jitter).  raypos: optional [R,D,3].
    parity_slot0: 1 = the voxel that wins occupancy slot 0 holds no points (query_worldcoords.cu:147, the reference's
    behaviour); 0 = it keeps them (the product's pnb_parity_slot0 0)."""
    lib = _load()
    xyz = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3)
    lo = np.ascontiguousarray(lo, np.float32); svs = np.ascontiguousarray(svs, np.float32)
    dim = np.ascontiguousarray(dim, np.int32)
    ks = np.ascontiguousarray(kernel_size, np.int32); qs = np.ascontiguousarray(query_size, np.int32)
    if raypos is not None:
        raypos = np.ascontiguousarray(raypos, np.float32)
        R, D = raypos.shape[0], raypos.shape[1]
        campos_a = np.zeros(3, np.float32); raydir_a = np.zeros((R, 3), np.float32)
        t_a = np.zeros(D, np.float32); stride = 0
    else:
        campos_a = np.ascontiguousarray(campos, np.float32).reshape(3)
        raydir_a = np.ascontiguousarray(raydir, np.float32).reshape(-1, 3)
        R = raydir_a.shape[0]
        t_a = np.ascontiguousarray(t, np.float32)
        D = t_a.shape[-1]
        stride = D if t_a.ndim == 2 else 0
        if t_a.ndim == 2:
            assert t_a.shape[0] == R
    ray_mask = np.zeros(R, np.int8)
    pidx = np.full((max(R, 1), SR, K), -1, np.int32)
    loc = np.zeros((max(R, 1), SR, 3), np.float32)
    counters = np.zeros(10, np.int32)
    rc = lib.pnb_oracle_query(
        _p(xyz, ctypes.c_float), ctypes.c_int(xyz.shape[0]),
        _p(lo, ctypes.c_float), _p(svs, ctypes.c_float), _p(dim, ctypes.c_int),
        _p(ks, ctypes.c_int), _p(qs, ctypes.c_int),
        ctypes.c_int(int(max_o)), ctypes.c_int(int(P)), ctypes.c_float(float(radius_limit)),
        _p(campos_a, ctypes.c_float), _p(raydir_a, ctypes.c_float), ctypes.c_int(R),
        _p(t_a, ctypes.c_float), ctypes.c_int(stride), ctypes.c_int(D),
        _p(raypos, ctypes.c_float),
        ctypes.c_int(SR), ctypes.c_int(K), ctypes.c_int(1 if parity_slot0 else 0),
        _p(ray_mask, ctypes.c_int8), _p(pidx, ctypes.c_int), _p(loc, ctypes.c_float),
        _p(counters, ctypes.c_int))
    if rc != 0:
        raise RuntimeError("pnb_oracle_query failed rc=%d" % rc)
    c = dict(zip(COUNTER_NAMES, (int(v) for v in counters)))
    R2 = c["R2"]
    return dict(sample_pidx=pidx[:R2].copy(), sample_loc_w=loc[:R2].copy(), ray_mask=ray_mask, counters=c)


last_counters = None


def woord_query_grid_point_index(pixel_idx, raypos, xyz, actual_numpoints, kernel_size, query_size,
                                 SR, K, R, D, scaled_vdim, max_o, P, radius_limit, ranges, scaled_vsize,
                                 kMaxThreadsPerBlock, NN):
    """Signature of query_worldcoords.cpp:34-52; tensors are CPU torch tensors here.  B must be 1 (Q7)."""
    import torch
    global last_counters
    assert xyz.shape[0] == 1, "B==1 only (SURVEY 8a Q7)"
    n = int(actual_numpoints[0])
    out = query(xyz[0, :n].detach().cpu().numpy(), ranges.detach().cpu().numpy()[:3],
                scaled_vsize.detach().cpu().numpy(), scaled_vdim.detach().cpu().numpy(),
                kernel_size.detach().cpu().numpy(), query_size.detach().cpu().numpy(),
                max_o, P, float(radius_limit), raypos=raypos[0].detach().cpu().numpy(), SR=SR, K=K)
    last_counters = out["counters"]
    return [torch.from_numpy(out["sample_pidx"])[None], torch.from_numpy(out["sample_loc_w"])[None],
            torch.from_numpy(out["ray_mask"])[None]]
