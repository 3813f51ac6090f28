"""TEST INFRASTRUCTURE ONLY -- Python face of oracle/frustum_oracle.c, the serial C restatement of the reference's perspective-frustum
query (query_point_indices.py, NN 2).  query(...) takes numpy inputs and returns the reference's outputs in numpy."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "frustum_oracle.c")
_SO = os.path.join(_HERE, "_build", "libfrustum_oracle.so")
_lib = None

COUNTER_NAMES = ("R2", "overflow_p", "overflow_o", "max_o", "max_pts", "n_bad_pixel", "n_col_capped")


def build(force=False):
    """gcc the C restatement; -ffp-contract=off: no a*b+c is fused unless the source says fmaf / fma."""
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        os.makedirs(os.path.dirname(_SO), exist_ok=True)
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-shared",
                               "-o", _SO, _SRC, "-lm"])
    return _SO


def _load():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        _lib.pnb_oracle_frustum.restype = ctypes.c_int
    return _lib


def _p(a, ty):
    return a.ctypes.data_as(ctypes.POINTER(ty))


def query(pers, lo, svs, dim, vscale, kernel_size, query_size, SR, K, P, pixel_idx, radius_limit2=0.0, depth_limit2=0.0, max_o=None):
    """pers [N,3] points in perspective coordinates, pixel_idx [R,2] int.  Returns dict(ray_mask [R] i8, pixel_idx_cur [R',2] i32,
    sample_pidx [R',SR,K] i32, sample_loc [R',SR,3] f32, counters{})."""
    lib = _load()
    pers = np.ascontiguousarray(pers, np.float32).reshape(-1, 3)
    pix = np.ascontiguousarray(pixel_idx, np.int32).reshape(-1, 2)
    R = pix.shape[0]
    f3 = lambda v: np.ascontiguousarray(v, np.float32).reshape(3)  # noqa: E731
    i3 = lambda v: np.ascontiguousarray(v, np.int32).reshape(3)    # noqa: E731
    lo, svs, dim, vs, ks, qs = f3(lo), f3(svs), i3(dim), i3(vscale), i3(kernel_size), i3(query_size)
    ray_mask = np.zeros(max(R, 1), np.int8)
    cur = np.zeros((max(R, 1), 2), np.int32)
    pidx = np.full((max(R, 1), SR, K), -1, np.int32)
    loc = np.zeros((max(R, 1), SR, 3), np.float32)
    counters = np.zeros(16, np.int32)
    rc = lib.pnb_oracle_frustum(
        _p(pers, ctypes.c_float), ctypes.c_int(pers.shape[0]), _p(lo, ctypes.c_float), _p(svs, ctypes.c_float), _p(dim, ctypes.c_int),
        _p(vs, ctypes.c_int), _p(ks, ctypes.c_int), _p(qs, ctypes.c_int), ctypes.c_int(SR), ctypes.c_int(K), ctypes.c_int(P),
        ctypes.c_int(int(max_o) if max_o else 0), ctypes.c_float(float(radius_limit2)), ctypes.c_float(float(depth_limit2)),
        _p(pix, ctypes.c_int), ctypes.c_int(R), _p(ray_mask, ctypes.c_int8), _p(cur, ctypes.c_int), _p(pidx, ctypes.c_int),
        _p(loc, ctypes.c_float), _p(counters, ctypes.c_int))
    if rc != 0:
        raise RuntimeError("pnb_oracle_frustum failed rc=%d" % rc)
    c = dict(zip(COUNTER_NAMES, (int(v) for v in counters)))
    R2 = c["R2"]
    return dict(ray_mask=ray_mask[:R].copy(), pixel_idx_cur=cur[:R2].copy(), sample_pidx=pidx[:R2].copy(), sample_loc=loc[:R2].copy(),
                counters=c)
