"""Host-side mirror of the reference's `lighting_fast_querier` (wcoord_query = -1 flavour),
/root/reference/models/neural_points/point_query.py:25-108, on top of libpnb200.so.

Same constructor (`lighting_fast_querier(device, opt)`), same `query_points(...)` signature and
7-tuple of returns, same `clean_up()`, same `get_hyperparameters()` -- so that
`NeuralPoints.__init__` (/root/reference/models/neural_points/neural_points.py:330-339) can pick
this class up unchanged (see INTEGRATION.md).  Differences, all deliberate:
  * the voxel grid is built once per point cloud (storage object, address, version, size) and cached (the
    reference rebuilds it on every ray chunk, query_worldcoords.cu:314-365);
  * ray positions are never materialised ([1,R,400,3] in the reference);
  * results are deterministic (canonical serial semantics, SURVEY.md 8a), overflow of max_o / P is
    reported (`last_grid_counters`) instead of resolved by wall-clock-seeded curand;
  * no CPU path: the CUDA library must be present, otherwise lib.load() raises.
"""
import weakref

import numpy as np
import torch

from . import lib as _lib


def same_storage(ref, t):
    """True when the weak reference `ref` (or None) points at the storage of tensor `t`.  The queriers cache their build on the points
    they were handed, which arrive as a new tensor object on every call (NeuralPoints passes `self.xyz[None]`, the fused module a
    detached `xyz`); every view and detached alias of one cloud shares its storage object, which lives exactly as long as the cloud's
    memory.  A key of (data_ptr, _version, N) alone also matches a NEW cloud that the caching allocator placed where a freed one was
    (both at version 0), which a feed-forward run (a new cloud from the network on every call) produces; its storage is another
    object."""
    return ref is not None and ref() is t.untyped_storage()


def host_t_table(near, far, D):
    """Mid-point table of near_far_linear_ray_generation with jitter 0
    (/root/reference/models/rendering/diff_ray_marching.py:369-385), evaluated with the same fp32
    torch CPU ops so that the table is bit-identical to what the reference's CPU path marches."""
    tvals = torch.linspace(0, 1, D + 1).view(1, -1)
    tvals = near * (1 - tvals) + far * tvals
    seg = (tvals[..., 1:] - tvals[..., :-1]) * (1 + 0.0 * (torch.zeros(1, 1, D) - 0.5))
    end = torch.cumsum(seg, dim=2)
    end = torch.cat([torch.zeros(1, 1, 1), end], dim=2)
    end = near + end
    return ((end[:, :, :-1] + end[:, :, 1:]) / 2).reshape(D).contiguous()


def device_t_table_jitter(near, far, D, R, jitter, device, generator=None):
    """Per-ray table [R, D] for is_train (jitter 0.3): same ops as diff_ray_marching.py:369-385 on device."""
    tvals = torch.linspace(0, 1, D + 1, device=device).view(1, -1)
    tvals = near * (1 - tvals) + far * tvals
    seg = (tvals[..., 1:] - tvals[..., :-1]) * (1 + jitter * (torch.rand((1, R, D), device=device, generator=generator) - 0.5))
    end = torch.cumsum(seg, dim=2)
    end = torch.cat([torch.zeros((1, R, 1), device=device), end], dim=2)
    end = near + end
    return ((end[:, :, :-1] + end[:, :, 1:]) / 2).reshape(R, D).contiguous()


class VoxelGrid:
    """Owns the device buffer of one pnb_grid_t."""

    def __init__(self, xyz, lo, svs, dim, query_size, max_o, P, parity_slot0=True, want_counters=True):
        lib = _lib.load()
        assert xyz.is_cuda and xyz.dtype == torch.float32 and xyz.is_contiguous()
        self.N = xyz.shape[0]
        dim_c = _lib.i3(dim)
        nbytes = lib.pnb_grid_bytes(self.N, dim_c)
        self.buf = torch.empty(nbytes, dtype=torch.uint8, device=xyz.device)
        self.desc = _lib.Grid()
        hc = (_lib.C.c_int32 * 16)() if want_counters else None
        stream = torch.cuda.current_stream(xyz.device).cuda_stream
        _lib.check(lib.pnb_grid_build(_lib.C.byref(self.desc), self.buf.data_ptr(), nbytes, xyz.data_ptr(), self.N,
                                      _lib.f3(lo), _lib.f3(svs), dim_c, _lib.i3(query_size), int(max_o), int(P),
                                      1 if parity_slot0 else 0, stream, hc), "pnb_grid_build")
        self.counters = {k: int(hc[i]) for k, i in _lib.GC.items()} if want_counters else None
        self.xyz_ref = xyz  # keep the storage alive while the grid is in use


class QueryResult:
    """Owns the workspace of one pnb_query_t (sample-compacted query output)."""

    def __init__(self, grid, campos, raydir, t, D, SR, K, radius_limit, kernel_size, cap_samples=0, ws=None,
                 want_counters=False):
        lib = _lib.load()
        assert raydir.is_cuda and raydir.dtype == torch.float32 and raydir.is_contiguous()
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
        R = raydir.shape[0]
        nbytes = lib.pnb_query_bytes(R, SR, K, cap_samples)
        if ws is None or ws.numel() < nbytes:
            ws = torch.empty(nbytes, dtype=torch.uint8, device=raydir.device)
        self.ws, self.grid, self.raydir, self.t = ws, grid, raydir, t
        self.desc = _lib.Query()
        hc = (_lib.C.c_int32 * 16)() if want_counters else None
        stride = D if t.dim() == 2 else 0
        stream = torch.cuda.current_stream(raydir.device).cuda_stream
        _lib.check(lib.pnb_query(_lib.C.byref(self.desc), ws.data_ptr(), ws.numel(), _lib.C.byref(grid.desc),
                                 _lib.f3(campos), raydir.data_ptr(), R, t.data_ptr(), stride, D, SR, K,
                                 float(radius_limit), _lib.i3(kernel_size), int(cap_samples), stream, hc), "pnb_query")
        self.counters = {k: int(hc[i]) for k, i in _lib.QC.items()} if want_counters else None
        self.R, self.SR, self.K, self.D = R, SR, K, D

    def counters_tensor(self):
        """The device int32[16] counters (PNB_QC_*) as a tensor view into the query workspace."""
        off = int(self.desc.counters) - self.ws.data_ptr()
        return self.ws[off:off + 64].view(torch.int32)

    def export(self, cam_opts, want_pers=True, want_dirs=True):
        """Dense reference layout (needs counters['R2'] -> the query must have been run with want_counters)."""
        lib = _lib.load()
        dev = self.raydir.device
        R2 = self.counters["R2"]
        ray_row = torch.empty(self.R, dtype=torch.int32, device=dev)
        ray_mask = torch.empty(self.R, dtype=torch.int8, device=dev)
        pidx = torch.empty((max(R2, 1), self.SR, self.K), dtype=torch.int32, device=dev)
        loc_w = torch.empty((max(R2, 1), self.SR, 3), dtype=torch.float32, device=dev)
        loc = torch.empty_like(loc_w) if want_pers else None
        dirs = torch.empty_like(loc_w) if want_dirs else None
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(lib.pnb_query_export(_lib.C.byref(self.desc), _lib.C.byref(cam_opts), ray_row.data_ptr(),
                                        ray_mask.data_ptr(), pidx.data_ptr(), loc_w.data_ptr(),
                                        loc.data_ptr() if loc is not None else None,
                                        dirs.data_ptr() if dirs is not None else None, stream), "pnb_query_export")
        return dict(sample_pidx=pidx[:R2], sample_loc_w=loc_w[:R2], sample_loc=None if loc is None else loc[:R2],
                    sample_ray_dirs=None if dirs is None else dirs[:R2], ray_mask=ray_mask, ray_row=ray_row)


def make_cam_opts(campos, camrotc2w, Rw2c=None, vsize_z=0.0, bg_color=(1., 1., 1.), raydist_mode_unit=1, agg_intrp_order=2):
    o = _lib.ShadeOpts()
    cp = [float(v) for v in torch.as_tensor(campos).reshape(-1).tolist()]
    rot = [float(v) for v in torch.as_tensor(camrotc2w).reshape(-1).tolist()]
    rw = [1., 0., 0., 0., 1., 0., 0., 0., 1.] if Rw2c is None else [float(v) for v in torch.as_tensor(Rw2c).reshape(-1).tolist()]
    bg = [float(v) for v in torch.as_tensor(bg_color).reshape(-1).tolist()]
    for i in range(3):
        o.campos[i] = cp[i]
        o.bg_color[i] = bg[i]
    for i in range(9):
        o.camrotc2w[i] = rot[i]
        o.Rw2c[i] = rw[i]
    o.vsize_z = float(vsize_z)
    o.raydist_mode_unit = int(raydist_mode_unit)
    o.agg_intrp_order = int(agg_intrp_order)
    return o


def grid_hyperparameters(point_xyz_w_tensor, vsize_np, scaled_vsize_np, vscale_np, kernel_size, ranges):
    """The world grid of point_query.py:47-71 (and query_point_indices_worldcoords.py:46-77, the same expressions): the points' box,
    clipped to `ranges` and padded by half a kernel of scaled voxels.  Returns ranges_tensor ([6] on the points' device), scaled_vdim_np
    (int32 [3]) and vdim_np (float64 [3], before the division by vscale)."""
    min_xyz, max_xyz = torch.min(point_xyz_w_tensor, dim=-2)[0][0], torch.max(point_xyz_w_tensor, dim=-2)[0][0]
    if ranges is not None:
        ranges_min = torch.as_tensor(ranges[:3], dtype=torch.float32, device=min_xyz.device)
        ranges_max = torch.as_tensor(ranges[3:], dtype=torch.float32, device=min_xyz.device)
        min_xyz, max_xyz = torch.maximum(min_xyz, ranges_min), torch.minimum(max_xyz, ranges_max)
    pad = torch.as_tensor(scaled_vsize_np * np.asarray(kernel_size) / 2, device=min_xyz.device, dtype=torch.float32)
    min_xyz = min_xyz - pad
    max_xyz = max_xyz + pad
    ranges_tensor = torch.cat([min_xyz, max_xyz], dim=-1)
    vdim_np = (max_xyz - min_xyz).cpu().numpy() / np.asarray(vsize_np, dtype=np.float64)
    scaled_vdim_np = np.ceil(vdim_np / vscale_np).astype(np.int32)
    return ranges_tensor, scaled_vdim_np, vdim_np


class lighting_fast_querier():
    """Drop-in for point_query.py:25-108 (same name on purpose)."""

    def __init__(self, device, opt):
        _lib.load()  # fail loudly at construction when the CUDA library is absent
        self.device = device if isinstance(device, torch.device) else torch.device(device)
        self.gpu = self.device.index
        self.opt = opt
        self.inverse = self.opt.inverse if hasattr(self.opt, "inverse") else 0
        if self.inverse > 0:
            raise NotImplementedError("pnb200: --inverse > 0 (disparity-linear ray generation) is outside the "
                                      "implemented hot path")
        self.count = 0
        self._read_options()
        self.scaled_vsize_tensor = torch.as_tensor(self.scaled_vsize_np, device=self.device)
        self.kernel_size_tensor = torch.as_tensor(self.kernel_size, device=self.device)
        self.query_size_tensor = torch.as_tensor(self.query_size, device=self.device)
        self.parity_slot0 = bool(getattr(self.opt, "pnb_parity_slot0", 1))
        self._grid = None
        self._grid_key = None
        self._grid_storage = None   # weak reference to the storage of the grid's points (same_storage)
        self._hyper = None
        self._ws = None
        self._t_cache = {}
        self.n_builds = 0
        self.last_grid_counters = None
        self.last_query_counters = None
        self.last_query = None

    def _read_options(self):
        """The query options, read here once at construction exactly like the reference (point_query.py:35-42)."""
        if self.opt.K > _lib.MAX_K:
            raise NotImplementedError("pnb200: K=%d > 8; the reference kernel's neighbour buffer is KN=8 "
                                      "(query_worldcoords.cu:14), larger K is undefined there" % self.opt.K)
        if self.opt.SR > _lib.MAX_SR:
            raise NotImplementedError("pnb200: SR=%d > %d" % (self.opt.SR, _lib.MAX_SR))
        self.radius_limit_np = np.asarray(self.opt.radius_limit_scale * max(self.opt.vsize[0], self.opt.vsize[1])).astype(np.float32)
        self.vscale_np = np.array(self.opt.vscale, dtype=np.int32)
        self.scaled_vsize_np = (np.asarray(self.opt.vsize, dtype=np.float64) * self.vscale_np).astype(np.float32)
        self.kernel_size = np.asarray(self.opt.kernel_size, dtype=np.int32)
        self.query_size = np.asarray(self.opt.query_size, dtype=np.int32)

    def clean_up(self):
        self._grid = None
        self._grid_key = None
        self._grid_storage = None
        self._hyper = None
        self._ws = None
        self.last_query = None

    # ------------------------------------------------------------------ point_query.py:47-71
    def get_hyperparameters(self, vsize_np, point_xyz_w_tensor, ranges=None):
        ranges_tensor, scaled_vdim_np, _ = grid_hyperparameters(point_xyz_w_tensor, vsize_np, self.scaled_vsize_np, self.vscale_np,
                                                                self.opt.kernel_size, ranges)
        return ranges_tensor, vsize_np, scaled_vdim_np

    def _grid_for(self, xyz):
        """xyz: [N,3] contiguous fp32 on the device.  Rebuilt only when the point cloud changed: another storage, address, version
        or size."""
        key = (xyz.data_ptr(), xyz._version, xyz.shape[0], tuple(float(v) for v in self.opt.ranges) if self.opt.ranges is not None else None)
        if self._grid is None or key != self._grid_key or not same_storage(self._grid_storage, xyz):
            vsize_np = self.opt.vsize
            ranges_tensor, scaled_vdim_np, _ = grid_hyperparameters(xyz[None], vsize_np, self.scaled_vsize_np, self.vscale_np,
                                                                    self.opt.kernel_size, self.opt.ranges)
            ranges_np = ranges_tensor.cpu().numpy()
            max_o = self.opt.max_o if self.opt.max_o is not None else xyz.shape[0]
            self._grid = VoxelGrid(xyz, ranges_np[:3], self.scaled_vsize_np, scaled_vdim_np, self.query_size, max_o,
                                   self.opt.P, parity_slot0=self.parity_slot0)
            self._grid_key = key
            self._grid_storage = weakref.ref(xyz.untyped_storage())
            self.n_builds += 1
            self._hyper = (ranges_tensor, ranges_np, vsize_np, scaled_vdim_np)
            self.last_grid_counters = self._grid.counters
        return self._grid

    def _t_for(self, near, far, R, device):
        D = int(self.opt.z_depth_dim)
        if getattr(self.opt, "is_train", False):
            return device_t_table_jitter(near, far, D, R, 0.3, device)  # point_query.py:81
        key = (float(near), float(far), D, str(device))
        if key not in self._t_cache:
            self._t_cache[key] = host_t_table(near, far, D).to(device)
        return self._t_cache[key]

    def run_query(self, xyz, raydir, campos, near, far, t=None, want_counters=True, cap_samples=0):
        """Sample-compacted query (the form the fused renderer consumes).  raydir [R,3], campos 3 floats."""
        grid = self._grid_for(xyz)
        R = raydir.shape[0]
        if t is None:
            t = self._t_for(near, far, R, raydir.device)
        q = QueryResult(grid, campos, raydir, t, int(self.opt.z_depth_dim), int(self.opt.SR), int(self.opt.K),
                        float(self.radius_limit_np), self.kernel_size, cap_samples=cap_samples, ws=self._ws,
                        want_counters=want_counters)
        self._ws = q.ws
        self.last_query_counters = q.counters
        self.last_query = q
        return q

    # ------------------------------------------------------------------ point_query.py:74-98
    def query_points(self, pixel_idx_tensor, point_xyz_pers_tensor, point_xyz_w_tensor, actual_numpoints_tensor, h, w,
                     intrinsic, near_depth, far_depth, ray_dirs_tensor, cam_pos_tensor, cam_rot_tensor):
        near_depth, far_depth = np.asarray(near_depth).item(), np.asarray(far_depth).item()
        if point_xyz_w_tensor.shape[0] != 1:
            raise NotImplementedError("pnb200: batch size must be 1 (the reference kernel's B>1 indexing is wrong, "
                                      "query_worldcoords.cu:265-266; every shipped script uses B=1)")
        xyz = point_xyz_w_tensor[0]
        if not xyz.is_contiguous():
            xyz = xyz.contiguous()
        raydir = ray_dirs_tensor[0].contiguous()
        q = self.run_query(xyz, raydir, cam_pos_tensor[0].tolist(), near_depth, far_depth, want_counters=True)
        cam = make_cam_opts(cam_pos_tensor[0], cam_rot_tensor[0])
        ex = q.export(cam)
        ranges_np = self._hyper[1]
        return ex["sample_pidx"][None], ex["sample_loc"][None], ex["sample_loc_w"][None], \
            ex["sample_ray_dirs"][None], ex["ray_mask"][None], self._hyper[2], ranges_np
