"""Drop-in for the reference's pycuda world-coordinate querier (wcoord_query 1), models/neural_points/query_point_indices_worldcoords.py:29-712,
on top of libpnb200.so (pnb_grid_build / pnb_query / pnb_query_export, the kernels of the wcoord_query -1 querier).

Same constructor (`lighting_fast_querier(device, opt)`), `get_hyperparameters(vsize_np, point_xyz_w_tensor, ranges=None)` (the
reference's 14-tuple), `query_points(...)` (12 arguments, 7-tuple), `w2pers` and `clean_up`, so that

    sys.modules["models.neural_points.query_point_indices_worldcoords"] = pointnerf_b200.query_point_indices_worldcoords

makes the reference's NeuralPoints use it unchanged, without pycuda (INTEGRATION.md).

The kernels of the two world-coordinate flavours are the same math (query_point_indices_worldcoords.py:237-522 and
cuda/query_worldcoords.cu, including the slot-0 condition of fill_occ2pnts, :366 vs :147), so this class is the wcoord_query -1 drop-in
(pointnerf_b200.point_query) with the one host difference of flavour 1: the -1 querier reads vsize, vscale, kernel_size, query_size and
radius_limit_scale once, in its constructor (point_query.py:33-42), while flavour 1 reads them from the shared `opt` on every call
(:47-95).  Training runs rely on that: probe_hole (run/train_ft.py:425-429, :517) sets `opt.query_size` to the probe tier and does not
restore it, so every later query of the run uses the tier's query size.  Here every call reads those options (and ranges, SR, K, P,
max_o, z_depth_dim and is_train, which the -1 drop-in already reads per call) and the voxel grid is cached on everything its build
depends on: the points (storage and version), ranges, vsize, vscale and kernel_size (which fix the grid's box and dimensions),
query_size, max_o and P.  A changed option rebuilds the grid once; a chunk loop over one view with unchanged options builds it once.

In the 14-tuple the reference's pycuda gpuarrays are device tensors with the same values (only its own query_points reads them).
depth_limit is computed and returned, and, as in the reference, no kernel reads it.  Refused (NotImplementedError) as by the -1 drop-in:
inverse > 0, K > 8, SR > 128, B > 1; and NN <= 0, for which the reference's kernel module has no query function
(query_rand_along_ray, :530).
"""
import numpy as np
import torch

from . import point_query as _wq


class lighting_fast_querier(_wq.lighting_fast_querier):
    """Drop-in for query_point_indices_worldcoords.py:29 (same name on purpose)."""

    def __init__(self, device, opt):
        if int(opt.NN) <= 0:
            raise NotImplementedError("pnb200: world-coordinate query with NN=%r (the reference's flavour 1 has no kernel for NN <= 0)"
                                      % opt.NN)
        super().__init__(device, opt)
        # the -1 querier's device copies of its constructor-time options: this flavour has none (get_hyperparameters returns them)
        del self.scaled_vsize_tensor, self.kernel_size_tensor, self.query_size_tensor
        self._options_key = None

    def _read_options(self):
        """The query options from the shared opt, on every call (query_point_indices_worldcoords.py:47-95)."""
        if getattr(self.opt, "inverse", 0) > 0:
            raise NotImplementedError("pnb200: --inverse > 0 (disparity-linear ray generation) is outside the implemented hot path")
        super()._read_options()

    # ------------------------------------------------------------------ query_point_indices_worldcoords.py:46-77
    def get_hyperparameters(self, vsize_np, point_xyz_w_tensor, ranges=None):
        self._read_options()
        vscale_np = self.vscale_np
        scaled_vsize_np = (np.asarray(vsize_np, dtype=np.float64) * vscale_np).astype(np.float32)
        ranges_tensor, scaled_vdim_np, vdim_np = _wq.grid_hyperparameters(point_xyz_w_tensor, vsize_np, scaled_vsize_np, vscale_np,
                                                                          self.opt.kernel_size, ranges)
        ranges_np = ranges_tensor.cpu().numpy().astype(np.float32)
        radius_limit_np = np.asarray(self.opt.radius_limit_scale * max(vsize_np[0], vsize_np[1])).astype(np.float32)
        depth_limit_np = np.asarray(self.opt.depth_limit_scale * vsize_np[2]).astype(np.float32)
        ranges_gpu = ranges_tensor
        scaled_vsize_gpu, scaled_vdim_gpu, vscale_gpu, kernel_size_gpu, query_size_gpu = (
            torch.as_tensor(a, device=ranges_tensor.device) for a in (scaled_vsize_np, scaled_vdim_np, vscale_np, self.kernel_size,
                                                                      self.query_size))
        return radius_limit_np, depth_limit_np, ranges_np, vsize_np, vdim_np, scaled_vsize_np, scaled_vdim_np, vscale_np, ranges_gpu, \
            scaled_vsize_gpu, scaled_vdim_gpu, vscale_gpu, kernel_size_gpu, query_size_gpu

    def _grid_for(self, xyz):
        """The -1 querier's grid, also rebuilt when an option the build depends on changed since it was built."""
        key = (tuple(float(v) for v in self.opt.vsize), tuple(self.vscale_np.tolist()), tuple(self.kernel_size.tolist()),
               tuple(self.query_size.tolist()), self.opt.max_o, int(self.opt.P))
        if key != self._options_key:
            self._grid = None
            self._options_key = key
        return super()._grid_for(xyz)

    def run_query(self, xyz, raydir, campos, near, far, t=None, want_counters=True, cap_samples=0):
        """The -1 querier's run_query (the fused module's entry point, and the one query_points goes through) on the options of now."""
        self._read_options()
        return super().run_query(xyz, raydir, campos, near, far, t=t, want_counters=want_counters, cap_samples=cap_samples)

    # ------------------------------------------------------------------ query_point_indices_worldcoords.py:96-103 (the reference's expression)
    def w2pers(self, point_xyz_w, camrotc2w, campos):
        xyz_w_shift = point_xyz_w - campos[:, None, :]
        xyz_c = torch.sum(xyz_w_shift[..., None, :] * torch.transpose(camrotc2w, 1, 2)[:, None, None, ...], dim=-1)
        z_pers = xyz_c[..., 2]
        x_pers = xyz_c[..., 0] / xyz_c[..., 2]
        y_pers = xyz_c[..., 1] / xyz_c[..., 2]
        return torch.stack([x_pers, y_pers, z_pers], dim=-1)
