"""Drop-in for the reference's perspective-frustum querier (wcoord_query 0), models/neural_points/query_point_indices.py:32-127, on top
of libpnb200.so (pnb_frustum_*).

Same constructor (`lighting_fast_querier(device, opt)`), `get_hyperparameters`, `query_points` (12 arguments, 7-tuple), `pers2w`,
`uniform`, `gaussian` and `clean_up`, so that

    sys.modules["models.neural_points.query_point_indices"] = pointnerf_b200.query_point_indices

makes the reference's NeuralPoints use it unchanged (INTEGRATION.md).  Differences, all deliberate (DESIGN.md §5 F1-F9):
  * deterministic: points in ascending index, the first P per voxel; overflow of P and of the per-column numbering is reported
    (`last_build_counters`) instead of resolved by wall-clock-seeded curand or int8 wrap-around;
  * the build is cached per (points, camera, h, w, intrinsic, near, far, options), so the chunk loop over one view builds it once.
    The camera is compared by value; a call on a cached view synchronises once (for R').  The points are identified by the storage
    object (a weak reference, point_query.same_storage), the address and the autograd version of `point_xyz_w_tensor` (NeuralPoints
    passes `self.xyz[None]`): in-place updates through autograd-visible ops, a new `self.xyz` Parameter and a new cloud from a
    feed-forward network (also one the caching allocator placed where the freed previous cloud was) rebuild, but a write through
    `.data` does not bump the version.  After such an edit, call `clean_up()`;
  * only NN 2, inverse 0, B 1, K <= 8 and SR <= 128 (the DTU scripts' configuration) are implemented: anything else raises;
  * no pycuda and no CPU path: the CUDA library must be present, otherwise lib.load() raises.
The jitter (`uniform`, `gaussian`) and `pers2w` are the reference's own torch expressions, so they round the same way.

`run_fused` is the entry point of the fused module (pointnerf_b200.ray_marching with wcoord_query 0): the same query and tuple, handed
to the shading kernels in the sample-compacted layout of pnb_frustum_samples.  Its one host synchronisation is the one that sizes R'.
"""
import weakref

import numpy as np
import torch

from . import lib as _lib
from .point_query import same_storage


def hyperparameters(opt, h, w, intrinsic, near_depth, far_depth):
    """The grid of query_point_indices.py:57-70 with the reference's numpy expressions (inverse 0): radius_limit, depth_limit,
    ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale."""
    x_rl, x_rh = -intrinsic[0, 2] / intrinsic[0, 0], (w - intrinsic[0, 2]) / intrinsic[0, 0]
    y_rl, y_rh = -intrinsic[1, 2] / intrinsic[1, 1], (h - intrinsic[1, 2]) / intrinsic[1, 1],
    z_r = far_depth - near_depth
    ranges = np.array([x_rl, y_rl, near_depth, x_rh, y_rh, far_depth], dtype=np.float32)
    vdim = np.array([w, h, opt.z_depth_dim], dtype=np.int32)
    vsize = np.array([(x_rh - x_rl) / vdim[0], (y_rh - y_rl) / vdim[1], z_r / vdim[2]], dtype=np.float32)
    vscale = np.array(opt.vscale, dtype=np.int32)
    scaled_vdim = np.ceil(vdim / vscale).astype(np.int32)
    scaled_vsize = (vsize * vscale).astype(np.float32)
    radius_limit, depth_limit = opt.radius_limit_scale * max(vsize[0], vsize[1]), opt.depth_limit_scale * vsize[2]
    return np.float32(radius_limit), np.float32(depth_limit), ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale


def w2pers(point_xyz, camrotc2w, campos):
    """NeuralPoints.w2pers (neural_points.py:604-610), the reference's expression: perspective coordinates (x/z, y/z, z) of [N,3] world
    points for camera [1,3,3] / [1,3]."""
    point_xyz_shift = point_xyz[None, ...] - campos[:, None, :]
    xyz = torch.sum(camrotc2w[:, None, :, :] * point_xyz_shift[:, :, :, None], dim=-2)
    xper = xyz[:, :, 0] / xyz[:, :, 2]
    yper = xyz[:, :, 1] / xyz[:, :, 2]
    return torch.stack([xper, yper, xyz[:, :, 2]], dim=-1)


class FrustumSamples:
    """One frustum query in the sample-compacted layout (pnb_query_t) the fused renderer reads: every slot of a hit ray is a
    candidate sample, its geometry read in place from the querier's tuple, which this object keeps alive."""

    def __init__(self, desc, ws, R, R2, SR, K, tup):
        self.desc, self.ws, self.R, self.R2, self.SR, self.K = desc, ws, R, R2, SR, K
        self.sample_pidx, self.sample_loc, self.sample_loc_w, self.sample_ray_dirs, self.ray_mask, self.vsize, self.ranges = tup
        self._counters = None

    def counters_tensor(self):
        """The device int32[16] counters (PNB_QC_*) as a tensor view into the workspace."""
        off = int(self.desc.counters) - self.ws.data_ptr()
        return self.ws[off:off + 64].view(torch.int32)

    @property
    def counters(self):
        """The counters on the host (PNB_QC_* names); the first access synchronises the stream."""
        if self._counters is None:
            h = self.counters_tensor().cpu()
            self._counters = {k: int(h[i]) for k, i in _lib.QC.items()}
        return self._counters


class lighting_fast_querier():
    """Drop-in for query_point_indices.py:32 (same name on purpose)."""

    def __init__(self, device, opt):
        self.opt = opt
        self.inverse = self.opt.inverse
        if int(self.opt.NN) != 2:
            raise NotImplementedError("pnb200: frustum query with NN=%r (only NN 2, the DTU scripts' value, is implemented)" % self.opt.NN)
        if self.inverse > 0:
            raise NotImplementedError("pnb200: frustum query with inverse > 0 (disparity grid) is not implemented")
        if self.opt.K > _lib.MAX_K:
            raise NotImplementedError("pnb200: K=%d > %d" % (self.opt.K, _lib.MAX_K))
        if self.opt.SR > _lib.MAX_SR:
            raise NotImplementedError("pnb200: SR=%d > %d" % (self.opt.SR, _lib.MAX_SR))
        _lib.load()  # fail loudly at construction when the CUDA library is absent
        self.device = device if isinstance(device, torch.device) else torch.device(device)
        self.gpu = self.device.index
        self.n_builds = 0
        self.last_build_counters = None
        self.last_query_counters = None
        self.last_pixel_idx_cur = None
        self._key = None
        self._storage = None     # weak reference to the storage of the build's points (same_storage)
        self._fr = None
        self._buf = None
        self._ws = None
        self._host = None

    def clean_up(self):
        self._key = self._storage = self._fr = self._buf = self._ws = None

    # ------------------------------------------------------------------ query_point_indices.py:50-73
    def get_hyperparameters(self, h, w, intrinsic, near_depth, far_depth):
        radius_limit, depth_limit, ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale = \
            hyperparameters(self.opt, h, w, intrinsic, near_depth, far_depth)
        # the reference returns pycuda gpuarrays here; these are device tensors with the same values
        range_gpu, scaled_vsize_gpu, scaled_vdim_gpu, vscale_gpu, kernel_size_gpu, query_size_gpu = (
            torch.as_tensor(np.asarray(a), device=self.device) for a in (ranges, scaled_vsize, scaled_vdim, vscale,
                                                                         np.asarray(self.opt.kernel_size, dtype=np.int32),
                                                                         np.asarray(self.opt.query_size, dtype=np.int32)))
        return radius_limit, depth_limit, ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale, range_gpu, scaled_vsize_gpu, \
            scaled_vdim_gpu, vscale_gpu, kernel_size_gpu, query_size_gpu

    def _build(self, pers, n, key, storage, ranges, scaled_vsize, scaled_vdim, vscale):
        """The frustum build of this view (synchronises once, for its counters)."""
        lib = _lib.load()
        pts = pers[0, :n].to(torch.float32).contiguous()
        dim = _lib.i3(scaled_vdim)
        nbytes = lib.pnb_frustum_bytes(n, dim, int(self.opt.SR))
        self._fr = self._key = None
        self._buf = torch.empty(nbytes, dtype=torch.uint8, device=pts.device)
        fr = _lib.Frustum()
        hc = (_lib.C.c_int32 * 16)()
        stream = torch.cuda.current_stream(pts.device).cuda_stream
        _lib.check(lib.pnb_frustum_build(_lib.C.byref(fr), self._buf.data_ptr(), nbytes, pts.data_ptr(), n, int(pers.shape[0]),
                                         _lib.f3(ranges[:3]), _lib.f3(scaled_vsize), dim, _lib.i3(vscale), _lib.i3(self.opt.kernel_size),
                                         _lib.i3(self.opt.query_size), int(self.opt.SR), int(self.opt.K), int(self.opt.P),
                                         int(self.opt.max_o) if self.opt.max_o is not None else 0, int(self.opt.NN), int(self.inverse),
                                         stream, hc), "pnb_frustum_build")
        self.last_build_counters = {k: int(hc[i]) for k, i in _lib.FB.items()}
        self._fr, self._key, self._storage = fr, key, weakref.ref(storage)
        self.n_builds += 1

    def _mask(self, pix, dev):
        """Ray mask + compaction scan of the current build; synchronises once, for R'."""
        lib = _lib.load()
        R = pix.shape[0]
        qbytes = lib.pnb_frustum_query_bytes(R)
        if self._ws is None or self._ws.numel() < qbytes:
            self._ws = torch.empty(qbytes, dtype=torch.uint8, device=dev)
        ray_mask = torch.empty(R, dtype=torch.int8, device=dev)
        hc = (_lib.C.c_int32 * 16)()
        _lib.check(lib.pnb_frustum_query(_lib.C.byref(self._fr), pix.data_ptr(), R, self._ws.data_ptr(), self._ws.numel(),
                                         ray_mask.data_ptr(), torch.cuda.current_stream(dev).cuda_stream, hc), "pnb_frustum_query")
        self.last_query_counters = {k: int(hc[i]) for k, i in _lib.FQ.items()}
        return ray_mask

    # ------------------------------------------------------------------ query_point_indices.py:76-100
    def query_points(self, pixel_idx_tensor, point_xyz_pers_tensor, point_xyz_w_tensor, actual_numpoints_tensor, h, w, intrinsic,
                     near_depth, far_depth, ray_dirs_tensor, cam_pos_tensor, cam_rot_tensor):
        radius_limit, depth_limit, ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale = \
            self.get_hyperparameters(h, w, intrinsic, near_depth, far_depth)[:8]
        self.radius_limit, self.depth_limit, self.ranges, self.vsize, self.vdim, self.scaled_vsize, self.scaled_vdim, self.vscale = \
            radius_limit, depth_limit, ranges, vsize, vdim, scaled_vsize, scaled_vdim, vscale
        B = point_xyz_pers_tensor.shape[0]
        if B != 1:
            raise NotImplementedError("pnb200: frustum query with batch size %d (only 1 is implemented)" % B)
        lib = _lib.load()
        dev = point_xyz_pers_tensor.device
        # The build depends on the points (identified by storage, address and version, see the module docstring), the camera, the grid
        # and the options.  The camera and the caller's point count live on the device: they are copied to pinned memory behind the work of
        # this call and compared after the synchronisation that sizes R', so a call whose view is cached synchronises once.
        static = (point_xyz_w_tensor.data_ptr(), point_xyz_w_tensor._version, tuple(point_xyz_w_tensor.shape), int(h), int(w),
                  np.asarray(intrinsic).tobytes(), float(near_depth), float(far_depth), tuple(self.opt.vscale),
                  tuple(self.opt.kernel_size), tuple(self.opt.query_size), int(self.opt.SR), int(self.opt.K), int(self.opt.P),
                  self.opt.max_o, int(self.opt.z_depth_dim))
        vals = torch.cat([cam_rot_tensor.reshape(-1).double(), cam_pos_tensor.reshape(-1).double(),
                          torch.as_tensor(actual_numpoints_tensor).reshape(-1)[:1].to(cam_rot_tensor.device).double()])
        if self._host is None or self._host.numel() != vals.numel():
            self._host = torch.empty(vals.numel(), dtype=torch.float64, pin_memory=True)
        self._host.copy_(vals, non_blocking=True)
        pix = pixel_idx_tensor.reshape(B, -1, 2)[0].to(torch.int32).contiguous()

        def build():
            v = self._host.tolist()
            self._build(point_xyz_pers_tensor, int(v[-1]), (static, tuple(v)), point_xyz_w_tensor.untyped_storage(), ranges,
                        scaled_vsize, scaled_vdim, vscale)

        if self._fr is None or self._key[0] != static or not same_storage(self._storage, point_xyz_w_tensor):
            torch.cuda.current_stream(dev).synchronize()       # a new view: the build needs the point count now
            build()
        ray_mask = self._mask(pix, dev)
        if self._key[1] != tuple(self._host.tolist()):         # same points and grid, another camera or point count: rebuild
            build()
            ray_mask = self._mask(pix, dev)

        R = pix.shape[0]
        R2 = self.last_query_counters["R2"]
        SR, K = int(self.opt.SR), int(self.opt.K)
        pixel_idx_cur = torch.empty((R2, 2), dtype=torch.int32, device=dev)
        sample_pidx_tensor = torch.empty((B, R2, SR, K), dtype=torch.int32, device=dev)
        sample_loc_tensor = torch.empty((B, R2, SR, 3), dtype=torch.float32, device=dev)
        _lib.check(lib.pnb_frustum_export(_lib.C.byref(self._fr), pix.data_ptr(), R, self._ws.data_ptr(), self._ws.numel(),
                                          ray_mask.data_ptr(), R2, float(np.float32(radius_limit ** 2)), float(np.float32(depth_limit ** 2)),
                                          pixel_idx_cur.data_ptr(), sample_pidx_tensor.data_ptr(), sample_loc_tensor.data_ptr(),
                                          torch.cuda.current_stream(dev).cuda_stream), "pnb_frustum_export")
        self.last_pixel_idx_cur = pixel_idx_cur[None]

        if self.opt.is_train:
            sample_loc_tensor = getattr(self, self.opt.shpnt_jitter, None)(sample_loc_tensor, vsize)
        sample_loc_w_tensor, sample_ray_dirs_tensor = self.pers2w(sample_loc_tensor, cam_rot_tensor, cam_pos_tensor)
        return sample_pidx_tensor, sample_loc_tensor, sample_loc_w_tensor, sample_ray_dirs_tensor, ray_mask[None], vsize, ranges

    # ------------------------------------------------------------------ the fused module's entry point
    def run_fused(self, xyz, campos, camrotc2w, pixel_idx, h, w, intrinsic, near, far):
        """The query of forward() / render_full() with wcoord_query 0: the points' perspective coordinates (w2pers), query_points (one
        host synchronisation for R'; the build is cached per view; jitter with opt.is_train, drawn as the reference draws it), then
        pnb_frustum_samples.  xyz [N,3]; campos [1,3] and camrotc2w [1,3,3] device tensors; pixel_idx [.., 2]; h, w, intrinsic [3,3],
        near, far as NeuralPoints.forward passes them to the querier.  Returns a FrustumSamples."""
        lib = _lib.load()
        dev = xyz.device
        pers = w2pers(xyz, camrotc2w, campos)
        pix = pixel_idx.reshape(1, -1, 2).to(torch.int32)
        tup = self.query_points(pix, pers, xyz[None], torch.tensor([xyz.shape[0]], dtype=torch.int32), h, w, intrinsic, near, far,
                                None, campos, camrotc2w)
        pidx, loc, loc_w, dirs, mask = (t[0].contiguous() for t in tup[:5])
        R, R2 = pix.shape[1], int(pidx.shape[0])
        SR, K = int(self.opt.SR), int(self.opt.K)
        nb = lib.pnb_frustum_samples_bytes(R, R2, SR)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)    # per call: a training step's backward still reads the previous one
        desc = _lib.Query()
        _lib.check(lib.pnb_frustum_samples(_lib.C.byref(desc), ws.data_ptr(), ws.numel(), mask.data_ptr(), R, R2, SR, K,
                                           pidx.data_ptr(), loc_w.data_ptr(), loc.data_ptr(), dirs.data_ptr(),
                                           torch.cuda.current_stream(dev).cuda_stream), "pnb_frustum_samples")
        return FrustumSamples(desc, ws, R, R2, SR, K, (pidx, loc, loc_w, dirs, mask, tup[5], tup[6]))

    # ------------------------------------------------------------------ query_point_indices.py:102-126 (the reference's expressions)
    def pers2w(self, point_xyz_pers, camrotc2w, campos):
        x_pers = point_xyz_pers[..., 0] * point_xyz_pers[..., 2]
        y_pers = point_xyz_pers[..., 1] * point_xyz_pers[..., 2]
        z_pers = point_xyz_pers[..., 2]
        xyz_c = torch.stack([x_pers, y_pers, z_pers], dim=-1)
        xyz_w_shift = torch.sum(xyz_c[..., None, :] * camrotc2w, dim=-1)
        ray_dirs = xyz_w_shift / (torch.linalg.norm(xyz_w_shift, dim=-1, keepdims=True) + 1e-7)
        xyz_w = xyz_w_shift + campos[:, None, :]
        return xyz_w, ray_dirs

    def gaussian(self, input, vsize):
        B, R, SR, _ = input.shape
        jitters = torch.normal(mean=torch.zeros([B, R, SR], dtype=torch.float32, device=input.device),
                               std=torch.full([B, R, SR], vsize[2] / 4, dtype=torch.float32, device=input.device))
        input[..., 2] = input[..., 2] + torch.clamp(jitters, min=-vsize[2] / 2, max=vsize[2] / 2)
        return input

    def uniform(self, input, vsize):
        B, R, SR, _ = input.shape
        jitters = torch.rand([B, R, SR], dtype=torch.float32, device=input.device) - 0.5
        input[..., 2] = input[..., 2] + jitters * vsize[2]
        return input
