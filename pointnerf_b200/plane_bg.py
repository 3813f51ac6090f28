"""The plane background of bgmodel plane on the GPU: drop-ins for mvs_utils.gen_bg_points / get_rayplane_cross and
MvsPointsVolumetricModel.set_bg (models/mvs/mvs_utils.py:380-408, models/mvs_points_volumetric_model.py:272-310).

Same signatures and return values as the reference.  set_bg projects the plane points into every view of img_lst, tests them against
each view's foreground mask, samples the view's image bilinearly (grid_sample, zeros padding, align_corners=True), keeps the samples
that fit the plane colour +- 0.03 and returns the max over the views -- all in csrc/plane_bg.cu, with every fp32 operation in a
documented order (DESIGN.md §5 "Plane background").  Nothing synchronises.

Kept from the reference: only imgs[0:1], w2c[:, 0], intrinsics and HDWD of each img_lst entry are read (c2ws_lst is not: the
reference projects with an identity c2w); the second return value is the fg_masks passed in (None when none was); the foreground
masks have no depth test.

Cached on the model (`self._pnb_plane_bg`, see `reset`), so that create_all_bg's per-frame loop pays for set-up once:
  * the device copies of imgs[0] of every entry, keyed on each tensor object (a weak reference) and its _version;
  * the stacked view matrices, keyed the same way on every w2c and intrinsics tensor and on the HDWD values;
  * the G foreground masks, keyed on the views and on self.neural_points.xyz by its storage (a weak reference), data_ptr, _version
    and size.  A new cloud, or an in-place edit autograd sees, rebuilds them; a write through `.data` does not: call
    `plane_bg.reset(model)` after one.
"""
import weakref

import torch

from . import lib as _lib
from .point_query import same_storage


def _check(t, name):
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s must be a torch.Tensor (got %s)" % (name, type(t).__name__))
    return t


def get_rayplane_cross(cam_pos, raydir, p_co, p_no, epsilon=1e-3):
    """cam_pos [1,3], raydir [1,R,3], p_co / p_no [1,1,3] (CUDA float32) -> intersections [1,R,3]; (0, 0, 0) where n . d < 0.001."""
    for t, name in ((cam_pos, "cam_pos"), (raydir, "raydir"), (p_co, "p_co"), (p_no, "p_no")):
        _check(t, name)
        if t.dtype != torch.float32 or not t.is_cuda:
            raise ValueError("%s must be a float32 CUDA tensor (got %s on %s)" % (name, t.dtype, t.device))
    if epsilon != 1e-3:
        raise NotImplementedError("get_rayplane_cross: epsilon=%r (the kernel tests n . d >= 0.001f, the reference's default)" % (epsilon,))
    if raydir.dim() != 3 or raydir.shape[0] != 1 or raydir.shape[2] != 3:
        raise ValueError("raydir must be [1,R,3] (got %s): the plane background takes one camera per call" % (tuple(raydir.shape),))
    if cam_pos.numel() != 3 or p_co.numel() != 3 or p_no.numel() != 3:
        raise ValueError("cam_pos, p_co and p_no must hold 3 values each (got %d, %d, %d)" % (cam_pos.numel(), p_co.numel(), p_no.numel()))
    dev = raydir.device
    R = int(raydir.shape[1])
    out = torch.empty((1, R, 3), dtype=torch.float32, device=dev)
    d = raydir.contiguous()
    c, p, n = (t.to(dev).reshape(3).contiguous() for t in (cam_pos, p_co, p_no))
    _lib.check(_lib.load().pnb_plane_cross(c.data_ptr(), d.data_ptr(), p.data_ptr(), n.data_ptr(), R, out.data_ptr(),
                                           torch.cuda.current_stream(dev).cuda_stream), "pnb_plane_cross")
    return out


def gen_bg_points(batch):
    """mvs_utils.gen_bg_points: the plane of batch["plane_pnt"][0], batch["plane_normal"][0] against batch["campos"] [1,3] and
    batch["raydir"] [1,R,3] -> [1,R,3]."""
    dev = batch["campos"].device
    plane_pnt = torch.as_tensor(batch["plane_pnt"][0], dtype=torch.float32, device=dev)
    plane_normal = torch.as_tensor(batch["plane_normal"][0], dtype=torch.float32, device=dev)
    return get_rayplane_cross(batch["campos"], batch["raydir"], plane_pnt[None, None, :], plane_normal[None, None, :])


class _Cache:
    """What set_bg reuses from frame to frame (see the module docstring)."""

    def __init__(self):
        self.n_image_builds = 0
        self.n_view_builds = 0
        self.n_mask_builds = 0
        self.img_src = None      # [(weak reference, _version)] of every imgs tensor
        self.img = None          # [G,3,H,W] float32 on the device
        self.view_src = None     # [(w2c weak ref, _version, intrinsics weak ref, _version, HD, WD)]
        self.views = None        # (w2c [G,4,4], K [G,3,3], hdwd int32 [G,2], mask_off int64 [G], total mask bytes)
        self.mask_key = None
        self.mask_storage = None
        self.masks = None        # int8, view g's [HD,WD] at mask_off[g]


def reset(model):
    """Forget everything set_bg cached on `model` (after a write through `.data` to its points, views or images)."""
    model._pnb_plane_bg = _Cache()


def _same(src, tensors):
    return src is not None and len(src) == len(tensors) and all(r() is t and v == t._version for (r, v), t in zip(src, tensors))


def _images(cache, img_lst, dev):
    imgs = [_check(t, "img_lst entry") for t in img_lst]
    if _same(cache.img_src, imgs) and cache.img.device == dev:
        return cache.img
    for t in imgs:
        if t.dtype != torch.float32:
            raise ValueError("set_bg: the views' images must be float32 (got %s)" % t.dtype)
        if t.dim() != 4 or t.shape[1] != 3:
            raise ValueError("set_bg: every img_lst entry must be [V,3,H,W] (got %s)" % (tuple(t.shape),))
        if tuple(t.shape[2:]) != tuple(imgs[0].shape[2:]):
            raise ValueError("set_bg: the views' images must share one size (got %s and %s)" % (tuple(t.shape[2:]), tuple(imgs[0].shape[2:])))
    cache.img = torch.stack([t[0].to(dev) for t in imgs]).contiguous()
    cache.img_src = [(weakref.ref(t), t._version) for t in imgs]
    cache.n_image_builds += 1
    return cache.img


def _views(cache, w2cs_lst, intrinsics_all, HDWD_lst, dev):
    w2cs = [_check(t, "w2cs_lst entry") for t in w2cs_lst]
    Ks = [_check(t, "intrinsics_all entry") for t in intrinsics_all]
    hdwd = [(int(h[0]), int(h[1])) for h in HDWD_lst]
    if not (len(w2cs) == len(Ks) == len(hdwd)):
        raise ValueError("set_bg: %d w2c, %d intrinsics and %d HDWD entries" % (len(w2cs), len(Ks), len(hdwd)))
    src = [(weakref.ref(w), w._version, weakref.ref(k), k._version, h) for w, k, h in zip(w2cs, Ks, hdwd)]
    if cache.view_src is not None and len(cache.view_src) == len(src) and cache.views[0].device == dev and all(
            a[0]() is w and a[1] == w._version and a[2]() is k and a[3] == k._version and a[4] == h
            for a, w, k, h in zip(cache.view_src, w2cs, Ks, hdwd)):
        return cache.views
    for t in w2cs + Ks:
        if t.dtype != torch.float32:
            raise ValueError("set_bg: w2c and intrinsics must be float32 (got %s)" % t.dtype)
    for HD, WD in hdwd:
        if HD < 2 or WD < 2:
            raise ValueError("set_bg: HDWD must be at least 2 x 2 (got %d x %d)" % (HD, WD))
    w2c = torch.stack([w[:, 0].reshape(4, 4) for w in w2cs]).to(dev).contiguous()
    K = torch.stack([k.reshape(3, 3) for k in Ks]).to(dev).contiguous()
    sizes = [HD * WD for HD, WD in hdwd]
    off = [0]
    for s in sizes[:-1]:
        off.append(off[-1] + s)
    cache.views = (w2c, K, torch.tensor(hdwd, dtype=torch.int32, device=dev), torch.tensor(off, dtype=torch.int64, device=dev),
                   sum(sizes))
    cache.view_src = src
    cache.mask_key = None
    cache.n_view_builds += 1
    return cache.views


def _masks(cache, xyz, views, dev):
    key = (xyz.data_ptr(), xyz._version, tuple(xyz.shape))
    if key == cache.mask_key and same_storage(cache.mask_storage, xyz):
        return cache.masks
    if xyz.dim() != 2 or xyz.shape[1] != 3 or xyz.dtype != torch.float32 or xyz.device != dev:
        raise ValueError("set_bg: neural_points.xyz must be float32 [N,3] on %s (got %s %s on %s)" % (dev, tuple(xyz.shape), xyz.dtype,
                                                                                                     xyz.device))
    w2c, K, hdwd, off, total = views
    pts = xyz.detach().contiguous()
    masks = torch.empty(total, dtype=torch.int8, device=dev)
    _lib.check(_lib.load().pnb_plane_fg_masks(pts.data_ptr(), int(pts.shape[0]), int(w2c.shape[0]), w2c.data_ptr(), K.data_ptr(),
                                              hdwd.data_ptr(), off.data_ptr(), masks.data_ptr(), total,
                                              torch.cuda.current_stream(dev).cuda_stream), "pnb_plane_fg_masks")
    cache.masks, cache.mask_key, cache.mask_storage = masks, key, weakref.ref(xyz.untyped_storage())
    cache.n_mask_builds += 1
    return masks


def _given_masks(fg_masks, hdwd_lst, dev):
    """A caller's fg_masks, indexed as the reference indexes it (fg_masks[:, count, ...]), as the kernel's int8 (1 where not < 1)."""
    out = []
    for g, (HD, WD) in enumerate(hdwd_lst):
        m = fg_masks[:, g, ...]
        if tuple(m.shape) != (HD, WD):
            raise ValueError("set_bg: fg_masks[:, %d] is %s, the view's HDWD %s" % (g, tuple(m.shape), (HD, WD)))
        out.append((~(m.to(dev) < 1)).to(torch.int8).reshape(-1))
    return torch.cat(out)


def set_bg(self, xyz_world_sect_plane, img_lst, c2ws_lst, w2cs_lst, intrinsics_all, HDWD_lst, plane_color, fg_masks=None, **kwargs):
    """MvsPointsVolumetricModel.set_bg: (bg_ray [1,R,3], fg_masks as passed)."""
    pts = _check(xyz_world_sect_plane, "xyz_world_sect_plane")
    if pts.dim() != 3 or pts.shape[0] != 1 or pts.shape[2] != 3:
        raise ValueError("set_bg: xyz_world_sect_plane must be [1,R,3] (got %s)" % (tuple(pts.shape),))
    if pts.dtype != torch.float32 or not pts.is_cuda:
        raise ValueError("set_bg: xyz_world_sect_plane must be a float32 CUDA tensor (got %s on %s)" % (pts.dtype, pts.device))
    pc = _check(plane_color, "plane_color")
    if pc.dtype != torch.float32 or pc.numel() != 3:
        raise ValueError("set_bg: plane_color must be a float32 tensor of 3 values (got %s, %d values)" % (pc.dtype, pc.numel()))
    if len(img_lst) == 0:
        raise ValueError("set_bg: img_lst is empty")
    dev = pts.device
    cache = getattr(self, "_pnb_plane_bg", None)
    if cache is None:
        reset(self)
        cache = self._pnb_plane_bg
    img = _images(cache, img_lst, dev)
    views = _views(cache, w2cs_lst, intrinsics_all, HDWD_lst, dev)
    w2c, K, hdwd, off, _ = views
    G = int(w2c.shape[0])
    if G != img.shape[0]:
        raise ValueError("set_bg: %d images for %d views" % (img.shape[0], G))
    if fg_masks is None:
        masks = _masks(cache, self.neural_points.xyz, views, dev)
    else:
        masks = _given_masks(fg_masks, [(int(h[0]), int(h[1])) for h in HDWD_lst], dev)
    R = int(pts.shape[1])
    out = torch.empty((1, R, 3), dtype=torch.float32, device=dev)
    p = pts.contiguous()
    c = pc.to(dev).reshape(3).contiguous()
    _lib.check(_lib.load().pnb_plane_bg(p.data_ptr(), R, G, w2c.data_ptr(), K.data_ptr(), hdwd.data_ptr(), off.data_ptr(), masks.data_ptr(),
                                        img.data_ptr(), int(img.shape[2]), int(img.shape[3]), c.data_ptr(), out.data_ptr(),
                                        torch.cuda.current_stream(dev).cuda_stream), "pnb_plane_bg")
    return out, fg_masks
