"""The initial point cloud's depth filter and visual-hull mask on the GPU: drop-ins for filter_utils.filter_by_masks_gpu and
mvs_utils.alpha_masking (models/mvs/filter_utils.py:157-291, models/mvs/mvs_utils.py:573-607), the two geometric steps of
gen_points_filter_embeddings between MVSNet and voxelization.

Same signatures and return values as the reference.  filter_by_masks_gpu tests every pixel of every ref view against every other view
(reproject, sample the source depth bilinearly with border padding, reproject back: |dp| < 1 px and |dd| / d < 0.01), averages the
matched depths, keeps the pixels that pass the confidence, mask and geo_cnsst_num tests and the inclusive range mask on their world
point, in row-major pixel order per view -- all in csrc/depth_filter.cu, with every fp32 operation in a documented order (DESIGN.md §5
"Depth filter and visual hull").  With device inputs a call makes one device-to-host copy of the view matrices and one synchronisation
to size its outputs (filter_by_masks_gpu's docstring has the cpu2gpu case).  alpha_masking returns the bool [N] visual-hull mask with no
per-view temporaries; on device points it does not synchronise, and host points get a host mask.

Kept from the reference: xyz_cam holds the input's raw camera x, y beside the averaged depth; with one view there is no geometric test.
The per-view `visible_*` sums, which the reference computes and never reads, are not computed.

Refused (NotImplementedError, no shipped script sets them): manual_depth_view > 1, default_conf > 1 (reassign_conf) and far_plane_shift.
"""
import numpy as np
import torch

from . import lib as _lib

HOST_CHUNK = 1 << 24     # host points alpha_masking stages on the device at a time (192 MiB of coordinates)


def _t(x):
    return x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))


def view_matrices(intrinsics, extrinsics):
    """K [V,3,3], Kinv [V,3,3], c2w [V,3,4] and pair [V,V,3,4] (pair (r, s) = rows 0..2 of E_s inv(E_r)) as float32 numpy arrays, from
    the fp32 intrinsics [V,3,3] and extrinsics [V,4,4]: formed in float64 (numpy.linalg.inv) and rounded once."""
    K = np.asarray(intrinsics, np.float32).astype(np.float64)
    E = np.asarray(extrinsics, np.float32).astype(np.float64)
    Einv = np.linalg.inv(E)
    pair = np.einsum("sij,rjk->rsik", E[:, :3], Einv)
    f = np.float32
    return K.astype(f), np.linalg.inv(K).astype(f), np.ascontiguousarray(Einv[:, :3]).astype(f), np.ascontiguousarray(pair).astype(f)


def _ptrs(ts, dev):
    return torch.tensor([t.data_ptr() for t in ts], dtype=torch.int64, device=dev)


def _filter_views(depth, confs, masks, xyzs, mats, r0, ranges, opt, V, H, W, dev, stream):
    """pnb_depth_filter_build + _outputs on ref views r0 .. r0 + len(confs) - 1: the per-view (xyz_cam, xyz_world, conf) on dev."""
    lib = _lib.load()
    nr = len(confs)
    K, Kinv, c2w, pair = mats
    ws = torch.empty(lib.pnb_depth_filter_bytes(nr, H, W), dtype=torch.uint8, device=dev)
    pc, pm, px = _ptrs(confs, dev), _ptrs(masks, dev), _ptrs(xyzs, dev)
    counts = (_lib.C.c_longlong * nr)()
    _lib.check(lib.pnb_depth_filter_build(ws.data_ptr(), ws.numel(), V, H, W, r0, nr, depth.data_ptr(), pc.data_ptr(), pm.data_ptr(),
                                          px.data_ptr(), K.data_ptr(), Kinv.data_ptr(), c2w.data_ptr(), pair.data_ptr(),
                                          ranges.data_ptr() if ranges is not None else None, float(opt.depth_conf_thresh),
                                          int(opt.geo_cnsst_num), stream, counts), "pnb_depth_filter_build")
    n = int(sum(counts))
    cam = torch.empty((n, 3), dtype=torch.float32, device=dev)
    world = torch.empty((n, 3), dtype=torch.float32, device=dev)
    conf = torch.empty((n,), dtype=torch.float32, device=dev)
    if n:
        _lib.check(lib.pnb_depth_filter_outputs(ws.data_ptr(), ws.numel(), H, W, r0, nr, px.data_ptr(), pc.data_ptr(), c2w.data_ptr(),
                                                cam.data_ptr(), world.data_ptr(), conf.data_ptr(), stream), "pnb_depth_filter_outputs")
    out, o = [], 0
    for c in counts:
        out.append((cam[o:o + c], world[o:o + c], conf[o:o + c]))
        o += c
    return out


def filter_by_masks_gpu(cam_xyz_all, intrinsics_all, extrinsics_all, confidence_all, points_mask_all, opt, vis=False, return_w=False,
                        cpu2gpu=False, near_fars_all=None):
    """filter_utils.filter_by_masks_gpu: (xyz_cam_lst, xyz_world_lst, conf_lst), one [n_v,3] / [n_v,3] / [n_v] entry per view.

    cam_xyz_all[v] [1,1,C,H,W,3] (slice C = 0 is read: raw camera x, y and the depth), confidence_all[v] [1,1,H,W] fp32,
    points_mask_all[v] [1,1,H,W], intrinsics_all[v] [1,3,3], extrinsics_all[v] [1,4,4].  vis, return_w and near_fars_all are accepted
    and unread, as in the reference for these options.

    Synchronisation: the view matrices are copied to the host once per call (one transfer when they are CUDA tensors); with device
    inputs the call then synchronises once more, to size its outputs; under cpu2gpu once per ref view, whose outputs are then copied to
    the host.

    Device inputs: the outputs are on the inputs' device; the device holds the V depth maps ([V,H,W] fp32), a workspace of 5 bytes
    per pixel of every view and the outputs.  cpu2gpu (host inputs): the depth maps are staged on the current CUDA device once per call,
    each ref view's x, y, confidence and mask are copied there when it is filtered, and the outputs are host tensors; the device then
    holds the depth maps, one view's inputs and workspace and one view's outputs."""
    if opt.manual_depth_view > 1:
        raise NotImplementedError("filter_by_masks_gpu: manual_depth_view %r > 1 is not implemented" % (opt.manual_depth_view,))
    if opt.default_conf > 1.0:
        raise NotImplementedError("filter_by_masks_gpu: default_conf %r > 1 (reassign_conf) is not implemented" % (opt.default_conf,))
    if getattr(opt, "far_plane_shift", None) is not None:
        raise NotImplementedError("filter_by_masks_gpu: far_plane_shift %r is not implemented" % (opt.far_plane_shift,))
    V = len(cam_xyz_all)
    if V == 0:
        return [], [], []
    if not (len(intrinsics_all) == len(extrinsics_all) == len(confidence_all) == len(points_mask_all) == V):
        raise ValueError("filter_by_masks_gpu: %d views of points, %d intrinsics, %d extrinsics, %d confidences and %d masks"
                         % (V, len(intrinsics_all), len(extrinsics_all), len(confidence_all), len(points_mask_all)))
    shape = tuple(cam_xyz_all[0].shape)
    if len(shape) != 6 or shape[0] != 1 or shape[1] != 1 or shape[5] != 3:
        raise ValueError("filter_by_masks_gpu: cam_xyz_all entries must be [1,1,C,H,W,3] (B = N = 1; got %s)" % (shape,))
    H, W = int(shape[3]), int(shape[4])
    xyzs, confs, masks = [], [], []
    for v in range(V):
        t = cam_xyz_all[v]
        if tuple(t.shape) != shape:
            raise ValueError("filter_by_masks_gpu: every view must be %s (view %d is %s)" % (shape, v, tuple(t.shape)))
        if t.dtype != torch.float32 or confidence_all[v].dtype != torch.float32:
            raise ValueError("filter_by_masks_gpu: points and confidences must be float32 (view %d: %s, %s)"
                             % (v, t.dtype, confidence_all[v].dtype))
        c, m = confidence_all[v][0, 0], points_mask_all[v][0, 0]
        if tuple(c.shape) != (H, W) or tuple(m.shape) != (H, W):
            raise ValueError("filter_by_masks_gpu: view %d's confidence / mask are %s / %s, not %s"
                             % (v, tuple(c.shape), tuple(m.shape), (H, W)))
        xyzs.append(t[0, 0, 0])
        confs.append(c)
        masks.append(m)
    if not cpu2gpu and not all(t.is_cuda for t in xyzs + confs + masks):
        raise ValueError("filter_by_masks_gpu: the inputs must be CUDA tensors (or pass cpu2gpu=True)")
    dev = xyzs[0].device if not cpu2gpu else torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.current_stream(dev).cuda_stream
    # every view's K and E in one [V,25] tensor, copied to the host once (the matrices are formed there in float64)
    src = _t(intrinsics_all[0]).device
    KE = torch.stack([torch.cat([_t(k).detach()[0].reshape(9).to(src, torch.float32), _t(e).detach()[0].reshape(16).to(src, torch.float32)])
                      for k, e in zip(intrinsics_all, extrinsics_all)]).cpu().numpy()
    mats = tuple(torch.from_numpy(a).to(dev) for a in view_matrices(KE[:, :9].reshape(V, 3, 3), KE[:, 9:].reshape(V, 4, 4)))
    ranges = None
    if opt.ranges[0] > -99.0:
        ranges = torch.as_tensor(opt.ranges, dtype=torch.float32).to(dev)
    depth = torch.stack([t[..., 2].to(dev) for t in xyzs]).contiguous()
    mask_u8 = [m if m.dtype == torch.bool else (m != 0) for m in masks]
    if not cpu2gpu:
        res = _filter_views(depth, [c.contiguous() for c in confs], [m.contiguous().view(torch.uint8) for m in mask_u8],
                            [t.contiguous() for t in xyzs], mats, 0, ranges, opt, V, H, W, dev, stream)
    else:
        res = []
        for r in range(V):
            out = _filter_views(depth, [confs[r].to(dev).contiguous()], [mask_u8[r].to(dev).contiguous().view(torch.uint8)],
                                [xyzs[r].to(dev).contiguous()], mats, r, ranges, opt, V, H, W, dev, stream)[0]
            res.append(tuple(a.cpu() for a in out))
    return [a for a, _, _ in res], [b for _, b, _ in res], [c for _, _, c in res]


def alpha_masking(points, alphas, intrinsics, c2ws, w2cs, near_far, opt=None):
    """mvs_utils.alpha_masking: bool [N] on the points' device, True where every view's alpha at the point's pixel exceeds 0.1 (and the
    point is within near_far, when given).  points [N,>=3] float32, on a CUDA device or on the host; alphas[v][0] [H,W];
    intrinsics[v] [3,3]; w2cs[v] [4,4] (numpy or tensors); c2ws is unread, as in the reference.

    Host points (gen_points_filter_embeddings' cloud under cpu2gpu) are masked on the current CUDA device, HOST_CHUNK points at a
    time: the device then holds the V alpha maps, one chunk of points and its mask, and the mask is copied back chunk by chunk."""
    if not isinstance(points, torch.Tensor) or points.dtype != torch.float32 or points.dim() != 2 or points.shape[1] < 3:
        raise ValueError("alpha_masking: points must be a float32 tensor [N, >=3]")
    V = len(alphas)
    if V == 0 or len(intrinsics) < V or len(w2cs) < V:
        raise ValueError("alpha_masking: %d alphas, %d intrinsics, %d w2cs" % (V, len(intrinsics), len(w2cs)))
    dev = points.device if points.is_cuda else torch.device("cuda", torch.cuda.current_device())
    H, W = (int(s) for s in _t(alphas[0][0]).shape)
    al = []
    for v in range(V):
        a = torch.as_tensor(alphas[v][0], dtype=torch.float32, device=dev)
        if tuple(a.shape) != (H, W):
            raise ValueError("alpha_masking: view %d's alpha is %s, view 0's %s" % (v, tuple(a.shape), (H, W)))
        al.append(a)
    alpha = torch.stack(al).contiguous()
    w2c = torch.stack([torch.as_tensor(w2cs[v], dtype=torch.float32).reshape(4, 4)[:3] for v in range(V)]).to(dev).contiguous()
    K = torch.stack([torch.as_tensor(intrinsics[v], dtype=torch.float32).reshape(3, 3) for v in range(V)]).to(dev).contiguous()
    nf = None
    if near_far is not None:
        nf = (_lib.C.c_float * 2)(float(np.float32(float(near_far[0]) - 1.0)), float(np.float32(float(near_far[1]))))
    range_test = int(opt is not None and (opt.alpha_range > 0 or opt.inall_img == 0))
    lib = _lib.load()
    stream = torch.cuda.current_stream(dev).cuda_stream
    N = int(points.shape[0])

    def run(pts, out):
        _lib.check(lib.pnb_alpha_mask(pts.data_ptr(), int(pts.shape[0]), V, w2c.data_ptr(), K.data_ptr(), alpha.data_ptr(), H, W, nf,
                                      range_test, out.data_ptr(), stream), "pnb_alpha_mask")

    if points.is_cuda:
        out = torch.empty(N, dtype=torch.bool, device=dev)
        run(points[:, :3].contiguous(), out)
        return out
    out = torch.empty(N, dtype=torch.bool)
    for i in range(0, N, HOST_CHUNK):
        m = torch.empty(min(HOST_CHUNK, N - i), dtype=torch.bool, device=dev)
        run(points[i:i + HOST_CHUNK, :3].to(dev).contiguous(), m)
        out[i:i + len(m)] = m.cpu()
    return out
