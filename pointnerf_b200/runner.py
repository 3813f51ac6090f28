"""Whole-image entry points either side of the seam (SURVEY.md 8(f) rank 2).

The reference renders an image as a host loop over `random_sample_size**2`-ray chunks
(`/root/reference/run/render_vid.py:45-71`, `/root/reference/run/train_ft.py:283-320`): per chunk `model.set_input`,
`model.test()`, `.cpu().numpy()` of every `*color` visual into a `[H*W,3]` host array, then `fill_invalid`
(`neural_points_volumetric_model.py:87-123`) — 278 launches + host syncs for an 800x800 frame at the shipped 2304-ray
chunk.  `render_image` is the same computation as ONE call (rays of the whole frame resident on the device, fill_invalid
applied in-kernel, no host sync until the caller reads the result); `render_image_chunked` reproduces the reference loop
through the drop-in `forward()` and is what the parity test compares it with (a ray's colour is bit-identical whichever
rays share its call).  `probe_image` / `probe_image_chunked` are the same pair for the probe pass of point growing
(`run/train_ft.py:417-530`, opt.prob = 1).

With the perspective-frustum query (wcoord_query 0, the DTU scripts) the data dict also carries `pixel_idx [1,H*W,2]`, `h`, `w` and
`intrinsic`, as the reference's dataset items do; the querier's synchronisation for the number of hit rays is then the one host
synchronisation of a frame.  `bg_ray [1,H*W,3]` (bgmodel plane) replaces the background colour the way the model shell's fill_invalid
does (`coarse_is_background * bg_ray`, plus the colour of a hit ray).
"""
import numpy as np
import torch


def _near_far(near, far):
    n = float(torch.min(near)) if isinstance(near, torch.Tensor) else float(near)
    f = float(torch.max(far)) if isinstance(far, torch.Tensor) else float(far)
    return n, f


def _full_kwargs(net, data, bg_ray):
    """The optional arguments of render_full for this frame: bg_ray, and under wcoord_query 0 the frustum query's view (pixel_idx, h,
    w, intrinsic); none of them for a world-query frame with a background colour."""
    kw = {} if bg_ray is None else dict(bg_ray=bg_ray)
    view = _view(net, data)
    if view is not None:
        kw["view"] = view
    return kw


def _view(net, data):
    """The frustum query's view (pixel_idx, h, w, intrinsic) from a data dict under wcoord_query 0, else None."""
    if int(getattr(getattr(net, "opt", None), "wcoord_query", -1)) != 0:
        return None
    return {k: data.get(k) for k in ("pixel_idx", "h", "w", "intrinsic")}


def _fill_bg_ray(color, is_bg, mask, bg_ray):
    """fill_invalid with bg_ray (neural_points_volumetric_model.py:101-103) on one chunk: coarse_is_background * bg_ray, then the colour
    of each hit ray added."""
    full_bg = torch.ones((mask.shape[0], 1), dtype=torch.float32, device=bg_ray.device)
    full_bg[mask] = is_bg
    out = full_bg * bg_ray
    out[mask] += color
    return out


def render_image(net, data, height, width, check=True, bg_ray=None):
    """data: the dict a reference dataset item carries (`campos [1,3]`, `raydir [1,H*W,3]`, `camrotc2w [1,3,3]`, `near`, `far`,
    `bg_color`).  Returns device tensors: `coarse_raycolor [H,W,3]`, `coarse_point_opacity [H,W,SR]`,
    `coarse_is_background [H,W,1]`, `ray_mask [H,W]` (all rays, background filled as fill_invalid does).
    check=True (default): the device status of the frame is read before returning (one stream synchronisation; the caller is
    about to read the image anyway) and a frame whose shading workspace was too small is rendered again with the exact size;
    check=False: fully asynchronous, the status surfaces at a later call or through `net.check_errors()`.
    bg_ray [1,H*W,3] (default: data["bg_ray"] if present): the per-ray background of bgmodel plane, applied in the kernel."""
    near, far = _near_far(data["near"], data["far"])
    raydir = data["raydir"]
    if raydir.shape[1] != height * width:
        raise ValueError("render_image: %d rays for a %dx%d image" % (raydir.shape[1], height, width))
    bg = data.get("bg_color", None)
    bg_ray = data.get("bg_ray", None) if bg_ray is None else bg_ray
    from .lib import PnbOverflow
    with torch.no_grad():
        for attempt in range(2):
            out = net.render_full(data["campos"], raydir, data["camrotc2w"], near, far, bg if bg is not None else torch.zeros(3),
                                  **_full_kwargs(net, data, bg_ray))
            if not check:
                break
            try:
                net.check_errors()
                break
            except PnbOverflow:
                if attempt == 1:
                    raise
    sr = out["coarse_point_opacity"].shape[-1]
    return dict(coarse_raycolor=out["coarse_raycolor"][0].view(height, width, 3),
                coarse_point_opacity=out["coarse_point_opacity"][0].view(height, width, sr),
                coarse_is_background=out["coarse_is_background"][0].view(height, width, 1),
                ray_mask=out["ray_mask"][0].view(height, width))


def render_image_chunked(net, data, height, width, chunk_size, bg_ray=None):
    """The reference chunk loop (render_vid.py:45-71) through the drop-in `forward()` + fill_invalid on the host:
    returns `{"coarse_raycolor": np.ndarray [H,W,3]}` exactly as the reference assembles `visuals`.  bg_ray [1,H*W,3] (default:
    data["bg_ray"] if present): each chunk's slice goes to forward() and fill_invalid adds coarse_is_background * bg_ray."""
    near, far = _near_far(data["near"], data["far"])
    raydir = data["raydir"]
    total = height * width
    bg = data.get("bg_color", None)
    bgv = (bg if bg is not None else torch.zeros(3)).reshape(-1)[:3].cpu().numpy().astype(np.float32)
    bg_ray = data.get("bg_ray", None) if bg_ray is None else bg_ray
    view = _view(net, data)
    img = np.zeros((total, 3), dtype=np.float32)
    with torch.no_grad():
        for start in range(0, total, chunk_size):
            end = min(start + chunk_size, total)
            kw = {} if bg_ray is None else dict(bg_ray=bg_ray[:, start:end])
            if view is not None:
                kw.update(pixel_idx=view["pixel_idx"][:, start:end], h=view["h"], w=view["w"], intrinsic=view["intrinsic"])
            out = net(data["campos"], raydir[:, start:end, :], bg_color=bg, camrotc2w=data["camrotc2w"],
                      near=near, far=far, **kw)
            if bg_ray is not None:
                mask = out["ray_mask"][0].bool()
                img[start:end] = _fill_bg_ray(out["coarse_raycolor"][0], out["coarse_is_background"][0], mask,
                                              bg_ray[0, start:end].to(mask.device, torch.float32)).cpu().numpy()
                continue
            mask = out["ray_mask"][0].bool().cpu().numpy()
            chunk = np.tile(bgv[None, :], (end - start, 1))                      # fill_invalid: background where no neighbour
            chunk[mask] = out["coarse_raycolor"][0].cpu().numpy()
            img[start:end] = chunk
    return dict(coarse_raycolor=img.reshape(height, width, 3))


# what probe_hole (run/train_ft.py:417-530) collects of every training frame, in its order
PROBE_MAP_KEYS = ("coarse_raycolor", "ray_mask", "ray_max_sample_loc_w", "ray_max_far_dist", "ray_max_shading_opacity",
                  "shading_avg_color", "shading_avg_dir", "shading_avg_conf", "shading_avg_embedding")


def probe_image(net, data, height, width, check=True, t=None, bg_ray=None):
    """The probe pass of point growing (opt.prob == 1) over a whole frame in one call: the maps probe_hole
    (run/train_ft.py:417-530) assembles from its 2304-ray chunks, as device tensors [H,W,C] under its keys (PROBE_MAP_KEYS):
    `coarse_raycolor` (background where a ray missed), `ray_mask` [H,W,1] (int8), `ray_max_sample_loc_w`, `ray_max_far_dist`,
    `ray_max_shading_opacity` and `shading_avg_{color,dir,conf,embedding}` (zeros where a ray missed).  probe_hole's selection
    (miss mask, bloat_inds, thresholds) runs unchanged on them.  check: as render_image (one stream synchronisation, a frame whose
    shading workspace was too small is probed again).  The depth table follows opt.is_train as forward() does; with jitter a
    chunked run agrees with this one only when both get the same table `t` ([R, D]).  bg_ray: as render_image."""
    near, far = _near_far(data["near"], data["far"])
    raydir = data["raydir"]
    if raydir.shape[1] != height * width:
        raise ValueError("probe_image: %d rays for a %dx%d image" % (raydir.shape[1], height, width))
    bg = data.get("bg_color", None)
    bg_ray = data.get("bg_ray", None) if bg_ray is None else bg_ray
    from .lib import PnbOverflow
    with torch.no_grad():
        for attempt in range(2):
            out = net.render_full(data["campos"], raydir, data["camrotc2w"], near, far, bg if bg is not None else torch.zeros(3),
                                  t=t, probe=True, **_full_kwargs(net, data, bg_ray))
            if not check:
                break
            try:
                net.check_errors()
                break
            except PnbOverflow:
                if attempt == 1:
                    raise
    maps = {k: out[k][0].view(height, width, -1) for k in PROBE_MAP_KEYS if k != "ray_mask"}
    maps["ray_mask"] = out["ray_mask"][0].view(height, width, 1)
    return {k: maps[k] for k in PROBE_MAP_KEYS}


def probe_image_chunked(net, data, height, width, chunk_size, bg_ray=None):
    """probe_hole's loop (run/train_ft.py:455-480) through the drop-in `forward()` with opt.prob = 1: chunks of `chunk_size` rays,
    each chunk's outputs filled as fill_invalid / unmask fill them (:87-131) and written into [H,W,C] device maps.  What
    probe_image replaces, and what it is compared with."""
    near, far = _near_far(data["near"], data["far"])
    raydir = data["raydir"]
    total = height * width
    bg = data.get("bg_color", None)
    bgv = (bg if bg is not None else torch.zeros(3)).reshape(-1)[:3].to(raydir.device, torch.float32)
    bg_ray = data.get("bg_ray", None) if bg_ray is None else bg_ray
    view = _view(net, data)
    maps = {}
    prob = getattr(net.opt, "prob", 0)
    net.opt.prob = 1
    try:
        with torch.no_grad():
            for start in range(0, total, chunk_size):
                end = min(start + chunk_size, total)
                kw = {} if bg_ray is None else dict(bg_ray=bg_ray[:, start:end])
                if view is not None:
                    kw.update(pixel_idx=view["pixel_idx"][:, start:end], h=view["h"], w=view["w"], intrinsic=view["intrinsic"])
                out = net(data["campos"], raydir[:, start:end, :], bg_color=bg, camrotc2w=data["camrotc2w"], near=near, far=far, **kw)
                mask = out["ray_mask"][0].bool()
                for key in PROBE_MAP_KEYS:
                    v = out["ray_mask"][0][:, None] if key == "ray_mask" else out[key].reshape(-1, out[key].shape[-1])
                    if key not in maps:
                        maps[key] = torch.zeros((total, v.shape[-1]), dtype=v.dtype, device=raydir.device)
                    if key == "coarse_raycolor" and bg_ray is not None:
                        maps[key][start:end] = _fill_bg_ray(out[key][0], out["coarse_is_background"][0], mask,
                                                            bg_ray[0, start:end].to(raydir.device, torch.float32))
                        continue
                    if key == "coarse_raycolor":
                        maps[key][start:end] = bgv
                    if key == "ray_mask":
                        maps[key][start:end] = v
                    elif v.shape[0] > 0:          # a chunk without a hit ray returns empty placeholders (:352-361): its rows stay 0
                        maps[key][start:end][mask] = v
    finally:
        net.opt.prob = prob
    return {k: v.view(height, width, -1) for k, v in maps.items()}
