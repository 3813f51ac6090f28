"""Checkpoint wire format of the reference (SURVEY.md 8(f) rank 3).

The reference writes, per saved iteration (`/root/reference/models/base_model.py:85-103`):
  `{epoch}_net_ray_marching.pth`  = `net_ray_marching.state_dict()` (after unwrapping `nn.DataParallel`): flat dict
      neural_points.xyz [N,3] | neural_points.points_embeding [1,N,F] (F = point_features_dim: 32, or 63 for the DTU scripts) | neural_points.points_conf [1,N,1] |
      neural_points.points_dir [1,N,3] | neural_points.points_color [1,N,3] | (neural_points.eulers, neural_points.Rw2c [3,3] or [N,3,3]) |
      aggregator.{block1.0,block1.2,block3.0,block3.2,alpha_branch.0,color_branch.0,.2,.4,.6}.{weight,bias}
  `{epoch}_states.pth`            = free-form dict of runner state (`epoch_count`, `total_steps`, optimiser states ...)
and reads them back with `NeuralPoints.__init__(checkpoint=...)` (`models/neural_points/neural_points.py:242-288`) and
`load_networks` (`base_model.py:105-121`, `strict=False`).  `pointnerf_b200.ray_marching.NeuralPointsRayMarching` keeps the
same attribute names, so its own `state_dict()` IS this format; the functions below add the validation the reference
leaves out (a `strict=False` load silently ignores a misspelt key) and build a module from a checkpoint alone.
"""
import os

import torch

from . import ray_marching

POINT_KEYS = {  # key -> (ndim, trailing shape); N is taken from xyz
    "neural_points.xyz": (2, (3,)),
    "neural_points.points_embeding": (3, None),
    "neural_points.points_conf": (3, (1,)),
    "neural_points.points_dir": (3, (3,)),
    "neural_points.points_color": (3, (3,)),
}
OPTIONAL_POINT_KEYS = ("neural_points.Rw2c", "neural_points.eulers")


class CheckpointError(ValueError):
    pass


def checkpoint_paths(resume_dir, epoch):
    """File names used by save_networks / load_networks (base_model.py:87,101,109)."""
    return (os.path.join(resume_dir, "%s_net_ray_marching.pth" % epoch), os.path.join(resume_dir, "%s_states.pth" % epoch))


def _strip_module(sd):
    """`nn.DataParallel` state dicts carry a `module.` prefix when saved without unwrapping."""
    if sd and all(k.startswith("module.") for k in sd):
        return {k[len("module."):]: v for k, v in sd.items()}
    return dict(sd)


def read_state_dict(path_or_dict, map_location="cpu"):
    sd = torch.load(path_or_dict, map_location=map_location) if isinstance(path_or_dict, (str, os.PathLike)) else path_or_dict
    if not isinstance(sd, dict):
        raise CheckpointError("checkpoint is not a state dict: %r" % type(sd))
    return _strip_module(sd)


def validate(sd, opt=None):
    """Checks the tensor inventory of a `*_net_ray_marching.pth` state dict; returns N."""
    missing = [k for k in POINT_KEYS if k not in sd]
    if missing:
        raise CheckpointError("checkpoint misses %s" % ", ".join(missing))
    n = sd["neural_points.xyz"].shape[0]
    for k, (nd, tail) in POINT_KEYS.items():
        t = sd[k]
        ok = t.dim() == nd and (t.shape[0] == n if nd == 2 else (t.shape[0] == 1 and t.shape[1] == n))
        if ok and tail is not None:
            ok = tuple(t.shape[-len(tail):]) == tail
        if not ok or t.dtype != torch.float32:
            raise CheckpointError("%s has shape %s / %s for N=%d" % (k, tuple(t.shape), t.dtype, n))
    if opt is not None:
        c = int(getattr(opt, "point_features_dim", sd["neural_points.points_embeding"].shape[-1]))
        if sd["neural_points.points_embeding"].shape[-1] != c:
            raise CheckpointError("points_embeding has %d channels, opt.point_features_dim=%d" % (sd["neural_points.points_embeding"].shape[-1], c))
    if "neural_points.Rw2c" in sd:
        # one rotation for the whole cloud, or one per point (a checkpoint saved after an edit, run/editing.py)
        R = sd["neural_points.Rw2c"]
        if tuple(R.shape) not in ((3, 3), (n, 3, 3)) or R.dtype != torch.float32:
            raise CheckpointError("neural_points.Rw2c has shape %s / %s; needs fp32 [3,3] or [N,3,3] for N=%d" % (tuple(R.shape), R.dtype, n))
    if "neural_points.eulers" in sd:
        raise NotImplementedError("pnb200: per-point euler rotations (neural_points.eulers) are outside the shipped hot path")
    unknown = [k for k in sd if not (k in POINT_KEYS or k in OPTIONAL_POINT_KEYS or k.startswith("aggregator."))]
    if unknown:
        raise CheckpointError("unexpected keys: %s" % ", ".join(sorted(unknown)[:8]))
    return n


def load_into(net, path_or_dict, strict=True):
    """Loads a reference checkpoint into an existing NeuralPointsRayMarching (points are re-created as parameters, the
    cached voxel grid is invalidated, the packed wgmma weight images are rebuilt on the next call)."""
    sd = read_state_dict(path_or_dict)
    validate(sd, getattr(net, "opt", None))
    dev = net.neural_points.device
    np_ = net.neural_points
    np_.set_points(sd["neural_points.xyz"].to(dev), sd["neural_points.points_embeding"].to(dev),
                   points_color=sd["neural_points.points_color"].to(dev), points_dir=sd["neural_points.points_dir"].to(dev),
                   points_conf=sd["neural_points.points_conf"].to(dev), parameter=True, as_stored=True,
                   Rw2c=sd["neural_points.Rw2c"].to(dev) if "neural_points.Rw2c" in sd else None)
    agg_sd = {k[len("aggregator."):]: v for k, v in sd.items() if k.startswith("aggregator.")}
    want = set(net.aggregator.state_dict().keys())
    if strict and set(agg_sd) != want:
        raise CheckpointError("aggregator keys differ: missing %s, unexpected %s" % (sorted(want - set(agg_sd)), sorted(set(agg_sd) - want)))
    net.aggregator.load_state_dict(agg_sd, strict=strict)
    return net


def load_checkpoint(path_or_dict, opt, device):
    """Builds the fused module from a checkpoint alone (what `create_network_models` + `load_networks` do in the reference,
    neural_points_volumetric_model.py:155-168)."""
    npts = ray_marching.NeuralPoints(opt, device)
    agg = ray_marching.PointAggregator(opt).to(device)
    net = ray_marching.NeuralPointsRayMarching(aggregator=agg, neural_points=npts, opt=opt)
    return load_into(net, path_or_dict)


def save_checkpoint(net, resume_dir, epoch, other_states=None):
    """Writes the two files the reference's `save_networks` writes (base_model.py:85-103); tensors go to the CPU first."""
    os.makedirs(resume_dir, exist_ok=True)
    net_path, states_path = checkpoint_paths(resume_dir, epoch)
    sd = {k: v.detach().cpu() for k, v in _strip_module(net.state_dict()).items()}
    validate(sd, getattr(net, "opt", None))
    torch.save(sd, net_path)
    torch.save(dict(other_states or {}), states_path)
    return net_path, states_path
