"""CPU, where the reference tree exists (skipped elsewhere): the feed-forward scripts (dev_scripts/ete/*.sh, run/train.py
--feedforward 1) against the fused module's option surface and point seam.

  options  check_opt accepts each ete script's full flag set as given, on the reference's argparse namespace: the one of
           oracle/ref_shim.make_opt (the shipped hot-path flags, then the script's), and the reference's own defaults with the
           script's flags alone (the F 63 script passes no --wcoord_query, so it runs the default perspective-frustum query)
  points   the reference's own NeuralPoints.set_points(parameter=False), fed non-leaf tensors shaped like query_embedding's outputs,
           installs tensors that the fused module reads in place: contiguous fp32, the network's own outputs (no copies) and, for
           point modes "01", one colour tensor both in the embedding and kept beside it
"""
import argparse
import re

import pytest
import torch

from oracle import ref_shim

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")

SCRIPTS = {32: "dtu_dgt_d012_img0123_conf_agg2_32_dirclr20", 63: "dtu_dgt_d012_img0123_conf_color_dir_agg2"}


def script_flags(name):
    """The argument list run/train.py receives from dev_scripts/ete/<name>.sh: the shell variables substituted into the python3
    command, word-split as bash splits an unquoted expansion."""
    import os
    src = open(os.path.join(ref_shim.REF, "dev_scripts", "ete", name + ".sh")).read()
    env = {}
    for m in re.finditer(r"""^\s*(\w+)=("[^"]*"|'[^']*'|\S*)""", src, re.M):
        v = m.group(2)
        env[m.group(1)] = v[1:-1] if v[:1] in "\"'" else v
    cmd = src[src.index("python3 train.py"):].replace("\\\n", " ").split("\n")[0]
    cmd = re.sub(r"\$\{?(\w+)\}?", lambda m: env.get(m.group(1), ""), cmd)
    return cmd.split()[2:]


def _reference_defaults(flags):
    ref_shim.install()
    from models.neural_points_volumetric_model import NeuralPointsVolumetricModel
    parser = argparse.ArgumentParser()
    NeuralPointsVolumetricModel.modify_commandline_options(parser, True)
    opt, _ = parser.parse_known_args(flags)
    opt.is_train = True
    return opt


@pytest.mark.parametrize("F", [32, 63])
def test_check_opt_accepts_the_ete_scripts(F):
    from pointnerf_b200.ray_marching import check_opt, is_frustum
    flags = script_flags(SCRIPTS[F])
    assert "--feedforward" in flags and flags[flags.index("--feedforward") + 1] == "1"
    shipped = ref_shim.make_opt(flags, is_train=True)
    own = _reference_defaults(flags)
    for opt in (shipped, own):
        assert int(opt.point_features_dim) == F and int(opt.SR) == 40 and int(opt.K) == 8 and int(opt.P) == 20
        check_opt(opt)
    if F == 32:
        assert int(own.wcoord_query) == 1 and list(own.kernel_size) == [5, 5, 5] and list(own.vsize) == [0.002] * 3
        assert own.point_conf_mode == own.point_dir_mode == own.point_color_mode == "1"
    else:
        assert is_frustum(own) and list(own.kernel_size) == [3, 3, 3]
        assert own.point_conf_mode == own.point_dir_mode == own.point_color_mode == "01"


def _network_outputs(N, F, g):
    """Non-leaf tensors shaped like MvsPointsModel.query_embedding's outputs (models/mvs/mvs_points_model.py:222-259): F 32, the premlp's
    [1,N,32] embedding; F 63, 56 image-feature channels; colour [1,N,3] (differentiable), dir [1,N,3] and conf [1,N,1] (computed
    under no_grad, plain tensors); xyz [N,3]."""
    src = torch.randn(1, N, 8, generator=g, requires_grad=True)
    w = torch.randn(8, 32 if F == 32 else 56, generator=g)
    emb = torch.tanh(src @ w)
    col = torch.sigmoid(src[..., :3] * 2.0)
    with torch.no_grad():
        pdir = torch.nn.functional.normalize(torch.randn(1, N, 3, generator=g), dim=-1)
        conf = torch.rand(1, N, 1, generator=g)
        xyz = torch.randn(N, 3, generator=g)
    return xyz, emb, col, pdir, conf


@pytest.mark.parametrize("F", [32, 63])
def test_reference_set_points_installs_the_network_tensors_in_place(F):
    from pointnerf_b200 import ray_marching as P
    flags = script_flags(SCRIPTS[F])
    opt = _reference_defaults(flags)
    opt.wcoord_query = -1        # the reference's CPU-importable querier; the point tensors do not depend on it
    opt.ranges = [-1.0, -1.0, -1.0, 1.0, 1.0, 1.0]
    from models.neural_points.neural_points import NeuralPoints as RefPoints
    npts = RefPoints(F, 8192, opt, torch.device("cpu"), feedforward=1)
    xyz, emb, col, pdir, conf = _network_outputs(500, F, torch.Generator().manual_seed(F))
    npts.set_points(xyz, emb, points_color=col, points_dir=pdir, points_conf=conf, parameter=False)
    assert npts.xyz is xyz and npts.points_color is col and npts.points_dir is pdir and npts.points_conf is conf
    if F == 32:
        assert npts.points_embeding is emb
    else:
        # "01": colour, dir and conf prepended ([color, dir, conf, emb]) and kept: the colour reaches the module twice
        assert torch.equal(npts.points_embeding, torch.cat([col, pdir, conf, emb], dim=-1))
        assert npts.points_embeding.grad_fn is not None
    assert npts.points_embeding.shape[-1] == F and npts.points_embeding.requires_grad and npts.points_color.requires_grad
    assert not npts.points_embeding.is_leaf and not npts.points_dir.requires_grad and not npts.points_conf.requires_grad
    # what points_desc_of reads in place, apart from the device: contiguous fp32 tensors of the width the kernels take
    for t in (npts.xyz, npts.points_embeding, npts.points_color, npts.points_dir, npts.points_conf):
        assert t.is_contiguous() and t.dtype == torch.float32
    assert npts.points_embeding.shape[-1] in P.FEAT_DIMS
    with pytest.raises(P._lib.PnbError, match="CUDA"):
        P.points_desc_of(npts)      # the device is the only thing it refuses on this machine
