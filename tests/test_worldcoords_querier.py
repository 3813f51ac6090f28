"""CPU checks of the world-coordinate querier of wcoord_query 1 (pointnerf_b200.query_point_indices_worldcoords): its public surface
against the reference's pycuda class, the reference's own NeuralPoints constructing it in place of that class, get_hyperparameters
against the reference's expressions and the wcoord_query -1 querier (also after the options change), and its refusals.

The reference class is imported with stub pycuda modules (it needs pycuda only to construct, which these tests never do); the tests
that read the reference need its tree and are skipped elsewhere."""
import inspect
import sys
import types
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ref_shim
from pointnerf_b200 import harness, scene
from pointnerf_b200 import point_query as wq
from pointnerf_b200 import query_point_indices_worldcoords as wc

needs_reference = pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree")
CPU = torch.device("cpu")
REF_MODULE = "models.neural_points.query_point_indices_worldcoords"


def _opt(name="tiny", **over):
    return harness.make_opt(scene.CONFIGS[name], **dict(dict(wcoord_query=1, depth_limit_scale=0.0), **over))


@pytest.fixture
def ref_class(monkeypatch):
    """The reference's flavour-1 lighting_fast_querier, imported with stub pycuda modules; gpuarray.to_gpu returns its numpy input, so
    the reference's get_hyperparameters runs on the CPU."""
    ref_shim.install()
    drv = types.ModuleType("pycuda.driver")
    drv.PointerHolderBase = object
    gpuarray = types.ModuleType("pycuda.gpuarray")
    gpuarray.to_gpu = lambda a: a
    compiler = types.ModuleType("pycuda.compiler")
    compiler.SourceModule = None
    pycuda = types.ModuleType("pycuda")
    pycuda.driver, pycuda.gpuarray, pycuda.compiler = drv, gpuarray, compiler
    for name, mod in (("pycuda", pycuda), ("pycuda.driver", drv), ("pycuda.gpuarray", gpuarray), ("pycuda.compiler", compiler)):
        monkeypatch.setitem(sys.modules, name, mod)
    monkeypatch.delitem(sys.modules, REF_MODULE, raising=False)
    import importlib
    mod = importlib.import_module(REF_MODULE)
    monkeypatch.delitem(sys.modules, REF_MODULE)       # the next import of the name finds the reference file again, not this object
    return mod.lighting_fast_querier


@needs_reference
def test_public_surface_matches_the_reference(ref_class):
    for m in ("__init__", "get_hyperparameters", "query_points", "w2pers", "clean_up"):
        ours = list(inspect.signature(getattr(wc.lighting_fast_querier, m)).parameters)
        assert ours == list(inspect.signature(getattr(ref_class, m)).parameters), m
    assert len(inspect.signature(ref_class.query_points).parameters) == 13     # self + 12
    # NeuralPoints resolves the class by name (neural_points.py:333-335)
    assert wc.lighting_fast_querier.__name__ == ref_class.__name__


@needs_reference
def test_reference_neural_points_builds_the_drop_in_without_pycuda(monkeypatch):
    from oracle import make_golden
    for name in ("pycuda", "pycuda.driver", "pycuda.gpuarray", "pycuda.compiler"):
        monkeypatch.delitem(sys.modules, name, raising=False)
    monkeypatch.setitem(sys.modules, REF_MODULE, wc)                # the registration INTEGRATION.md gives for wcoord_query 1
    net, agg, npts, pts, opt = make_golden.build_reference_net(scene.CONFIGS["tiny"], 4.0, extra_flags=["--wcoord_query", "1"])
    assert opt.wcoord_query == 1
    assert type(npts.querier) is wc.lighting_fast_querier and npts.querier.opt is opt
    assert "pycuda" not in sys.modules
    npts.reset_querier()                                            # the model shell's clean_up + construct again (neural_points.py:341-344)
    assert type(npts.querier) is wc.lighting_fast_querier


def _assert_same_hyper(ours, ref):
    assert len(ours) == len(ref) == 14
    for i, (a, b) in enumerate(zip(ours[:8], ref[:8])):
        if i == 3:
            assert a is b                                           # vsize_np is returned as passed
            continue
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and np.array_equal(a, b), i
    for i, (a, b) in enumerate(zip(ours[8:], ref[8:])):             # device tensors here, gpuarrays there (numpy under the stub)
        assert isinstance(a, torch.Tensor) and a.dtype == torch.from_numpy(np.asarray(b)).dtype, 8 + i
        assert np.array_equal(a.cpu().numpy(), np.asarray(b)), 8 + i


@needs_reference
@pytest.mark.parametrize("name", ["tiny", "chair_plumbing", "lego_render", "truck_8gpu"])
def test_get_hyperparameters_is_the_reference_expression(name, ref_class):
    cfg = scene.CONFIGS[name]
    xyz = scene.make_points(cfg)["xyz"][None]
    for over in ({}, dict(query_size=[1, 1, 1], radius_limit_scale=2.5, depth_limit_scale=1.5), dict(vsize=[0.007, 0.005, 0.011])):
        opt = _opt(name, **over)
        ours = wc.lighting_fast_querier(CPU, opt).get_hyperparameters(opt.vsize, xyz, ranges=opt.ranges)
        _assert_same_hyper(ours, ref_class.get_hyperparameters(SimpleNamespace(opt=opt), opt.vsize, xyz, ranges=opt.ranges))
        ours = wc.lighting_fast_querier(CPU, opt).get_hyperparameters(opt.vsize, xyz)
        _assert_same_hyper(ours, ref_class.get_hyperparameters(SimpleNamespace(opt=opt), opt.vsize, xyz))


@pytest.mark.parametrize("name", ["tiny", "lego_render", "truck_8gpu"])
def test_get_hyperparameters_gives_the_minus_one_numbers_and_follows_the_options(name):
    cfg = scene.CONFIGS[name]
    xyz = scene.make_points(cfg)["xyz"][None]
    opt = _opt(name)
    q = wc.lighting_fast_querier(CPU, opt)

    def check():
        ref = wq.lighting_fast_querier(CPU, opt)                    # the -1 querier reads the options of now at construction
        rl, dl, ranges_np, vsize_np, vdim, svs, sdim, vscale, ranges_gpu, svs_gpu, sdim_gpu, vscale_gpu, ks_gpu, qs_gpu = \
            q.get_hyperparameters(opt.vsize, xyz, ranges=opt.ranges)
        r_ranges, r_vsize, r_sdim = ref.get_hyperparameters(opt.vsize, xyz, ranges=opt.ranges)
        assert np.array_equal(ranges_np, r_ranges.numpy()) and torch.equal(ranges_gpu, r_ranges)
        assert vsize_np is r_vsize and np.array_equal(sdim, r_sdim) and np.array_equal(sdim_gpu.numpy(), r_sdim)
        assert np.array_equal(svs, ref.scaled_vsize_np) and np.array_equal(svs_gpu.numpy(), ref.scaled_vsize_np)
        assert rl == ref.radius_limit_np and rl.dtype == np.float32
        assert np.array_equal(vscale, ref.vscale_np) and np.array_equal(vscale_gpu.numpy(), ref.vscale_np)
        assert np.array_equal(ks_gpu.numpy(), ref.kernel_size) and np.array_equal(qs_gpu.numpy(), ref.query_size)
        assert np.array_equal(np.ceil(vdim / vscale).astype(np.int32), sdim)
        assert dl == np.float32(opt.depth_limit_scale * opt.vsize[2])
        # the attributes the fused path reads follow the options too
        assert np.array_equal(q.scaled_vsize_np, ref.scaled_vsize_np) and q.radius_limit_np == ref.radius_limit_np
        assert np.array_equal(q.kernel_size, ref.kernel_size) and np.array_equal(q.query_size, ref.query_size)

    check()
    opt.query_size = [1, 1, 1]
    check()
    opt.vsize = [v * 1.5 for v in opt.vsize]
    check()
    opt.kernel_size, opt.radius_limit_scale, opt.depth_limit_scale = [5, 3, 1], 1.5, 2.0
    check()
    opt.vscale = [1, 2, 3]
    check()


def test_refusals():
    for over in (dict(NN=0), dict(NN=-1), dict(inverse=1), dict(K=9), dict(SR=129)):
        with pytest.raises(NotImplementedError, match=next(iter(over))):
            wc.lighting_fast_querier(CPU, _opt(**over))
    # the options are read on every call: a value set after construction is refused at the next call
    xyz = scene.make_points(scene.CONFIGS["tiny"])["xyz"][None]
    for k, v in (("inverse", 1), ("K", 9), ("SR", 129)):
        opt = _opt()
        q = wc.lighting_fast_querier(CPU, opt)
        setattr(opt, k, v)
        with pytest.raises(NotImplementedError, match=k):
            q.get_hyperparameters(opt.vsize, xyz, ranges=opt.ranges)
    q = wc.lighting_fast_querier(CPU, _opt())
    with pytest.raises(NotImplementedError, match="batch size"):
        q.query_points(None, None, torch.zeros((2, 10, 3)), None, 0, 0, None, 2.0, 6.0, torch.zeros((2, 4, 3)), torch.zeros((2, 3)),
                       torch.zeros((2, 3, 3)))


def test_the_minus_one_querier_keeps_its_constructor_options():
    """wcoord_query -1 reads the options once, at construction (point_query.py:33-42); changing them afterwards changes nothing."""
    opt = harness.make_opt(scene.CONFIGS["tiny"])
    q = wq.lighting_fast_querier(CPU, opt)
    before = (q.scaled_vsize_np.copy(), q.radius_limit_np.copy(), q.kernel_size.copy(), q.query_size.copy())
    opt.query_size, opt.kernel_size, opt.vsize, opt.radius_limit_scale = [1, 1, 1], [5, 5, 5], [0.05] * 3, 1.0
    xyz = scene.make_points(scene.CONFIGS["tiny"])["xyz"][None]
    q.get_hyperparameters(opt.vsize, xyz, ranges=opt.ranges)
    after = (q.scaled_vsize_np, q.radius_limit_np, q.kernel_size, q.query_size)
    assert all(np.array_equal(a, b) for a, b in zip(before, after))


def test_fused_module_builds_the_flavour_of_wcoord_query():
    from pointnerf_b200 import query_point_indices as qpi
    from pointnerf_b200.ray_marching import NeuralPoints
    for wcq, cls in ((-1, wq.lighting_fast_querier), (1, wc.lighting_fast_querier), (2, wc.lighting_fast_querier)):
        assert type(NeuralPoints(_opt(wcoord_query=wcq), CPU).querier) is cls
    assert type(NeuralPoints(scene.frustum_opt(scene.FRUSTUM_CONFIGS["dtu_surface"]), CPU).querier) is qpi.lighting_fast_querier
