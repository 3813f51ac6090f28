"""TEST INFRASTRUCTURE ONLY -- compiles the REFERENCE's own CUDA query extension (two source files, read in place in the
reference tree named by oracle/ref_shim.py; nothing is copied) into oracle/_ref/ (git-ignored).  It is the un-modified
`query_worldcoords_cuda` torch extension that models/neural_points/point_query.py:15-22 of the reference JIT-builds at import;
oracle/record_ref_kernel.py runs it on an H100 to record the reference kernel's query results that tests/test_gpu_ref_kernel.py
compares libpnb200 with (tests/golden/ref_kernel_*.npz).

    python -m oracle.build_ref        # needs the reference tree; nvcc cross-compiles for sm_90a
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from oracle.ref_shim import REF  # noqa: E402

REF_SRC = os.path.join(REF, "models", "neural_points", "cuda")
OUT = os.path.join(ROOT, "oracle", "_ref")
NAME = "query_worldcoords_cuda"


def build(verbose=False):
    if not os.path.isdir(REF_SRC):
        raise RuntimeError("oracle.build_ref needs the reference sources at %s" % REF_SRC)
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")       # the build machine may have no GPU: name the target instead of probing one
    from torch.utils.cpp_extension import load
    return load(name=NAME, sources=[os.path.join(REF_SRC, f) for f in ("query_worldcoords.cpp", "query_worldcoords.cu")],
                build_directory=OUT, verbose=verbose, extra_cuda_cflags=["-lineinfo"])


def load_prebuilt():
    """Import the extension built by build() (no compiler, no reference tree needed)."""
    import importlib.util
    import torch  # noqa: F401  (libtorch symbols must be loaded first)
    path = os.path.join(OUT, NAME + ".so")
    if not os.path.isfile(path):
        return None
    spec = importlib.util.spec_from_file_location(NAME, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    m = build(verbose=True)
    print("built", os.path.join(OUT, NAME + ".so"), "exports", [n for n in dir(m) if not n.startswith("_")])
