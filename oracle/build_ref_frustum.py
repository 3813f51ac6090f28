"""TEST INFRASTRUCTURE ONLY -- compiles the REFERENCE's own perspective-frustum query kernels
(models/neural_points/query_point_indices.py:131-600, the CUDA source string it hands to pycuda's SourceModule) with a launcher of
ours (oracle/frustum_ref_launch.cu) into oracle/_ref/libref_frustum.so (git-ignored).

The source string is read from the reference file at build time (parsed with `ast`, never copied into this repository), written to
oracle/_ref/frustum_ref_kernels.cu and compiled with nvcc's defaults for sm_90a, as pycuda compiles it (no -use_fast_math, FMA
contraction on).  oracle/record_ref_frustum.py runs the result on an H100 to record tests/golden/ref_frustum_*.npz.

    python -m oracle.build_ref_frustum        # needs the reference tree; nvcc cross-compiles for sm_90a
"""
import ast
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.join(ROOT, "oracle")
from oracle.ref_shim import REF  # noqa: E402

REF_FILE = os.path.join(REF, "models", "neural_points", "query_point_indices.py")
OUT = os.path.join(ROOT, "oracle", "_ref")
KERNELS = os.path.join(OUT, "frustum_ref_kernels.cu")
LIB = os.path.join(OUT, "libref_frustum.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
KN = 8   # the DTU scripts' K; the string is specialised with `#define KN <opt.K>`


def kernel_source(K=KN):
    """The CUDA string of build_cuda() with opt.K = K: `\"\"\"...#define KN \"\"\" + str(self.opt.K) + \"\"\"...\"\"\"`."""
    with open(REF_FILE) as f:
        tree = ast.parse(f.read())
    for node in ast.walk(tree):
        if isinstance(node, ast.Call) and getattr(node.func, "id", None) == "SourceModule":
            parts = []

            def flat(n):
                if isinstance(n, ast.BinOp) and isinstance(n.op, ast.Add):
                    flat(n.left)
                    flat(n.right)
                elif isinstance(n, ast.Constant) and isinstance(n.value, str):
                    parts.append(n.value)
                else:                      # str(self.opt.K)
                    parts.append(str(K))
            flat(node.args[0])
            return "".join(parts)
    raise RuntimeError("no SourceModule(...) call in %s" % REF_FILE)


def build(verbose=False):
    if not os.path.isfile(REF_FILE):
        raise RuntimeError("oracle.build_ref_frustum needs the reference source at %s" % REF_FILE)
    os.makedirs(OUT, exist_ok=True)
    with open(KERNELS, "w") as f:
        f.write(kernel_source())
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC", "-I", OUT,
           os.path.join(HERE, "frustum_ref_launch.cu"), "-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode:
        raise RuntimeError("nvcc failed on the reference frustum kernels")
    return LIB


if __name__ == "__main__":
    print("built", build(verbose=True))
