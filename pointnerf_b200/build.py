"""Compile libpnb200.so (hand-written sm_90a CUDA + C ABI) in-tree with nvcc.  No torch involved.
Also builds libpnb200_selftest.so (test-only wgmma / GEMM-engine self-tests, csrc/selftest/)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libpnb200.so")
LIB_SELFTEST = os.path.join(CSRC, "libpnb200_selftest.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "--fmad=true", "-Xptxas", "-v"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def selftest_sources():
    return sorted(glob.glob(os.path.join(CSRC, "selftest", "*.cu")))


def _headers():
    return glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "selftest", "*.h")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h"))


def _stale(lib, srcs):
    if not os.path.exists(lib):
        return True
    t = os.path.getmtime(lib)
    return any(os.path.getmtime(d) > t for d in srcs + _headers())


def needs_build():
    return _stale(LIB, sources()) or _stale(LIB_SELFTEST, selftest_sources() + sources())


def _compile(srcs, lib, log):
    objs = []
    procs = []
    for src in srcs:                                   # the translation units are independent: compile them concurrently
        obj = src[:-3] + ".o"
        procs.append((src, obj, subprocess.Popen([NVCC] + FLAGS + ["-c", src, "-o", obj], stdout=subprocess.PIPE,
                                                 stderr=subprocess.PIPE, text=True)))
    for src, obj, pr in procs:
        out, err = pr.communicate()
        log.append(err)
        if pr.returncode != 0:
            sys.stderr.write(out + err)
            raise RuntimeError("nvcc failed on %s" % src)
        objs.append(obj)
    r = subprocess.run([NVCC, "-shared", "-o", lib] + objs + ["-lcudart"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed: %s" % lib)


def build(force=False, verbose=False):
    log = []
    if force or _stale(LIB, sources()):
        _compile(sources(), LIB, log)
    if force or _stale(LIB_SELFTEST, selftest_sources() + sources()):     # gemm_selftest.cu includes ../gemm_tc.cu
        _compile(selftest_sources(), LIB_SELFTEST, log)
    if log:
        with open(os.path.join(CSRC, "build.log"), "w") as f:
            f.write("\n".join(log))
        if verbose:
            print("\n".join(log))
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
