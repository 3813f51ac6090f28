"""CPU: every C entry point that picks a kernel instantiation from its inputs rejects the inputs no instantiation serves, with
the return code and pnb_last_error text of the C ABI, and accepts the ones it accepted before.

The calls pass placeholder addresses and run in a child process that sees no CUDA device, so every case is one that returns
before any CUDA call: a check that goes missing shows up as a CUDA error (no device) instead of a launch on host addresses."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

OK, INVALID, UNSUPPORTED = 0, -1, -4
FAKE = 0x10000            # placeholder device address; never dereferenced
BIG = 1 << 40             # workspace / buffer size that passes every size check
XS = {"none": (0, 0, 0), "all": (1, 1, 1), "no_loc": (1, 0, 1), "no_dir": (1, 1, 0)}   # xs_loc_w, xs_loc, xs_dir given


def _inputs(lib, F, mlp_F, xs, frames):
    q = lib.Query()
    q.R, q.SR, q.K, q.cap_samples = 1, 4, 8, 1
    q.xs_loc_w, q.xs_loc, q.xs_dir = [FAKE if g else None for g in XS[xs]]
    pts = lib.Points()
    pts.xyz = pts.emb = pts.color = pts.dir = pts.conf = FAKE
    pts.N, pts.rw2c, pts.feat_dim = 1, FAKE if frames else None, F
    mlp = lib.Mlp()
    for i in range(9):
        mlp.w[i] = mlp.b[i] = FAKE
    mlp.feat_dim = F if mlp_F is None else mlp_F
    return q, pts, mlp


def _call(lib, l, fn, F=32, mlp_F=None, xs="none", frames=False, n_rows=1):
    """The return value of fn on these inputs (every other argument valid)."""
    q, pts, mlp = _inputs(lib, F, mlp_F, xs, frames)
    opts = lib.ShadeOpts()
    if fn == "pnb_shade_forward":
        return l.pnb_shade_forward(q, pts, mlp, opts, FAKE, None, 0, None)
    if fn == "pnb_shade_forward_tc":
        return l.pnb_shade_forward_tc(q, pts, mlp, FAKE, None, opts, FAKE, FAKE, BIG, 1, lib.TC_PAIRS | lib.TC_COLOR, FAKE, None)
    if fn == "pnb_shade_backward":
        grads = (C.c_void_p * 9)(*[FAKE] * 9)
        return l.pnb_shade_backward(q, pts, mlp, opts, FAKE, FAKE, None, None, 1, 1, FAKE, FAKE, FAKE, FAKE, grads, grads, FAKE, BIG,
                                    0, FAKE, None)
    if fn == "pnb_point_pre":
        return l.pnb_point_pre(pts, mlp, FAKE, BIG, None)
    if fn == "pnb_aux_outputs":
        return l.pnb_aux_outputs(q, pts, FAKE, n_rows, FAKE, FAKE, FAKE, FAKE, None)
    if fn == "pnb_probe_outputs":
        return l.pnb_probe_outputs(q, pts, FAKE, n_rows, FAKE, *([FAKE] * 9), None)
    if fn == "pnb_mlp_pack":
        return l.pnb_mlp_pack(mlp, FAKE, BIG, None)
    if fn == "pnb_backward_tables":
        out = (C.c_void_p * 10)()
        return l.pnb_backward_tables(FAKE, BIG, 1, 1, F, out)
    if fn == "pnb_mlp_pack_bytes":
        return l.pnb_mlp_pack_bytes(F)
    if fn == "pnb_backward_bytes":
        return l.pnb_backward_bytes(1, 1, F)
    raise KeyError(fn)


FRAMES_XS = "the frustum query's samples are shaded with point_features_dim 63 and a uniform Rw2c only"
PROBE_XS = "the frustum query's samples need point_features_dim 63"

# (entry point, inputs, expected return value, expected pnb_last_error text or None)
CASES = []
for _fn in ("pnb_shade_forward", "pnb_shade_forward_tc", "pnb_shade_backward"):     # the frame-reading kernels
    CASES += [
        (_fn, dict(F=64), UNSUPPORTED, _fn + ": point_features_dim 64 unsupported (32 or 63)"),
        (_fn, dict(F=63, mlp_F=0), INVALID, _fn + ": the MLP was built for point_features_dim 32, the points have 63"),
        (_fn, dict(F=32, mlp_F=63), INVALID, _fn + ": the MLP was built for point_features_dim 63, the points have 32"),
        (_fn, dict(F=63, xs="no_loc"), INVALID, _fn + ": explicit samples need xs_loc_w, xs_loc and xs_dir"),
        (_fn, dict(F=63, xs="no_dir"), INVALID, _fn + ": explicit samples need xs_loc_w, xs_loc and xs_dir"),
        (_fn, dict(F=32, xs="no_loc"), INVALID, _fn + ": explicit samples need xs_loc_w, xs_loc and xs_dir"),
        (_fn, dict(F=32, xs="all"), UNSUPPORTED, _fn + ": " + FRAMES_XS),
        (_fn, dict(F=63, xs="all", frames=True), UNSUPPORTED, _fn + ": " + FRAMES_XS),
    ]
CASES += [
    ("pnb_point_pre", dict(F=64), UNSUPPORTED, "pnb_point_pre: point_features_dim 64 unsupported (32 or 63)"),
    ("pnb_point_pre", dict(F=63, mlp_F=0), INVALID, "pnb_point_pre: the MLP was built for point_features_dim 32, the points have 63"),
    # the aux outputs check F but have no F axis, and no check on explicit samples (n_rows = 0: accepted before any CUDA call)
    ("pnb_aux_outputs", dict(F=64), UNSUPPORTED, "pnb_aux_outputs: point_features_dim 64 unsupported (32 or 63)"),
    ("pnb_aux_outputs", dict(F=64, n_rows=0), UNSUPPORTED, "pnb_aux_outputs: point_features_dim 64 unsupported (32 or 63)"),
    ("pnb_aux_outputs", dict(F=32, xs="no_loc", frames=True, n_rows=0), OK, None),
    # the probe: explicit samples need F = 63 only (frames allowed, xs_loc / xs_dir unread), checked only when there are rows
    ("pnb_probe_outputs", dict(F=64), UNSUPPORTED, "pnb_probe_outputs: point_features_dim 64 unsupported (32 or 63)"),
    ("pnb_probe_outputs", dict(F=64, n_rows=0), UNSUPPORTED, "pnb_probe_outputs: point_features_dim 64 unsupported (32 or 63)"),
    ("pnb_probe_outputs", dict(F=32, xs="all"), UNSUPPORTED, "pnb_probe_outputs: " + PROBE_XS),
    ("pnb_probe_outputs", dict(F=32, xs="no_loc"), UNSUPPORTED, "pnb_probe_outputs: " + PROBE_XS),
    ("pnb_probe_outputs", dict(F=32, xs="all", frames=True), UNSUPPORTED, "pnb_probe_outputs: " + PROBE_XS),
    ("pnb_probe_outputs", dict(F=32, xs="all", n_rows=0), OK, None),
    ("pnb_mlp_pack", dict(F=64), UNSUPPORTED, "pnb_mlp_pack: point_features_dim 64 unsupported (32 or 63)"),
    ("pnb_mlp_pack", dict(F=-1), UNSUPPORTED, "pnb_mlp_pack: point_features_dim -1 unsupported (32 or 63)"),
    ("pnb_backward_tables", dict(F=64), UNSUPPORTED, "pnb_backward_tables: point_features_dim 64 unsupported"),
    # the *_bytes functions: 0 for a width without an instantiation
    ("pnb_mlp_pack_bytes", dict(F=64), 0, None),
    ("pnb_mlp_pack_bytes", dict(F=31), 0, None),
    ("pnb_backward_bytes", dict(F=64), 0, None),
    ("pnb_backward_bytes", dict(F=31), 0, None),
]


def _case_id(case):
    fn, kw, _, _ = case
    return fn + "-" + "-".join("%s=%s" % kv for kv in sorted(kw.items()))


def _run_cases():
    """Child process: the return value and error text of every case, as JSON on stdout."""
    sys.path.insert(0, ROOT)
    from pointnerf_b200 import lib
    l = lib.load()
    out = {}
    for case in CASES:
        rc = _call(lib, l, case[0], **case[1])
        out[_case_id(case)] = [rc, l.pnb_last_error().decode()]
    print(json.dumps(out))


@pytest.fixture(scope="module")
def results():
    from pointnerf_b200 import build
    build.build()
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, os.path.abspath(__file__)], env=env, cwd=ROOT, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_variant_inputs(results, case):
    fn, kw, want_rc, want_err = case
    rc, err = results[_case_id(case)]
    assert rc == want_rc, "%s: returned %d, expected %d (%s)" % (fn, rc, want_rc, err)
    if want_err is not None:
        assert err == want_err


def test_sizes_of_the_instantiated_widths():
    """0 is read as 32; both instantiated widths have a size (the zero above is the rejection, not an empty buffer)."""
    from pointnerf_b200 import build, lib
    build.build()
    l = lib.load()
    assert l.pnb_mlp_pack_bytes(0) == l.pnb_mlp_pack_bytes(32) > 0 and l.pnb_mlp_pack_bytes(63) > 0
    assert l.pnb_backward_bytes(1, 1, 0) == l.pnb_backward_bytes(1, 1, 32) > 0 and l.pnb_backward_bytes(1, 1, 63) > 0


if __name__ == "__main__":
    _run_cases()
