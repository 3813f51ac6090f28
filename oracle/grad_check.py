"""TEST INFRASTRUCTURE ONLY -- comparison of gradients with a float64 oracle that ran with the LeakyReLU masks of the computation under
test (oracle/shade_oracle.py, `slopes=`).  Once the masks agree, nothing but rounding separates the two, so every point and every MLP
tensor is held to one strict bound relative to its tensor's scale, without an allowance for outliers.

The one exception is points_conf of point 0: every empty neighbour slot gathers point 0 (clamp(pidx, 0), neural_points.py:707), so
a loss on conf_coefficient adds one term per padded slot into it, tens of thousands in an fp32 sum.  Its bound follows from that count.
"""
import numpy as np
import torch

LAYERS = ("block1.0", "block1.2", "block3.0", "block3.2", "color_branch.0", "color_branch.2", "color_branch.4")
U32 = 2.0 ** -24    # unit roundoff of fp32


def rel_point_errors(a, ref):
    """[N] largest |a - ref| of each point (over its channels) relative to max |ref| of the tensor.  a, ref: [1,N,C] or [N,C]."""
    a = np.asarray(a, np.float64)
    ref = np.asarray(ref, np.float64).reshape(a.shape)
    a, ref = a.reshape(-1, a.shape[-1]), ref.reshape(-1, a.shape[-1])
    scale = max(np.abs(ref).max(), 1e-30)
    return np.abs(a - ref).max(axis=-1) / scale


def rel_error(a, ref):
    a = np.asarray(a, np.float64)
    ref = np.asarray(ref, np.float64).reshape(a.shape)
    return float(np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30))


def check_points(a, ref, name, rtol):
    """Every point within rtol of the tensor's scale.  Returns the largest relative error."""
    e = rel_point_errors(a, ref)
    bad = np.nonzero(e > rtol)[0]
    assert bad.size == 0, "%s: %d points beyond %.1e of scale (worst %.3e at point %d)" % (name, bad.size, rtol, e.max(), int(e.argmax()))
    return float(e.max())


def point0_conf_bound(n0, ref0, term=1e-3):
    """Bound of the error of an fp32 sum into point 0's conf gradient: n0 terms (one per gathered slot), each rounding step off by at
    most U32 of the partial sum, which stays below |ref0| plus the padded terms' `term` each (1e-3: the loss's
    1e-3 * conf_coefficient.sum())."""
    return n0 * U32 * (abs(float(ref0)) + term * n0)


def check_conf(a, ref, n0, rtol):
    """points_conf: points 1.. within rtol of their scale (point 0 left out of it: its padded terms would dominate the scale), point 0
    within point0_conf_bound.  n0: number of [R',SR,K] slots whose clamped index is 0.  Returns the largest relative error of 1.."""
    a = np.asarray(a, np.float64).reshape(-1)
    ref = np.asarray(ref, np.float64).reshape(-1)
    e = check_points(a[1:, None], ref[1:, None], "points_conf (points 1..)", rtol)
    d0, b0 = abs(a[0] - ref[0]), point0_conf_bound(n0, ref[0])
    assert d0 <= b0, "points_conf of point 0: |diff| %.3e > %.3e (%d accumulated terms)" % (d0, b0, n0)
    return e


class MaskRecorder:
    """Stands in for torch.nn.functional in oracle/shade_oracle.py (monkeypatch its `F`): records the slope each LeakyReLU unit takes
    (1 above zero, else the negative slope, as torch's derivative does) in call order, which is the layer order of `slopes=`."""

    def __init__(self, functional):
        self._f, self.slopes = functional, []

    def __getattr__(self, k):
        return getattr(self._f, k)

    def leaky_relu(self, x, negative_slope):
        self.slopes.append(torch.where(x > 0, 1.0, negative_slope).to(torch.float64).detach())
        return self._f.leaky_relu(x, negative_slope)


def flipped_rows(slopes_a, slopes_b):
    """Per layer, the rows in which some unit has a different slope in the two mask sets."""
    return [(sa != sb).any(dim=-1) for sa, sb in zip(slopes_a, slopes_b)]
