"""Monotonic rational-quadratic splines (Durkan et al. 2019) -- function API of the reference
(nflows/transforms/splines/rational_quadratic.py:13-181).

CUDA fp32 inputs without autograd are evaluated by `nfk_rqs_elementwise` (one thread per element, all knots in
registers).  Other inputs (CPU, fp64, training) use the differentiable torch formulation below."""
import numpy as np
import torch
from torch.nn import functional as F

from ... import _native as N
from ... import config
from ... import kernels as K
from ..base import InputOutsideDomain

DEFAULT_MIN_BIN_WIDTH = 1e-3
DEFAULT_MIN_BIN_HEIGHT = 1e-3
DEFAULT_MIN_DERIVATIVE = 1e-3


def _use_native(inputs, *params):
    ts = (inputs,) + params
    return all(K.native_ok(t) for t in ts)


def _native_call(desc, inverse, inputs, uw, uh, ud):
    lead = inputs.shape
    with K.on_device_of(inputs):
        flags = K.new_flags(inputs.device)
        k = uw.shape[-1]
        y, lad = K.rqs_elementwise(desc, inverse, inputs, uw.expand(*lead, k), uh.expand(*lead, k),
                                   ud.expand(*lead, ud.shape[-1]), flags=flags)
        if config.check_domain:
            K.raise_for_flags(flags)
    return y, lad


def _bin_edges(unnormalized, lo, hi, min_size):
    k = unnormalized.shape[-1]
    sizes = min_size + (1 - min_size * k) * F.softmax(unnormalized, dim=-1)
    edges = F.pad(torch.cumsum(sizes, dim=-1), pad=(1, 0), mode="constant", value=0.0)
    edges = (hi - lo) * edges + lo
    edges[..., 0] = lo
    edges[..., -1] = hi
    return edges, edges[..., 1:] - edges[..., :-1]


def rational_quadratic_spline(inputs, unnormalized_widths, unnormalized_heights, unnormalized_derivatives, inverse=False,
                              left=0.0, right=1.0, bottom=0.0, top=1.0, min_bin_width=DEFAULT_MIN_BIN_WIDTH,
                              min_bin_height=DEFAULT_MIN_BIN_HEIGHT, min_derivative=DEFAULT_MIN_DERIVATIVE,
                              enable_identity_init=False):
    """Spline on [left,right] -> [bottom,top] with K bins; derivatives has K+1 entries.  Returns (outputs, logabsdet)
    elementwise.  Raises InputOutsideDomain for inputs outside [left, right]."""
    num_bins = unnormalized_widths.shape[-1]
    if _use_native(inputs, unnormalized_widths, unnormalized_heights, unnormalized_derivatives):
        desc = N.spline_desc(num_bins, None, 1.0, left, right, bottom, top, min_bin_width, min_bin_height, min_derivative,
                             enable_identity_init)
        return _native_call(desc, inverse, inputs, unnormalized_widths, unnormalized_heights, unnormalized_derivatives)

    if inputs.numel() and (torch.min(inputs) < left or torch.max(inputs) > right):
        raise InputOutsideDomain()
    N.check_bin_sizes(num_bins, min_bin_width, min_bin_height)
    from ...utils.torchutils import searchsorted

    cw, w = _bin_edges(unnormalized_widths, left, right, min_bin_width)
    ch, h = _bin_edges(unnormalized_heights, bottom, top, min_bin_height)
    beta = np.log(2) / (1 - min_derivative) if enable_identity_init else 1
    d = min_derivative + F.softplus(unnormalized_derivatives, beta=beta)
    idx = searchsorted(ch if inverse else cw, inputs)[..., None]
    at = lambda t: t.gather(-1, idx)[..., 0]
    k_cw, k_w, k_ch, k_h, k_delta = at(cw), at(w), at(ch), at(h), at(h / w)
    d0, d1 = at(d), at(d[..., 1:])
    curv = d0 + d1 - 2 * k_delta
    if inverse:
        u = inputs - k_ch
        qa = u * curv + k_h * (k_delta - d0)
        qb = k_h * d0 - u * curv
        qc = -k_delta * u
        disc = qb.pow(2) - 4 * qa * qc
        assert (disc >= 0).all()
        theta = (2 * qc) / (-qb - torch.sqrt(disc))
        outputs = theta * k_w + k_cw
    else:
        theta = (inputs - k_cw) / k_w
    tt = theta * (1 - theta)
    den = k_delta + curv * tt
    if not inverse:
        outputs = k_ch + k_h * (k_delta * theta.pow(2) + d0 * tt) / den
    dnum = k_delta.pow(2) * (d1 * theta.pow(2) + 2 * k_delta * tt + d0 * (1 - theta).pow(2))
    logabsdet = torch.log(dnum) - 2 * torch.log(den)
    return outputs, (-logabsdet if inverse else logabsdet)


def unconstrained_rational_quadratic_spline(inputs, unnormalized_widths, unnormalized_heights, unnormalized_derivatives,
                                            inverse=False, tails="linear", tail_bound=1.0,
                                            min_bin_width=DEFAULT_MIN_BIN_WIDTH, min_bin_height=DEFAULT_MIN_BIN_HEIGHT,
                                            min_derivative=DEFAULT_MIN_DERIVATIVE, enable_identity_init=False):
    """Spline on [-B, B] with identity (linear) tails outside; derivatives has K-1 entries (the two boundary
    derivatives are fixed so the tails join smoothly)."""
    if tails != "linear":
        raise RuntimeError("{} tails are not implemented.".format(tails))
    num_bins = unnormalized_widths.shape[-1]
    if _use_native(inputs, unnormalized_widths, unnormalized_heights, unnormalized_derivatives):
        desc = N.spline_desc(num_bins, "linear", tail_bound, 0, 0, 0, 0, min_bin_width, min_bin_height, min_derivative,
                             enable_identity_init)
        return _native_call(desc, inverse, inputs, unnormalized_widths, unnormalized_heights, unnormalized_derivatives)

    inside = (inputs >= -tail_bound) & (inputs <= tail_bound)
    outputs = torch.zeros_like(inputs)
    logabsdet = torch.zeros_like(inputs)
    edge = np.log(np.exp(1 - min_derivative) - 1)
    derivs = F.pad(unnormalized_derivatives, pad=(1, 1))
    derivs[..., 0] = edge
    derivs[..., -1] = edge
    outputs[~inside] = inputs[~inside]
    if torch.any(inside):
        outputs[inside], logabsdet[inside] = rational_quadratic_spline(
            inputs[inside], unnormalized_widths[inside, :], unnormalized_heights[inside, :], derivs[inside, :],
            inverse=inverse, left=-tail_bound, right=tail_bound, bottom=-tail_bound, top=tail_bound,
            min_bin_width=min_bin_width, min_bin_height=min_bin_height, min_derivative=min_derivative,
            enable_identity_init=enable_identity_init)
    return outputs, logabsdet
