"""CPU oracle for the nflows coupling-flow hot path.  TEST INFRASTRUCTURE ONLY.

This module is a *restatement* (functional, weight-dict driven, no nn.Module classes) of the
arithmetic the reference performs on the path SURVEY.md section 8 names.  It exists to CHECK the
CUDA path; the product (`nflows_b200/`) never imports it.  Only `tests/`,
`__graft_entry__.smoke()` and the `cpu_baseline` / `--impl reference` legs of `bench.py` may use it.

Pinning: `oracle/make_golden.py` imports the real reference (a checkout of bayesiains/nflows),
runs both on identical weights/inputs and stores the reference's outputs in
`tests/golden/*.pt`; `tests/test_oracle_golden.py` replays them.  The arithmetic is executed by the
same library the reference uses (PyTorch ATen CPU kernels, fp32), in the same order, so the
agreement is expected to be bit-exact and is asserted at <= 1e-6 relative.

Every function cites the reference lines (relative to the reference's nflows/ package) it follows.

Weights are addressed by the reference's own ``state_dict`` keys, e.g. for a coupling under prefix
``p``: ``p.identity_features``, ``p.transform_features``, ``p.transform_net.initial_layer.weight`` ...
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

DEFAULT_MIN = 1e-3


# --------------------------------------------------------------------------------------------
# spline core
# --------------------------------------------------------------------------------------------
def searchsorted(bin_locations, inputs, eps=1e-6):
    """utils/torchutils.py:134-136.  NOTE: mutates the last knot in place, like the reference."""
    bin_locations[..., -1] += eps
    return torch.sum(inputs[..., None] >= bin_locations, dim=-1) - 1


#: ATen's CPU cumsum accumulates float inputs in DOUBLE (acc_type<float, false>), its CUDA cumsum in float.  The
#: reference run on a GPU therefore has less accurate knots than the CPU goldens; set this to emulate the CUDA
#: semantics (sequential float accumulation) when calibrating tolerances for sharp-bin stress vectors.
F32_CUMSUM = False


def _cumsum(frac):
    if not F32_CUMSUM or frac.dtype != torch.float32:
        return torch.cumsum(frac, dim=-1)
    out = torch.empty_like(frac)
    run = torch.zeros_like(frac[..., 0])
    for i in range(frac.shape[-1]):
        run = run + frac[..., i]
        out[..., i] = run
    return out


def _knots(unnormalized, lo, hi, min_size):
    """transforms/splines/rational_quadratic.py:91-98 (widths) and :106-113 (heights)."""
    k = unnormalized.shape[-1]
    frac = F.softmax(unnormalized, dim=-1)
    frac = min_size + (1 - min_size * k) * frac
    cum = _cumsum(frac)
    cum = F.pad(cum, pad=(1, 0), mode="constant", value=0.0)
    cum = (hi - lo) * cum + lo
    cum[..., 0] = lo
    cum[..., -1] = hi
    return cum, cum[..., 1:] - cum[..., :-1]


def rq_spline(x, uw, uh, ud, inverse=False, left=0.0, right=1.0, bottom=0.0, top=1.0,
              min_bin_width=DEFAULT_MIN, min_bin_height=DEFAULT_MIN, min_derivative=DEFAULT_MIN,
              enable_identity_init=False, check_domain=True):
    """transforms/splines/rational_quadratic.py:66-181.  Returns (outputs, logabsdet) elementwise.

    Raises ValueError("domain") where the reference raises InputOutsideDomain (:81-82) and
    AssertionError for a negative discriminant (:142)."""
    if check_domain and x.numel() and (torch.min(x) < left or torch.max(x) > right):
        raise ValueError("domain")
    k = uw.shape[-1]
    if min_bin_width * k > 1.0:
        raise ValueError("Minimal bin width too large for the number of bins")
    if min_bin_height * k > 1.0:
        raise ValueError("Minimal bin height too large for the number of bins")

    cw, w = _knots(uw, left, right, min_bin_width)
    beta = np.log(2) / (1 - min_derivative) if enable_identity_init else 1
    d = min_derivative + F.softplus(ud, beta=beta)
    ch, h = _knots(uh, bottom, top, min_bin_height)

    idx = searchsorted(ch if inverse else cw, x)[..., None]
    pick = lambda t: t.gather(-1, idx)[..., 0]
    x_cw, x_w, x_ch, x_h = pick(cw), pick(w), pick(ch), pick(h)
    x_delta = pick(h / w)
    x_d, x_d1 = pick(d), pick(d[..., 1:])
    s = x_d + x_d1 - 2 * x_delta

    if inverse:
        u = x - x_ch
        a = u * s + x_h * (x_delta - x_d)
        b = x_h * x_d - u * s
        c = -x_delta * u
        disc = b.pow(2) - 4 * a * c
        assert (disc >= 0).all()
        theta = (2 * c) / (-b - torch.sqrt(disc))
        out = theta * x_w + x_cw
    else:
        theta = (x - x_cw) / x_w
    t1mt = theta * (1 - theta)
    den = x_delta + s * t1mt
    if not inverse:
        num = x_h * (x_delta * theta.pow(2) + x_d * t1mt)
        out = x_ch + num / den
    dnum = x_delta.pow(2) * (x_d1 * theta.pow(2) + 2 * x_delta * t1mt + x_d * (1 - theta).pow(2))
    lad = torch.log(dnum) - 2 * torch.log(den)
    return out, (-lad if inverse else lad)


def rq_spline_unconstrained(x, uw, uh, ud, inverse=False, tails="linear", tail_bound=1.0,
                            min_bin_width=DEFAULT_MIN, min_bin_height=DEFAULT_MIN,
                            min_derivative=DEFAULT_MIN, enable_identity_init=False):
    """transforms/splines/rational_quadratic.py:13-63 (linear tails, boundary derivative constant,
    inside-mask compaction and scatter)."""
    if tails != "linear":
        raise RuntimeError("{} tails are not implemented.".format(tails))
    inside = (x >= -tail_bound) & (x <= tail_bound)
    out = torch.zeros_like(x)
    lad = torch.zeros_like(x)
    ud = F.pad(ud, pad=(1, 1))
    const = np.log(np.exp(1 - min_derivative) - 1)
    ud[..., 0] = const
    ud[..., -1] = const
    out[~inside] = x[~inside]
    if torch.any(inside):
        o, l = rq_spline(x[inside], uw[inside, :], uh[inside, :], ud[inside, :], inverse=inverse,
                         left=-tail_bound, right=tail_bound, bottom=-tail_bound, top=tail_bound,
                         min_bin_width=min_bin_width, min_bin_height=min_bin_height,
                         min_derivative=min_derivative, enable_identity_init=enable_identity_init)
        out[inside] = o
        lad[inside] = l
    return out, lad


# --------------------------------------------------------------------------------------------
# conditioner nets
# --------------------------------------------------------------------------------------------
def residual_net(sd, p, x, num_blocks):
    """nn/nets/resnet.py:39-53 (block) and :92-100 (net); relu, no context, no BN, dropout 0."""
    t = F.linear(x, sd[p + "initial_layer.weight"], sd[p + "initial_layer.bias"])
    for i in range(num_blocks):
        q = "{}blocks.{}.linear_layers.".format(p, i)
        r = F.relu(t)
        r = F.linear(r, sd[q + "0.weight"], sd[q + "0.bias"])
        r = F.relu(r)
        r = F.linear(r, sd[q + "1.weight"], sd[q + "1.bias"])
        t = t + r
    return F.linear(t, sd[p + "final_layer.weight"], sd[p + "final_layer.bias"])


def count_blocks(sd, p):
    n = 0
    while "{}blocks.{}.linear_layers.0.weight".format(p, n) in sd:
        n += 1
    return n


# --------------------------------------------------------------------------------------------
# transforms; each returns (outputs, logabsdet[B])
# --------------------------------------------------------------------------------------------
def rq_coupling(sd, p, x, num_bins, tails="linear", tail_bound=1.0, inverse=False,
                min_bin_width=DEFAULT_MIN, min_bin_height=DEFAULT_MIN, min_derivative=DEFAULT_MIN):
    """transforms/coupling.py:73-130 (split / conditioner / scatter), :279-293 (param reshape,
    column j*M+k = param k of transformed feature j), :549-582 (slices, in-place 1/sqrt(H))."""
    idf, trf = sd[p + "identity_features"], sd[p + "transform_features"]
    xi, xt = x[:, idf], x[:, trf]
    net = p + "transform_net."
    hidden = sd[net + "initial_layer.weight"].shape[0]
    params = residual_net(sd, net, xi, count_blocks(sd, net))
    params = params.reshape(x.shape[0], xt.shape[1], -1)
    uw = params[..., :num_bins]
    uh = params[..., num_bins:2 * num_bins]
    ud = params[..., 2 * num_bins:]
    uw /= np.sqrt(hidden)
    uh /= np.sqrt(hidden)
    kw = dict(inverse=inverse, min_bin_width=min_bin_width, min_bin_height=min_bin_height,
              min_derivative=min_derivative)
    if tails is None:
        yt, lad = rq_spline(xt, uw, uh, ud, **kw)
    else:
        yt, lad = rq_spline_unconstrained(xt, uw, uh, ud, tails=tails, tail_bound=tail_bound, **kw)
    y = torch.empty_like(x)
    y[:, idf] = xi
    y[:, trf] = yt
    return y, torch.sum(lad, dim=1)


def affine_coupling(sd, p, x, inverse=False, additive=False, scale_activation="default"):
    """transforms/coupling.py:212-269.  Blocked param layout: shift = p[:, :d_t], raw scale =
    p[:, d_t:] (:234-238); scale = sigmoid(u+2)+1e-3 (DEFAULT) or clamp(softplus(u)+1e-3, 0, 3)."""
    idf, trf = sd[p + "identity_features"], sd[p + "transform_features"]
    xi, xt = x[:, idf], x[:, trf]
    net = p + "transform_net."
    params = residual_net(sd, net, xi, count_blocks(sd, net))
    dt = xt.shape[1]
    if additive:
        shift, scale = params, torch.ones_like(params)
    else:
        shift, u = params[:, :dt], params[:, dt:]
        if scale_activation == "default":
            scale = torch.sigmoid(u + 2) + 1e-3
        else:
            scale = (F.softplus(u) + 1e-3).clamp(0, 3)
    log_scale = torch.log(scale)
    if inverse:
        yt, lad = (xt - shift) / scale, -torch.sum(log_scale, dim=1)
    else:
        yt, lad = xt * scale + shift, torch.sum(log_scale, dim=1)
    y = torch.empty_like(x)
    y[:, idf] = xi
    y[:, trf] = yt
    return y, lad


def actnorm(sd, p, x, inverse=False):
    """transforms/normalization.py:171-204 (2-D inputs)."""
    scale, shift = torch.exp(sd[p + "log_scale"]).view(1, -1), sd[p + "shift"].view(1, -1)
    total = torch.sum(sd[p + "log_scale"])
    if inverse:
        y = (x - shift) / scale
        return y, -total * y.new_ones(x.shape[0])
    y = scale * x + shift
    return y, total * y.new_ones(x.shape[0])


def lu_factors(sd, p, eps=1e-3):
    """transforms/lu.py:44-54 and :119-121 (np.tril_indices / np.triu_indices entry order)."""
    bias = sd[p + "bias"]
    n = bias.shape[0]
    lo = np.tril_indices(n, k=-1)
    up = np.triu_indices(n, k=1)
    dg = np.diag_indices(n)
    lower = bias.new_zeros(n, n)
    lower[lo[0], lo[1]] = sd[p + "lower_entries"]
    lower[dg[0], dg[1]] = 1.0
    upper = bias.new_zeros(n, n)
    upper[up[0], up[1]] = sd[p + "upper_entries"]
    diag = F.softplus(sd[p + "unconstrained_upper_diag"]) + eps
    upper[dg[0], dg[1]] = diag
    return lower, upper, diag


def lu_linear(sd, p, x, inverse=False, eps=1e-3):
    """transforms/lu.py:56-91: y = (x U^T) L^T + b; inverse by two triangular solves."""
    lower, upper, diag = lu_factors(sd, p, eps)
    lad = torch.sum(torch.log(diag))
    if inverse:
        y = x - sd[p + "bias"]
        y = torch.linalg.solve_triangular(lower, y.t(), upper=False, unitriangular=True)
        y = torch.linalg.solve_triangular(upper, y, upper=True, unitriangular=False).t()
        return y, -lad * x.new_ones(x.shape[0])
    y = F.linear(F.linear(x, upper), lower, sd[p + "bias"])
    return y, lad * x.new_ones(x.shape[0])


def permutation(sd, p, x, inverse=False):
    """transforms/permutations.py:22-45 (index_select; inverse permutation = argsort)."""
    perm = sd[p + "_permutation"]
    if inverse:
        perm = torch.argsort(perm)
    return torch.index_select(x, 1, perm), x.new_zeros(x.shape[0])


def std_normal_log_prob(x):
    """distributions/normal.py:23-33; _log_z is a float64 0-dim tensor, result stays fp32."""
    log_z = torch.tensor(0.5 * np.prod(x.shape[1:]) * np.log(2 * np.pi), dtype=torch.float64)
    return -0.5 * torch.sum(x ** 2, dim=list(range(1, x.dim()))) - log_z


def made(sd, p, x):
    """transforms/made.py:17-283: MADE with residual blocks, relu, no context / BN / dropout; masks are stored buffers."""
    lin = lambda q, t: F.linear(t, sd[q + "weight"] * sd[q + "mask"], sd[q + "bias"])
    t = lin(p + "initial_layer.", x)
    n = 0
    while "{}blocks.{}.linear_layers.0.weight".format(p, n) in sd:
        q = "{}blocks.{}.linear_layers.".format(p, n)
        r = lin(q + "0.", F.relu(t))
        r = lin(q + "1.", F.relu(r))
        t = t + r
        n += 1
    return lin(p + "final_layer.", t)


def ar_rq(sd, p, x, num_bins, tails=None, tail_bound=1.0, inverse=False):
    """transforms/autoregressive.py:37-52 (forward = one MADE pass; inverse = D passes, keeping the last logabsdet) and
    :453-495 (params viewed [B, D, M]; no 1/sqrt(H) rescale because transforms.made.MADE has no hidden_features)."""
    net = p + "autoregressive_net."

    def elementwise(inp, params, inv):
        prm = params.view(inp.shape[0], inp.shape[1], -1)
        uw, uh, ud = prm[..., :num_bins], prm[..., num_bins:2 * num_bins], prm[..., 2 * num_bins:]
        if tails is None:
            y, lad = rq_spline(inp, uw, uh, ud, inverse=inv)
        else:
            y, lad = rq_spline_unconstrained(inp, uw, uh, ud, inverse=inv, tails=tails, tail_bound=tail_bound)
        return y, torch.sum(lad, dim=1)

    if not inverse:
        return elementwise(x, made(sd, net, x), False)
    out = torch.zeros_like(x)
    lad = None
    for _ in range(x.shape[1]):
        out, lad = elementwise(x, made(sd, net, out), True)
    return out, lad


# --------------------------------------------------------------------------------------------
# composite / flow driven by a spec: list of (kind, prefix, kwargs)
# --------------------------------------------------------------------------------------------
_KINDS = {
    "actnorm": actnorm,
    "lu": lu_linear,
    "perm": permutation,
    "rq_coupling": rq_coupling,
    "affine_coupling": affine_coupling,
    "ar_rq": ar_rq,
}


def apply_step(sd, step, x, inverse=False):
    kind, prefix, kwargs = step
    return _KINDS[kind](sd, prefix, x, inverse=inverse, **kwargs)


def composite(sd, spec, x, inverse=False):
    """transforms/base.py:44-60 (_cascade): total starts at zeros and is += per transform."""
    total = x.new_zeros(x.shape[0])
    steps = reversed(spec) if inverse else spec
    for step in steps:
        x, lad = apply_step(sd, step, x, inverse=inverse)
        total += lad
    return x, total


def flow_log_prob(sd, spec, x):
    """flows/base.py:42-49 with a StandardNormal base."""
    z, lad = composite(sd, spec, x)
    return std_normal_log_prob(z) + lad


def flow_log_prob_chunked(sd, spec, x, chunk=4096):
    return torch.cat([flow_log_prob(sd, spec, x[i:i + chunk]) for i in range(0, x.shape[0], chunk)])


def flow_sample_from_noise(sd, spec, noise):
    """flows/base.py:51-75 with the noise given (the reference draws torch.randn itself)."""
    return composite(sd, spec, noise, inverse=True)[0]


def nsf_spec(num_layers, num_bins=8, tail_bound=3.0, prefix="_transform._transforms."):
    """Spec of the cfg-3 recipe (SURVEY.md section 8d): per layer ActNorm, Composite[RandomPermutation,
    LULinear], RQ coupling; prefixes follow the reference state_dict of that construction."""
    spec = []
    for i in range(num_layers):
        b = "{}{}.".format(prefix, 3 * i)
        spec.append(("actnorm", b, {}))
        b = "{}{}._transforms.".format(prefix, 3 * i + 1)
        spec.append(("perm", b + "0.", {}))
        spec.append(("lu", b + "1.", {}))
        b = "{}{}.".format(prefix, 3 * i + 2)
        spec.append(("rq_coupling", b, dict(num_bins=num_bins, tails="linear", tail_bound=tail_bound)))
    return spec
