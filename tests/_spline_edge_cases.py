"""One case table of the spline's settings and edge inputs, shared by test_spline_edges_host.py (the kernel source built for the
CPU) and test_spline_edges_gpu.py (the fused coupling kernels, the row kernel and its backward on a GPU).

  * SETTINGS: the minimum bin sizes and derivative, the tail bound and the divisor of the width and height logits, each with a
    name.  Every one of them reaches the kernels only through the spline descriptor (SplineParams: min_w, mix_w, edge_ud ...).
  * VECTORS: crafted raw parameter vectors in the reference's layout [K widths | K heights | K-1 (linear tails) or K+1
    derivatives]: saturated softmax arguments, one dominant bin, derivative logits at and around softplus's threshold of 20.
  * edge inputs of each vector, computed in fp64 from its exact parameters: the interior knots and the fp32 values either side
    of them, the ends of the interval, the tail bound and what lies past it, then random fill.

The fused kernels evaluate the spline on (packed final-layer weight rows) x (trunk output) + bias.  A feature whose weight rows
are zero sees exactly its bias (the epilogue computes fmaf(0, inv_acc_scale, b) == b): crafted_coupling writes the crafted
vectors there, so the spline inside the tensor-core kernels runs on known parameters whatever the trunk computes.

Truth is the fp64 oracle on the exact parameters; the yardstick is the same oracle in fp32 with the CUDA reference's float
prefix sum (O.F32_CUMSUM), as in _spline_cases.py."""
from collections import namedtuple

import torch

from nflows_b200 import _native as N
from nflows_b200 import transforms as T
from nflows_b200.nn.nets import ResidualNet
from oracle import flow_oracle as O

BINS = (4, 8, 10, 16)                 # the bin counts the fused kernels are instantiated for (10: the padded binary search)
DEFAULT_MINS = (1e-3, 1e-3, 1e-3)

# name, (min_bin_width, min_bin_height, min_derivative), tail bound, divisor of the width / height logits.  full_mins depends on K.
Setting = namedtuple("Setting", "name mins tail_bound divisor")
SETTING_NAMES = ("default", "mins", "full_mins", "steep_min_derivative", "tail_bound_0.5", "tail_bound_8", "divisor_1",
                 "divisor_8")


def setting(name, bins):
    base = dict(mins=DEFAULT_MINS, tail_bound=3.0, divisor=4.0)
    over = {
        "default": {},
        "mins": dict(mins=(1e-2, 5e-3, 5e-2)),
        # every bin at its minimum: mix 0, uniform bins whatever the logits (K = 10: 0.1 * 10 is 1.0 in double)
        "full_mins": dict(mins=(1.0 / bins, 1.0 / bins, 1e-3)),
        "steep_min_derivative": dict(mins=(1e-3, 1e-3, 0.5)),     # moves the boundary logit edge_ud far from its default
        "tail_bound_0.5": dict(tail_bound=0.5),
        "tail_bound_8": dict(tail_bound=8.0),
        "divisor_1": dict(divisor=1.0),
        "divisor_8": dict(divisor=8.0),                           # sqrt(64): a conditioner of hidden width 64
    }[name]
    return Setting(name, **dict(base, **over))


def settings(bins, tails):
    """The settings that change something for this tail mode (the tail bound means nothing to a spline on [0, 1])."""
    names = SETTING_NAMES if tails == "linear" else tuple(n for n in SETTING_NAMES if not n.startswith("tail_bound"))
    return [setting(n, bins) for n in names]


def desc(bins, tails, s):
    return N.spline_desc(bins, tails, s.tail_bound, 0.0, 1.0, 0.0, 1.0, *s.mins, False, s.divisor)


def num_derivatives(bins, tails):
    return bins - 1 if tails == "linear" else bins + 1


def num_params(bins, tails):
    return 3 * bins - 1 if tails == "linear" else 3 * bins + 1


def interval(tails, s):
    return (-s.tail_bound, s.tail_bound) if tails == "linear" else (0.0, 1.0)


# ---- crafted raw parameter vectors -------------------------------------------------------------------------------------------
VECTORS = ("zero", "random", "one_wide_bin", "one_tall_bin", "shift_minus_1000", "shift_plus_1000", "steep", "flat")


def _f32_next(v, toward):
    return float(torch.nextafter(torch.tensor(v, dtype=torch.float32), torch.tensor(toward, dtype=torch.float32)))


STEEP_LOGITS = (25.0, 20.5, 20.0, _f32_next(20.0, 30.0), _f32_next(20.0, 0.0))   # around F.softplus's threshold of 20


def vector(name, bins, tails, s):
    """(uw, uh, ud) of one crafted vector, fp32, raw (the kernels and the oracle divide uw, uh by the setting's divisor)."""
    g = torch.Generator().manual_seed(17 * bins + (tails is None) + 101 * VECTORS.index(name))
    nd = num_derivatives(bins, tails)
    moderate = lambda n, scale: torch.randn(n, generator=g) * scale
    uw, uh = moderate(bins, 1.5 * s.divisor), moderate(bins, 1.5 * s.divisor)
    ud = moderate(nd, 1.5)
    if name == "zero":
        uw, uh, ud = torch.zeros(bins), torch.zeros(bins), torch.zeros(nd)
    elif name == "one_wide_bin":                  # the other bins at their minimum width
        uw = torch.zeros(bins)
        uw[bins // 2] = 40.0 * s.divisor
    elif name == "one_tall_bin":                  # the last bin: the inverse's top end
        uh = torch.zeros(bins)
        uh[bins - 1] = 40.0 * s.divisor
    elif name == "shift_minus_1000":              # exp underflows unless the softmax subtracts the maximum
        uw, uh = uw - 1000.0, uh - 1000.0
    elif name == "shift_plus_1000":               # ... or overflows
        uw, uh = uw + 1000.0, uh + 1000.0
    elif name == "steep":
        ud = torch.tensor([STEEP_LOGITS[k % len(STEEP_LOGITS)] for k in range(nd)])
    elif name == "flat":
        ud = torch.full((nd,), -30.0)
    return uw.float(), uh.float(), ud.float()


# ---- edge inputs -------------------------------------------------------------------------------------------------------------
PER_VECTOR = 384                  # elements of each vector: its edge inputs, then random fill


def knots64(u, lo, hi, min_size, divisor):
    """The fp64 knots of one raw width or height vector (first and last forced to lo, hi)."""
    return O._knots(u.double()[None] / divisor, lo, hi, min_size)[0][0]


def edge_inputs(uw, uh, bins, tails, inverse, s, seed):
    """(x fp32 [PER_VECTOR], kind list): the edge inputs of one vector in the direction's input space, then random fill."""
    lo, hi = interval(tails, s)
    u, min_size = (uh, s.mins[1]) if inverse else (uw, s.mins[0])
    kn = knots64(u, lo, hi, min_size, s.divisor)
    xs, kinds = [], []
    for k in range(1, bins):
        v = float(torch.tensor(float(kn[k]), dtype=torch.float32))
        for x, kind in ((v, "knot"), (_f32_next(v, hi + 1.0), "knot_up"), (_f32_next(v, lo - 1.0), "knot_down")):
            xs.append(x)
            kinds.append(kind)
    xs += [lo, hi]
    kinds += ["left", "right"]
    if tails == "linear":
        B = s.tail_bound
        far = [(_f32_next(B, 2 * B), "ulp_out"), (_f32_next(-B, -2 * B), "ulp_out"), (2 * B, "out"), (-2 * B, "out"),
               (1e30, "huge"), (-1e30, "huge"), (float("nan"), "nan")]
        xs += [x for x, _ in far]
        kinds += [k for _, k in far]
    g = torch.Generator().manual_seed(seed)
    n_fill = PER_VECTOR - len(xs)
    fill = lo + (hi - lo) * torch.rand(n_fill, generator=g)
    x = torch.cat([torch.tensor(xs, dtype=torch.float32), fill.float()])
    return x, kinds + ["random"] * n_fill


Table = namedtuple("Table", "x uw uh ud vec kind")


def table(bins, tails, inverse, s, vectors=VECTORS):
    """Every crafted element of one (K, tails, direction, setting): x [n], uw, uh [n, K], ud [n, K -/+ 1] (fp32, raw), the
    index of each element's vector, and the kind of each input ("knot", "left", "out", "random", ...)."""
    xs, ps, vec, kinds = [], [], [], []
    for i, name in enumerate(vectors):
        uw, uh, ud = vector(name, bins, tails, s)
        x, kind = edge_inputs(uw, uh, bins, tails, inverse, s, seed=1000 * bins + 10 * i + inverse)
        xs.append(x)
        ps.append([t[None].expand(len(x), -1) for t in (uw, uh, ud)])
        vec += [i] * len(x)
        kinds += kind
    cat = lambda j: torch.cat([p[j] for p in ps]).contiguous()
    return Table(torch.cat(xs), cat(0), cat(1), cat(2), torch.tensor(vec), kinds)


def kind_mask(tab, *names):
    return torch.tensor([k in names for k in tab.kind])


KNOTS = ("knot", "knot_up", "knot_down")


def assert_as_accurate(got, ref32, truth, tab, what):
    """assert_statistically_as_accurate (test_native_parity.py) with the knot inputs and the right end (top) held to its
    worst-element bar only (check_edges holds the right end to its own bar).  Next to
    a knot any fp32 evaluation is ill-conditioned (a 1-ulp knot difference moves theta by percents, and the fp32 and fp64 knots
    may put the input in neighbouring bins), so which evaluation errs most there is luck; the table puts 3 (K - 1) such inputs
    in every vector -- up to a tenth of the elements -- and they would set the percentiles; so would the eight right ends, a
    quarter of a percent, whose inverse a flat or steep last bin makes ill-conditioned.  The percentiles are those of the other
    elements (the left end, the tails, the random fill), held to 5x the reference's instead of 2x: with the steep and flat
    vectors the host build of the scan form reached 4.2x-4.4x at the 99.9th percentile of a table (its third-worst element, a
    log|det| of 6e-5 against 1.5e-5), at K = 4 without tails.  The worst element over all of them
    stays within 15x the reference's."""
    from test_native_parity import TOL, _elementwise_err
    got, ref32, truth = got.detach().cpu(), ref32.detach().cpu(), truth.detach().cpu()
    # where the reference has no result (NaN for a finite truth: the log|det| of its inverse on the height knots of a flat bin,
    # theta rounded past 1) there is no bar to scale: the kernel's value must be finite, and the element leaves the comparison
    failed = torch.isnan(ref32) & torch.isfinite(truth)
    assert bool(torch.isfinite(got[failed]).all()), (what, "where the reference fails")
    got, ref32, truth = got[~failed], ref32[~failed], truth[~failed]
    keep = ~kind_mask(tab, "right", *KNOTS)[~failed]
    e, r = _elementwise_err(got[keep], truth[keep]), _elementwise_err(ref32[keep], truth[keep])
    n = len(e)
    for q in (0.99, 0.999):
        i = min(n - 1, int(q * n))
        assert e[i] <= 5 * r[i] + TOL, (what, q, float(e[i]), float(r[i]))
    e, r = _elementwise_err(got, truth), _elementwise_err(ref32, truth)
    assert e[-1] <= 15 * r[-1] + TOL, (what, "max", float(e[-1]), float(r[-1]))


def assert_inverse_backward_error(got_y, ref_y, truth_y, truth_lad, tab, what):
    """assert_as_accurate's bars on the inverse's error measured in its input space, |y - y64| times the forward's slope
    exp(-log|det| of the inverse), off the knots and the top, for the kernel and the reference alike.  Where a bin is nearly
    flat in the forward (inverse log|det| up to +8: slope 3e-4) an x error of 1e-4 is an input error below one fp32 ulp, and
    which fp32 evaluation lands closest in x is luck."""
    from test_native_parity import TOL
    keep = ~kind_mask(tab, "right", *KNOTS)
    slope = torch.exp(-truth_lad[keep].double())
    e = ((got_y.detach().cpu().double() - truth_y)[keep].abs() * slope).sort().values
    r = ((ref_y.double() - truth_y)[keep].abs() * slope).sort().values
    n = len(e)
    for q in (0.99, 0.999):
        i = min(n - 1, int(q * n))
        assert e[i] <= 5 * r[i] + TOL, (what, "input space", q, float(e[i]), float(r[i]))
    assert e[-1] <= 15 * r[-1] + TOL, (what, "input space", "max", float(e[-1]), float(r[-1]))


def params_of(tab):
    """[n, M]: the raw parameters of each element in the row kernel's layout."""
    return torch.cat([tab.uw, tab.uh, tab.ud], -1).contiguous()


def oracle(x, uw, uh, ud, tails, inverse, s, dtype):
    """(y, log|det|) of the oracle in `dtype` on the CPU at setting s; uw, uh are divided by the divisor as the reference does."""
    x, uw, uh, ud = (t.detach().cpu().to(dtype) for t in (x, uw, uh, ud))
    kw = dict(inverse=inverse, min_bin_width=s.mins[0], min_bin_height=s.mins[1], min_derivative=s.mins[2])
    if tails == "linear":
        return O.rq_spline_unconstrained(x, uw / s.divisor, uh / s.divisor, ud.clone(), tail_bound=s.tail_bound, **kw)
    return O.rq_spline(x, uw / s.divisor, uh / s.divisor, ud.clone(), **kw)


def truth_and_yardstick(tab, tails, inverse, s):
    """((y, lad) fp64, (y, lad) fp32 with the CUDA reference's float prefix sum) of every element.  The caller sets O.F32_CUMSUM."""
    assert O.F32_CUMSUM, "the yardstick is the reference as it runs on CUDA: set O.F32_CUMSUM (monkeypatch)"
    args = (tab.x, tab.uw, tab.uh, tab.ud, tails, inverse, s)
    truth = oracle(*args, torch.float64)
    return truth, yardstick(tab, tails, inverse, s, truth)


def yardstick(tab, tails, inverse, s, truth):
    """The fp32 oracle on every element.  Where it has no result -- the inverse's discriminant rounds below zero, so the
    reference itself raises (K = 8, one dominant width bin, inputs on a height knot) -- the element gets the fp64 truth rounded
    to fp32: the best any fp32 evaluation can do, so such an element only makes the bar stricter."""
    try:
        return oracle(tab.x, tab.uw, tab.uh, tab.ud, tails, inverse, s, torch.float32)
    except AssertionError:
        pass
    y, lad = (t.float().clone() for t in truth)
    for i in range(len(tab.x)):
        one = lambda t: t[i:i + 1]
        try:
            y[i:i + 1], lad[i:i + 1] = oracle(one(tab.x), one(tab.uw), one(tab.uh), one(tab.ud), tails, inverse, s, torch.float32)
        except AssertionError:
            pass
    return y, lad


# ---- the crafted coupling ----------------------------------------------------------------------------------------------------
def crafted_coupling(bins, tails, s, vectors, d_id=8, n_random=8, hidden=64, num_blocks=1, seed=0):
    """A PiecewiseRationalQuadraticCouplingTransform (CPU, eval) with the setting's minimum sizes and tail bound on d_id identity
    features followed by len(vectors) crafted and n_random random transformed features.  Crafted feature j has its final-layer
    rows j*M .. j*M + M - 1 zeroed and its bias entries set to the vector: the spline sees exactly the vector.  The random
    features keep the conditioner's weights (times 2, as _coupling_checks.build), so the final layer stays a real GEMM.
    The module divides the width / height logits by sqrt(hidden), not by s.divisor."""
    torch.manual_seed(seed)
    d_t = len(vectors) + n_random
    mask = torch.cat([-torch.ones(d_id), torch.ones(d_t)])
    t = T.PiecewiseRationalQuadraticCouplingTransform(
        mask, lambda i, o: ResidualNet(i, o, hidden_features=hidden, num_blocks=num_blocks), num_bins=bins, tails=tails,
        tail_bound=s.tail_bound, min_bin_width=s.mins[0], min_bin_height=s.mins[1], min_derivative=s.mins[2]).eval()
    m = num_params(bins, tails)
    final = t.transform_net.final_layer
    with torch.no_grad():
        final.weight.mul_(2.0)
        final.bias.mul_(2.0)
        for j, v in enumerate(vectors):
            final.weight[j * m:(j + 1) * m].zero_()
            final.bias[j * m:(j + 1) * m] = torch.cat(v)
    return t


# ---- module-level cases: one per route of the coupling's spline head ---------------------------------------------------------
# route "step": the coupling-step kernel (hidden 64); "final": the trunk, then the fused final-layer kernel (hidden 288, wider than
# the step kernel takes); "rows": config.fuse_coupling off, the last layer into HBM and nfk_rqs_rows.
ModuleCase = namedtuple("ModuleCase", "name route hidden bins tails tail_bound")
MODULE_CASES = [ModuleCase("{}_B{}".format(route, b), route, hidden, bins, "linear", b)
                for route, hidden in (("step", 64), ("final", 288), ("rows", 64))
                for b, bins in ((0.5, 10), (8.0, 16))]


def module_setting(case):
    """The "mins" setting with the case's tail bound and the divisor the module applies (sqrt(hidden))."""
    return setting("mins", case.bins)._replace(name="mins_B{}".format(case.tail_bound), tail_bound=case.tail_bound,
                                               divisor=float(case.hidden) ** 0.5)


def module_coupling(case, seed=0):
    s = module_setting(case)
    vectors = [vector(name, case.bins, case.tails, s) for name in VECTORS]
    return crafted_coupling(case.bins, case.tails, s, vectors, hidden=case.hidden, seed=seed), s
