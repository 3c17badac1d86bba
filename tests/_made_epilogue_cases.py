"""Case table of the two MADE epilogues of the coupling-step kernel: the mixture of MixtureOfGaussiansMADE
(nfk_mog_made_step_f16x3, fused_spline.cuh: mog_tile) and the affine map of MaskedAffineAutoregressiveTransform
(nfk_affine_ar_step_f16x3, affine_tile).  test_made_epilogue_cases.py runs it on the CPU through the emulated kernels and checks
what each case claims; test_made_epilogues_gpu.py runs it on the device through the wrappers.

  * Shape cases, derived from the library: for every packed-row instance MP of the mixture (kernels.mog_made_padded_rows over
    every component count) the smallest and the largest C that packs to it, each at feature counts giving one column tile, two,
    an odd count >= 3 and a partial last tile, over hidden widths 32, 160 (a two-chunk trunk whose second chunk is partial) and
    256.  The affine map's tiles hold TF = 64 features and its inputs are loaded G = 8 at a time: d_t runs across both.
  * Crafted parameters: a helper zeroes the final-layer rows of chosen features and writes a vector into their bias, so the
    epilogue sees exactly that vector (fmaf(0, inv_acc_scale, b) == b): saturated, shifted and underflowing logits, softplus at
    its threshold of 20, sigma at epsilon, means far from x, and for the sampler components picked at exact cumulative-weight
    boundaries.
  * Truth: the fp64 MADE of _mademog_oracle with the module's formulas; the yardstick is the same formulation in fp32, and an
    output passes when its error is at most max(floor, 3 x the fp32 formulation's error)."""
import copy
import math
from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F

import _mademog_oracle as oracle
from conftest import rel_err
from nflows_b200 import _native as N
from nflows_b200 import dense as D
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.nn.nde import MixtureOfGaussiansMADE

BN = 128                  # packed final-layer rows of the widest column tile (fused_spline.cuh: FusedCfg)
AFFINE_TF = 64            # affine features per column tile: 2 rows each
AFFINE_G = 8              # affine inputs loaded together by a thread
HIDDEN = (32, 160, 256)
TILE_CLASSES = ("one", "two", "odd", "partial")
MODES = ("log_prob", "sample")
MARGIN = 1e-5             # draws whose u lies this close to a cumulative-weight boundary (fp64) may pick either neighbour
FLOOR = 1e-5


# ---- layouts ------------------------------------------------------------------------------------------------------------------
def instances():
    """The packed-row counts with a mixture instance, from the library."""
    return sorted({K.mog_made_padded_rows(c) for c in range(1, N.MOG_MAX_COMPONENTS + 1)})


def components_of(mp):
    return [c for c in range(1, N.MOG_MAX_COMPONENTS + 1) if K.mog_made_padded_rows(c) == mp]


def mog_tile_features(mp):
    """TF: features per column tile, FPT = BN / (2 MP) per thread and two threads per row."""
    return 2 * (BN // (2 * mp))


def n_tiles(d_t, tf):
    return (d_t + tf - 1) // tf


def path(tiles):
    """The kernel shares a single column tile between both warpgroups by rows, and ping-pongs two or more between them."""
    return "single" if tiles == 1 else "pingpong"


def class_features(cls, tf):
    """A feature count of tile class `cls`.  The partial tile fills the first half-row and one feature of the second; at one
    feature per thread (MP >= 48) it leaves the second half-row empty."""
    fpt = tf // 2
    return {"one": tf, "two": 2 * tf, "odd": 3 * tf, "partial": tf + (fpt + 1 if fpt > 1 else 1)}[cls]


# ---- shape cases --------------------------------------------------------------------------------------------------------------
MogCase = namedtuple("MogCase", "name mp tf tiles path cls components features hidden")
AffineCase = namedtuple("AffineCase", "name tiles path group_rem features hidden")


def _mog_cases():
    out = []
    for i, mp in enumerate(instances()):
        cs = components_of(mp)
        tf = mog_tile_features(mp)
        for j, cls in enumerate(TILE_CLASSES):
            for k, c in enumerate((cs[0], cs[-1])):
                d = class_features(cls, tf)
                h = HIDDEN[(i + 2 * j + k) % len(HIDDEN)]
                t = n_tiles(d, tf)
                out.append(MogCase("mp{}_c{}_{}_d{}_h{}".format(mp, c, cls, d, h), mp, tf, t, path(t), cls, c, d, h))
    return out


MOG_CASES = _mog_cases()
AFFINE_FEATURES = (1, 7, 8, 9, 33, 63, 64, 65, 129)
AFFINE_CASES = [AffineCase("d{}_h{}".format(d, h), n_tiles(d, AFFINE_TF), path(n_tiles(d, AFFINE_TF)), d % AFFINE_G, d, h)
                for d in AFFINE_FEATURES for h in HIDDEN]


# ---- models -------------------------------------------------------------------------------------------------------------------
def _perturb(module, seed):
    """Every bias + 0.1 N(0, 1), the residual blocks' second linear + 0.05 N(0, 1) (as the golden scripts)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "linear_layers.1" in name:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return module


def mog_model(features, hidden, components, epsilon=1e-2, seed=0):
    torch.manual_seed(seed)
    m = MixtureOfGaussiansMADE(features, hidden, num_blocks=1, num_mixture_components=components, epsilon=epsilon)
    return _perturb(m, seed + 1).eval()


def affine_model(features, hidden, seed=0):
    torch.manual_seed(seed)
    t = T.MaskedAffineAutoregressiveTransform(features=features, hidden_features=hidden, num_blocks=1)
    return _perturb(t, seed + 1).eval()


def craft(final_layer, vectors, rows):
    """Feature j of `vectors` ({feature: vector of `rows` values}): final-layer weight rows j * rows .. + rows - 1 zeroed, the
    vector in their bias.  The epilogue then sees exactly the vector."""
    with torch.no_grad():
        for j, v in vectors.items():
            final_layer.weight[j * rows:(j + 1) * rows].zero_()
            final_layer.bias[j * rows:(j + 1) * rows] = v.reshape(-1).to(final_layer.bias.dtype)


# ---- crafted mixture vectors: [C, 3] of (logit, mean, unconstrained std) --------------------------------------------------------
def _f32(v):
    return float(np.float32(v))


SOFTPLUS_T = 20.0
NEAR_T = (_f32(np.nextafter(np.float32(SOFTPLUS_T), np.float32(0))), SOFTPLUS_T,
          _f32(np.nextafter(np.float32(SOFTPLUS_T), np.float32(np.inf))))


def mog_vectors(c, seed=0):
    """{name: [C, 3]} of the crafted mixture parameters at C components (those that need two components only when C >= 2)."""
    g = torch.Generator().manual_seed(seed + c)
    r = lambda *s: torch.randn(*s, generator=g)
    base = lambda: torch.stack([r(c), r(c), 0.5 * r(c)], -1)

    def with_col(k, vals, v=None):
        v = base() if v is None else v
        v[:, k] = torch.as_tensor(vals, dtype=torch.float32).expand(c)
        return v

    out = {
        "uniform": with_col(0, 0.0),
        "dominant": with_col(0, torch.cat([torch.tensor([40.0]), torch.zeros(c - 1)])),
        "shift+1000": with_col(0, 1000.0 + r(c)),
        "shift-1000": with_col(0, -1000.0 + r(c)),
        "sigma_eps": with_col(2, -30.0),
        "std80": with_col(2, 80.0),
        "far+1e3": with_col(2, -30.0, with_col(1, 1e3)),
        "far-1e3": with_col(2, -30.0, with_col(1, -1e3)),
        "random": base(),
    }
    for i, t in enumerate(NEAR_T):
        out["std20_{}".format(i)] = with_col(2, t)
    if c >= 2:
        out["underflow"] = with_col(0, torch.cat([torch.zeros(c - 1), torch.tensor([-200.0])]))
        v = base()
        v[1] = v[0]
        out["twins"] = v
    return out


# ---- sample boundaries: equal live logits make the cumulative weights exact ----------------------------------------------------
U_BOUNDARY = (0.0, _f32(np.nextafter(np.float32(0.25), np.float32(0))), 0.25, 0.5, 0.75,
              _f32(np.nextafter(np.float32(1.0), np.float32(0))))


def pick_fp32(logits, u):
    """The kernel's rule in fp32: c* = the first c with u < sum_{c' <= c} exp(l_c' - lmax) / se, C - 1 when rounding leaves u
    above the total.  Exact for the boundary vectors (every exp is of 0 or of -200)."""
    l = np.asarray(logits, dtype=np.float32)
    w = np.exp(l - l.max()).astype(np.float32)
    se = np.float32(0)
    for x in w:
        se = np.float32(se + x)
    cum = np.float32(0)
    for c in range(len(l)):
        cum = np.float32(cum + np.float32(w[c] / se))
        if np.float32(u) < cum:
            return c
    return len(l) - 1


def fallback_components():
    """Component counts whose equal logits leave the fp32 cumulative total below nextafter(1, 0): u = nextafter(1, 0) then takes
    the C - 1 fallback rather than a boundary."""
    out = []
    for c in range(1, N.MOG_MAX_COMPONENTS + 1):
        w = np.float32(1) / np.float32(c)
        cum = np.float32(0)
        for _ in range(c):
            cum = np.float32(cum + w)
        if np.float32(U_BOUNDARY[-1]) >= cum:
            out.append(c)
    return out


def boundary_logits(c):
    """{name: logits [C]} of the boundary cases at C components: four live components of weight 0.25 (the rest at -200, so a
    zero weight at the end), the same with a zero-weight component in the middle, two live halves, and all equal."""
    z = lambda live: torch.tensor([0.0 if i in live else -200.0 for i in range(c)])
    out = {"all_equal": torch.zeros(c)}
    if c >= 2:
        out["halves"] = z({0, 1})
    if c >= 4:
        out["quarters"] = z({0, 1, 2, 3})
    if c >= 5:
        out["quarters_zero_middle"] = z({0, 1, 3, 4})
    return out


def boundary_vector(logits):
    """Means 100 c (distinct, exact) and unit-ish sigma: with e = 0 the draw is the chosen component's mean exactly."""
    c = logits.numel()
    return torch.stack([logits, 100.0 * torch.arange(c, dtype=torch.float32), torch.zeros(c)], -1)


def mog_crafted(c, seed=0):
    """(vectors {name: [C, 3]}, boundary names) of the crafted mixture table at C components."""
    vec = mog_vectors(c, seed)
    bnd = {"bnd_" + k: boundary_vector(v) for k, v in boundary_logits(c).items()}
    vec.update(bnd)
    return vec, list(bnd)


# ---- crafted affine vectors: (u, shift) ---------------------------------------------------------------------------------------
AFFINE_U = (0.0,) + NEAR_T + (-30.0, 15.0, 80.0)
AFFINE_SHIFT = (0.0, 1e3, -1e3, None)      # None: random


def affine_vectors(seed=0):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for u in AFFINE_U:
        for s in AFFINE_SHIFT:
            out["u{}_s{}".format(u, "rand" if s is None else s)] = torch.tensor(
                [u, float(torch.randn(1, generator=g)) if s is None else s])
    return out


# ---- truth and yardstick ------------------------------------------------------------------------------------------------------
def mixture_params(out, n, d, c, eps):
    o = out.reshape(n, d, c, 3)
    return o[..., 0], o[..., 1], F.softplus(o[..., 2]) + eps


def mixture_terms(params, x):
    """Per-feature log-density [n, D] (the module's formulation, in the parameters' dtype)."""
    logits, means, stds = params
    x = x.to(logits.dtype)
    t = torch.log_softmax(logits, -1) - 0.5 * (math.log(2 * math.pi) + 2 * torch.log(stds) + ((x[..., None] - means) / stds) ** 2)
    return torch.logsumexp(t, -1)


def mixture_draws(params, u, e):
    """(y [n, D], component [n, D], margin [n, D]): c* = the first c with u < cumulative weight, C - 1 above the total; margin =
    distance of u to the nearest inner boundary."""
    logits, means, stds = params
    c = logits.shape[-1]
    u, e = u.to(logits.dtype), e.to(logits.dtype)
    cdf = torch.cumsum(torch.softmax(logits, -1), -1)
    comp = torch.clamp((u[..., None] >= cdf).sum(-1), max=c - 1)
    margin = (cdf[..., :-1] - u[..., None]).abs().min(-1).values if c > 1 else torch.full_like(u, math.inf)
    pick = lambda t: t.gather(-1, comp[..., None])[..., 0]
    return pick(means) + pick(stds) * e, comp, margin


class MogTruth:
    """fp64 parameters of every feature from the oracle's MADE, fp32 ones from the module; m and x on the CPU."""

    def __init__(self, m, x):
        n, d = x.shape
        c, eps = m.num_mixture_components, m.epsilon
        sd = {k: v.detach() for k, v in m.state_dict().items()}
        self.p64 = mixture_params(oracle.made_outputs(sd, x, None, prefix=""), n, d, c, eps)
        with torch.no_grad():
            self.p32 = mixture_params(m(x), n, d, c, eps)
        self.t64, self.t32 = mixture_terms(self.p64, x), mixture_terms(self.p32, x)

    def log_prob(self, c0, dt):
        """(fp64, fp32) sums over features c0 .. c0 + dt - 1 of each row."""
        return self.t64[:, c0:c0 + dt].sum(-1), self.t32[:, c0:c0 + dt].sum(-1)

    def sample(self, u, e, c0, dt):
        """(y64, y32, margin) of features c0 .. c0 + dt - 1 with noise u, e [n, dt]."""
        sl = lambda p: tuple(t[:, c0:c0 + dt] for t in p)
        y64, _, margin = mixture_draws(sl(self.p64), u.cpu(), e.cpu())
        y32, _, _ = mixture_draws(sl(self.p32), u.cpu(), e.cpu())
        return y64, y32, margin


def affine_truth(t, x, inverse):
    """((y, lad) fp64, (y, lad) fp32) per feature of the direct launch, t and x on the CPU: the parameters come from MADE(x) and
    both directions map x (the inverse's one pass: y = (x - shift) / scale)."""
    out = []
    for dt in (torch.float64, torch.float32):
        m = copy.deepcopy(t).to(dt)
        xx = x.to(dt)
        with torch.no_grad():
            scale, shift = m._scale_shift(m.autoregressive_net(xx))
        y = (xx - shift) / scale if inverse else scale * xx + shift
        lad = torch.log(scale)
        out.append((y, -lad if inverse else lad))
    return out


def within(got, truth, yard, floor=FLOOR):
    """(ok, kernel error, fp32 error): the sandwich."""
    e_got, e_ref = rel_err(got.detach().cpu(), truth), rel_err(yard, truth)
    return e_got <= max(floor, 3 * e_ref), e_got, e_ref


def ratio(e_got, e_ref, floor=FLOOR):
    """The error as a share of its bar (<= 1 passes)."""
    return e_got / max(floor, 3 * e_ref)


# ---- direct launches ----------------------------------------------------------------------------------------------------------
def mog_launch(m, x, cols, mode, lad=None, y=None, noise=None, epsilon=None, a=None):
    """One call of kernels.mog_made_step on the model's padded chain and packed final layer, features cols = (first, count):
    the final rows of those features only (a sub-range of the packed operands, as the sampler's passes take).  a: the input pair
    (default: m.input_pair(x)).  Returns the flag word."""
    chain = m.padded_chain(None)
    c = m.num_mixture_components
    wf, bias, mp = D.mog_operands(chain[-1][0], chain[-1][1], c)
    c0, dt = cols
    w = K.Pair16(wf.hi[c0 * mp:(c0 + dt) * mp], wf.lo[c0 * mp:(c0 + dt) * mp], wf.exp)
    flags = torch.zeros(1, dtype=torch.int32, device=x.device)
    a = m.input_pair(x, flags) if a is None else a
    eps = m.epsilon if epsilon is None else epsilon
    if mode == "log_prob":
        K.mog_made_step(D.step_plan(chain), a, w, bias[c0 * mp:(c0 + dt) * mp], c, eps, cols, x=x, lad_accum=lad, flags=flags)
    else:
        K.mog_made_step(D.step_plan(chain), a, w, bias[c0 * mp:(c0 + dt) * mp], c, eps, cols, y=y, noise=noise, flags=flags)
    return flags


def affine_launch(t, x, cols, y, lad, inverse, a=None):
    """One call of kernels.affine_ar_step on the transform's padded chain, features cols = (first, count) of x and y (the MADE
    final rows 2 first .. 2 (first + count) - 1).  Returns the flag word."""
    net = t.autoregressive_net
    chain = net.padded_chain(None)
    wf, bias, _ = D.ar_affine_operands(chain[-1][0], chain[-1][1])
    c0, dt = cols
    w = K.Pair16(wf.hi[2 * c0:2 * (c0 + dt)], wf.lo[2 * c0:2 * (c0 + dt)], wf.exp)
    flags = torch.zeros(1, dtype=torch.int32, device=x.device)
    a = net.input_pair(x, flags) if a is None else a
    K.affine_ar_step(D.step_plan(chain), a, w, bias[2 * c0:2 * (c0 + dt)], x, cols, y, lad, flags, inverse)
    return flags


def noise(n, d, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, d, generator=g), torch.randn(n, d, generator=g)


# ---- runners shared by the CPU and GPU tests ----------------------------------------------------------------------------------
N_ROWS = 257              # two full row tiles of 128 and one of a single row


def inputs(n, d, seed):
    return torch.randn(n, d, generator=torch.Generator().manual_seed(seed))


def run_mog_case(case, mode, device, seed=0):
    """One direct launch of a shape case over all its features.  Returns (flag word, kernel error, fp32 error)."""
    m = mog_model(case.features, case.hidden, case.components, seed=seed)
    x = inputs(N_ROWS, case.features, seed + 2)
    truth = MogTruth(m, x)
    m, xd, d = m.to(device), x.to(device), case.features
    if mode == "log_prob":
        lad = torch.zeros(N_ROWS, device=device)
        flags = mog_launch(m, xd, (0, d), mode, lad=lad)
        want, yard = truth.log_prob(0, d)
        _, e, r = within(lad, want, yard)
        return int(flags.item()), e, r
    u, e = noise(N_ROWS, d, seed + 3)
    y = torch.zeros(N_ROWS, d, device=device)
    flags = mog_launch(m, xd, (0, d), mode, y=y, noise=(u.to(device), e.to(device)))
    y64, y32, margin = truth.sample(u, e, 0, d)
    keep = margin > MARGIN
    assert keep.double().mean() >= 0.99, keep.double().mean()
    _, err, r = within(y.cpu()[keep], y64[keep], y32[keep])
    return int(flags.item()), err, r


def crafted_components():
    """The component counts of the crafted mixture table: the largest C of every instance (the most crafted vectors), C = 4
    (four equal components and nothing else) and the first C whose equal weights take the C - 1 fallback."""
    return sorted({components_of(mp)[-1] for mp in instances()} | {4, fallback_components()[0]})


def run_mog_crafted(c, epsilon, device, hidden=64, n_random=3, seed=0):
    """The crafted vectors of C components in features 0 .. V - 1 of one model, n_random ordinary features after them.
    log_prob: one launch of every feature, then one launch per crafted feature (d_t = 1 at t_col0 = j), each against its own
    fp64 truth.  sample: one launch of every feature; boundary features draw with e = 0 and u cycling through U_BOUNDARY and
    must return the mean (100 c*) of the component the kernel's fp32 rule picks, exactly.
    Returns {what: (flag word, kernel error, fp32 error)} and the boundary checks' failures."""
    vec, bnd = mog_crafted(c, seed)
    names = list(vec)
    d, n = len(names) + n_random, N_ROWS
    m = mog_model(d, hidden, c, epsilon=epsilon, seed=seed)
    craft(m.final_layer, {j: vec[k] for j, k in enumerate(names)}, 3 * c)
    x = inputs(n, d, seed + 2)
    u, e = noise(n, d, seed + 3)
    ub = torch.tensor(U_BOUNDARY)[torch.arange(n) % len(U_BOUNDARY)]
    for j, k in enumerate(names):
        if k in bnd:
            u[:, j], e[:, j] = ub, 0.0
    truth = MogTruth(m, x)
    m, xd = m.to(device), x.to(device)
    out = {}
    lad = torch.zeros(n, device=device)
    f = mog_launch(m, xd, (0, d), "log_prob", lad=lad)
    out["log_prob_all"] = (int(f.item()),) + within(lad, *truth.log_prob(0, d))[1:]
    for j, k in enumerate(names):
        lad = torch.zeros(n, device=device)
        f = mog_launch(m, xd, (j, 1), "log_prob", lad=lad)
        out["log_prob_" + k] = (int(f.item()),) + within(lad, *truth.log_prob(j, 1))[1:]
    y = torch.zeros(n, d, device=device)
    f = mog_launch(m, xd, (0, d), "sample", y=y, noise=(u.to(device), e.to(device)))
    y = y.cpu()
    y64, y32, margin = truth.sample(u, e, 0, d)
    keep = margin > MARGIN
    plain = [j for j, k in enumerate(names) if k not in bnd] + list(range(len(names), d))
    out["sample"] = (int(f.item()),) + within(y[:, plain][keep[:, plain]], y64[:, plain][keep[:, plain]],
                                              y32[:, plain][keep[:, plain]])[1:]
    misses = []
    for j, k in enumerate(names):
        if k in bnd:
            want = torch.tensor([100.0 * pick_fp32(vec[k][:, 0].numpy(), float(uu)) for uu in ub])
            if not torch.equal(y[:, j], want):
                bad = (y[:, j] != want).nonzero()[:3, 0].tolist()
                misses.append((k, [(float(ub[i]), float(y[i, j]), float(want[i])) for i in bad]))
    return out, misses


def run_affine_case(case, inverse, device, seed=0):
    """One direct launch of an affine shape case over all its features: ((y error, fp32 error), (lad error, fp32 error), flags)."""
    t = affine_model(case.features, case.hidden, seed=seed)
    x = inputs(N_ROWS, case.features, seed + 2)
    return run_affine(t, x, inverse, device)


def run_affine(t, x, inverse, device):
    (y64, l64), (y32, l32) = affine_truth(t, x, inverse)
    t, xd = t.to(device), x.to(device)
    y = torch.zeros_like(xd)
    lad = torch.zeros(x.shape[0], device=device)
    flags = affine_launch(t, xd, (0, x.shape[1]), y, lad, inverse)
    return within(y, y64, y32)[1:], within(lad, l64.sum(-1), l32.sum(-1))[1:], int(flags.item())


def affine_crafted(seed=0, hidden=64, n_random=41):
    """A transform whose first features carry the crafted (u, shift) vectors and n_random ordinary ones after them (65 features:
    two column tiles, the second partial), and its inputs."""
    vec = affine_vectors(seed)
    d = len(vec) + n_random
    t = affine_model(d, hidden, seed=seed)
    craft(t.autoregressive_net.final_layer, dict(enumerate(vec.values())), 2)
    return t, inputs(N_ROWS, d, seed + 2)
