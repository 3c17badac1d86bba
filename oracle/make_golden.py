"""Generate tests/golden/*.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows).

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python oracle/make_golden.py

Each fixture stores the reference's weights (its own ``state_dict``), the seeded inputs and the
reference's outputs, so parity tests can replay them anywhere.  The full-shape cfg-3 layer is too
large to commit (10.7 MB of weights), so that fixture stores only (seed, inputs, outputs, a weight
checksum): the weights are re-created from the seed by ``nflows_b200`` (whose constructors consume
the torch CPU RNG in the same order as the reference; checked by tests/test_api_reference_parity.py).
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REFERENCE_SRC = os.environ.get("NFLOWS_REFERENCE_SRC")
if not REFERENCE_SRC or not os.path.isdir(os.path.join(REFERENCE_SRC, "nflows")):
    sys.exit("set NFLOWS_REFERENCE_SRC to a checkout of bayesiains/nflows (the directory that contains nflows/)")
sys.path[:0] = [os.path.join(ROOT, "tests", "_shims"), REFERENCE_SRC]

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from nflows import transforms as T  # noqa: E402
from nflows.distributions import StandardNormal  # noqa: E402
from nflows.flows import Flow  # noqa: E402
from nflows.nn.nets import ResidualNet  # noqa: E402
from nflows.transforms.splines import rational_quadratic as rq  # noqa: E402
from nflows.utils import torchutils  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def save(name, obj):
    path = os.path.join(OUT, name + ".pt")
    torch.save(obj, path)
    print("{:32s} {:8.1f} KB".format(name, os.path.getsize(path) / 1024))


def weight_checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values() if v.is_floating_point()))


def perturb(flow, seed=2):
    """SURVEY.md section 8d 'well-conditioned perturbed variant'."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in flow.named_parameters():
            if name.endswith("lower_entries") or name.endswith("upper_entries"):
                d = (1 + int(np.sqrt(1 + 8 * p.numel()))) // 2
                p.add_((0.1 / np.sqrt(d)) * torch.randn(p.shape, generator=g))
            elif name.split(".")[-1] in ("log_scale", "shift", "unconstrained_upper_diag") or (
                    name.endswith(".bias") and "transform_net" not in name):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "final_layer" in name:
                p.mul_(3.0)


def nsf(features, hidden, layers, num_bins=8, tail_bound=3.0, num_blocks=2):
    ts = []
    for i in range(layers):
        ts.append(T.ActNorm(features))
        ts.append(T.CompositeTransform([T.RandomPermutation(features), T.LULinear(features, identity_init=True)]))
        ts.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(features, even=(i % 2 == 0)),
            transform_net_create_fn=lambda i_, o_: ResidualNet(i_, o_, hidden_features=hidden, num_blocks=num_blocks),
            num_bins=num_bins, tails="linear", tail_bound=tail_bound))
    return Flow(T.CompositeTransform(ts), StandardNormal([features]))


@torch.no_grad()
def main():
    # ---- g_searchsorted: reference known-answer (tests/utils/torchutils_test.py:80-90) ----------
    locs = torch.linspace(0, 1, 10)
    left, right = locs[:-1], locs[1:]
    mid = (left + right) / 2
    queries = torch.stack([left, right - 1e-7, mid])
    save("searchsorted", {
        "bin_locations": torch.linspace(0, 1, 10),
        "inputs": queries,
        "idx": torch.stack([torchutils.searchsorted(torch.linspace(0, 1, 10).repeat(9, 1), v) for v in queries]),
    })

    # ---- g_spline: function-level vectors, both directions, constrained + linear tails ----------
    torch.manual_seed(10)
    n, k = 4096, 8
    uw, uh = torch.randn(n, k) * 2, torch.randn(n, k) * 2
    ud_t, ud_c = torch.randn(n, k - 1) * 2, torch.randn(n, k + 1) * 2
    ud_t[:16] = 25.0  # softplus linear branch (threshold 20)
    ud_t[16:32] = -30.0
    x_t = torch.randn(n) * 2.2
    b = 3.0
    x_t[:8] = torch.tensor([-b, b, np.nextafter(np.float32(b), np.float32(4)), np.nextafter(np.float32(-b), np.float32(-4)),
                            np.nextafter(np.float32(b), np.float32(0)), 0.0, float("nan"), 1e30])
    x_c = torch.rand(n)
    x_c[:3] = torch.tensor([0.0, 1.0, 0.5])
    fx = {}
    for inv in (False, True):
        y, l = rq.unconstrained_rational_quadratic_spline(x_t.clone(), uw.clone(), uh.clone(), ud_t.clone(), inverse=inv,
                                                          tails="linear", tail_bound=b)
        fx["tails_inv%d" % inv] = (y, l)
        y, l = rq.rational_quadratic_spline(x_c.clone(), uw.clone(), uh.clone(), ud_c.clone(), inverse=inv)
        fx["constrained_inv%d" % inv] = (y, l)
        y, l = rq.rational_quadratic_spline(x_c.clone() * 4 - 1, uw.clone(), uh.clone(), ud_c.clone(), inverse=inv,
                                            left=-1.0, right=3.0, bottom=-1.0, top=3.0,
                                            min_bin_width=1e-2, min_bin_height=2e-2, min_derivative=5e-2)
        fx["constrained_box_inv%d" % inv] = (y, l)
    save("spline", dict(uw=uw, uh=uh, ud_tails=ud_t, ud_constrained=ud_c, x_tails=x_t, x_constrained=x_c,
                        tail_bound=b, **fx))

    # ---- g_cfg1: 2-layer affine coupling D=2 (BASELINE configs[0]) -------------------------------
    torch.manual_seed(0)
    f = lambda i, o: ResidualNet(i, o, hidden_features=8)
    flow = Flow(T.CompositeTransform([T.AffineCouplingTransform(mask=[1, 0], transform_net_create_fn=f),
                                      T.AffineCouplingTransform(mask=[0, 1], transform_net_create_fn=f)]),
                StandardNormal([2])).eval()
    torch.manual_seed(0)
    x = torch.randn(1024, 2)
    z, lad = flow._transform(x)
    xr, ladr = flow._transform.inverse(z)
    save("cfg1_affine", dict(sd=flow.state_dict(), x=x, z=z, lad=lad, log_prob=flow.log_prob(x), x_roundtrip=xr,
                             lad_inverse=ladr))

    # ---- g_affine_general: GENERAL scale activation + additive, D=10 ------------------------------
    torch.manual_seed(3)
    f = lambda i, o: ResidualNet(i, o, hidden_features=16)
    mask = torchutils.create_mid_split_binary_mask(10)
    tg = T.AffineCouplingTransform(mask, f, scale_activation=T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION).eval()
    ta = T.AdditiveCouplingTransform(mask, f).eval()
    for t in (tg, ta):
        for name, p in t.named_parameters():
            if "final_layer" in name or "blocks.1.linear_layers.1" in name:
                p.mul_(4.0)
    x = torch.randn(512, 10) * 2
    yg, lg = tg(x)
    ya, la = ta(x)
    save("affine_variants", dict(sd_general=tg.state_dict(), sd_additive=ta.state_dict(), x=x, y_general=yg, lad_general=lg,
                                 y_additive=ya, lad_additive=la, xinv_general=tg.inverse(x)[0],
                                 ladinv_general=tg.inverse(x)[1]))

    # ---- g_cfg2: single RQ coupling D=64 K=8 H=128 (BASELINE configs[1]); default and x3 ---------
    torch.manual_seed(0)
    t = T.PiecewiseRationalQuadraticCouplingTransform(
        mask=torchutils.create_alternating_binary_mask(64),
        transform_net_create_fn=lambda i, o: ResidualNet(i, o, hidden_features=128, num_blocks=2),
        num_bins=8, tails="linear", tail_bound=3.0).eval()
    torch.manual_seed(1)
    x = torch.randn(512, 64)
    x[0, :8] = torch.tensor([-3.0, 3.0, 3.0000002, -3.0000002, 2.9999998, 0.0, 100.0, -1e-30])
    out = dict(sd={k: v.clone() for k, v in t.state_dict().items()}, x=x, checksum=weight_checksum(t.state_dict()))
    out["y"], out["lad"] = t(x)
    out["xinv"], out["ladinv"] = t.inverse(x)
    for name, p in t.named_parameters():
        if "final_layer" in name:
            p.mul_(3.0)
    out["y_x3"], out["lad_x3"] = t(x)
    out["xinv_x3"], out["ladinv_x3"] = t.inverse(x)
    save("cfg2_rq_coupling", out)

    # ---- g_rq_constrained: tails=None coupling on U[0,1), odd D, K=5, mid-split mask -------------
    torch.manual_seed(4)
    t = T.PiecewiseRationalQuadraticCouplingTransform(
        mask=torchutils.create_mid_split_binary_mask(11),
        transform_net_create_fn=lambda i, o: ResidualNet(i, o, hidden_features=24, num_blocks=1),
        num_bins=5, tails=None, min_bin_width=2e-3, min_bin_height=3e-3, min_derivative=4e-3).eval()
    for name, p in t.named_parameters():
        if "final_layer" in name:
            p.mul_(5.0)
    x = torch.rand(300, 11)
    y, l = t(x)
    xi, li = t.inverse(x)
    save("rq_coupling_constrained", dict(sd=t.state_dict(), x=x, y=y, lad=l, xinv=xi, ladinv=li))

    # ---- g_linear: ActNorm / LULinear / Permutation standalone, D=37 ------------------------------
    torch.manual_seed(5)
    d = 37
    an, lu, pm = T.ActNorm(d).eval(), T.LULinear(d, identity_init=False).eval(), T.RandomPermutation(d).eval()
    an.log_scale.add_(0.3 * torch.randn(d))
    an.shift.add_(torch.randn(d))
    lu.bias.add_(torch.randn(d))
    x = torch.randn(257, d)
    rec = dict(x=x, sd_actnorm=an.state_dict(), sd_lu=lu.state_dict(), sd_perm=pm.state_dict())
    for nm, m in (("actnorm", an), ("lu", lu), ("perm", pm)):
        rec[nm + "_y"], rec[nm + "_lad"] = m(x)
        rec[nm + "_xinv"], rec[nm + "_ladinv"] = m.inverse(x)
    rec["lu_weight"], rec["lu_weight_inverse"], rec["lu_logabsdet"] = lu.weight(), lu.weight_inverse(), lu.logabsdet()
    save("linear_transforms", rec)

    # ---- g_nsf_small: 3-layer NSF D=24 H=32, perturbed; log_prob + inverse ------------------------
    torch.manual_seed(0)
    flow = nsf(24, 32, 3).eval()
    perturb(flow)
    torch.manual_seed(1)
    x = torch.randn(384, 24)
    z, lad = flow._transform(x)
    noise = torch.randn(384, 24)
    xs, lads = flow._transform.inverse(noise)
    save("nsf_small", dict(sd=flow.state_dict(), x=x, z=z, lad=lad, log_prob=flow.log_prob(x), noise=noise,
                           sample=xs, lad_inverse=lads, features=24, hidden=32, layers=3))

    # ---- g_nsf784_layer: ONE full-shape cfg-3 layer (D=784 H=256 K=8), weights by seed ------------
    torch.manual_seed(0)
    flow = nsf(784, 256, 1).eval()
    perturb(flow)
    torch.manual_seed(1)
    x = torch.randn(96, 784)
    z, lad = flow._transform(x)
    xi, li = flow._transform.inverse(x)
    zd, ladd = flow.double()._transform(x.double())
    save("nsf784_layer", dict(seed=0, perturb_seed=2, x=x, z=z, lad=lad, log_prob=flow.float().log_prob(x), xinv=xi, ladinv=li,
                              z_fp64=zd, lad_fp64=ladd, checksum=weight_checksum(flow.float().state_dict()),
                              features=784, hidden=256, layers=1))

    # ---- g_nsf784_full: the 10-layer cfg-3 flow, 32 rows, weights by seed -------------------------
    torch.manual_seed(0)
    flow = nsf(784, 256, 10).eval()
    perturb(flow)
    torch.manual_seed(1)
    x = torch.randn(32, 784)
    lp = flow.log_prob(x)
    z = flow.transform_to_noise(x)
    ck = weight_checksum(flow.state_dict())
    lpd = flow.double().log_prob(x.double())
    save("nsf784_full", dict(seed=0, perturb_seed=2, x=x, log_prob=lp, z=z, log_prob_fp64=lpd, checksum=ck,
                             features=784, hidden=256, layers=10))

    # ---- g_ar_rq: BASELINE configs[3] shape -- MaskedPiecewiseRationalQuadraticAutoregressiveTransform D=64 H=256 K=8
    # (weights by seed; final layer x3: non-trivial splines, log|det| ~ -30, yet the 64-step inverse stays well conditioned),
    # forward and the D-pass inverse
    torch.manual_seed(0)
    ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=64, hidden_features=256, num_bins=8,
                                                                   tails="linear", tail_bound=3.0, num_blocks=2).eval()
    for name, p in ar.named_parameters():
        if "final_layer" in name:
            p.mul_(3.0)
    torch.manual_seed(1)
    x = torch.randn(96, 64) * 1.3
    y, lad = ar(x)
    xi, li = ar.inverse(x)
    yd, ladd = ar.double()(x.double())
    xid, lid = ar.inverse(x.double())
    save("ar_rq", dict(seed=0, final_scale=3.0, x=x, y=y, lad=lad, xinv=xi, ladinv=li, y_fp64=yd, lad_fp64=ladd,
                       xinv_fp64=xid, ladinv_fp64=lid,
                       checksum=weight_checksum(ar.float().state_dict())))
    # small variant with the weights stored, for the CPU oracle
    torch.manual_seed(2)
    ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=6, hidden_features=16, num_bins=4, tails=None,
                                                                   num_blocks=1).eval()
    for name, p in ar.named_parameters():
        if "final_layer" in name:
            p.mul_(20.0)
    x = torch.rand(40, 6)
    y, lad = ar(x)
    xi, li = ar.inverse(x)
    save("ar_rq_small", dict(sd=ar.state_dict(), x=x, y=y, lad=lad, xinv=xi, ladinv=li))


def next_rows():
    """Round 2: reference outputs for the SURVEY section 8 'next' rows that were only compared with this package's own CPU path
    in round 1 -- OneByOneConvolution on an image batch, PiecewiseRationalQuadraticCDF (both tail modes), an RQ coupling with
    apply_unconditional_transform, SimpleRealNVP, and an MLP-conditioned RQ coupling.  Weights travel as reference state_dicts."""
    from nflows.flows.realnvp import SimpleRealNVP
    from nflows.nn.nets import MLP
    rec = {}
    with torch.no_grad():
        torch.manual_seed(10)
        conv = T.OneByOneConvolution(3, identity_init=False).eval()
        x = torch.randn(10, 3, 28, 28)
        y, lad = conv(x)
        xi, li = conv.inverse(x)
        rec["conv1x1"] = dict(sd=conv.state_dict(), x=x, y=y, lad=lad, xinv=xi, ladinv=li)
        torch.manual_seed(11)
        conv = T.OneByOneConvolution(12, identity_init=False).eval()
        x = torch.randn(5, 12, 6, 6)
        y, lad = conv(x)
        rec["conv1x1_c12"] = dict(sd=conv.state_dict(), x=x, y=y, lad=lad)
        for tails in (None, "linear"):
            torch.manual_seed(12)
            cdf = T.PiecewiseRationalQuadraticCDF(shape=[7], num_bins=6, tails=tails, tail_bound=2.0).eval()
            for p_ in cdf.parameters():
                p_.copy_(torch.randn(p_.shape) * 1.5)
            x = torch.rand(300, 7) if tails is None else torch.randn(300, 7) * 1.5
            y, lad = cdf(x)
            xi, li = cdf.inverse(x if tails == "linear" else y)
            rec["rq_cdf_%s" % (tails or "none")] = dict(sd=cdf.state_dict(), x=x, y=y, lad=lad, inv_in=(x if tails == "linear" else y),
                                                        xinv=xi, ladinv=li)
        torch.manual_seed(13)
        t = T.PiecewiseRationalQuadraticCouplingTransform(
            torchutils.create_alternating_binary_mask(16), lambda i, o: ResidualNet(i, o, hidden_features=32, num_blocks=1),
            num_bins=8, tails="linear", tail_bound=3.0, apply_unconditional_transform=True).eval()
        for name, p_ in t.named_parameters():
            if "final_layer" in name or "unnormalized" in name:
                p_.copy_(p_ * 3.0 + 0.3 * torch.randn(p_.shape))
        x = torch.randn(200, 16) * 1.2
        y, lad = t(x)
        xi, li = t.inverse(x)
        rec["rq_coupling_unconditional"] = dict(sd=t.state_dict(), x=x, y=y, lad=lad, xinv=xi, ladinv=li)
        torch.manual_seed(14)
        flow = SimpleRealNVP(features=10, hidden_features=16, num_layers=3, num_blocks_per_layer=2).eval()
        for p_ in flow.parameters():
            p_.add_(0.05 * torch.randn(p_.shape))
        x = torch.randn(257, 10)
        rec["simple_realnvp"] = dict(sd=flow.state_dict(), x=x, log_prob=flow.log_prob(x))
        torch.manual_seed(15)
        class CtxMLP(torch.nn.Module):        # the reference's MLP takes no context argument: the usual user-side adapter
            def __init__(self, i, o):
                super().__init__()
                self.mlp = MLP([i], [o], [64, 64, 64])

            def forward(self, inputs, context=None):
                return self.mlp(inputs)

        t = T.PiecewiseRationalQuadraticCouplingTransform(
            torchutils.create_alternating_binary_mask(32), lambda i, o: CtxMLP(i, o),
            num_bins=8, tails="linear", tail_bound=3.0).eval()
        for name, p_ in t.named_parameters():
            if "_final_layer" in name:
                p_.mul_(3.0)
        x = torch.randn(500, 32) * 1.2
        y, lad = t(x)
        xi, li = t.inverse(x)
        yd, ladd = t.double()(x.double())
        rec["rq_coupling_mlp"] = dict(sd=t.float().state_dict(), x=x, y=y, lad=lad, xinv=xi, ladinv=li, y_fp64=yd, lad_fp64=ladd)
    save("next_rows", rec)


def context_rows():
    """Round 2: the context-conditioned surface (SURVEY section 8 row f4): a Flow with an embedding net whose RQ couplings use
    context-conditioned ResidualNets (GLU gates, resnet.py:50-51), log_prob / sample_and_log_prob with a context batch."""
    rec = {}
    with torch.no_grad():
        torch.manual_seed(20)
        features, ctx_raw, ctx = 16, 5, 6
        steps = []
        for i in range(3):
            steps.append(T.ActNorm(features))
            steps.append(T.CompositeTransform([T.RandomPermutation(features), T.LULinear(features, identity_init=True)]))
            steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
                mask=torchutils.create_alternating_binary_mask(features, even=(i % 2 == 0)),
                transform_net_create_fn=lambda i_, o_: ResidualNet(i_, o_, hidden_features=32, context_features=ctx, num_blocks=2),
                num_bins=8, tails="linear", tail_bound=3.0))
        flow = Flow(T.CompositeTransform(steps), StandardNormal([features]), embedding_net=torch.nn.Linear(ctx_raw, ctx)).eval()
        perturb(flow)
        x = torch.randn(300, features)
        c = torch.randn(300, ctx_raw)
        lp = flow.log_prob(x, context=c)
        z = flow.transform_to_noise(x, context=c)
        lp64 = flow.double().log_prob(x.double(), context=c.double())
        flow.float()
        noise = torch.randn(300, features)
        xs, _ = flow._transform.inverse(noise, context=flow._embedding_net(c))
        rec["context_flow"] = dict(sd=flow.state_dict(), x=x, context=c, log_prob=lp, z=z, log_prob_fp64=lp64, noise=noise, sample=xs)
    save("context_rows", rec)


def glow_multiscale(image_shape=(3, 16, 16), levels=3, steps=2, hidden_channels=32, num_bins=8, tail_bound=3.0):
    """BASELINE cfg 5 in small: `levels` x [SqueezeTransform, `steps` x [ActNorm, OneByOneConvolution, RQ coupling over channels
    (mid-split mask alternated with its complement, ConvResidualNet conditioner)]] under a MultiscaleCompositeTransform."""
    from nflows.nn.nets import ConvResidualNet
    c, h, w = image_shape
    mct = T.MultiscaleCompositeTransform(num_transforms=levels)
    for _ in range(levels):
        squeeze = T.SqueezeTransform()
        c, h, w = squeeze.get_output_shape(c, h, w)
        layers = [squeeze]
        for i in range(steps):
            mask = torchutils.create_mid_split_binary_mask(c)
            if i % 2:
                mask = 1 - mask
            layers.append(T.CompositeTransform([
                T.ActNorm(c), T.OneByOneConvolution(c),
                T.PiecewiseRationalQuadraticCouplingTransform(
                    mask=mask, transform_net_create_fn=lambda i_, o_: ConvResidualNet(i_, o_, hidden_channels=hidden_channels, num_blocks=2),
                    num_bins=num_bins, tails="linear", tail_bound=tail_bound)]))
        shape = mct.add_transform(T.CompositeTransform(layers), (c, h, w))
        if shape is not None:
            c, h, w = shape
    return Flow(mct, StandardNormal([int(np.prod(image_shape))]))


def image_rows():
    """Round 2: the image path (SURVEY section 8 row f3, BASELINE cfg 5 in small): 3 x 16 x 16 images, 3 levels x 2 steps, 32 hidden
    channels -- squeezed channel counts 12 / 24 / 48, i.e. 6 / 12 / 24 identity channels (padded and unpadded initial layers,
    gathered and packed coupling paths)."""
    rec = {}
    with torch.no_grad():
        torch.manual_seed(30)
        flow = glow_multiscale().eval()
        perturb(flow)
        g = torch.Generator().manual_seed(31)
        for name, p in flow.named_parameters():          # the zero-initialised 3x3 convolutions must matter in the outputs
            if "conv_layers" in name and name.endswith("weight"):
                p.add_(0.05 * torch.randn(p.shape, generator=g))
        x = torch.randn(6, 3, 16, 16)
        z = flow.transform_to_noise(x)
        lp = flow.log_prob(x)
        lp64 = flow.double().log_prob(x.double())
        z64 = flow.transform_to_noise(x.double())
        flow.float()
        noise = torch.randn(6, 3 * 16 * 16)
        xs, lad_inv = flow._transform.inverse(noise)
        xs64, lad_inv64 = flow.double()._transform.inverse(noise.double())
        flow.float()
        rec["glow_small"] = dict(sd=flow.state_dict(), x=x, z=z, z_fp64=z64, log_prob=lp, log_prob_fp64=lp64, noise=noise, sample=xs,
                                 sample_fp64=xs64, lad_inv=lad_inv, lad_inv_fp64=lad_inv64)
    save("image_rows", rec)


def affine_rows():
    """Round 2 (row ns2): affine / additive couplings at sizes the tensor-core dense path takes -- D = 48 (alternating mask: 24
    identity columns: packed path) and D = 20 (8 identity / 12 transformed columns: gathered path), hidden 64, both scale activations -- and a
    small RealNVP-style flow of them behind ActNorm + LU layers (column layouts)."""
    rec = {}
    with torch.no_grad():
        torch.manual_seed(40)
        f = lambda i, o: ResidualNet(i, o, hidden_features=64, num_blocks=2)
        for name, d, mask_fn, kw in (
                ("default48", 48, torchutils.create_alternating_binary_mask, {}),
                ("general48", 48, torchutils.create_alternating_binary_mask,
                 dict(scale_activation=T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION)),
                ("default20", 20, lambda d: torch.tensor([0] * 8 + [1] * 12), {})):
            t = T.AffineCouplingTransform(mask_fn(d), f, **kw).eval()
            for n_, p in t.named_parameters():
                if "final_layer" in n_ or "blocks.1.linear_layers.1" in n_:
                    p.mul_(4.0)
            x = torch.randn(700, d) * 1.5
            y, lad = t(x)
            xi, li = t.inverse(x)
            y64, lad64 = t.double()(x.double())
            t.float()
            rec[name] = dict(sd=t.state_dict(), x=x, y=y, lad=lad, xinv=xi, ladinv=li, y_fp64=y64, lad_fp64=lad64)
        ta = T.AdditiveCouplingTransform(torchutils.create_alternating_binary_mask(48), f).eval()
        for n_, p in ta.named_parameters():
            if "final_layer" in n_:
                p.mul_(4.0)
        x = torch.randn(700, 48)
        y, lad = ta(x)
        rec["additive48"] = dict(sd=ta.state_dict(), x=x, y=y, lad=lad, xinv=ta.inverse(x)[0])
        steps = []
        for i in range(3):
            steps += [T.ActNorm(48), T.CompositeTransform([T.RandomPermutation(48), T.LULinear(48, identity_init=True)]),
                      T.AffineCouplingTransform(torchutils.create_alternating_binary_mask(48, even=(i % 2 == 0)), f)]
        flow = Flow(T.CompositeTransform(steps), StandardNormal([48])).eval()
        perturb(flow)
        x = torch.randn(700, 48)
        lp = flow.log_prob(x)
        lp64 = flow.double().log_prob(x.double())
        flow.float()
        rec["flow48"] = dict(sd=flow.state_dict(), x=x, log_prob=lp, log_prob_fp64=lp64, z=flow.transform_to_noise(x))
    save("affine_rows", rec)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "affine_rows":
        affine_rows()
    elif len(sys.argv) > 1 and sys.argv[1] == "image_rows":
        image_rows()
    elif len(sys.argv) > 1 and sys.argv[1] == "next_rows":
        next_rows()
    elif len(sys.argv) > 1 and sys.argv[1] == "context_rows":
        context_rows()
    else:
        main()
        next_rows()
        context_rows()
        image_rows()
        affine_rows()
