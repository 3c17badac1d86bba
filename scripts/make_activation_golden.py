"""Generate tests/golden/activation_rows.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows).

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python scripts/make_activation_golden.py

Conditioners with activations other than relu, and feed-forward MADE blocks (use_residual_blocks=False), fp32 and fp64:
  "maf_flow":    a Flow of 5 x [MaskedAffineAutoregressiveTransform(D = 5, H = 50, feed-forward, torch.tanh, 7-wide context),
                 RandomPermutation] on a standard normal -- the shape of sbi's MAF; log_prob, and the inverse of fixed noise;
  "maf_rq":      MaskedPiecewiseRationalQuadraticAutoregressiveTransform(D = 8, H = 64, K = 8, linear tails, feed-forward,
                 torch.tanh, 6-wide context); forward and inverse;
  "made_gelu":   MaskedAffineAutoregressiveTransform(D = 8, H = 64) with residual blocks and F.gelu; forward and inverse;
  "rq_elu", "rq_elu_ctx": PiecewiseRationalQuadraticCouplingTransform(D = 8, K = 8, linear tails) with a
                 ResidualNet(H = 64, activation=F.elu), without and with a 6-wide context; forward and inverse;
  "affine_leaky": AffineCouplingTransform(D = 8) with an MLP(hidden [64, 64], activation=F.leaky_relu); forward and inverse;
  "mademog_silu": MADEMoG(D = 5, H = 50, C = 10, 7-wide context) with feed-forward blocks and nn.SiLU(); log_prob;
  "cfg4_tanh":   the cfg-4 shape (MAF-RQ, D = 64, H = 256, K = 8, linear tails, tail bound 3, 2 residual blocks) with torch.tanh.
"affine_leaky" and "mademog_silu" store the reference's state_dict; the others, like ar_rq.pt, store (seed, weight checksum): the
package's constructors consume the torch CPU RNG in the same order as the reference's, so the tests re-create its weights (and
the fixture stays small).
Weights are perturbed (`perturb`: every bias + 0.1 N(0, 1), the residual blocks' zero-initialised second linear + 0.05 N(0, 1)),
so every layer shows in the outputs.  tests/test_activations_host.py builds the same modules (BUILDERS there)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as MG  # noqa: E402  (exits with a message when NFLOWS_REFERENCE_SRC is not set)

from nflows.distributions.mixture import MADEMoG  # noqa: E402
from nflows.nn.nets import MLP as ReferenceMLP  # noqa: E402

torch, T, Flow, StandardNormal, ResidualNet = MG.torch, MG.T, MG.Flow, MG.StandardNormal, MG.ResidualNet
F = torch.nn.functional

ROWS = 160
MASK8 = [1, 0, 1, 0, 1, 0, 1, 0]


class MLP(ReferenceMLP):
    """The reference's MLP as a coupling conditioner: the coupling passes a context, which its forward does not take (the
    package's MLP takes and ignores it).  Same parameters and state_dict keys."""

    def forward(self, inputs, context=None):
        return super().forward(inputs)


def perturb(module, seed):
    g = torch.Generator().manual_seed(seed)
    for name, p in module.named_parameters():
        if name.endswith(".bias"):
            p.add_(0.1 * torch.randn(p.shape, generator=g))
        elif "linear_layers.1" in name:
            p.add_(0.05 * torch.randn(p.shape, generator=g))


BUILDERS = {
    "maf_flow": lambda: Flow(T.CompositeTransform(
        [t for _ in range(5) for t in (T.MaskedAffineAutoregressiveTransform(5, 50, context_features=7, use_residual_blocks=False,
                                                                             activation=torch.tanh), T.RandomPermutation(5))]),
        StandardNormal([5])),
    "maf_rq": lambda: T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
        8, 64, context_features=6, num_bins=8, tails="linear", tail_bound=3.0, use_residual_blocks=False, activation=torch.tanh),
    "made_gelu": lambda: T.MaskedAffineAutoregressiveTransform(8, 64, activation=F.gelu),
    "rq_elu": lambda: T.PiecewiseRationalQuadraticCouplingTransform(
        MASK8, lambda i, o: ResidualNet(i, o, 64, num_blocks=2, activation=F.elu), num_bins=8, tails="linear", tail_bound=3.0),
    "rq_elu_ctx": lambda: T.PiecewiseRationalQuadraticCouplingTransform(
        MASK8, lambda i, o: ResidualNet(i, o, 64, context_features=6, num_blocks=2, activation=F.elu), num_bins=8, tails="linear",
        tail_bound=3.0),
    "affine_leaky": lambda: T.AffineCouplingTransform(MASK8, lambda i, o: MLP([i], [o], [64, 64], activation=F.leaky_relu)),
    "mademog_silu": lambda: MADEMoG(5, 50, 7, num_mixture_components=10, use_residual_blocks=False,
                                    activation=torch.nn.SiLU()),
    "cfg4_tanh": lambda: T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
        64, 256, num_bins=8, tails="linear", tail_bound=3.0, num_blocks=2, activation=torch.tanh),
}
FEATURES = {"maf_flow": 5, "maf_rq": 8, "made_gelu": 8, "rq_elu": 8, "rq_elu_ctx": 8, "affine_leaky": 8, "mademog_silu": 5,
            "cfg4_tanh": 64}
STORED = ("affine_leaky", "mademog_silu")
CONTEXT = {"maf_flow": 7, "maf_rq": 6, "rq_elu_ctx": 6, "mademog_silu": 7}


def outputs(name, m, x, c, noise):
    """The case's outputs: {key: tensor}."""
    if name == "maf_flow":
        s, lad = m._transform.inverse(noise, context=c)
        return dict(log_prob=m.log_prob(x, context=c), sample=s, lad_inv=lad)
    if name == "mademog_silu":
        return dict(log_prob=m.log_prob(x, context=c))
    y, lad = m(x, context=c)
    xi, li = m.inverse(x, context=c)
    return dict(y=y, lad=lad, xinv=xi, ladinv=li)


def case(name, seed, store_weights=True, rows=ROWS):
    torch.manual_seed(seed)
    m = BUILDERS[name]().eval()
    perturb(m, seed + 1)
    d, cf = FEATURES[name], CONTEXT.get(name)
    x = torch.randn(rows, d)
    c = None if cf is None else torch.randn(rows, cf)
    noise = torch.randn(rows, d)
    rec = dict(seed=seed, perturb_seed=seed + 1, features=d, context_features=cf, checksum=MG.weight_checksum(m.state_dict()),
               x=x, context=c, noise=noise)
    rec.update(outputs(name, m, x, c, noise))
    if store_weights:
        rec["state_dict"] = {k: v.clone() for k, v in m.state_dict().items()}
    m.double()
    out64 = outputs(name, m, x.double(), None if c is None else c.double(), noise.double())
    rec.update({k + "_fp64": v for k, v in out64.items()})
    return rec


@torch.no_grad()
def main():
    rec = {}
    for i, name in enumerate(BUILDERS):
        rec[name] = case(name, 100 + 2 * i, store_weights=name in STORED, rows=64 if name == "cfg4_tanh" else ROWS)
    MG.save("activation_rows", rec)


if __name__ == "__main__":
    main()
