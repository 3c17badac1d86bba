"""Generate tests/golden/mademog_rows.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows).

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python scripts/make_mademog_golden.py

Mixture-of-Gaussians MADE log-densities (reference nn/nde/made.py:284-427, distributions/mixture.py), fp32 and fp64:
  "sbi":    MADEMoG(D = 5, H = 50, 7-wide context, C = 10) -- the shape of sbi's `made` density estimator;
  "uncond": MixtureOfGaussiansMADE(D = 8, H = 64, C = 5, custom_initialization=True), no context; also the checksum of the
            weights as constructed from the seed (before the perturbation);
  "flow":   a Flow of [ReversePermutation, MaskedAffineAutoregressiveTransform(context_features=5)] x 3 on a MADEMoG base
            (D = 6, H = 32, C = 3) behind an nn.Linear(7, 5) embedding net;
  "large":  MADEMoG(D = 64, H = 256, C = 10, 16-wide context), stored like ar_rq.pt as (seed, weight checksum): the package's
            constructors consume the torch CPU RNG in the same order as the reference's, so the tests re-create its weights.
Weights are perturbed (`perturb`: every bias, and the residual blocks' zero-initialised second linear), so every layer shows in
the outputs."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as MG  # noqa: E402  (exits with a message when NFLOWS_REFERENCE_SRC is not set)

from nflows.distributions.mixture import MADEMoG  # noqa: E402
from nflows.nn.nde.made import MixtureOfGaussiansMADE  # noqa: E402

torch, T, Flow = MG.torch, MG.T, MG.Flow

ROWS = 160
CTX_RAW, CTX = 7, 5


def perturb(module, seed):
    """Every bias + 0.1 N(0, 1); the residual blocks' second linear, which starts near zero (made.py:183-185), + 0.05 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    for name, p in module.named_parameters():
        if name.endswith(".bias"):
            p.add_(0.1 * torch.randn(p.shape, generator=g))
        elif "linear_layers.1" in name:
            p.add_(0.05 * torch.randn(p.shape, generator=g))


def density_case(seed, build, features, context, store_weights, rows=ROWS):
    torch.manual_seed(seed)
    m = build().eval()
    init_checksum = MG.weight_checksum(m.state_dict())
    perturb(m, seed + 1)
    x = torch.randn(rows, features)
    c = None if context is None else torch.randn(rows, context)
    lp = m.log_prob(x, context=c)
    rec = dict(seed=seed, perturb_seed=seed + 1, features=features, context_features=context, init_checksum=init_checksum,
               checksum=MG.weight_checksum(m.state_dict()), x=x, context=c, log_prob=lp)
    if store_weights:
        rec["state_dict"] = {k: v.clone() for k, v in m.state_dict().items()}
    m.double()
    rec["log_prob_fp64"] = m.log_prob(x.double(), context=None if c is None else c.double())
    return rec


@torch.no_grad()
def main():
    rec = {
        "sbi": density_case(80, lambda: MADEMoG(5, 50, 7, num_mixture_components=10), 5, 7, True),
        "uncond": density_case(82, lambda: MixtureOfGaussiansMADE(8, 64, num_mixture_components=5, custom_initialization=True),
                               8, None, True),
        "large": density_case(84, lambda: MADEMoG(64, 256, 16, num_mixture_components=10), 64, 16, False, rows=64),
    }
    torch.manual_seed(86)
    features = 6
    layers = []
    for _ in range(3):
        layers += [T.ReversePermutation(features), T.MaskedAffineAutoregressiveTransform(features=features, hidden_features=64,
                                                                                          context_features=CTX)]
    flow = Flow(T.CompositeTransform(layers), MADEMoG(features, 32, CTX, num_mixture_components=3),
                embedding_net=torch.nn.Linear(CTX_RAW, CTX)).eval()
    perturb(flow, 87)
    x = torch.randn(ROWS, features)
    c = torch.randn(ROWS, CTX_RAW)
    lp = flow.log_prob(x, context=c)
    sd = {k: v.clone() for k, v in flow.state_dict().items()}
    flow.double()
    lp64 = flow.log_prob(x.double(), context=c.double())
    rec["flow"] = dict(features=features, state_dict=sd, x=x, context=c, log_prob=lp, log_prob_fp64=lp64)
    MG.save("mademog_rows", rec)


if __name__ == "__main__":
    main()
