"""Generate tests/golden/maf_affine_rows.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows).

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python scripts/make_maf_affine_golden.py

Masked affine autoregressive transforms (reference transforms/autoregressive.py:64-128: scale = softplus(u) + 1e-3 with
u = params.view(B, D, 2)[..., 0], shift = [..., 1]) on MADE (made.py), fp32 and fp64 outputs of forward, inverse and log_prob:
  "single":  one transform, D = 16, H = 64, 2 blocks;
  "flow":    a Flow of [ReversePermutation, MaskedAffineAutoregressiveTransform(context_features=5)] x 3 behind an nn.Linear
             embedding net (a 5-wide context: not a multiple of 8), D = 8, H = 64;
  "small":   one transform, D = 5 (not a multiple of 8), H = 32, unconditional;
  "cfg4":    the cfg-4 shape D = 64, H = 256, 2 blocks.
Weights are perturbed (`perturb` below: every bias, and the residual blocks' zero-initialised second linear, so every layer shows
in the outputs).  The final layer keeps its initialisation: scaled up, the scales of the inverse reach 1e-3 and its outputs 1e15.
"single", "flow" and "small" store the reference's state_dict; "cfg4", like ar_rq.pt, stores (seed, weight checksum): the package's constructors consume the torch CPU RNG in the same order as the reference's, so the tests
re-create its weights from the seed."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as MG  # noqa: E402  (exits with a message when NFLOWS_REFERENCE_SRC is not set)

torch, T, Flow, StandardNormal = MG.torch, MG.T, MG.Flow, MG.StandardNormal

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


def maf(features, hidden, context=None, num_blocks=2):
    return T.MaskedAffineAutoregressiveTransform(features=features, hidden_features=hidden, context_features=context,
                                                 num_blocks=num_blocks)


def transform_case(seed, features, hidden, store_weights, rows=ROWS):
    torch.manual_seed(seed)
    t = maf(features, hidden).eval()
    perturb(t, seed + 1)
    x = torch.randn(rows, features)
    y, lad = t(x)
    xi, li = t.inverse(x)
    rec = dict(seed=seed, perturb_seed=seed + 1, features=features, hidden=hidden, checksum=MG.weight_checksum(t.state_dict()),
               x=x, y=y, lad=lad, xinv=xi, ladinv=li)
    if store_weights:
        rec["state_dict"] = {k: v.clone() for k, v in t.state_dict().items()}
    t.double()
    y64, lad64 = t(x.double())
    xi64, li64 = t.inverse(x.double())
    rec.update(y_fp64=y64, lad_fp64=lad64, xinv_fp64=xi64, ladinv_fp64=li64)
    return rec


@torch.no_grad()
def main():
    rec = {"single": transform_case(60, 16, 64, True), "small": transform_case(62, 5, 32, True),
           "cfg4": transform_case(64, 64, 256, False, rows=64)}

    torch.manual_seed(66)
    features = 8
    layers = []
    for _ in range(3):
        layers += [T.ReversePermutation(features), maf(features, 64, context=CTX)]
    flow = Flow(T.CompositeTransform(layers), StandardNormal([features]), embedding_net=torch.nn.Linear(CTX_RAW, CTX)).eval()
    perturb(flow, 67)
    x = torch.randn(ROWS, features)
    c = torch.randn(ROWS, CTX_RAW)
    lp = flow.log_prob(x, context=c)
    e = flow._embedding_net(c)
    # the inverse runs on the image of fresh inputs: standard normal noise drives some rows of this untrained flow to 1e7
    noise = flow._transform(torch.randn(ROWS, features), context=e)[0]
    z, lad = flow._transform(x, context=e)
    xs, lad_inv = flow._transform.inverse(noise, context=e)
    sd = {k: v.clone() for k, v in flow.state_dict().items()}
    flow.double()
    lp64 = flow.log_prob(x.double(), context=c.double())
    e64 = flow._embedding_net(c.double())
    z64, lad64 = flow._transform(x.double(), context=e64)
    xs64, lad_inv64 = flow._transform.inverse(noise.double(), context=e64)
    rec["flow"] = dict(features=features, state_dict=sd, x=x, context=c, log_prob=lp, log_prob_fp64=lp64, z=z, lad=lad, z_fp64=z64,
                       lad_fp64=lad64, noise=noise, sample=xs, lad_inv=lad_inv, sample_fp64=xs64, lad_inv_fp64=lad_inv64)
    MG.save("maf_affine_rows", rec)


if __name__ == "__main__":
    main()
