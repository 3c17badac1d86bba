"""Generate tests/golden/conditional_ar_rows.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows).

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python scripts/make_conditional_ar_golden.py

Context-conditioned masked autoregressive RQ transforms (SURVEY section 8 row f4 on the autoregressive side): MADE with context
layers (made.py:187-202, 274-283), D = 16, H = 64, a 5-wide context (not a multiple of 8).  "linear": a Flow of RandomPermutations
and two such transforms with linear tails behind an embedding net; "none": one transform without tails on inputs in [0, 1].  fp32
and fp64 outputs of forward, inverse and log_prob.

Like ar_rq.pt, the fixture stores no weights: (seed, weight checksum) -- the package's constructors consume the torch CPU RNG in
the same order as the reference's, so the tests re-create the weights from the seed and compare the checksum.  The shared helpers
(reference import, `perturb`, `save`) are those of oracle/make_golden.py."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as MG  # noqa: E402  (exits with a message when NFLOWS_REFERENCE_SRC is not set)

torch, T, Flow, StandardNormal = MG.torch, MG.T, MG.Flow, MG.StandardNormal

FEATURES, CTX_RAW, CTX, ROWS = 16, 7, 5, 120


def maf(tails):
    kw = dict(tails="linear", tail_bound=3.0) if tails == "linear" else dict(tails=None)
    return T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=FEATURES, hidden_features=64, context_features=CTX,
                                                                    num_bins=8, num_blocks=2, **kw)


def sharpen(module, seed):
    """The residual blocks' second linear starts near zero (made.py:183-185): give it weight, so the block context terms show in
    the outputs."""
    g = torch.Generator().manual_seed(seed)
    for name, p in module.named_parameters():
        if "linear_layers.1" in name:
            p.add_(0.05 * torch.randn(p.shape, generator=g))


@torch.no_grad()
def main():
    rec = {}
    torch.manual_seed(50)
    flow = Flow(T.CompositeTransform([T.RandomPermutation(FEATURES), maf("linear"), T.RandomPermutation(FEATURES), maf("linear")]),
                StandardNormal([FEATURES]), embedding_net=torch.nn.Linear(CTX_RAW, CTX)).eval()
    MG.perturb(flow)
    sharpen(flow, 51)
    x = torch.randn(ROWS, FEATURES)
    c = torch.randn(ROWS, CTX_RAW)
    noise = torch.randn(ROWS, FEATURES)
    lp = flow.log_prob(x, context=c)
    e = flow._embedding_net(c)
    z, lad = flow._transform(x, context=e)
    xs, lad_inv = flow._transform.inverse(noise, context=e)
    checksum = MG.weight_checksum(flow.state_dict())
    flow.double()
    lp64 = flow.log_prob(x.double(), context=c.double())
    e64 = flow._embedding_net(c.double())
    z64, lad64 = flow._transform(x.double(), context=e64)
    xs64, lad_inv64 = flow._transform.inverse(noise.double(), context=e64)
    rec["linear"] = dict(seed=50, sharpen_seed=51, checksum=checksum, x=x, context=c, log_prob=lp, log_prob_fp64=lp64, z=z, lad=lad,
                         z_fp64=z64, lad_fp64=lad64, noise=noise, sample=xs, lad_inv=lad_inv, sample_fp64=xs64, lad_inv_fp64=lad_inv64)

    torch.manual_seed(52)
    t = maf(None).eval()
    MG.perturb(t)
    sharpen(t, 53)
    x = torch.rand(ROWS, FEATURES)
    c = torch.randn(ROWS, CTX)
    y, lad = t(x, context=c)
    xi, li = t.inverse(x, context=c)
    checksum = MG.weight_checksum(t.state_dict())
    t.double()
    y64, lad64 = t(x.double(), context=c.double())
    xi64, li64 = t.inverse(x.double(), context=c.double())
    rec["none"] = dict(seed=52, sharpen_seed=53, checksum=checksum, x=x, context=c, y=y, lad=lad, y_fp64=y64, lad_fp64=lad64,
                       xinv=xi, ladinv=li, xinv_fp64=xi64, ladinv_fp64=li64)
    MG.save("conditional_ar_rows", rec)


if __name__ == "__main__":
    main()
