"""Generate tests/golden/image_affine_rows.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows).

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python scripts/make_image_affine_golden.py

Glow / RealNVP-style image flows whose couplings are affine or additive (reference transforms/coupling.py:212-269) with a
ConvResidualNet conditioner, behind ActNorm + OneByOneConvolution, fp32 and fp64:
  "glow_affine":   3 x 16 x 16 images, 3 levels x 2 steps, 32 hidden channels, AffineCouplingTransform with the default scale
                   activation -- squeezed widths 12 / 24 / 48 (6 / 12 / 24 identity channels: padded and unpadded initial layers,
                   gathered and packed coupling paths);
  "glow_general":  the same flow with GENERAL_SCALE_ACTIVATION;
  "glow_additive": the same flow with AdditiveCouplingTransform;
  "glow_mixed":    one level on 4 x 16 x 16 images (16 channels after the squeeze, 8 identity: packed path), 4 steps alternating
                   affine and RQ couplings -- the column layout handed from one head to the other;
  "flat_affine":   CompositeTransform([ActNorm, OneByOneConvolution, AffineCouplingTransform]) on 4 x 8 x 8 images, no squeeze and
                   no multiscale split (2 identity channels).
Every case stores the seed, the weight checksum after the perturbation, the state_dict's keys and shapes, 4 input images x,
z = transform(x), log_prob, the base noise, the sample inverse(noise) and its log|det| `lad_inv`, each with its fp64 twin.  No
weights are stored (they would be ~1 MB per case): nflows_b200's constructors consume the torch CPU RNG in the reference's
order, so the tests re-create them from the seed and the perturbation below and check the checksum.  "rq_default_init"
is the weight checksum of the RQ flow of oracle/make_golden.py's `glow_multiscale` as constructed from seed 99 (the recipe's
default coupling).
The perturbation (`perturb`) moves ActNorm, the LU factors, the biases outside the conditioners and the 3x3 convolution weights, so
every layer shows in the outputs."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as MG  # noqa: E402  (exits with a message when NFLOWS_REFERENCE_SRC is not set)

from nflows.nn.nets import ConvResidualNet  # noqa: E402

torch, T, Flow, np, torchutils = MG.torch, MG.T, MG.Flow, MG.np, MG.torchutils
StandardNormal = MG.StandardNormal
BATCH = 4


def coupling(kind, mask, hidden, scale_activation=None):
    net = lambda i_, o_: ConvResidualNet(i_, o_, hidden_channels=hidden, num_blocks=2)
    if kind == "rq":
        return T.PiecewiseRationalQuadraticCouplingTransform(mask=mask, transform_net_create_fn=net, num_bins=8, tails="linear",
                                                             tail_bound=3.0)
    if kind == "additive":
        return T.AdditiveCouplingTransform(mask=mask, transform_net_create_fn=net)
    kw = {} if scale_activation is None else dict(scale_activation=scale_activation)
    return T.AffineCouplingTransform(mask=mask, transform_net_create_fn=net, **kw)


def glow(kinds, image_shape=(3, 16, 16), levels=3, steps=2, hidden=32, scale_activation=None):
    """The module tree of nflows_b200.flows.recipes.glow_multiscale; step i of every level has coupling kinds[i % len(kinds)]."""
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
            layers.append(T.CompositeTransform([T.ActNorm(c), T.OneByOneConvolution(c),
                                                coupling(kinds[i % len(kinds)], mask, hidden, scale_activation)]))
        shape = mct.add_transform(T.CompositeTransform(layers), (c, h, w))
        if shape is not None:
            c, h, w = shape
    return Flow(mct, StandardNormal([int(np.prod(image_shape))]))


def flat_affine():
    c = 4
    return Flow(T.CompositeTransform([T.ActNorm(c), T.OneByOneConvolution(c),
                                      coupling("affine", torchutils.create_mid_split_binary_mask(c), 32)]),
                StandardNormal([c, 8, 8]))


def perturb(flow, seed):
    """oracle/make_golden.py's `perturb` without its x3 on the final conditioner layers (the inverse of an affine coupling divides
    by scales down to 1e-3; with larger raw scales the samples of these flows reach 1e9), plus 0.05 N(0, 1) on the 3x3 convolution
    weights, whose second layer starts near zero."""
    g = torch.Generator().manual_seed(seed)
    for name, p in flow.named_parameters():
        leaf = name.split(".")[-1]
        if leaf in ("lower_entries", "upper_entries"):
            d = (1 + int(np.sqrt(1 + 8 * p.numel()))) // 2
            p.add_((0.1 / np.sqrt(d)) * torch.randn(p.shape, generator=g))
        elif leaf in ("log_scale", "shift", "unconstrained_upper_diag") or (leaf == "bias" and "transform_net" not in name):
            p.add_(0.1 * torch.randn(p.shape, generator=g))
        elif "conv_layers" in name and leaf == "weight":
            p.add_(0.05 * torch.randn(p.shape, generator=g))


def case(seed, build, image_shape):
    torch.manual_seed(seed)
    flow = build().eval()
    perturb(flow, seed + 1)
    x = torch.randn(BATCH, *image_shape)
    rec = dict(seed=seed, perturb_seed=seed + 1, image_shape=tuple(image_shape), checksum=MG.weight_checksum(flow.state_dict()), x=x)
    rec["shapes"] = [(k, tuple(v.shape)) for k, v in flow.state_dict().items()]
    noise = torch.randn(BATCH, int(np.prod(image_shape)))
    for suffix, dtype in (("", torch.float32), ("_fp64", torch.float64)):
        flow.to(dtype)
        rec["z" + suffix] = flow._transform(x.to(dtype))[0]
        rec["log_prob" + suffix] = flow.log_prob(x.to(dtype))
        rec["sample" + suffix], rec["lad_inv" + suffix] = flow._transform.inverse(
            noise.to(dtype).reshape(-1, *flow._distribution._shape))
    rec["noise"] = noise
    return rec


@torch.no_grad()
def main():
    general = T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION
    rec = {
        "glow_affine": case(90, lambda: glow(["affine"]), (3, 16, 16)),
        "glow_general": case(92, lambda: glow(["affine"], scale_activation=general), (3, 16, 16)),
        "glow_additive": case(94, lambda: glow(["additive"]), (3, 16, 16)),
        "glow_mixed": case(96, lambda: glow(["affine", "rq"], image_shape=(4, 16, 16), levels=1, steps=4), (4, 16, 16)),
        "flat_affine": case(98, flat_affine, (4, 8, 8)),
    }
    torch.manual_seed(99)
    rec["rq_default_init"] = dict(seed=99, checksum=MG.weight_checksum(MG.glow_multiscale().state_dict()))
    MG.save("image_affine_rows", rec)


if __name__ == "__main__":
    main()
