"""Constructors for the flows BASELINE.json names (SURVEY.md section 8d).  Pure composition of the public classes."""
from torch.nn import functional as F

from .. import transforms as T
from ..distributions.normal import StandardNormal
from ..nn.nets import ResidualNet
from ..utils import torchutils
from .base import Flow


def rq_nsf(features, hidden_features=256, num_layers=10, num_bins=8, tail_bound=3.0, num_blocks=2):
    """cfg 3: num_layers x [ActNorm, Composite[RandomPermutation, LULinear], RQ coupling (alternating mask,
    ResidualNet conditioner)], StandardNormal base.  Consumes the torch RNG in the same order as building the
    same stack from the reference's classes, so a seed reproduces the reference's weights."""
    steps = []
    for i in range(num_layers):
        steps.append(T.ActNorm(features))
        steps.append(T.CompositeTransform([T.RandomPermutation(features), T.LULinear(features, identity_init=True)]))
        steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(features, even=(i % 2 == 0)),
            transform_net_create_fn=lambda i_, o_: ResidualNet(i_, o_, hidden_features=hidden_features,
                                                               num_blocks=num_blocks, activation=F.relu),
            num_bins=num_bins, tails="linear", tail_bound=tail_bound))
    return Flow(T.CompositeTransform(steps), StandardNormal([features]))


def rq_coupling_layer(features=64, hidden_features=128, num_bins=8, tail_bound=3.0, num_blocks=2):
    """cfg 2: a single RQ coupling with an alternating mask."""
    return T.PiecewiseRationalQuadraticCouplingTransform(
        mask=torchutils.create_alternating_binary_mask(features),
        transform_net_create_fn=lambda i_, o_: ResidualNet(i_, o_, hidden_features=hidden_features, num_blocks=num_blocks),
        num_bins=num_bins, tails="linear", tail_bound=tail_bound)


def affine_flow_2d(hidden_features=8):
    """cfg 1: two affine couplings on 2-D data with complementary masks."""
    f = lambda i_, o_: ResidualNet(i_, o_, hidden_features=hidden_features)
    return Flow(T.CompositeTransform([T.AffineCouplingTransform(mask=[1, 0], transform_net_create_fn=f),
                                      T.AffineCouplingTransform(mask=[0, 1], transform_net_create_fn=f)]),
                StandardNormal([2]))


def glow_multiscale(image_shape=(3, 32, 32), levels=4, steps=8, hidden_channels=96, num_bins=8, tail_bound=3.0, coupling="rq",
                    scale_activation=None):
    """cfg 5: `levels` x [SqueezeTransform, `steps` x [ActNorm, OneByOneConvolution, coupling over channels (mid-split mask
    alternated with its complement, ConvResidualNet conditioner)]] combined by a MultiscaleCompositeTransform; same module tree
    (state_dict keys) and RNG consumption as the same stack built from the reference's classes.
    coupling: "rq" (PiecewiseRationalQuadraticCouplingTransform with num_bins, linear tails at tail_bound), "affine" (Glow /
    RealNVP: AffineCouplingTransform with `scale_activation`, None = the class default) or "additive" (NICE:
    AdditiveCouplingTransform)."""
    import numpy as np
    from ..nn.nets import ConvResidualNet
    if coupling not in ("rq", "affine", "additive"):
        raise ValueError("coupling must be 'rq', 'affine' or 'additive', got {!r}".format(coupling))
    net = lambda i_, o_: ConvResidualNet(i_, o_, hidden_channels=hidden_channels, num_blocks=2)

    def make_coupling(mask):
        if coupling == "rq":
            return T.PiecewiseRationalQuadraticCouplingTransform(mask=mask, transform_net_create_fn=net, num_bins=num_bins,
                                                                 tails="linear", tail_bound=tail_bound)
        cls = T.AffineCouplingTransform if coupling == "affine" else T.AdditiveCouplingTransform
        kw = {} if scale_activation is None else dict(scale_activation=scale_activation)
        return cls(mask=mask, transform_net_create_fn=net, **kw)

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
            layers.append(T.CompositeTransform([T.ActNorm(c), T.OneByOneConvolution(c), make_coupling(mask)]))
        shape = mct.add_transform(T.CompositeTransform(layers), (c, h, w))
        if shape is not None:
            c, h, w = shape
    return Flow(mct, StandardNormal([int(np.prod(image_shape))]))


def perturb_(flow, seed=2):
    """The well-conditioned perturbation of SURVEY.md section 8d (makes ActNorm / LU / splines non-trivial)."""
    import numpy as np
    import torch
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in flow.named_parameters():
            leaf = name.split(".")[-1]
            if leaf in ("lower_entries", "upper_entries"):
                d = (1 + int(np.sqrt(1 + 8 * p.numel()))) // 2
                p.add_((0.1 / np.sqrt(d)) * torch.randn(p.shape, generator=g))
            elif leaf in ("log_scale", "shift", "unconstrained_upper_diag") or (leaf == "bias" and "transform_net" not in name):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "final_layer" in name:
                p.mul_(3.0)
    return flow
