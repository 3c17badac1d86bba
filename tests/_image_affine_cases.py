"""The flows of tests/golden/image_affine_rows.pt (scripts/make_image_affine_golden.py) built from nflows_b200's classes, with the
reference's weights re-created from the seed and the same perturbation (the golden stores no weights, only their checksum)."""
import torch

from conftest import load_golden
from nflows_b200 import transforms as T
from nflows_b200.distributions.normal import StandardNormal
from nflows_b200.flows import Flow, recipes
from nflows_b200.nn.nets import ConvResidualNet
from nflows_b200.utils import torchutils

CASES = ("glow_affine", "glow_general", "glow_additive", "glow_mixed", "flat_affine")
GENERAL = T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION


def golden():
    return load_golden("image_affine_rows")


def conv_net(hidden=32, **kw):
    return lambda i_, o_: ConvResidualNet(i_, o_, hidden_channels=hidden, num_blocks=2, **kw)


def mixed_flow():
    """One level on 4 x 16 x 16 images: squeeze, then 4 steps alternating affine and RQ couplings."""
    c = 16
    layers = [T.SqueezeTransform()]
    for i in range(4):
        mask = torchutils.create_mid_split_binary_mask(c)
        if i % 2:
            mask = 1 - mask
        # constructed in the reference's order (the 1x1 convolution draws its permutation and LU factors before the coupling)
        act, conv = T.ActNorm(c), T.OneByOneConvolution(c)
        coupling = (T.AffineCouplingTransform(mask, conv_net()) if i % 2 == 0 else
                    T.PiecewiseRationalQuadraticCouplingTransform(mask, conv_net(), num_bins=8, tails="linear", tail_bound=3.0))
        layers.append(T.CompositeTransform([act, conv, coupling]))
    mct = T.MultiscaleCompositeTransform(num_transforms=1)
    mct.add_transform(T.CompositeTransform(layers), (c, 8, 8))
    return Flow(mct, StandardNormal([4 * 16 * 16]))


def flat_flow(c=4):
    """CompositeTransform([ActNorm, OneByOneConvolution, affine coupling]) on c x 8 x 8 images."""
    act, conv = T.ActNorm(c), T.OneByOneConvolution(c)           # before the coupling: the reference's RNG order
    coupling = T.AffineCouplingTransform(torchutils.create_mid_split_binary_mask(c), conv_net())
    return Flow(T.CompositeTransform([act, conv, coupling]), StandardNormal([c, 8, 8]))


def unperturbed(key):
    small = dict(image_shape=(3, 16, 16), levels=3, steps=2, hidden_channels=32)
    if key == "glow_affine":
        return recipes.glow_multiscale(coupling="affine", **small)
    if key == "glow_general":
        return recipes.glow_multiscale(coupling="affine", scale_activation=GENERAL, **small)
    if key == "glow_additive":
        return recipes.glow_multiscale(coupling="additive", **small)
    if key == "glow_mixed":
        return mixed_flow()
    return flat_flow()


def perturb(flow, seed):
    """scripts/make_image_affine_golden.py's perturbation: recipes.perturb_ without the x3 on the final conditioner layers, plus
    noise on the 3x3 convolution weights."""
    import numpy as np
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in flow.named_parameters():
            leaf = name.split(".")[-1]
            if leaf in ("lower_entries", "upper_entries"):
                d = (1 + int(np.sqrt(1 + 8 * p.numel()))) // 2
                p.add_((0.1 / np.sqrt(d)) * torch.randn(p.shape, generator=g))
            elif leaf in ("log_scale", "shift", "unconstrained_upper_diag") or (leaf == "bias" and "transform_net" not in name):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "conv_layers" in name and leaf == "weight":
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return flow


def weight_checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values() if v.is_floating_point()))


def build(key, rec):
    """The golden case's flow in eval mode with the reference's weights (CPU, fp32): same state_dict keys and shapes, and the same
    weights from the seed (checksum)."""
    torch.manual_seed(rec["seed"])
    flow = perturb(unperturbed(key), rec["perturb_seed"]).eval()
    assert [(k, tuple(v.shape)) for k, v in flow.state_dict().items()] == [(k, tuple(s)) for k, s in rec["shapes"]], key
    assert abs(weight_checksum(flow.state_dict()) - rec["checksum"]) <= 1e-9 * rec["checksum"], key
    return flow


def noise_input(flow, rec):
    """The stored base noise in the shape the flow's inverse takes."""
    return rec["noise"].reshape(-1, *flow._distribution._shape)
