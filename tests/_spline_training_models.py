"""The flows of tests/golden/spline_training_grads.pt (scripts/make_spline_training_golden.py) built from nflows_b200's classes,
with the same seeds, perturbation and losses, for the CPU and GPU tests of the image-coupling and CDF training paths."""
import numpy as np
import torch

from nflows_b200 import transforms as T
from nflows_b200.distributions import StandardNormal
from nflows_b200.flows import recipes
from nflows_b200.flows.base import Flow
from nflows_b200.nn.nets import ConvResidualNet, ResidualNet
from nflows_b200.utils import torchutils


def glow_rq(image_shape=(3, 8, 8), levels=2, steps=2, hidden=16):
    return recipes.glow_multiscale(image_shape=image_shape, levels=levels, steps=steps, hidden_channels=hidden)


def nsf_uncond(tails, features=6, hidden=16, bins=5):
    steps = []
    for i in range(2):
        steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(features, even=(i % 2 == 0)),
            transform_net_create_fn=lambda a, b: ResidualNet(a, b, hidden_features=hidden, num_blocks=1),
            num_bins=bins, tails=tails, tail_bound=3.0, apply_unconditional_transform=True))
        steps.append(T.ReversePermutation(features))
    return Flow(T.CompositeTransform(steps), StandardNormal([features]))


def image_uncond(channels=4, size=8, hidden=16):
    coupling = T.PiecewiseRationalQuadraticCouplingTransform(
        mask=torchutils.create_mid_split_binary_mask(channels),
        transform_net_create_fn=lambda a, b: ConvResidualNet(a, b, hidden_channels=hidden, num_blocks=2),
        num_bins=8, tails="linear", tail_bound=3.0, apply_unconditional_transform=True, img_shape=[size, size])
    return Flow(T.CompositeTransform([coupling]), StandardNormal([channels, size, size]))


GOLDEN_BUILDERS = {
    "glow_rq": (glow_rq, False),
    "nsf_uncond_linear": (lambda: nsf_uncond("linear"), False),
    "nsf_uncond_sample": (lambda: nsf_uncond("linear"), True),
    "nsf_uncond_none": (lambda: nsf_uncond(None), False),
    "image_uncond": (image_uncond, False),
}


def weight_checksum(sd):
    return float(sum(v.double().abs().sum() for v in sd.values() if v.is_floating_point()))


def golden_flow(key, rec):
    """The flow of golden case `key`: built from its seed and perturbed as the generator did."""
    build, _ = GOLDEN_BUILDERS[key]
    torch.manual_seed(rec["seed"])
    flow = build().eval()
    recipes.perturb_(flow, rec["perturb_seed"])
    return flow


def sample_loss(flow, noise):
    samples, lad = flow._transform.inverse(noise.reshape(-1, *flow._distribution._shape))
    log_base = -0.5 * noise.square().sum(1) - 0.5 * noise.shape[1] * np.log(2 * np.pi)
    return (0.5 * samples.reshape(samples.shape[0], -1).square().sum(1) - (log_base - lad)).mean()


def loss(flow, x, sample):
    return sample_loss(flow, x) if sample else -flow.log_prob(x).mean()


def grads(flow, x, sample):
    """{name: gradient} of the loss (None entries dropped) and the loss."""
    flow.zero_grad()
    value = loss(flow, x, sample)
    value.backward()
    return {n: p.grad.detach().clone() for n, p in flow.named_parameters() if p.grad is not None}, value.detach()
