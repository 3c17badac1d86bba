"""fp64 oracle of the mixture-of-Gaussians MADE (reference nn/nde/made.py:208-427), driven by a state_dict alone: the nde MADE
with relu residual blocks, the mixture log-density and a sampler that takes its uniforms and normals as arguments."""
import math

import torch


def _w(sd, key):
    w = sd[key + ".weight"].double()
    return w * sd[key + ".mask"].double() if key + ".mask" in sd else w


def made_outputs(sd, x, context=None, prefix="_made."):
    """MADE.forward (made.py:274-283) and MaskedResidualBlock.forward (made.py:187-202), fp64."""
    p = prefix
    lin = lambda key, v: v @ _w(sd, p + key).t() + sd[p + key + ".bias"].double()
    t = lin("initial_layer", x.double())
    c = None if context is None else context.double()
    if c is not None:
        t = t + lin("context_layer", c)                  # no activation (made.py:276-277)
    b = 0
    while p + "blocks.%d.linear_layers.0.weight" % b in sd:
        u = lin("blocks.%d.linear_layers.0" % b, torch.relu(t))
        if c is not None:
            u = u + lin("blocks.%d.context_layer" % b, c)
        t = t + lin("blocks.%d.linear_layers.1" % b, torch.relu(u))
        b += 1
    return lin("final_layer", t)


def _params(sd, rows, context, num_components, epsilon, prefix):
    out = made_outputs(sd, rows, context, prefix).reshape(rows.shape[0], rows.shape[1], num_components, 3)
    logits, means, stds = out[..., 0], out[..., 1], torch.nn.functional.softplus(out[..., 2]) + epsilon
    return logits, means, stds


def log_prob(sd, x, context, num_components, epsilon=1e-2, prefix="_made."):
    """MixtureOfGaussiansMADE.log_prob (made.py:333-360)."""
    x = x.double()
    logits, means, stds = _params(sd, x, context, num_components, epsilon, prefix)
    terms = torch.log_softmax(logits, -1) - 0.5 * (math.log(2 * math.pi) + 2 * torch.log(stds) + ((x[..., None] - means) / stds) ** 2)
    return torch.logsumexp(terms, -1).sum(-1)


def sample(sd, u, e, context, num_components, epsilon=1e-2, prefix="_made."):
    """MixtureOfGaussiansMADE.sample (made.py:362-401) with the draws given: feature i takes component c* = the first c with
    u[:, i] < cumulative softmax weight (the last when u is above the total) and mean + std * e[:, i].  Returns the samples and,
    per row, the smallest distance of a u to a cumulative-weight boundary (fp64)."""
    n, d = u.shape
    samples = torch.zeros(n, d, dtype=torch.float64)
    margin = torch.full((n,), math.inf, dtype=torch.float64)
    for i in range(d):
        logits, means, stds = _params(sd, samples, context, num_components, epsilon, prefix)
        cdf = torch.cumsum(torch.softmax(logits[:, i], -1), -1)
        ui = u[:, i].double()
        c = torch.clamp((ui[:, None] >= cdf).sum(-1), max=num_components - 1)
        margin = torch.minimum(margin, (cdf[:, :-1] - ui[:, None]).abs().min(-1).values if num_components > 1 else margin)
        rows = torch.arange(n)
        samples[:, i] = means[rows, i, c] + stds[rows, i, c] * e[:, i].double()
    return samples, margin
