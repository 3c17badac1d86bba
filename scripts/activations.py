"""Conditioner activations on the native kernels, at 2^18 rows, against the torch formulation on the same GPU in the same run:
  "sbi":  a Flow of 5 x [MaskedAffineAutoregressiveTransform(D = 5, H = 50, feed-forward, torch.tanh, 7-wide context),
          RandomPermutation] -- the shape of sbi's MAF: log_prob and sample (one sample per context row);
  "cfg4": the cfg-4 shape (MAF-RQ, D = 64, H = 256, K = 8, linear tails, 2 residual blocks) forward and inverse with relu, tanh
          and GELU -- what the activation costs in the trunk.
The native runs have config.native_activations on.  Prints one JSON line with the card name and its power limit read in this
run.

    python scripts/activations.py [--rows N] [--iters K]"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import config  # noqa: E402
from nflows_b200 import transforms as T  # noqa: E402
from nflows_b200.distributions import StandardNormal  # noqa: E402
from nflows_b200.flows import Flow  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402


def sbi_flow():
    layers = []
    for _ in range(5):
        layers += [T.MaskedAffineAutoregressiveTransform(5, 50, context_features=7, use_residual_blocks=False, activation=torch.tanh),
                   T.RandomPermutation(5)]
    return Flow(T.CompositeTransform(layers), StandardNormal([5]))


def torch_formulation(module, fn):
    """fn() with every autoregressive transform of `module` on its torch formulation."""
    cls = [T.MaskedAffineAutoregressiveTransform, T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform]
    saved = [c._native_ready for c in cls]
    for c in cls:
        c._native_ready = lambda self, inputs, context: False
    try:
        return fn()
    finally:
        for c, s in zip(cls, saved):
            c._native_ready = s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    config.native_activations = True
    dev = torch.device("cuda:0")
    n = args.rows
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "rows": n}
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        torch.manual_seed(0)
        flow = sbi_flow().eval().to(dev)
        x, c = torch.randn(n, 5, generator=g).to(dev), torch.randn(n, 7, generator=g).to(dev)
        res["sbi_log_prob_ms"] = timed(lambda: flow.log_prob(x, context=c), args.iters)
        res["sbi_sample_ms"] = timed(lambda: flow.sample(1, context=c), args.iters)
        res["sbi_torch_log_prob_ms"] = torch_formulation(flow, lambda: timed(lambda: flow.log_prob(x, context=c), args.iters))
        res["sbi_torch_sample_ms"] = torch_formulation(flow, lambda: timed(lambda: flow.sample(1, context=c), args.iters))
        lp = flow.log_prob(x, context=c)
        ref = torch_formulation(flow, lambda: flow.log_prob(x, context=c))
        res["sbi_log_prob_max_abs_diff"] = float((lp - ref).abs().max())
        z = torch.randn(n, 64, generator=g).to(dev)
        for name, act in (("relu", F.relu), ("tanh", torch.tanh), ("gelu", F.gelu)):
            torch.manual_seed(0)
            ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(64, 256, num_bins=8, tails="linear", tail_bound=3.0,
                                                                            num_blocks=2, activation=act).eval().to(dev)
            res["cfg4_forward_ms_" + name] = timed(lambda: ar(z), args.iters)
            res["cfg4_inverse_ms_" + name] = timed(lambda: ar.inverse(z), max(1, args.iters - 1))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
