"""Glow-style image flows with affine and additive couplings at the cfg-5 shape (3 x 32 x 32 images, 4 levels x 8 steps, 96 hidden
channels), on the batch bench.py's cfg-5 leg uses (512 images): native log_prob and sample (pixel-row chain)
against the torch formulation of the same modules on the same GPU in the same run (autograd on, cuDNN convolutions), CUDA events
after warm-up.  Also reports the share of the native log_prob's tagged launches (kernels.TIMELINE) per kernel family, and the
largest |native - torch fp64| log_prob difference on 32 images.  The weights are perturbed (`perturb`) with the
final conditioner layers scaled by 0.1: `sample` runs 32 affine inverses, each dividing by scales down to 1e-3, and with the
constructor's final layers the samples of this untrained flow leave the float32 range (NaN on the torch formulation too).
Prints one JSON line with the card name and its power limit read in this run.

    python scripts/image_affine.py [--images N] [--iters K]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import kernels as K  # noqa: E402
from nflows_b200.flows import recipes  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402

FAMILIES = ("im2col3x3_", "linear_", "affine_coupling_final", "split_")


def perturb(flow, seed=2):
    """ActNorm, the LU factors and the biases outside the conditioners (as recipes.perturb_), noise on the 3x3 convolution weights,
    whose second layer starts near zero, and the final conditioner layers x 0.1 (raw scales near 0: scales near sigmoid(2))."""
    import numpy as np
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
        elif "final_layer" in name:
            p.mul_(0.1)
    return flow


def timeline_share(fn):
    """(ms per kernel family, its share of the call) over one call with CUDA events around every tagged launch."""
    K.TIMELINE = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    try:
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        total = e0.elapsed_time(e1)
        ms = {f: 0.0 for f in FAMILIES}
        for tag, _, t0, t1 in K.TIMELINE:
            for f in FAMILIES:
                if tag.startswith(f):
                    ms[f] += t0.elapsed_time(t1)
    finally:
        K.TIMELINE = None
    return {f.rstrip("_"): {"ms": round(v, 3), "share": round(v / total, 4)} for f, v in ms.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=512)
    ap.add_argument("--iters", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n = args.images
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "images": n, "shape": [3, 32, 32],
           "levels": 4, "steps": 8, "hidden_channels": 96}
    with torch.no_grad():
        for coupling in ("affine", "additive"):
            torch.manual_seed(0)
            glow = perturb(recipes.glow_multiscale(coupling=coupling)).eval().to(dev)
            img = torch.randn(n, 3, 32, 32, device=dev)
            r = {"log_prob_ms": timed(lambda: glow.log_prob(img), args.iters, warm=2),
                 "sample_ms": timed(lambda: glow.sample(n), args.iters, warm=2)}
            with torch.enable_grad():           # autograd on: the differentiable torch formulation of the same modules
                r["torch_log_prob_ms"] = timed(lambda: glow.log_prob(img).detach(), args.iters, warm=1)
                r["torch_sample_ms"] = timed(lambda: glow.sample(n).detach(), args.iters, warm=1)
            r["timeline"] = timeline_share(lambda: glow.log_prob(img))
            got = glow.log_prob(img[:32])
            want = glow.double().log_prob(img[:32].double())
            glow.float()
            r["log_prob_max_abs_diff_vs_torch_fp64"] = float((got.double() - want).abs().max())
            r["log_prob_max_rel_diff_vs_torch_fp64"] = float(((got.double() - want).abs() / want.abs().clamp_min(1.0)).max())
            res[coupling] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
