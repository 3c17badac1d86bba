"""Training step of Glow-RQ image flows and of RQ couplings with apply_unconditional_transform=True, with the spline on the kernels
(config.native_training) against the torch formulation, on the same GPU in the same process: the two arms are built from the same
seed and timed in alternating windows on the same batch.  One step = -flow.log_prob(x).mean(), backward, SGD step.  Models:
  "glow_cfg5_b64" / "glow_cfg5_b256": recipes.glow_multiscale() (cfg 5: 3 x 32 x 32, 4 levels x 8 steps, 96 hidden channels,
      K = 8, linear tails) at 64 and 256 images;
  "uncond_x5_b65536": 5 x [RQ coupling (D = 64, H = 128, K = 8, linear tails, 2 residual blocks, apply_unconditional_transform),
      RandomPermutation] at batch 2^16.
For each: the median over the windows of milliseconds per step, and torch.cuda.max_memory_allocated over one step above the
resident model, per arm.  Then each backward kernel alone: nfk_rqs_planes_backward at the level-1 shape of cfg 5 (512 images,
C_t = 6, P = 256, K = 8: reads x, grad_y and 23 parameters, writes grad_x and 23 parameter gradients, 4 bytes each, plus grad_lad)
and nfk_rqs_shared_backward at 2^20 x 32 (K = 8: reads x and grad_y, writes grad_x, plus grad_lad; the 23 x 32 shared parameters
and their gradients are negligible), as GB/s and as a share of the H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  Prints one
JSON line with the card name and its power limit read in this run.

    python scripts/train_image_spline.py [--iters K] [--rounds R]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import _native as N  # noqa: E402
from nflows_b200 import config  # noqa: E402
from nflows_b200 import kernels as K  # noqa: E402
from nflows_b200 import transforms as T  # noqa: E402
from nflows_b200.distributions import StandardNormal  # noqa: E402
from nflows_b200.flows import Flow, recipes  # noqa: E402
from nflows_b200.nn.nets import ResidualNet  # noqa: E402
from nflows_b200.utils import torchutils  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402

HBM_PEAK_GBS = 3350.0


def uncond_x5():
    steps = []
    for i in range(5):
        steps += [T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(64, even=(i % 2 == 0)),
            transform_net_create_fn=lambda a, b: ResidualNet(a, b, hidden_features=128, num_blocks=2),
            num_bins=8, tails="linear", tail_bound=3.0, apply_unconditional_transform=True), T.RandomPermutation(64)]
    return Flow(T.CompositeTransform(steps), StandardNormal([64]))


def measure(make, x, iters, rounds, dev):
    arms = {}
    for arm in ("torch", "native"):
        torch.manual_seed(0)
        model = make().to(dev)
        arms[arm] = (model, torch.optim.SGD(model.parameters(), lr=1e-5))

    def step(arm):
        config.native_training = arm == "native"
        model, opt = arms[arm]
        opt.zero_grad(set_to_none=True)
        (-model.log_prob(x).mean()).backward()
        opt.step()

    out = {}
    for arm in arms:                          # warm-up, then the peak of one step above what is resident before it
        step(arm)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        step(arm)
        torch.cuda.synchronize()
        out[arm] = {"peak_mib_above_resident": round((torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20, 1)}
    times = {arm: [] for arm in arms}
    for _ in range(rounds):
        for arm in arms:
            times[arm].append(timed(lambda: step(arm), iters, warm=0))
    config.native_training = False
    for arm in arms:
        out[arm]["ms_per_step"] = round(statistics.median(times[arm]), 3)
        out[arm]["ms_windows"] = [round(t, 3) for t in times[arm]]
    out["speedup"] = round(out["torch"]["ms_per_step"] / out["native"]["ms_per_step"], 3)
    out["memory_ratio"] = round(out["torch"]["peak_mib_above_resident"] / max(out["native"]["peak_mib_above_resident"], 1e-9), 3)
    del arms
    torch.cuda.empty_cache()
    return out


def rate(ms, nbytes):
    gbs = nbytes / (ms * 1e-3) / 1e9
    return {"ms": round(ms, 4), "GB_per_s": round(gbs, 1), "share_of_hbm_peak": round(gbs / HBM_PEAK_GBS, 3)}


def planes_backward(iters, dev):
    n, c, h, w, m = 512, 6, 16, 16, 23
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(n, c, h, w, device=dev, generator=g) * 2
    params = torch.randn(n, c * m, h, w, device=dev, generator=g)
    gy = torch.randn(n, c, h, w, device=dev, generator=g)
    gl = torch.randn(n, device=dev, generator=g)
    desc = N.spline_desc(8, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3, False, 96 ** 0.5)
    ms = timed(lambda: K.rqs_planes_backward(desc, False, x, params, gy, gl), iters, warm=3)
    el = n * c * h * w
    return dict(elements=el, **rate(ms, el * (2 * m + 4) * 4 + n * 4))


def shared_backward(iters, dev):
    rows, f, k = 1 << 20, 32, 8
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(rows, f, device=dev, generator=g) * 2
    uw, uh, ud = (torch.rand(f, d, device=dev, generator=g) for d in (k, k, k - 1))
    gy = torch.randn(rows, f, device=dev, generator=g)
    gl = torch.randn(rows, device=dev, generator=g)
    desc = N.spline_desc(k, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3)
    ms = timed(lambda: K.rqs_shared_backward(desc, False, x, uw, uh, ud, gy, gl), iters, warm=3)
    return dict(elements=rows * f, **rate(ms, rows * f * 12 + rows * 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_image_spline.py measures on a GPU; none is available")
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w()}
    for batch in (64, 256):
        torch.manual_seed(1)
        x = torch.randn(batch, 3, 32, 32, device=dev)
        res["glow_cfg5_b%d" % batch] = measure(recipes.glow_multiscale, x, args.iters, args.rounds, dev)
    torch.manual_seed(1)
    res["uncond_x5_b65536"] = measure(uncond_x5, torch.randn(1 << 16, 64, device=dev), args.iters, args.rounds, dev)
    res["rqs_planes_backward_512x6x256"] = planes_backward(max(args.iters, 20), dev)
    res["rqs_shared_backward_2p20x32"] = shared_backward(max(args.iters, 20), dev)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
