"""Training step with the spline on the kernels (config.native_training) against the torch formulation, on the same GPU in the
same run.  One step = -flow.log_prob(x).mean(), backward, SGD step.  Models:
  "cfg2x5": 5 x [cfg-2 RQ coupling (D = 64, H = 128, K = 8, linear tails, 2 residual blocks), RandomPermutation], batch 2^16;
  "cfg4":   MAF-RQ (D = 64, H = 256, K = 8, linear tails, 2 residual blocks), batch 2^14.
For each: milliseconds per step and torch.cuda.max_memory_allocated over one step, native and torch.  Then nfk_rqs_rows_backward
alone at 2^20 x 32 elements (K = 8, tails): achieved GB/s with 92 + 8 bytes read and 92 + 4 written per element, over the H100
SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  Prints one JSON line with the card name and its power limit read in this run.

    python scripts/train_spline.py [--iters K]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import _native as N  # noqa: E402
from nflows_b200 import config  # noqa: E402
from nflows_b200 import kernels as K  # noqa: E402
from nflows_b200 import transforms as T  # noqa: E402
from nflows_b200.distributions import StandardNormal  # noqa: E402
from nflows_b200.flows import Flow, recipes  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402

HBM_PEAK_GBS = 3350.0


def cfg2x5():
    steps = []
    for _ in range(5):
        steps += [recipes.rq_coupling_layer(features=64, hidden_features=128), T.RandomPermutation(64)]
    return Flow(T.CompositeTransform(steps), StandardNormal([64]))


def cfg4():
    return Flow(T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=64, hidden_features=256, num_bins=8, tails="linear",
                                                                         tail_bound=3.0), StandardNormal([64]))


def measure(make, batch, iters, dev):
    out = {}
    x = torch.randn(batch, 64, device=dev)
    for arm, native in (("torch", False), ("native", True)):
        config.native_training = native
        torch.manual_seed(0)
        model = make().to(dev)
        opt = torch.optim.SGD(model.parameters(), lr=1e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            (-model.log_prob(x).mean()).backward()
            opt.step()
        step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        step()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev) - base
        ms = timed(step, iters)
        out[arm] = {"ms_per_step": round(ms, 3), "peak_mib_above_resident": round(peak / 2 ** 20, 1)}
        del model, opt
        torch.cuda.empty_cache()
    config.native_training = False
    out["speedup"] = round(out["torch"]["ms_per_step"] / out["native"]["ms_per_step"], 3)
    out["memory_ratio"] = round(out["torch"]["peak_mib_above_resident"] / max(out["native"]["peak_mib_above_resident"], 1e-9), 3)
    return out


def backward_kernel(iters, dev):
    rows, d_t, bins, m = 1 << 20, 32, 8, 23
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(rows, d_t, device=dev, generator=g) * 2
    params = torch.randn(rows, d_t * m, device=dev, generator=g)
    gy = torch.randn(rows, d_t, device=dev, generator=g)
    gl = torch.randn(rows, device=dev, generator=g)
    desc = N.spline_desc(bins, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3, False, 16.0)
    ms = timed(lambda: K.rqs_rows_backward(desc, False, x, params, gy, gl), iters, warm=3)
    nbytes = rows * d_t * (92 + 8 + 92 + 4) + rows * 4
    gbs = nbytes / (ms * 1e-3) / 1e9
    return {"elements": rows * d_t, "ms": round(ms, 4), "GB_per_s": round(gbs, 1), "share_of_hbm_peak": round(gbs / HBM_PEAK_GBS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_spline.py measures on a GPU; none is available")
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
           "cfg2x5_b65536": measure(cfg2x5, 1 << 16, args.iters, dev),
           "cfg4_b16384": measure(cfg4, 1 << 14, args.iters, dev),
           "rqs_rows_backward_2p20x32": backward_kernel(max(args.iters, 20), dev)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
