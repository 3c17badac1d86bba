"""Mixture-of-Gaussians MADE (MADEMoG) at 2^18 rows: native log_prob and sample (nfk_mog_made_step_f16x3) against the torch
formulation on the same GPU in the same run, for two shapes:
  "d64":  D = 64, H = 256, C = 10, a 16-wide context, 2 residual blocks;
  "sbi":  D = 5, H = 50, C = 10, a 20-wide context, 2 residual blocks (the shape of sbi's `made` density estimator).
sample draws one sample per context row (2^18 context rows).  The torch formulation runs in row chunks (its temporaries of
[rows, D, C, 3] would not fit otherwise).  Also reports how far the native log_prob is from the torch formulation's.  Prints one
JSON line with the card name and its power limit read in this run.

    python scripts/mademog.py [--rows N] [--iters K]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200.distributions import MADEMoG  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402

SHAPES = {"d64": (64, 256, 10, 16), "sbi": (5, 50, 10, 20)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--torch-chunk", type=int, default=1 << 14, help="rows per torch formulation call")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n, k = args.rows, args.torch_chunk
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "rows": n, "num_blocks": 2}
    with torch.no_grad():
        for name, (d, h, comps, cf) in SHAPES.items():
            torch.manual_seed(0)
            m = MADEMoG(d, h, cf, num_mixture_components=comps).eval().to(dev)
            made = m._made
            g = torch.Generator().manual_seed(1)
            x = torch.randn(n, d, generator=g).to(dev)
            c = torch.randn(n, cf, generator=g).to(dev)
            res["log_prob_ms_" + name] = timed(lambda: m.log_prob(x, context=c), args.iters)
            res["sample_ms_" + name] = timed(lambda: m.sample(1, context=c), args.iters)
            res["torch_log_prob_ms_" + name] = timed(lambda: [made._torch_log_prob(x[r:r + k], c[r:r + k]) for r in range(0, n, k)],
                                                     args.iters)
            native = made.__class__._native_sample_ready
            made.__class__._native_sample_ready = lambda self, ctx: False       # the torch formulation of sample
            try:
                res["torch_sample_ms_" + name] = timed(lambda: [m.sample(1, context=c[r:r + k]) for r in range(0, n, k)], args.iters)
            finally:
                made.__class__._native_sample_ready = native
            lp = m.log_prob(x, context=c)
            ref = torch.cat([made._torch_log_prob(x[r:r + k], c[r:r + k]) for r in range(0, n, k)])
            res["log_prob_max_abs_diff_" + name] = float((lp - ref).abs().max())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
