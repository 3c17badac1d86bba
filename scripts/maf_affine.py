"""Masked affine autoregressive transform (MAF) at BASELINE cfg 4's shape (2^18 rows x D = 64, hidden 256, two residual blocks),
without a context and with a 16-wide one: native forward and inverse (nfk_affine_ar_step_f16x3), beside the MAF-RQ step path on the
same trunk (8 bins, linear tails) and the torch formulation of the affine transform (forward, in row chunks) on the same GPU in the
same run.  Prints one JSON line with the card name and its power limit read in this run.

    python scripts/maf_affine.py [--rows N] [--iters K]"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import transforms as T  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--torch-chunk", type=int, default=1 << 15, help="rows per torch forward call")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n, d, h = args.rows, 64, 256
    g = torch.Generator().manual_seed(0)
    x = torch.randn(n, d, generator=g).to(dev)
    c = torch.randn(n, 16, generator=g).to(dev)
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(), "rows": n, "features": d, "hidden": h,
           "num_blocks": 2}
    with torch.no_grad():
        for name, ctx in (("uncond", None), ("ctx16", 16)):
            torch.manual_seed(1)
            aff = T.MaskedAffineAutoregressiveTransform(features=d, hidden_features=h, context_features=ctx, num_blocks=2).eval().to(dev)
            torch.manual_seed(1)
            rq = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=d, hidden_features=h, context_features=ctx,
                                                                          num_bins=8, tails="linear", tail_bound=3.0,
                                                                          num_blocks=2).eval().to(dev)
            cc = None if ctx is None else c
            res["affine_fwd_ms_" + name] = timed(lambda: aff(x, context=cc), args.iters)
            res["affine_inv_ms_" + name] = timed(lambda: aff.inverse(x, context=cc), args.iters)
            res["rq_fwd_ms_" + name] = timed(lambda: rq(x, context=cc), args.iters)
            res["rq_inv_ms_" + name] = timed(lambda: rq.inverse(x, context=cc), args.iters)
            k = args.torch_chunk
            res["torch_fwd_ms_" + name] = timed(lambda: [aff._eager(x[r:r + k], None if cc is None else cc[r:r + k], False)
                                                         for r in range(0, n, k)], args.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
