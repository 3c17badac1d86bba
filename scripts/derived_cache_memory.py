#!/usr/bin/env python
"""Device memory of a MAF-RQ (D = 64, H = 256, K = 8, linear tails, 2 blocks) across parameter updates: each cycle adds 1e-3
to every parameter in place, then runs a no-grad forward and inverse, and prints torch.cuda.memory_allocated().  The operands
the native path derives from the parameters (masked weights, step plans, packed final layers, sorted sub-networks) are
rebuilt in place on each update, so the series stays flat after the first cycle.

    python scripts/derived_cache_memory.py [--cycles 50] [--rows 4096]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from nflows_b200 import transforms as T  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cycles", type=int, default=50)
    ap.add_argument("--rows", type=int, default=4096)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    torch.manual_seed(0)
    t = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=64, hidden_features=256, num_bins=8, tails="linear",
                                                                  tail_bound=3.0, num_blocks=2).cuda().eval()
    x = torch.randn(args.rows, 64, device="cuda")
    series = []
    with torch.no_grad():
        for cycle in range(args.cycles):
            for p in t.parameters():
                p.add_(1e-3)
            t(x)
            t.inverse(x)
            torch.cuda.synchronize()
            series.append(torch.cuda.memory_allocated())
            print("cycle {:2d}: memory_allocated {} bytes".format(cycle + 1, series[-1]), flush=True)
    print(json.dumps({"workload": "MAF-RQ D=64 H=256 K=8 linear tails", "rows": args.rows, "cycles": args.cycles,
                      "gpu": torch.cuda.get_device_name(), "memory_allocated": series}))


if __name__ == "__main__":
    main()
