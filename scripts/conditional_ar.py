"""Context-conditioned masked autoregressive RQ transform at BASELINE cfg 4's shape (2^18 rows x D = 64, hidden 256, 8 bins, linear
tails, two residual blocks) with a 16-wide context: native forward and inverse, beside the unconditional transform of the same shape
and the torch formulation of the conditional one on the same GPU (autograd on, in row chunks the D-pass graph fits in).  Prints one
JSON line with the card name and its power limit read in this run.

    python scripts/conditional_ar.py [--rows N] [--iters K]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import kernels as K  # noqa: E402
from nflows_b200 import transforms as T  # noqa: E402


def power_limit_w(index=0):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out)
    except (OSError, ValueError, subprocess.SubprocessError):
        return None


def timed(fn, iters, warm=1):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def tag_ms(fn, tags):
    """Milliseconds per tag over one call (kernels.TIMELINE: CUDA events around the tagged launches)."""
    K.TIMELINE = []
    fn()
    torch.cuda.synchronize()
    out = {}
    for tag, _, e0, e1 in K.TIMELINE:
        if tag in tags:
            out[tag] = out.get(tag, 0.0) + e0.elapsed_time(e1)
    K.TIMELINE = None
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 18)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--torch-chunk", type=int, default=1 << 15, help="rows per torch forward call")
    ap.add_argument("--torch-inverse-chunk", type=int, default=1 << 12,
                    help="rows per torch inverse call (autograd keeps the graphs of all D passes)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    n, d, h, bins, c = args.rows, 64, 256, 8, 16

    def make(context):
        torch.manual_seed(0)
        return T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=d, hidden_features=h, context_features=context,
                                                                        num_bins=bins, tails="linear", tail_bound=3.0,
                                                                        num_blocks=2).eval().to(dev)

    cond, plain = make(c), make(None)
    z = torch.randn(n, d, device=dev)
    ctx = torch.randn(n, c, device=dev)
    rec = {"workload": "conditional MAF-RQ D=%d H=%d K=%d C=%d" % (d, h, bins, c), "rows": n}
    with torch.no_grad():
        rec["forward_ms"] = timed(lambda: cond(z, context=ctx), args.iters)
        rec["inverse_ms"] = timed(lambda: cond.inverse(z, context=ctx), args.iters)
        rec["unconditional_forward_ms"] = timed(lambda: plain(z), args.iters)
        rec["unconditional_inverse_ms"] = timed(lambda: plain.inverse(z), args.iters)
        rec["inverse_breakdown_ms"] = tag_ms(lambda: cond.inverse(z, context=ctx), ("ar_context_terms", "rq_coupling_step"))
        rec["unconditional_inverse_breakdown_ms"] = tag_ms(lambda: plain.inverse(z), ("rq_coupling_step",))
    rec["inverse_vs_unconditional"] = rec["inverse_ms"] / rec["unconditional_inverse_ms"]
    rec["inverse_samples_per_s"] = n / (rec["inverse_ms"] * 1e-3)

    def torch_path(inverse):
        step = min(n, args.torch_inverse_chunk if inverse else args.torch_chunk)
        for r0 in range(0, n, step):
            out = cond.inverse(z[r0:r0 + step], context=ctx[r0:r0 + step]) if inverse else cond(z[r0:r0 + step], context=ctx[r0:r0 + step])
            del out

    with torch.enable_grad():       # parameters that need a gradient: the differentiable torch formulation
        K._warned_eager[0] = True
        rec["torch_same_gpu_forward_ms"] = timed(lambda: torch_path(False), 1)
        rec["torch_same_gpu_inverse_ms"] = timed(lambda: torch_path(True), 1, warm=0)
    rec["torch_chunk_rows"] = {"forward": min(n, args.torch_chunk), "inverse": min(n, args.torch_inverse_chunk)}
    rec["inverse_speedup_vs_torch"] = rec["torch_same_gpu_inverse_ms"] / rec["inverse_ms"]
    rec["gpu"] = torch.cuda.get_device_name(dev)
    rec["power_limit_w"] = power_limit_w(dev.index or 0)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
