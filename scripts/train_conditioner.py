"""Training step with the conditioners on the tensor-core dense layers (config.native_training, dense.DenseChainTraining) against
the spline-only native path and the torch formulation, in one process with alternating timing windows.  One step =
-flow.log_prob(x).mean(), backward, SGD step.  Models:
  "cfg2x5":   5 x [cfg-2 RQ coupling (D = 64, H = 128, K = 8, linear tails, 2 residual blocks), RandomPermutation], batch 2^16;
  "nsf784":   3-layer NSF (D = 784, H = 256, K = 8, 2 residual blocks per coupling), batch 2^12.
Arms: "torch" (native_training off), "spline" (on, conditioner gate closed: the splines on the kernels, the conditioners on
cuBLAS under autograd), "spline_conditioner" (both on the kernels).  For each: ms per step (median of alternating windows) and
torch.cuda.max_memory_allocated over one step.  Then a torch.profiler split of one native step (CUDA time per kernel family),
the host-read cost of the gradient exponents, and nfk_linear_f16x3_wgrad alone at 2^16 x 128 x 128 and 2^16 x 736 x 128: achieved
FLOP/s (2 B out in per product, three MMAs each) against the data-sheet 989 TFLOP/s dense FP16 / 3.  Prints one JSON line with
the card name, its power limit and torch.backends.cuda.matmul.allow_tf32, read in this run.

    python scripts/train_conditioner.py [--windows W] [--iters K] [--out DIR]"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from nflows_b200 import config  # noqa: E402
from nflows_b200 import kernels as K  # noqa: E402
from nflows_b200 import transforms as T  # noqa: E402
from nflows_b200.distributions import StandardNormal  # noqa: E402
from nflows_b200.flows import Flow, recipes  # noqa: E402
from nflows_b200.transforms.splines import training  # noqa: E402
from scripts.conditional_ar import power_limit_w, timed  # noqa: E402
from scripts.train_spline import cfg2x5  # noqa: E402

FP16_DENSE_TFLOPS = 989.0
_GATE = training.routed_conditioner


def nsf784():
    return recipes.rq_nsf(features=784, hidden_features=256, num_layers=3)


def set_arm(arm):
    config.native_training = arm != "torch"
    training.routed_conditioner = _GATE if arm == "spline_conditioner" else (lambda net, inputs, context: False)


ARMS = ("torch", "spline", "spline_conditioner")


def measure(make, batch, d, windows, iters, dev):
    x = torch.randn(batch, d, device=dev)
    steps, mem = {}, {}
    for arm in ARMS:
        torch.manual_seed(0)
        model = make().to(dev)
        opt = torch.optim.SGD(model.parameters(), lr=1e-5)

        def step(model=model, opt=opt):
            opt.zero_grad(set_to_none=True)
            (-model.log_prob(x).mean()).backward()
            opt.step()
        steps[arm] = step
    times = {arm: [] for arm in ARMS}
    for arm in ARMS:                                   # warm-up and peak memory of one step
        set_arm(arm)
        steps[arm]()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        steps[arm]()
        torch.cuda.synchronize()
        mem[arm] = round((torch.cuda.max_memory_allocated(dev) - base) / 2 ** 20, 1)
    for _ in range(windows):                           # alternating windows: drift hits every arm alike
        for arm in ARMS:
            set_arm(arm)
            times[arm].append(timed(steps[arm], iters, warm=0))
    out = {arm: {"ms_per_step": round(statistics.median(times[arm]), 3), "steps_per_s": round(1e3 / statistics.median(times[arm]), 2),
                 "ms_windows": [round(t, 3) for t in times[arm]], "peak_mib_above_resident": mem[arm]} for arm in ARMS}
    set_arm("spline_conditioner")
    out["profile"] = profile(steps["spline_conditioner"])
    out["exponent_reads"] = exponent_reads(steps["spline_conditioner"])
    set_arm("spline")
    out["profile_spline_only"] = profile(steps["spline"])
    set_arm("torch")
    return out


def family(name):
    n = name.lower()
    for key in ("linear_wgrad", "wgrad_reduce", "bias_partial", "mask_split", "absmax", "linear_f16x3", "split_f16", "rqs_rows_backward",
                "rqs_rows", "gemm", "sgemm", "cutlass", "ampere", "sm90", "nvjet"):
        if key in n:
            return "cublas_gemm" if key in ("gemm", "sgemm", "cutlass", "ampere", "sm90", "nvjet") else key
    return "other"


def profile(step):
    from torch.profiler import ProfilerActivity, profile as prof
    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        step()
        torch.cuda.synchronize()
    split = {}
    for e in p.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t:
            f = family(e.key)
            split[f] = split.get(f, 0.0) + t / 1e3
    total = sum(split.values())
    return {"gpu_ms_total": round(total, 3), "ms_by_family": {k: round(v, 3) for k, v in sorted(split.items(), key=lambda kv: -kv[1])}}


def exponent_reads(step):
    """The number of gradient-exponent host reads in one step."""
    count = [0]
    real = K.absmax_start

    def counted(x):
        count[0] += 1
        return real(x)
    K.absmax_start = counted
    try:
        step()
        torch.cuda.synchronize()
    finally:
        K.absmax_start = real
    return {"host_reads_per_step": count[0]}


def wgrad_rate(n, out, inp, iters, dev):
    g32 = torch.randn(n, out, device=dev) * 1e-4
    a32 = torch.relu(torch.randn(n, inp, device=dev))
    g = K.split_f16(g32, K.gradient_exp(K.absmax(g32)))
    a = K.split_f16(a32, 6)
    ms = timed(lambda: K.linear_wgrad(g, a), iters, warm=3)
    flop = 2.0 * n * out * inp
    tflops = flop / (ms * 1e-3) / 1e12
    return {"shape": [n, out, inp], "ms": round(ms, 4), "fp32_equivalent_TFLOP_per_s": round(tflops, 2),
            "fp16_mma_TFLOP_per_s": round(3 * tflops, 2), "share_of_989_over_3": round(tflops / (FP16_DENSE_TFLOPS / 3), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_conditioner.py measures on a GPU; none is available")
    dev = torch.device("cuda:0")
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
           "allow_tf32": bool(torch.backends.cuda.matmul.allow_tf32),
           "cfg2x5_b65536": measure(cfg2x5, 1 << 16, 64, args.windows, args.iters, dev),
           "nsf784_b4096": measure(nsf784, 1 << 12, 784, args.windows, args.iters, dev),
           "wgrad": [wgrad_rate(1 << 16, 128, 128, 50, dev), wgrad_rate(1 << 16, 736, 128, 50, dev),
                     wgrad_rate(1 << 20, 256, 256, 10, dev)]}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "train_conditioner.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
