"""Shared pieces of the spline-kernel tests (test_kernel_source_on_host.py on the CPU, test_spline_kernels_gpu.py on a GPU): the
bin counts that reach every instance of the HBM spline kernels, random parameters, and the fp64 truth / fp32 yardstick.

Truth is the fp64 oracle.  The yardstick is the same oracle in fp32 with O.F32_CUMSUM = True: the knots as the reference
computes them on CUDA (sequential float prefix sum), which is what these kernels replace on a GPU.  The CPU reference (double
accumulation in ATen's cumsum) has knots that are up to ~3x more accurate at large K; no fp32 scan of the bin sizes matches
that, so it is not the bar for a kernel."""
import torch

from nflows_b200._native import spline_desc
from oracle import flow_oracle as O

# every dispatch branch of nfk_rqs_elementwise (8 exact, < 8, 16 exact, < 16, <= 32, <= 64), its edges, and K = 1
BINS = (1, 2, 3, 5, 7, 8, 9, 12, 15, 16, 17, 24, 31, 32, 33, 48, 63, 64)
TAIL_BOUND = 3.0
DIVISOR = 4.0                       # wh_divisor: widths and heights are divided by it before the softmax (exact in fp32)
DEFAULT_MINS = (1e-3, 1e-3, 1e-3)

# parameter variants held to the same bar at a few bin counts: softplus beta != 1, and non-default minimum sizes
VARIANTS = {5: "identity_init", 17: "identity_init", 48: "identity_init", 7: "mins", 24: "mins", 63: "mins"}
VARIANT_MINS = (1e-2, 5e-3, 5e-2)


def variant_kw(variant):
    """(enable_identity_init, (min_bin_width, min_bin_height, min_derivative)) of a variant name (None: the defaults)."""
    return variant == "identity_init", VARIANT_MINS if variant == "mins" else DEFAULT_MINS


def num_derivatives(bins, tails):
    return bins - 1 if tails == "linear" else bins + 1


def desc(bins, tails, identity_init=False, mins=DEFAULT_MINS):
    return spline_desc(bins, tails, TAIL_BOUND, 0.0, 1.0, 0.0, 1.0, *mins, identity_init, DIVISOR)


def params(n, bins, tails, generator, scale=2.0):
    """Moderate random parameters: unnormalised widths, heights (before the divisor) and derivatives, fp32 [n, ...] on the
    generator's device.  The last sixteenth of the rows has its width and height logits shifted by -1000: the softmax is
    invariant to that only when it subtracts the maximum over the K real bins (exp(-250) underflows fp32)."""
    dev = generator.device
    uw = torch.randn(n, bins, generator=generator, device=dev) * scale
    uh = torch.randn(n, bins, generator=generator, device=dev) * scale
    ud = torch.randn(n, num_derivatives(bins, tails), generator=generator, device=dev) * scale
    uw[n - n // 16:] -= 1000.0
    uh[n - n // 16:] -= 1000.0
    return uw, uh, ud


def inputs(n, tails, generator):
    """Inside the interval, plus (linear tails) a share outside it: N(0, 2^2) against the tail bound 3."""
    dev = generator.device
    if tails == "linear":
        return torch.randn(n, generator=generator, device=dev) * 2.0
    return torch.rand(n, generator=generator, device=dev)


def oracle(x, uw, uh, ud, tails, inverse, dtype, identity_init=False, mins=DEFAULT_MINS):
    """(y, log|det|) of the oracle evaluated in `dtype` on the CPU; uw, uh are divided by DIVISOR as the reference does."""
    x, uw, uh, ud = (t.detach().cpu().to(dtype) for t in (x, uw, uh, ud))
    kw = dict(inverse=inverse, min_bin_width=mins[0], min_bin_height=mins[1], min_derivative=mins[2],
              enable_identity_init=identity_init)
    if tails == "linear":
        return O.rq_spline_unconstrained(x, uw / DIVISOR, uh / DIVISOR, ud.clone(), tail_bound=TAIL_BOUND, **kw)
    return O.rq_spline(x, uw / DIVISOR, uh / DIVISOR, ud.clone(), **kw)


def truth_and_yardstick(x, uw, uh, ud, tails, inverse, identity_init=False, mins=DEFAULT_MINS):
    """((y, lad) in fp64, (y, lad) in fp32 with the CUDA reference's float prefix sum).  The caller has set O.F32_CUMSUM."""
    assert O.F32_CUMSUM, "the yardstick is the reference as it runs on CUDA: set O.F32_CUMSUM (monkeypatch)"
    args = (x, uw, uh, ud, tails, inverse)
    return oracle(*args, torch.float64, identity_init, mins), oracle(*args, torch.float32, identity_init, mins)
