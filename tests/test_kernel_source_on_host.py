"""The per-element spline source of the CUDA kernels (nflows_b200/csrc/rq_spline.cuh) compiled for the HOST
(oracle/rqs_host.cpp) and checked against the reference's golden vectors and the fp64 oracle -- kernel numerics
without a GPU.  (The GPU run of the same source is checked in test_native_parity.py.)"""
import ctypes
import os
import subprocess

import pytest
import torch

from conftest import ROOT, load_golden
from nflows_b200._native import spline_desc
from oracle import flow_oracle as O


@pytest.fixture(scope="module")
def host_lib():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle")], check=True, capture_output=True)
    return ctypes.CDLL(os.path.join(ROOT, "oracle", "_build", "librqs_host.so"))


def run(lib, desc, inverse, x, uw, uh, ud, lean=False):
    x, uw, uh, ud = (t.contiguous().float() for t in (x, uw, uh, ud))
    y, lad, flag = torch.empty_like(x), torch.empty_like(x), ctypes.c_int(0)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    fn = lib.rqs_host_eval_lean if lean else lib.rqs_host_eval
    rc = fn(ctypes.byref(desc), int(inverse), p(x), p(uw), p(uh), p(ud), ctypes.c_longlong(x.numel()), p(y), p(lad),
            ctypes.byref(flag))
    assert rc == 0
    return y, lad, flag.value


def errs(a, b):
    a, b = a.double(), b.double()
    nan = torch.isnan(a) & torch.isnan(b)
    e = (a - b).abs() / torch.maximum(torch.maximum(a.abs(), b.abs()), torch.ones_like(a))
    return torch.where(nan, torch.zeros_like(e), e).flatten().sort().values


@pytest.mark.parametrize("lean", [False, True])
def test_kernel_source_matches_reference_distribution(host_lib, lean):
    """lean=True: the binary-search multi-feature form the tensor-core epilogues and the row kernel evaluate (rqs_eval_lean)."""
    g = load_golden("spline")
    cases = [("tails", g["x_tails"], g["ud_tails"], spline_desc(8, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3)),
             ("constrained", g["x_constrained"], g["ud_constrained"], spline_desc(8, None, 1.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3))]
    for name, x, ud, desc in cases:
        for inv in (False, True):
            y, lad, _ = run(host_lib, desc, inv, x, g["uw"], g["uh"], ud, lean=lean)
            if name == "tails":
                ty, tl = O.rq_spline_unconstrained(x.double(), g["uw"].double(), g["uh"].double(), ud.double(), inverse=inv,
                                                   tail_bound=3.0)
            else:
                ty, tl = O.rq_spline(x.double(), g["uw"].double(), g["uh"].double(), ud.double(), inverse=inv)
            wy, wl = g["%s_inv%d" % (name, inv)]
            for got, ref, truth in ((y, wy, ty), (lad, wl, tl)):
                e, r = errs(got, truth), errs(ref, truth)
                n = len(e)
                for q in (0.5, 0.99, 0.999):
                    i = min(n - 1, int(q * n))
                    assert e[i] <= 2 * r[i] + 1e-5, (name, inv, q, float(e[i]), float(r[i]))
                assert e[-1] <= 15 * r[-1] + 1e-5          # the same allowance as the GPU parity tests


def test_kernel_source_identity_and_domain_flag(host_lib):
    k = 10
    x = torch.rand(500)
    z, zd = torch.zeros(500, k), torch.zeros(500, k + 1)
    desc = spline_desc(k, None, 1.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3, enable_identity_init=True)
    y, lad, flag = run(host_lib, desc, False, x, z, z, zd)
    assert float((y - x).abs().max()) <= 1e-6 and float(lad.abs().max()) <= 1e-6 and flag == 0
    _, _, flag = run(host_lib, desc, False, x + 1.0, z, z, zd)
    assert flag & 1


@pytest.mark.parametrize("bins", [4, 8, 10, 16])
def test_lean_form_agrees_with_the_scan_form(host_lib, bins):
    """rqs_eval_lean (knots first, binary search, template direction) against rqs_eval (bin found by a scan) on random, moderately
    sharp parameters: same bins, same values up to the rounding of the re-associated softmax argument -- every bin count the
    fused kernels are instantiated for (10 exercises the padded search), both tail modes, both directions, bin edges included."""
    torch.manual_seed(bins)
    n = 4001
    uw, uh = torch.randn(n, bins) * 2.0, torch.randn(n, bins) * 2.0
    for tails in ("linear", None):
        ud = torch.randn(n, bins - 1 if tails else bins + 1) * 1.5
        desc = spline_desc(bins, tails, 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3, False, 4.0)
        x = torch.randn(n) * 2.0 if tails else torch.rand(n)
        if tails:
            x[:8] = torch.tensor([-3.0, 3.0, -3.0000002, 3.0000002, 0.0, float("nan"), 1e30, -1e30])
        else:
            x[:3] = torch.tensor([0.0, 1.0, 0.5])
        for inv in (False, True):
            y0, l0, f0 = run(host_lib, desc, inv, x, uw, uh, ud)
            y1, l1, f1 = run(host_lib, desc, inv, x, uw, uh, ud, lean=True)
            assert f0 == f1
            ey, el = errs(y1, y0), errs(l1, l0)
            i99 = int(0.99 * len(ey))
            assert ey[i99] <= 2e-6 and el[i99] <= 2e-5, (bins, tails, inv, float(ey[i99]), float(el[i99]))
            # a knot within one rounding of x may put the two forms in neighbouring bins: same spline, same value to ~1e-5
            assert ey[-1] <= 5e-5, (bins, tails, inv, float(ey[-1]))


def test_lean_form_inverse_is_the_inverse_of_its_forward(host_lib):
    """Round trip of the kernel's own spline source: inverse(forward(x)) = x and the two log-determinants cancel, for every
    bin count the fused kernels are instantiated for, moderately sharp parameters, both tail modes."""
    for bins in (4, 8, 10, 16):
        torch.manual_seed(100 + bins)
        n = 3000
        uw, uh = torch.randn(n, bins) * 1.5, torch.randn(n, bins) * 1.5
        for tails in ("linear", None):
            ud = torch.randn(n, bins - 1 if tails else bins + 1)
            desc = spline_desc(bins, tails, 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3, False, 2.0)
            x = torch.randn(n) * 2.5 if tails else torch.rand(n)
            y, lad, f = run(host_lib, desc, False, x, uw, uh, ud, lean=True)
            back, lad_back, f2 = run(host_lib, desc, True, y, uw, uh, ud, lean=True)
            assert f == 0 and f2 == 0
            e = errs(back, x)
            assert e[int(0.999 * n)] <= 2e-5 and e[-1] <= 2e-3, (bins, tails, float(e[int(0.999 * n)]), float(e[-1]))
            el = errs(lad_back, -lad)
            assert el[int(0.99 * n)] <= 2e-4, (bins, tails, float(el[int(0.99 * n)]))
