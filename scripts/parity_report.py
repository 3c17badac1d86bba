"""Parity calibration report (run on the GPU box): for every golden case prints
   err(native vs fp64 truth), err(reference fp32 vs fp64 truth), err(native vs reference fp32)
with rel_err = max |a-b| / max(|a|,|b|,1).  The fp64 truth is the CPU oracle evaluated in float64 on the same
weights/inputs.  Prints the error distribution behind the tolerances used in tests/."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from conftest import load_golden, rel_err  # noqa: E402
from nflows_b200.flows import recipes  # noqa: E402
from nflows_b200.transforms.splines import rational_quadratic as rq  # noqa: E402
from oracle import flow_oracle as O  # noqa: E402

dev = torch.device("cuda:0")


def line(name, got, ref32, truth):
    print("{:44s} native-vs-fp64 {:.2e}   ref32-vs-fp64 {:.2e}   native-vs-ref32 {:.2e}".format(
        name, rel_err(got.cpu(), truth), rel_err(ref32, truth), rel_err(got.cpu(), ref32)))


def tail(name, got, ref32, truth):
    """Error percentiles of the deliberately sharp-bin stress vectors: what tests/test_native_parity.py's
    assert_statistically_as_accurate bounds (p99 / p99.9 within 2x, worst element within a small multiple of the reference's)."""
    def errs(a):
        a, b = a.double().cpu().flatten(), truth.double().flatten()
        fin = torch.isfinite(a) & torch.isfinite(b)
        e = (a[fin] - b[fin]).abs() / torch.maximum(torch.maximum(a[fin].abs(), b[fin].abs()), torch.ones_like(b[fin]))
        return e.sort().values
    e, r = errs(got), errs(ref32)
    n = len(e)
    q = lambda v, f: float(v[min(n - 1, int(f * n))])
    print("{:44s} native p99 {:.2e} p99.9 {:.2e} max {:.2e} | reference p99 {:.2e} p99.9 {:.2e} max {:.2e} | max ratio {:.2f}".format(
        name, q(e, 0.99), q(e, 0.999), float(e[-1]), q(r, 0.99), q(r, 0.999), float(r[-1]), float(e[-1]) / max(float(r[-1]), 1e-30)))


def dbl(sd):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}


@torch.no_grad()
def main():
    print("GEMM backend:", os.environ.get("NFLOWS_B200_GEMM", "tc"))
    g = load_golden("spline")
    for inv in (False, True):
        y, l = rq.unconstrained_rational_quadratic_spline(g["x_tails"].to(dev), g["uw"].to(dev), g["uh"].to(dev),
                                                          g["ud_tails"].to(dev), inverse=inv, tail_bound=g["tail_bound"])
        ty, tl = O.rq_spline_unconstrained(g["x_tails"].double(), g["uw"].double(), g["uh"].double(), g["ud_tails"].double(),
                                           inverse=inv, tail_bound=g["tail_bound"])
        wy, wl = g["tails_inv%d" % inv]
        line("spline tails inv=%d  y" % inv, y, wy, ty)
        line("spline tails inv=%d  lad" % inv, l, wl, tl)
        tail("  stress tails inv=%d y" % inv, y, wy, ty)
        tail("  stress tails inv=%d lad" % inv, l, wl, tl)
        box = dict(left=-1.0, right=3.0, bottom=-1.0, top=3.0, min_bin_width=1e-2, min_bin_height=2e-2, min_derivative=5e-2)
        for key, xin, kw in (("constrained_inv%d", g["x_constrained"], {}), ("constrained_box_inv%d", g["x_constrained"] * 4 - 1, box)):
            yc, lc = rq.rational_quadratic_spline(xin.to(dev), g["uw"].to(dev), g["uh"].to(dev), g["ud_constrained"].to(dev), inverse=inv, **kw)
            wyc, wlc = g[key % inv]
            tyc, tlc = O.rq_spline(xin.double(), g["uw"].double(), g["uh"].double(), g["ud_constrained"].double(), inverse=inv, **kw)
            tail("  stress %s y" % (key % inv), yc, wyc, tyc)
            tail("  stress %s lad" % (key % inv), lc, wlc, tlc)
    g = load_golden("cfg2_rq_coupling")
    t = recipes.rq_coupling_layer()
    t.load_state_dict(g["sd"])
    t = t.eval().to(dev)
    kw = dict(num_bins=8, tails="linear", tail_bound=3.0)
    sd64 = dbl(g["sd"])
    for suffix in ("", "_x3"):
        if suffix:
            for name, p in t.named_parameters():
                if "final_layer" in name:
                    p.mul_(3.0)
            sd64 = {k: (v * 3.0 if "final_layer" in k else v) for k, v in sd64.items()}
        y, l = t(g["x"].to(dev))
        ty, tl = O.rq_coupling({k: v.clone() for k, v in sd64.items()}, "", g["x"].double(), **kw)
        line("cfg2 coupling%s fwd y" % suffix, y, g["y" + suffix], ty)
        line("cfg2 coupling%s fwd lad" % suffix, l, g["lad" + suffix], tl)
        y, l = t.inverse(g["x"].to(dev))
        ty, tl = O.rq_coupling({k: v.clone() for k, v in sd64.items()}, "", g["x"].double(), inverse=True, **kw)
        line("cfg2 coupling%s inv x" % suffix, y, g["xinv" + suffix], ty)
        line("cfg2 coupling%s inv lad" % suffix, l, g["ladinv" + suffix], tl)
    g = load_golden("nsf_small")
    flow = recipes.rq_nsf(g["features"], g["hidden"], g["layers"])
    flow.load_state_dict(g["sd"])
    flow = flow.eval().to(dev)
    spec = O.nsf_spec(g["layers"])
    z, lad = flow._transform(g["x"].to(dev))
    tz, tlad = O.composite(dbl(g["sd"]), spec, g["x"].double())
    line("nsf_small z", z, g["z"], tz)
    line("nsf_small lad", lad, g["lad"], tlad)
    line("nsf_small log_prob", flow.log_prob(g["x"].to(dev)), g["log_prob"], O.flow_log_prob(dbl(g["sd"]), spec, g["x"].double()))
    for name in ("nsf784_layer", "nsf784_full"):
        g = load_golden(name)
        torch.manual_seed(g["seed"])
        flow = recipes.perturb_(recipes.rq_nsf(g["features"], g["hidden"], g["layers"]).eval(), g["perturb_seed"]).to(dev)
        x = g["x"].to(dev)
        if name == "nsf784_layer":
            z, lad = flow._transform(x)
            line(name + " z", z, g["z"], g["z_fp64"])
            line(name + " lad", lad, g["lad"], g["lad_fp64"])
        else:
            line(name + " log_prob", flow.log_prob(x), g["log_prob"], g["log_prob_fp64"])


if __name__ == "__main__":
    main()
