"""On an H100: the spline inside the fused coupling kernels, the row kernel and the row kernel's backward at the settings and
edge inputs of _spline_edge_cases.py -- exact parameters through the real kernels.

A crafted feature has its final-layer rows zeroed and the crafted vector in its bias, so the tensor-core epilogue evaluates the
spline on exactly that vector (fmaf(0, inv_acc_scale, b) == b) while the trunk and, with linear tails, eight random features keep
the GEMM real.  With linear tails every row has ONE active crafted element; the other crafted features sit at 2B, in the identity
region (y = x, log|det| exactly 0), so the row's log|det| is that element's.  Without tails there is no identity region: the
launch carries the eight crafted features only, y is checked per element and the log|det| per row.

  A. nfk_rq_coupling_final_f16x3 and nfk_rq_coupling_step_f16x3, launched directly: flags, exact edges, per element against fp64,
     the fp16 pair output against the fp32 output, and the two kernels against each other;
  B. nfk_rqs_rows on the same parameters (the lean form at K = 8 / 16, the scan form at K = 4 / 10);
  C. nfk_rqs_rows_backward on the table, against fp64 autograd;
  D. a coupling with non-default minimum sizes on each route of its spline head, against the fp64 oracle."""
import pytest
import torch

import _coupling_checks as C
import _spline_edge_cases as E
from conftest import rel_err
from nflows_b200 import config
from nflows_b200 import dense as D
from nflows_b200 import kernels as K
from oracle import flow_oracle as O
from test_spline_edges_host import KNOWN_MISSES, KNOWN_VJP_MISSES, check_vjp, cotangents

pytestmark = pytest.mark.gpu

D_ID = 8


def bits(t):
    return t.contiguous().view(torch.int32)


class Launches:
    """The crafted coupling of one (K, tails, setting) on the device and its two fused kernels, launched directly."""

    def __init__(self, bins, tails, s, dev):
        self.bins, self.tails, self.s, self.dev = bins, tails, s, dev
        vectors = [E.vector(name, bins, tails, s) for name in E.VECTORS]
        self.n_random = 8 if tails == "linear" else 0
        self.t = E.crafted_coupling(bins, tails, s, vectors, d_id=D_ID, n_random=self.n_random, seed=bins).to(dev)
        self.d_t = len(vectors) + self.n_random
        self.desc = E.desc(bins, tails, s)
        self.chain = self.t.transform_net.dense_chain(None)
        self.wp, self.bias, _ = D.spline_operands(self.chain[-1][0], self.chain[-1][1], bins, tails, self.d_t)

    def run(self, route, x, inverse, pair=False):
        """(y fp32 or Pair16, lad, flag word) of one launch on x [n, D_ID + d_t]."""
        n = x.shape[0]
        a = K.split_f16(x[:, :D_ID], D.act_exp())
        lad = torch.zeros(n, device=self.dev)
        flags = torch.zeros(1, dtype=torch.int32, device=self.dev)
        y = None if pair else torch.full_like(x, -7.0)
        y_pair = K.Pair16.zeros(n, x.shape[1], D.act_exp(), self.dev) if pair else None
        cols = (D_ID, self.d_t)
        if route == "step":
            K.rq_coupling_step(D.step_plan(self.chain), a, self.desc, inverse, self.wp, self.bias, x, cols, y, lad, flags,
                               y_pair=y_pair)
        else:
            trunk = D.run_trunk(self.chain, x, None, True, x_pair=a).pair
            K.rq_coupling_final(self.desc, inverse, trunk, self.wp, self.bias, x, cols, y, lad, flags, y_pair=y_pair)
        torch.cuda.synchronize()
        return (y_pair if pair else y), lad, int(flags.item())


def layout(tab, tails, s, seed):
    """x [n, D_ID + d_t] on the CPU and, per crafted element, its (row, column).  Linear tails: one active crafted element per
    row, then 256 rows with the random features active (N(0, 1.3^2), the input of the coupling tests); no tails: row r carries element r of every vector."""
    B = s.tail_bound
    nv = len(E.VECTORS)
    g = torch.Generator().manual_seed(seed)
    if tails == "linear":
        n_el = len(tab.x)
        n = n_el + 256
        x = torch.full((n, D_ID + 2 * nv), 2 * B)
        rows = torch.arange(n_el)
        cols = D_ID + tab.vec
        x[rows, cols] = tab.x
        x[n_el:, D_ID + nv:] = torch.randn(256, nv, generator=g) * 1.3       # as _coupling_checks.inputs
    else:
        n = E.PER_VECTOR
        x = torch.empty(n, D_ID + nv)
        rows = torch.arange(len(tab.x)) % n
        cols = D_ID + tab.vec
        x[rows, cols] = tab.x
    x[:, :D_ID] = torch.randn(n, D_ID, generator=g)
    return x, rows, cols


CASES = [(bins, tails) for bins in E.BINS for tails in ("linear", None)]


# ---- A / B. the fused kernels and the row kernel ---------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("bins,tails", CASES, ids=["{}-{}".format(b, t or "none") for b, t in CASES])
def test_fused_kernels_on_the_edge_table(cuda_device, bins, tails, monkeypatch):
    monkeypatch.setattr(O, "F32_CUMSUM", True)
    for s in E.settings(bins, tails):
        L = Launches(bins, tails, s, cuda_device)
        for inverse in (False, True):
            what = (bins, tails, s.name, inverse)
            tab = E.table(bins, tails, inverse, s)
            (ty, tl), (ry, rl) = E.truth_and_yardstick(tab, tails, inverse, s)
            x, rows, cols = layout(tab, tails, s, bins + inverse)
            xd = x.to(cuda_device)
            out = {}
            for route in ("step", "final"):
                y, lad, flag = L.run(route, xd, inverse)
                assert flag == 0, what + (route, flag)
                assert torch.equal(bits(y[:, :D_ID]), bits(torch.full_like(y[:, :D_ID], -7.0))), what + (route, "identity columns")
                ye = y.cpu()[rows, cols]
                assert_edges(tab, ye, ry, tails, s, inverse, what + (route,))
                if what + ("lean", "y") in KNOWN_MISSES:        # the host build's known miss: conditioning (see there)
                    E.assert_inverse_backward_error(ye, ry, ty, tl, tab, what + (route, "y"))
                else:
                    E.assert_as_accurate(ye, ry, ty, tab, what + (route, "y"))
                if tails == "linear":
                    le = lad.cpu()[rows]
                    outside = E.kind_mask(tab, "ulp_out", "out", "huge", "nan")
                    assert torch.equal(bits(le[outside]), bits(torch.zeros(int(outside.sum())))), what + (route, "lad 0")
                    E.assert_as_accurate(le, rl, tl, tab, what + (route, "lad"))
                    # the rows of the random features: identity elsewhere, bit for bit
                    assert torch.equal(bits(y[len(tab.x):, D_ID:D_ID + len(E.VECTORS)]),
                                       bits(xd[len(tab.x):, D_ID:D_ID + len(E.VECTORS)])), what + (route,)
                else:
                    want64 = torch.zeros(x.shape[0], dtype=torch.float64).index_add_(0, rows, tl)
                    want32 = torch.zeros(x.shape[0], dtype=torch.float64).index_add_(0, rows, rl.double())
                    got = lad.cpu().double()
                    ok = torch.isfinite(want32)
                    assert rel_err(got[ok], want64[ok]) <= max(3e-5, 5 * rel_err(want32[ok], want64[ok])), what + (route, "lad")
                out[route] = (y, lad)
            # the two kernels evaluate the same rqs_eval_lean instance on the same parameters
            (y1, l1), (y2, l2) = out["step"], out["final"]
            cc = slice(D_ID, D_ID + len(E.VECTORS))
            assert torch.equal(bits(y1[:, cc]), bits(y2[:, cc])), what + ("step vs final", float((y1[:, cc] - y2[:, cc]).abs().max()))
            if tails == "linear":
                assert torch.equal(bits(l1[:len(tab.x)]), bits(l2[:len(tab.x)])), what + ("step vs final lad",)
            else:
                # eight elements per row: the two kernels add the row's shares in different orders
                assert rel_err(l1, l2) <= 2e-6, what + ("step vs final lad", rel_err(l1, l2))
            check_pair(L, xd, tails, s, inverse, what)
            check_rows(L, tab, xd, y2, l2, rows, cols, tails, inverse, what, ry, ty, rl, tl)
            if tails is None:
                bad = xd.clone()
                bad[3, D_ID + 2], bad[7, D_ID + 5] = -1e-6, 1.0 + 1e-6
                for route in ("step", "final"):
                    assert L.run(route, bad, inverse)[2] == 1, what + (route, "domain flag")


def assert_edges(tab, ye, ry, tails, s, inverse, what):
    lo, hi = E.interval(tails, s)
    assert bool((ye[E.kind_mask(tab, "left")] == lo).all()), what + ("left",)
    right = E.kind_mask(tab, "right")
    bar = 1e-6 * max(1.0, abs(hi)) + (15 * (ry[right].double() - hi).abs() if inverse else 0.0)
    assert bool(((ye[right].double() - hi).abs() <= bar).all()), what + ("right", ye[right])
    if tails == "linear":
        out = E.kind_mask(tab, "ulp_out", "out", "huge", "nan")
        assert torch.equal(bits(ye[out]), bits(tab.x[out])), what + ("identity",)


def check_pair(L, xd, tails, s, inverse, what):
    """The fp16 pair output: bit for bit the split of the fp32 output at the same exponent, the same log|det|; no flag on valid
    inputs; ±1e30 and NaN in the identity region raise exactly the fp16-range flag (4)."""
    finite = torch.isfinite(xd) & (xd.abs() < 1e20)
    xv = torch.where(finite, xd, torch.full_like(xd, 2 * s.tail_bound if tails == "linear" else 0.5))
    for route in ("step", "final"):
        y_ref, l_ref, flag = L.run(route, xv, inverse)
        assert flag == 0
        pair, lad, flag = L.run(route, xv, inverse, pair=True)
        assert flag == 0, what + (route, "pair", flag)
        want = K.split_f16(y_ref[:, D_ID:].contiguous(), D.act_exp())
        assert torch.equal(pair.hi[:, D_ID:], want.hi) and torch.equal(pair.lo[:, D_ID:], want.lo), what + (route, "pair")
        assert torch.equal(bits(lad), bits(l_ref)), what + (route, "pair lad")
        if tails == "linear" and not bool(finite.all()):
            assert L.run(route, xd, inverse, pair=True)[2] == 4, what + (route, "range flag")


def check_rows(L, tab, xd, y, lad, rows, cols, tails, inverse, what, ry, ty, rl, tl):
    """nfk_rqs_rows on the crafted columns with the same parameters: the lean form (K = 8 / 16) bit for bit, the scan form
    (K = 4 / 10) within the lean-vs-scan bars of test_kernel_source_on_host.py."""
    nv, m = len(E.VECTORS), E.num_params(L.bins, L.tails)
    vec = torch.cat([torch.cat(E.vector(name, L.bins, L.tails, L.s)) for name in E.VECTORS]).to(xd.device)
    n = xd.shape[0]
    xc = xd[:, D_ID:D_ID + nv].contiguous()
    params = vec[None].expand(n, nv * m).contiguous()
    lr = torch.zeros(n, device=xd.device)
    flags = torch.zeros(1, dtype=torch.int32, device=xd.device)
    yr = K.rqs_rows(L.desc, inverse, xc, params, None, None, lr, flags)
    torch.cuda.synchronize()
    assert int(flags.item()) == 0, what + ("rows flag",)
    yf = y[:, D_ID:D_ID + nv]
    n_el = len(tab.x) if tails == "linear" else n
    if L.bins in (8, 16):
        assert torch.equal(bits(yr), bits(yf)), what + ("rows y", float((yr - yf).abs().max()))
        if tails == "linear":
            assert torch.equal(bits(lr[:n_el]), bits(lad[:n_el])), what + ("rows lad",)
        else:       # eight elements per row: the row kernel adds them in another order
            assert rel_err(lr, lad) <= 2e-6, what + ("rows lad", rel_err(lr, lad))
    else:
        # the scan form finds the bin by another arithmetic: held to fp64 per element with the fused kernels' bar
        E.assert_as_accurate(yr.cpu()[rows, cols - D_ID], ry, ty, tab, what + ("rows y",))
        if tails == "linear":
            E.assert_as_accurate(lr.cpu()[rows], rl, tl, tab, what + ("rows lad",))


# ---- C. the backward -------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("bins,tails", CASES, ids=["{}-{}".format(b, t or "none") for b, t in CASES])
def test_row_backward_on_the_edge_table(cuda_device, bins, tails, monkeypatch):
    monkeypatch.setattr(O, "F32_CUMSUM", True)
    missed = []
    for s in E.settings(bins, tails):
        d = E.desc(bins, tails, s)
        for inverse in (False, True):
            tab = E.table(bins, tails, inverse, s)
            gy, gl = cotangents(len(tab.x), bins + 2 * inverse)
            gx, gp = K.rqs_rows_backward(d, inverse, tab.x[:, None].to(cuda_device), E.params_of(tab).to(cuda_device),
                                         gy[:, None].to(cuda_device), gl.to(cuda_device))
            with torch.enable_grad():
                ok = check_vjp(tab, gx[:, 0].cpu(), gp.cpu(), gy, gl, tails, inverse, s, (bins, tails, s.name, inverse))
            if not ok:
                missed.append((bins, tails, s.name, inverse))
    assert set(missed) <= {k for k in KNOWN_VJP_MISSES if k[:2] == (bins, tails)}, missed


# ---- D. module level, one case per route -------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("case", E.MODULE_CASES, ids=lambda c: c.name)
def test_coupling_with_minimum_sizes_on_each_route(cuda_device, case, monkeypatch):
    monkeypatch.setattr(config, "fuse_coupling", case.route != "rows")
    t, s = E.module_coupling(case, seed=3)
    sd = {k: v.detach().clone() for k, v in t.state_dict().items()}
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    kw = dict(num_bins=case.bins, tails=case.tails, tail_bound=case.tail_bound, min_bin_width=s.mins[0],
              min_bin_height=s.mins[1], min_derivative=s.mins[2])
    t = t.to(cuda_device)
    for inverse in (False, True):
        tab = E.table(case.bins, case.tails, inverse, s)
        x, rows, cols = layout(tab, case.tails, s, 5 + inverse)
        x = torch.where(torch.isfinite(x) & (x.abs() < 1e20), x, torch.full_like(x, 2 * case.tail_bound))
        with C.timeline() as tags:
            y, lad = (t.inverse if inverse else t)(x.to(cuda_device))
        torch.cuda.synchronize()
        want, truth = O.rq_coupling(sd, "", x, inverse=inverse, **kw), O.rq_coupling(sd64, "", x.double(), inverse=inverse, **kw)
        y, lad = y.cpu(), lad.cpu()
        # the crafted elements, one per row: per element, with the bar of the direct launches
        what = (case.name, inverse)
        E.assert_as_accurate(y[rows, cols], want[0][rows, cols], truth[0][rows, cols], tab, what + ("y",))
        E.assert_as_accurate(lad[rows], want[1][rows], truth[1][rows], tab, what + ("lad",))
        # the rows of the random features (parameters from the conditioner): the fp64 sandwich of the coupling tests
        r = slice(len(tab.x), None)
        tol_y, tol_l = C.sandwich((want[0][r], want[1][r]), (truth[0][r], truth[1][r]))
        assert rel_err(y[r], truth[0][r]) <= tol_y and rel_err(lad[r], truth[1][r]) <= tol_l, what
        if case.route == "rows":
            assert "spline_epilogue" in tags and not any(g.startswith("rq_coupling") for g in tags), tags
        else:
            assert any(g.startswith("rq_coupling_" + case.route) for g in tags), tags
