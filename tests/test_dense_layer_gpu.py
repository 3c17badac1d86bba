"""The dense-layer kernels against fp64 on the H100: the split-fp16 tensor-core layer (nfk_linear_f16x3) over the case table of
_dense_cases.py, the FFMA layer (nfk_linear), the operand passes that feed them (split_f16, weight_exp / nfk_absmax, glu_skip,
im2col3x3), one 3x3 convolution end to end, and the argument checks of the wrappers.

Accuracy criterion, per output element (scale-invariant: an output far below 1 is held to its own scale):

    err = |y - y64| / (|b| + sum_k |a_k| |w_k| + |r|)

y64 is the same operation in fp64 on the fp32 operands.  BAR is calibrated on one H100 80GB HBM3 (700 W power limit) over the
case table: the kernel's worst err was 8.6e-7, torch's fp32 GEMM (F.linear, allow_tf32=False) measured the same way 5.2e-6, both
on n200_o9016_k4608_same_sign (elsewhere both stay below 3e-7).  BAR is the kernel's worst with a 2x margin.  The FFMA layer's
worst on its shapes was 3.5e-7 (torch: 2.6e-7); it is held to the same BAR.  The same-sign cases (non-negative activations times non-negative
weights at K = 2304 and 4608) are where the tensor core's round-toward-zero accumulation adds up instead of cancelling: there a
partial sum drained every 64 slabs instead of every 2 (tc_common.cuh: DRAIN_SLABS_LINEAR) lands far above the bar."""
import math

import pytest
import torch
import torch.nn.functional as F

import _dense_cases as D
from conftest import rel_err
from nflows_b200 import _native
from nflows_b200 import kernels as K

pytestmark = pytest.mark.gpu

MEASURED_KERNEL = 8.6e-7       # worst err of the case table on the H100 (module docstring)
BAR = 2 * MEASURED_KERNEL
ACT_TOL = 2.0 ** -20            # the fp32 activations' own error, relative to |pre| + |act(pre)| (test_activations_gpu.py)
ACT_LIPSCHITZ = 1.2             # max |act'| of the codes (GELU: 1.13)
ACT64 = {0: lambda t: t, 1: F.relu, 2: torch.tanh, 3: F.elu, 4: lambda t: F.leaky_relu(t, 0.01), 5: F.gelu, 6: F.silu}
SPLIT_EXP = 6

F32_SENTINEL = 0x7FA5A5A5       # NaN bit patterns no kernel writes
F16_SENTINEL = 0x7E5A


def sentinel(rows, cols, dtype, device):
    if dtype == torch.float32:
        return torch.full((rows, cols), F32_SENTINEL, dtype=torch.int32, device=device).view(torch.float32)
    return torch.full((rows, cols), F16_SENTINEL, dtype=torch.int16, device=device).view(torch.float16)


def untouched(t):
    bits = t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)
    return bool((bits == (F32_SENTINEL if t.dtype == torch.float32 else F16_SENTINEL)).all())


def bits(t):
    return t.contiguous().view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def split_torch(v, exp, code=0):
    """The fp16 pair of pre(v) * 2^exp as the kernels split it: hi = rn(s), lo = rn(s - hi); s - hi is exact in fp32."""
    v = F.relu(v) if code == 1 else v
    s = v * 2.0 ** exp
    hi = s.half()
    return hi, (s - hi.float()).half()


def torch_fp32_linear(x, w, b):
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return F.linear(x, w, b)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


# ---- the split-fp16 tensor-core layer over the case table ----------------------------------------------------------------
class Built:
    """Operands and destinations of one case: fp32 x, w, b, r; the pairs the kernel multiplies (views as the case asks)."""

    def __init__(self, c, device, seed=0):
        g = torch.Generator(device=device).manual_seed(seed)
        rnd = lambda *s: torch.randn(*s, generator=g, device=device)
        n, k, o = c.n, c.k, c.o
        if c.a_layout == "col_view":
            xb = rnd(n, k + 16)
            self.x, cols = xb[:, 8:8 + k], (8, 8 + k)
        elif c.a_layout == "row_slice":
            xb = rnd(n + 70, k)
            self.x, cols = xb[37:37 + n], None
        else:
            xb = rnd(n, k)
            self.x, cols = xb, None
        wb = rnd(o, k + 8) if c.w_layout == "col_view" else rnd(o, k)
        if c.data == "nonneg":
            xb.abs_(), wb.abs_()
        a_scale = 2.0 ** 28 if c.a_exp < 0 else 1.0
        xb.mul_(a_scale)
        wb.div_(math.sqrt(k))
        if c.w_max is not None:
            wb.mul_(2.0 ** c.w_max / float(wb[:, :k].abs().max()))
        self.w = wb[:, :k]
        w_scale = 2.0 ** c.w_max if c.w_max is not None else 1.0
        self.b = rnd(o) * a_scale * w_scale if c.bias else None
        self.r = rnd(n, o) * a_scale * w_scale if c.residual else None
        pair = K.split_f16(xb, c.a_exp)
        self.a = pair.cols(*cols) if cols else (pair.rows(37, 37 + n) if c.a_layout == "row_slice" else pair)
        self.wp = K.split_f16(wb, K.weight_exp(self.w)).cols(0, k)
        assert 2.0 ** 13 <= float(self.wp.hi.abs().max()) <= 2.0 ** 14 or c.w_max is not None
        self.c, self.device = c, device

    def destinations(self):
        """(y view, y buffer, pair view, (hi buffer, lo buffer)) filled with sentinels, per the case's layouts."""
        c, n, o = self.c, self.c.n, self.c.o
        rows = D.ROWS_ABOVE + n + D.ROWS_BELOW
        ld, col0, _ = D.dest_geometry(c.y_layout, o, 4)
        ybuf = sentinel(rows, ld, torch.float32, self.device)
        ld, s0, _ = D.dest_geometry(c.s_layout, o, 2)
        hi, lo = sentinel(rows, ld, torch.float16, self.device), sentinel(rows, ld, torch.float16, self.device)
        r = slice(D.ROWS_ABOVE, D.ROWS_ABOVE + n)
        self.y_col0, self.s_col0 = col0, s0
        return (ybuf[r, col0:col0 + o], ybuf, K.Pair16(hi[r, s0:s0 + o], lo[r, s0:s0 + o], SPLIT_EXP), (hi, lo))

    def launch(self, want_y, want_pair, y_out=None, pair_out=None, rows=None, y_first_col=None, flags=None):
        c = self.c
        a, r = self.a, self.r
        if rows is not None:
            a = a.rows(*rows)
            r = None if r is None else r[rows[0]:rows[1]]
            y_out = None if y_out is None else y_out[rows[0]:rows[1]]
            pair_out = None if pair_out is None else pair_out.rows(*rows)
        return K.linear_f16x3(a, self.wp, self.b, residual=r, relu_out=c.relu_out, want_y=want_y, want_split=want_pair,
                              split_relu=c.split_relu, split_exp=SPLIT_EXP, split_cols=c.split_cols, y_out=y_out, pair_out=pair_out,
                              flags=flags, y_first_col=c.y_first_col if y_first_col is None else y_first_col)

    def truth(self):
        """(y64, pre64, denominator) in fp64."""
        x64, w64 = self.x.double(), self.w.double()
        pre = x64 @ w64.t()
        den = x64.abs() @ w64.abs().t()
        if self.b is not None:
            pre += self.b.double()
            den += self.b.double().abs()
        post = ACT64[self.c.relu_out](pre)
        if self.r is not None:
            post = post + self.r.double()
            den += self.r.double().abs()
        return post, pre, den

    def errors(self, y, cols):
        """max err of y over the columns `cols`, and the element-wise check against BAR (activation codes add their own error)."""
        y64, pre, den = self.truth()
        y64, pre, den, y = y64[:, cols], pre[:, cols], den[:, cols], y[:, cols].double()
        diff = (y - y64).abs()
        err = float((diff / den.clamp_min(1e-300)).max())
        if self.c.relu_out > 1:
            act = ACT64[self.c.relu_out](pre)
            ok = diff <= BAR * ACT_LIPSCHITZ * den + ACT_TOL * (pre.abs() + act.abs())
        else:
            ok = diff <= BAR * den
        return err, bool(ok.all())

    def torch_error(self, cols):
        y = torch_fp32_linear(self.x.contiguous(), self.w.contiguous(), self.b)
        y = ACT64[self.c.relu_out](y)
        if self.r is not None:
            y = y + self.r
        y64, _, den = self.truth()
        return float(((y.double() - y64).abs() / den.clamp_min(1e-300))[:, cols].max())


CASE_ERRORS = {}


def test_every_branch_is_reached_on_this_device(cuda_device):
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    assert D.BRANCHES - set().union(*(D.plan(c, sms) for c in D.CASES)) == set()


@torch.no_grad()
@pytest.mark.parametrize("case", D.CASES, ids=lambda c: c.id)
def test_linear_f16x3_case(cuda_device, case):
    c = case
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    b = Built(c, cuda_device, seed=len(c.id))
    want_y, want_pair = D.want_y(c), D.want_pair(c)
    y_view, ybuf, p_view, (hibuf, lobuf) = b.destinations()
    # the plan's store paths are the ones these pointers take (nfk_linear_tc.cu: vec_y / vec_s)
    if want_y:
        assert (y_view.stride(0) % 2 == 0 and y_view.data_ptr() % 8 == 0) == ("y_vec" in D.plan(c, sms) or c.o - c.y_first_col < 2)
    if want_pair:
        vec_s = p_view.hi.stride(0) % 2 == 0 and p_view.hi.data_ptr() % 4 == 0 and p_view.lo.data_ptr() % 4 == 0
        assert vec_s == ("pair_vec" in D.plan(c, sms) or D.split_n(c) < 2)
    flags = K.new_flags(cuda_device)
    before = _native.launch_count()
    y, pair = b.launch(want_y, want_pair, y_view if want_y else None, p_view if want_pair else None, flags=flags)
    assert _native.launch_count() == before + 1
    assert int(flags.item()) == 0
    sn = D.split_n(c)

    # fp32 result: every column from y_first_col on, against fp64; nothing written outside the rows and columns of the view
    y_full, _ = b.launch(True, False, y_first_col=0)            # all columns (the reference of the pair below)
    cols = slice(c.y_first_col, c.o)
    err, ok = b.errors(y_full if not want_y else y, cols if want_y else slice(0, c.o))
    CASE_ERRORS[c.id] = (err, b.torch_error(slice(0, c.o)))
    print("dense case {}: kernel err {:.3e}, torch fp32 err {:.3e}".format(c.id, *CASE_ERRORS[c.id]))
    assert ok, (c.id, err)
    ymask = torch.ones_like(ybuf, dtype=torch.bool)
    ymask[D.ROWS_ABOVE:D.ROWS_ABOVE + c.n, b.y_col0:b.y_col0 + c.o] = False
    if want_y:
        assert untouched(ybuf[ymask]), c.id
        assert torch.equal(bits(y[:, cols]), bits(y_full[:, cols])), c.id
    else:
        assert untouched(ybuf), c.id

    if want_pair:
        # the pair: bit-identical to the split of the kernel's own fp32 output (relu / none), within the activation bar else
        if c.split_relu in (0, 1):
            hi, lo = split_torch(y_full[:, :sn], SPLIT_EXP, c.split_relu)
            assert torch.equal(bits(pair.hi[:, :sn]), bits(hi)) and torch.equal(bits(pair.lo[:, :sn]), bits(lo)), c.id
        else:
            want = ACT64[c.split_relu](y_full[:, :sn].double())
            assert rel_err(pair.cols(0, sn).float(), want) <= 1e-6, c.id
        pmask = torch.ones_like(hibuf, dtype=torch.bool)
        pmask[D.ROWS_ABOVE:D.ROWS_ABOVE + c.n, b.s_col0:b.s_col0 + sn] = False
        assert untouched(hibuf[pmask]) and untouched(lobuf[pmask]), c.id       # rows outside, pitch padding, >= split_cols
        # pair-only and both: the same pair, bit for bit
        _, other = b.launch(not want_y, True)
        assert torch.equal(bits(other.hi[:, :sn]), bits(pair.hi[:, :sn])) and torch.equal(bits(other.lo[:, :sn]), bits(pair.lo[:, :sn]))

    # determinism: a second launch, and the rows in two launches, give the same bits
    y2, p2 = b.destinations()[0], b.destinations()[2]
    b.launch(want_y, want_pair, y2 if want_y else None, p2 if want_pair else None)
    if c.n > 1:
        y3, p3 = b.destinations()[0], b.destinations()[2]
        m = c.n // 2 + 3 if c.n > 8 else 1
        for rows in ((0, m), (m, c.n)):
            b.launch(want_y, want_pair, y3 if want_y else None, p3 if want_pair else None, rows=rows)
    else:
        y3, p3 = y2, p2
    if want_y:
        assert torch.equal(bits(y2[:, cols]), bits(y[:, cols])) and torch.equal(bits(y3[:, cols]), bits(y[:, cols])), c.id
    if want_pair:
        for p in (p2, p3):
            assert torch.equal(bits(p.hi[:, :sn]), bits(pair.hi[:, :sn])) and torch.equal(bits(p.lo[:, :sn]), bits(pair.lo[:, :sn]))


@torch.no_grad()
def test_f16_range_flag_of_the_pair_output(cuda_device):
    """Flag 4 when a pair value leaves the fp16 range; never when only the fp32 result is asked for."""
    x = torch.randn(200, 64, device=cuda_device)
    w = torch.randn(40, 64, device=cuda_device)
    a, wp = K.split_f16(x, 0), K.split_f16(w, K.weight_exp(w))
    big = torch.zeros(40, device=cuda_device)
    big[17] = 5000.0                                              # 5000 * 2^6 > 65000
    for want_split, expect in ((False, 0), (True, 4)):
        flags = K.new_flags(cuda_device)
        K.linear_f16x3(a, wp, big, want_y=True, want_split=want_split, split_exp=SPLIT_EXP, flags=flags)
        assert int(flags.item()) == expect
    flags = K.new_flags(cuda_device)                             # the column is past split_cols: not split, no flag
    K.linear_f16x3(a, wp, big, want_y=False, want_split=True, split_exp=SPLIT_EXP, split_cols=16, flags=flags)
    assert int(flags.item()) == 0


# ---- the FFMA layer ---------------------------------------------------------------------------------------------------------
def ffma_truth(x, w, b, r, relu_in, relu_out):
    xa = ACT64[relu_in](x.double())
    pre = xa @ w.double().t()
    den = xa.abs() @ w.double().abs().t()
    if b is not None:
        pre, den = pre + b.double(), den + b.double().abs()
    y = ACT64[relu_out](pre)
    if r is not None:
        y, den = y + r.double(), den + r.double().abs()
    slack = torch.zeros_like(den)
    if relu_in > 1:        # the fp32 activation of x: its own error, through |w|
        slack += ACT_TOL * ((x.double().abs() + xa.abs()) @ w.double().abs().t())
    if relu_out > 1:
        slack += ACT_TOL * (pre.abs() + ACT64[relu_out](pre).abs())
    return y, den, slack


FFMA_CASES = [  # n, k, o, relu_in, relu_out, bias, residual, x at an odd column
    (1000, 392, 256, 0, 0, True, False, False),
    (300, 5, 7, 1, 1, True, True, False),          # K % 4, N % 4
    (257, 13, 130, 2, 0, False, False, True),      # scalar x loads
    (129, 64, 5, 3, 3, True, False, True),
    (64, 31, 9, 4, 4, True, True, False),
    (65, 100, 33, 5, 5, True, False, True),
    (70, 6, 128, 6, 6, True, True, False),
    (20000, 36, 17, 0, 1, True, True, True),       # 157 row tiles
    (40, 4608, 64, 0, 0, True, False, False),
]


@torch.no_grad()
@pytest.mark.parametrize("n,k,o,relu_in,relu_out,bias,residual,odd", FFMA_CASES)
def test_linear_simt(cuda_device, n, k, o, relu_in, relu_out, bias, residual, odd):
    g = torch.Generator(device=cuda_device).manual_seed(n + k + o)
    xb = torch.randn(n, k + 1, device=cuda_device, generator=g)
    x = xb[:, 1:] if odd else xb[:, :k].contiguous()
    w = torch.randn(o, k, device=cuda_device, generator=g) / k ** 0.5
    b = torch.randn(o, device=cuda_device, generator=g) if bias else None
    r = torch.randn(n, o, device=cuda_device, generator=g) if residual else None
    y = K.linear(x, w, b, residual=r, relu_in=relu_in, relu_out=relu_out)
    y64, den, slack = ffma_truth(x, w, b, r, relu_in, relu_out)
    lip = ACT_LIPSCHITZ if relu_out > 1 else 1.0
    assert bool(((y.double() - y64).abs() <= BAR * lip * den + slack).all())
    yt = ACT64[relu_out](torch_fp32_linear(ACT64[relu_in](x), w, b)) + (r if r is not None else 0)
    print("ffma {}: kernel err {:.3e}, torch err {:.3e}".format((n, k, o), float(((y.double() - y64).abs() / den).max()),
                                                                 float(((yt.double() - y64).abs() / den).max())))


@torch.no_grad()
def test_linear_simt_residual_aliasing_the_output(cuda_device):
    """hidden = linear(branch, W, b, residual=hidden, out=hidden), the skip connection of the FFMA chain (dense.py)."""
    torch.manual_seed(0)
    branch, hidden = torch.randn(500, 96, device=cuda_device), torch.randn(500, 80, device=cuda_device)
    w, b = torch.randn(80, 96, device=cuda_device) / 10, torch.randn(80, device=cuda_device)
    before = hidden.clone()
    out = K.linear(branch, w, b, residual=hidden, relu_in=1, relu_out=1, out=hidden)
    assert out.data_ptr() == hidden.data_ptr()
    y64, den, _ = ffma_truth(branch, w, b, before, 1, 1)
    assert bool(((out.double() - y64).abs() <= BAR * den).all())


@torch.no_grad()
def test_linear_simt_past_the_row_super_block(cuda_device):
    """More than 65535 row tiles: the launcher loops over super-blocks of 65535 * 128 rows."""
    n = 65535 * 128 + 300
    g = torch.Generator(device=cuda_device).manual_seed(1)
    x = torch.randn(n, 3, device=cuda_device, generator=g)
    w, b = torch.randn(5, 3, device=cuda_device, generator=g), torch.randn(5, device=cuda_device, generator=g)
    r = torch.randn(n, 5, device=cuda_device, generator=g)
    y = K.linear(x, w, b, residual=r)
    edge = 65535 * 128
    pick = torch.cat([torch.arange(edge - 200, n, device=cuda_device), torch.arange(0, 100, device=cuda_device),
                      torch.randint(0, n, (4096,), device=cuda_device, generator=g)])
    y64, den, _ = ffma_truth(x[pick], w, b, r[pick], 0, 0)
    assert bool(((y[pick].double() - y64).abs() <= BAR * den).all())
    del x, r, y


# ---- the operand passes -----------------------------------------------------------------------------------------------------
def split_cases(device):
    """(name, fp32 source view, destination Pair16 view) over the vec4 and scalar instances."""
    g = torch.Generator(device=device).manual_seed(5)
    rnd = lambda *s: torch.randn(*s, device=device, generator=g) * 3
    out = []
    for name, src, dst_cols, dst_off in (
            ("vec4", rnd(300, 64), 64, 0),
            ("cols%4", rnd(300, 66)[:, :62], 62, 0),
            ("ld%4", rnd(301, 70)[:, :64], 64, 0),
            ("odd_view", rnd(77, 40)[:, 1:33], 32, 0),
            ("strided_dst", rnd(129, 32), 32, 8),
            ("strided_dst_odd", rnd(129, 31), 31, 3),
            ("subnormal_lo", (1.0 + torch.arange(1, 2049, device=device, dtype=torch.float32).reshape(64, 32) * 2.0 ** -23), 32, 0)):
        hi = torch.empty(src.shape[0], dst_cols + dst_off + 8, dtype=torch.float16, device=device)
        lo = torch.empty_like(hi)
        out.append((name, src, K.Pair16(hi[:, dst_off:dst_off + dst_cols], lo[:, dst_off:dst_off + dst_cols], 0)))
    return out


@torch.no_grad()
@pytest.mark.parametrize("code", range(7))
def test_split_f16_instances(cuda_device, code):
    for name, src, dst in split_cases(cuda_device):
        exp = 0 if name == "subnormal_lo" else 4
        dst.exp = exp
        flags = K.new_flags(cuda_device)
        K.split_f16(src, exp, relu=code, out=dst, flags=flags)
        assert int(flags.item()) == 0, name
        if code in (0, 1):
            hi, lo = split_torch(src, exp, code)
            assert torch.equal(bits(dst.hi), bits(hi)) and torch.equal(bits(dst.lo), bits(lo)), (name, code)
        else:
            assert rel_err(dst.float(), ACT64[code](src.double())) <= 1e-6, (name, code)
        if name == "subnormal_lo" and code == 0:
            sub = (dst.lo.float().abs() < 2.0 ** -14) & (dst.lo != 0)
            assert bool(sub.any()) and bool((dst.hi == 1).all())


@torch.no_grad()
def test_split_f16_flag_boundary(cuda_device):
    """|v * 2^e| <= 65000 passes; the next float, NaN and +-Inf raise flag 4 (both instances)."""
    nxt = float(torch.nextafter(torch.tensor(65000.0), torch.tensor(math.inf)))
    for cols in (8, 7):
        for v, expect in ((65000.0, 0), (-65000.0, 0), (nxt, 4), (-nxt, 4), (math.nan, 4), (math.inf, 4), (-math.inf, 4)):
            x = torch.ones(3, cols, device=cuda_device)
            x[1, cols - 1] = v
            flags = K.new_flags(cuda_device)
            K.split_f16(x, 0, flags=flags)
            assert int(flags.item()) == expect, (cols, v)


@torch.no_grad()
def test_weight_exp_and_absmax(cuda_device):
    dev = cuda_device
    wide = torch.randn(50, 40, device=dev)
    wide[:, 20:] *= 1000.0                                        # outside the view: must not count
    view = wide[:, :20]
    assert K.weight_exp(view) == 14 - math.ceil(math.log2(float(view.abs().max())))
    for p in (-30, -26, -1, 0, 3, 13, 20, 54):
        for mult in (1.0, 1.0 + 2.0 ** -23, 1.0 - 2.0 ** -24):
            w = torch.randn(33, 17, device=dev)
            w = w / w.abs().max() * 0.5 * 2.0 ** p
            w[7, 3] = -(2.0 ** p) * mult                          # the maximum magnitude, negative
            e = K.weight_exp(w)
            assert e == max(-40, min(40, 14 - math.ceil(math.log2(abs(float(w[7, 3])))))), (p, mult)
            if -40 < 14 - p < 40:
                assert 2.0 ** 13 <= 2.0 ** p * mult * 2.0 ** e <= 2.0 ** 14, (p, mult, e)
    nan = torch.randn(9, 9, device=dev)
    nan[4, 4] = math.nan
    assert K.weight_exp(nan) == 14 - math.ceil(math.log2(float(nan.nan_to_num(0).abs().max())))       # NaN skipped
    assert K.weight_exp(torch.full((4, 4), -0.0, device=dev)) == 0
    assert K.weight_exp(torch.zeros(4, 4, device=dev)) == 0
    inf = torch.ones(4, 4, device=dev)
    inf[1, 1] = math.inf
    assert K.weight_exp(inf) == 0


@torch.no_grad()
@pytest.mark.parametrize("skip,want_y,code", [(True, True, 0), (False, True, 1), (True, False, 1), (True, True, 6)])
def test_glu_skip(cuda_device, skip, want_y, code):
    g = torch.Generator(device=cuda_device).manual_seed(3)
    n, c = 1000, 37
    tg = torch.randn(n, 2 * c + 5, device=cuda_device, generator=g) * 4                  # t and gate: views of one tensor
    t, gate = tg[:, :c], tg[:, c + 5:]
    s = torch.randn(n, c + 3, device=cuda_device, generator=g)[:, 3:] if skip else None
    y, pair = K.glu_skip(t, gate, s, want_y=want_y, want_split=True, split_relu=code, split_exp=SPLIT_EXP)
    y_ref, none = K.glu_skip(t, gate, s, want_y=True)
    assert none is None and (y is None) == (not want_y)
    prod = t.double() * torch.sigmoid(gate.double())
    want = prod + (s.double() if skip else 0)
    scale = prod.abs() + (s.double().abs() if skip else 0)
    assert bool(((y_ref.double() - want).abs() <= 2.0 ** -20 * scale).all())
    if want_y:
        assert torch.equal(bits(y), bits(y_ref))
    if code in (0, 1):
        hi, lo = split_torch(y_ref, SPLIT_EXP, code)
        assert torch.equal(bits(pair.hi), bits(hi)) and torch.equal(bits(pair.lo), bits(lo))
    else:
        assert rel_err(pair.float(), ACT64[code](y_ref.double())) <= 1e-6


def im2col_torch(t, n_images, h, w):
    """The pad-and-slice formulation of the 3x3 / padding-1 operand (tests/emulated_kernels.py)."""
    n, c = t.shape
    img = F.pad(t.reshape(n_images, h, w, c), (0, 0, 1, 1, 1, 1))
    return torch.cat([img[:, ky:ky + h, kx:kx + w, :] for ky in range(3) for kx in range(3)], dim=-1).reshape(n, 9 * c)


@torch.no_grad()
def test_im2col3x3(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(9)
    chans = [(8, 0, 8), (64, 0, 64), (3, 0, 3), (5, 0, 5), (12, 0, 12), (8, 0, 16), (8, 1, 10)]   # C, first column, pitch
    for gi, (h, w) in enumerate(((1, 1), (1, 7), (7, 1), (5, 9), (7, 7), (28, 28))):
        for bi, nb in enumerate((1, 3, 130)):
            sel = chans if nb == 3 else [chans[(gi + bi) % len(chans)]]
            for c, c0, ld in sel:
                src = (torch.randn(nb * h * w, ld, device=cuda_device, generator=g) * 100).half()
                src_lo = torch.randn(nb * h * w, ld, device=cuda_device, generator=g).half()
                pair = K.Pair16(src[:, c0:c0 + c], src_lo[:, c0:c0 + c], 3)
                vec = c % 8 == 0 and ld % 8 == 0 and c0 == 0
                out = K.im2col3x3(pair, nb, h, w)
                assert out.exp == 3 and tuple(out.shape) == (nb * h * w, 9 * c)
                for got, t in ((out.hi, pair.hi), (out.lo, pair.lo)):
                    assert torch.equal(bits(got), bits(im2col_torch(t.contiguous(), nb, h, w))), (h, w, nb, c, c0, ld, vec)


@torch.no_grad()
@pytest.mark.parametrize("nb,c,o,h,w", [(3, 8, 16, 7, 7), (2, 64, 40, 5, 9), (130, 16, 8, 6, 6)])
def test_conv3x3_end_to_end(cuda_device, nb, c, o, h, w):
    """Dense layer on im2col3x3 == F.conv2d(padding=1), weight stored [out, (ky, kx, c)] (dense.ConvChain)."""
    g = torch.Generator(device=cuda_device).manual_seed(c + o)
    x = torch.randn(nb, c, h, w, device=cuda_device, generator=g)
    wt = torch.randn(o, c, 3, 3, device=cuda_device, generator=g) / (3 * c ** 0.5)
    b = torch.randn(o, device=cuda_device, generator=g)
    rows = K.nchw_to_rows(x)
    wd = wt.permute(0, 2, 3, 1).reshape(o, 9 * c).contiguous()
    y, _ = K.linear_f16x3(K.im2col3x3(K.split_f16(rows, SPLIT_EXP), nb, h, w), K.split_f16(wd, K.weight_exp(wd)), b)
    want = F.conv2d(x.double(), wt.double(), b.double(), padding=1)
    den = F.conv2d(x.double().abs(), wt.double().abs(), b.double().abs(), padding=1)
    got = K.rows_to_nchw(y, nb, o, h, w).double()
    assert bool(((got - want).abs() <= BAR * den).all())


# ---- the wrappers reject wrong destinations before anything is launched ----------------------------------------------------
@torch.no_grad()
def test_wrappers_check_residual_and_destinations(cuda_device):
    dev = cuda_device
    x, w, b = torch.randn(64, 32, device=dev), torch.randn(24, 32, device=dev), torch.randn(24, device=dev)
    a, wp = K.split_f16(x, SPLIT_EXP), K.split_f16(w, K.weight_exp(w))
    good_r = torch.randn(64, 24, device=dev)
    bad_tensors = {
        "shape": torch.randn(64, 23, device=dev), "rows": torch.randn(63, 24, device=dev),
        "dtype": good_r.double(), "device": good_r.cpu(), "column stride": torch.randn(24, 64, device=dev).t(),
    }
    torch.cuda.synchronize()
    for what, bad in bad_tensors.items():
        before = _native.launch_count()
        with pytest.raises(ValueError):
            K.linear(x, w, b, residual=bad)
        with pytest.raises(ValueError):
            K.linear_f16x3(a, wp, b, residual=bad)
        with pytest.raises(ValueError):
            K.linear_f16x3(a, wp, b, y_out=bad)
        with pytest.raises(ValueError):
            K.linear(x, w, b, out=bad)
        assert _native.launch_count() == before, what
    for bad in (torch.randn(23, device=dev), b.double(), b.cpu()):
        before = _native.launch_count()
        with pytest.raises(ValueError):
            K.linear(x, w, bad)
        with pytest.raises(ValueError):
            K.linear_f16x3(a, wp, bad)
        assert _native.launch_count() == before
    bad_pairs = [K.Pair16.empty(64, 23, SPLIT_EXP, dev), K.Pair16.empty(63, 24, SPLIT_EXP, dev),
                 K.Pair16(torch.empty(64, 24, device=dev), torch.empty(64, 24, device=dev), SPLIT_EXP),
                 K.Pair16(torch.empty(24, 64, dtype=torch.float16, device=dev).t(), torch.empty(24, 64, dtype=torch.float16, device=dev).t(), SPLIT_EXP),
                 K.Pair16(torch.empty(64, 24, dtype=torch.float16, device=dev), torch.empty(64, 32, dtype=torch.float16, device=dev)[:, :24], SPLIT_EXP)]
    for bad in bad_pairs:
        before = _native.launch_count()
        with pytest.raises(ValueError):
            K.linear_f16x3(a, wp, b, want_split=True, split_exp=SPLIT_EXP, pair_out=bad)
        assert _native.launch_count() == before
    # the good ones still run
    y, pair = K.linear_f16x3(a, wp, b, residual=good_r, y_out=torch.empty(64, 24, device=dev), want_split=True,
                             pair_out=K.Pair16.empty(64, 24, SPLIT_EXP, dev))
    assert pair is not None and y.shape == (64, 24)
