"""The row-wise kernels (nfk_rowwise.cu) and the index kernels of the image path (nfk_image.cu) on the H100, each against a plain
torch formulation of the same operation: bit for bit where the kernel's arithmetic allows it (gathers, transposes, squeezes,
fills, ActNorm's correctly rounded mul / add / div, the identity columns of a coupling), else against fp64.

The sums (std_normal_log_prob, segment_sum, a coupling's log|det|) are held to the classic bound of m fp32 additions,
|err| <= m * 2^-24 * sum |terms|, with m the additions one lane makes (ceil(len / 32)) plus the five-step warp reduction and the
final adds: a kernel that drops or repeats a term is orders of magnitude outside it.  Measured on an H100 80GB HBM3 (700 W),
std_normal_log_prob's worst err relative to sum |terms| was 1.7e-7 over every d and layout here, the same as torch's fp32
formulation (1.7e-7); the bound is at least 1.3e-6."""
import math

import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from nflows_b200 import kernels as K
from nflows_b200.transforms.reshape import SqueezeTransform

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def bits(t):
    return t.contiguous().view(torch.int32)


def sum_bound(length, extra=8):
    return (math.ceil(length / 32) + extra) * U


def more_than_one_round():
    """Elements past one grid-stride round of the row-wise kernels (grid capped at 64 blocks of 256 threads per SM)."""
    return torch.cuda.get_device_properties(0).multi_processor_count * 64 * 256 + 12345


@torch.no_grad()
def test_gather_cols(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(0)
    x = torch.randn(40000, 90, device=cuda_device, generator=g)[:, 3:80]                       # strided input
    cols = torch.cat([torch.randperm(77, generator=g, device=cuda_device), torch.tensor([5, 5, 76, 0], device=cuda_device)])
    assert x.shape[0] * cols.numel() > more_than_one_round()
    out_buf = torch.full((40000, cols.numel() + 6), 123.0, device=cuda_device)
    out = K.gather_cols(x, K.index_tensor(cols, cuda_device), out=out_buf[:, 2:2 + cols.numel()])
    assert torch.equal(bits(out), bits(x[:, cols]))
    assert bool((out_buf[:, :2] == 123.0).all()) and bool((out_buf[:, 2 + cols.numel():] == 123.0).all())
    assert torch.equal(bits(K.gather_cols(x[:7], K.index_tensor(cols[:3], cuda_device))), bits(x[:7, cols[:3]]))


@torch.no_grad()
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("with_lad", [False, True])
def test_actnorm(cuda_device, inverse, with_lad):
    g = torch.Generator(device=cuda_device).manual_seed(1)
    for n, d in ((1, 1), (333, 7), (20000, 129)):
        x = torch.randn(n, d + 2, device=cuda_device, generator=g)[:, 1:1 + d] * 3
        scale = torch.rand(d, device=cuda_device, generator=g) * 2 + 0.1
        shift = torch.randn(d, device=cuda_device, generator=g)
        lad0 = torch.randn(n, device=cuda_device, generator=g)
        lad = lad0.clone() if with_lad else None
        c = -1.2345678
        y = K.actnorm(x, scale, shift, lad, c, inverse)
        want = (x - shift) / scale if inverse else x * scale + shift
        assert torch.equal(bits(y), bits(want)), (n, d)
        if with_lad:
            assert torch.equal(bits(lad), bits(lad0 + torch.tensor(c, dtype=torch.float32))), (n, d)      # exactly once per row


def coupling_truth(x, params, mult, act, inverse, t_cols, dtype):
    """(y of the transformed columns, sum log scale) of the affine / additive coupling in `dtype`."""
    x, params = x.to(dtype), params.to(dtype)
    d_t = t_cols.numel()
    xt = x[:, t_cols.long()]
    shift = params[:, :d_t]
    if mult == 1:
        return (xt - shift if inverse else xt + shift), torch.zeros(x.shape[0], dtype=dtype, device=x.device)
    u = params[:, d_t:2 * d_t]
    scale = torch.sigmoid(u + 2.0) + 1e-3 if act == 0 else torch.clamp(F.softplus(u) + 1e-3, 0.0, 3.0)
    y = (xt - shift) / scale if inverse else xt * scale + shift
    return y, torch.log(scale).sum(1)


@torch.no_grad()
@pytest.mark.parametrize("d_t", [1, 31, 32, 33, 100])
@pytest.mark.parametrize("mult,act", [(1, 0), (2, 0), (2, 1)])
@pytest.mark.parametrize("inverse", [False, True])
def test_affine_coupling_rows(cuda_device, d_t, mult, act, inverse):
    g = torch.Generator(device=cuda_device).manual_seed(d_t * 7 + mult + act)
    d_id = 13
    n = 3000
    perm = torch.randperm(d_t + d_id, generator=g, device=cuda_device)
    t_cols, id_cols = perm[:d_t], perm[d_t:]                                        # arbitrary order
    x = torch.randn(n, d_t + d_id + 3, device=cuda_device, generator=g)[:, :d_t + d_id] * 2
    params = torch.randn(n, mult * d_t, device=cuda_device, generator=g) * 3
    if mult == 2:      # raw scales across the softplus threshold (20) and the clamp at 3 (softplus(u) + 1e-3 = 3 near u = 2.95)
        edge = torch.tensor([19.99, 20.0, 20.01, 2.94, 2.9459, 2.95, 2.96, -30.0, 30.0], device=cuda_device)
        params[:edge.numel(), d_t:] = edge[:, None].expand(-1, d_t) if d_t > 1 else edge[:, None]
        params[-edge.numel():, d_t] = edge
    lad0 = torch.randn(n, device=cuda_device, generator=g)
    for with_lad in (True, False):
        lad = lad0.clone() if with_lad else None
        y = K.affine_coupling_rows(x, params, mult, act, inverse, K.index_tensor(t_cols, cuda_device),
                                   K.index_tensor(id_cols, cuda_device), lad)
        assert torch.equal(bits(y[:, id_cols]), bits(x[:, id_cols]))
        (y32, s32), (y64, s64) = (coupling_truth(x, params, mult, act, inverse, t_cols, dt) for dt in (torch.float32, torch.float64))
        # the fp64 sandwich: within 3x (outputs) / 5x (log|det|) the fp32 torch formulation's own distance from fp64
        assert rel_err(y[:, t_cols], y64) <= max(2e-6, 3 * rel_err(y32, y64))
        if with_lad:
            sign = -1.0 if inverse else 1.0
            want = lad0.double() + sign * s64
            assert rel_err(lad, want) <= max(1e-5, 5 * rel_err(lad0 + sign * s32, want))
            if mult == 1:
                assert torch.equal(bits(lad), bits(lad0))


@torch.no_grad()
@pytest.mark.parametrize("d", [1, 3, 4, 127, 128, 3072])
@pytest.mark.parametrize("layout", ["dense", "ld%4", "misaligned"])
@pytest.mark.parametrize("with_lad", [False, True])
def test_std_normal_log_prob(cuda_device, d, layout, with_lad):
    g = torch.Generator(device=cuda_device).manual_seed(d)
    n = 2000
    if layout == "dense":
        z = torch.randn(n, d, device=cuda_device, generator=g)                       # float4 path when d % 4 == 0
    elif layout == "ld%4":
        z = torch.randn(n, d + 1, device=cuda_device, generator=g)[:, :d]
    else:
        z = torch.randn(n, d + 8, device=cuda_device, generator=g)[:, 1:1 + d]
    z = z * 1.5
    lad = torch.randn(n, device=cuda_device, generator=g) * 10 if with_lad else None
    log_z = 0.5 * d * math.log(2 * math.pi)
    out = K.std_normal_log_prob(z, log_z, lad)
    z64 = z.double()
    want = -0.5 * (z64 * z64).sum(1) - float(torch.tensor(log_z, dtype=torch.float32))
    scale = 0.5 * (z64 * z64).sum(1) + abs(log_z)
    if with_lad:
        want, scale = want + lad.double(), scale + lad.double().abs()
    err = (out.double() - want).abs()
    assert bool((err <= 2 * sum_bound(d, 10) * scale).all()), float((err / scale).max())
    torch32 = -0.5 * (z * z).sum(1) - log_z + (lad if with_lad else 0)
    print("std_normal_log_prob d={} {}: kernel {:.2e}, torch fp32 {:.2e}".format(
        d, layout, float((err / scale).max()), float(((torch32.double() - want).abs() / scale).max())))


@torch.no_grad()
@pytest.mark.parametrize("length", [1, 31, 32, 33, 1024, 3072])
def test_segment_sum(cuda_device, length):
    g = torch.Generator(device=cuda_device).manual_seed(length)
    segs = 5000
    v = torch.randn(segs * length, device=cuda_device, generator=g)
    out0 = torch.randn(segs, device=cuda_device, generator=g) * 100
    out = out0.clone()
    K.segment_sum_(v, out, length)
    want = out0.double() + v.double().reshape(segs, length).sum(1)
    scale = out0.double().abs() + v.double().abs().reshape(segs, length).sum(1)
    assert bool(((out.double() - want).abs() <= sum_bound(length) * scale).all())


@torch.no_grad()
def test_nchw_rows_round_trip(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(4)
    for b in (1, 3, 64):
        for c in (1, 3, 33, 40, 70):
            for h, w in ((7, 7), (5, 9), (28, 28), (1, 1)):
                x = torch.randn(b, c, h, w, device=cuda_device, generator=g)
                rows = K.nchw_to_rows(x)
                assert torch.equal(bits(rows), bits(x.permute(0, 2, 3, 1).reshape(b * h * w, c))), (b, c, h, w)
                back = K.rows_to_nchw(rows, b, c, h, w)
                assert torch.equal(bits(back), bits(x)), (b, c, h, w)


@torch.no_grad()
def test_squeeze_rows(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(6)
    for b, c, h, w in ((1, 1, 2, 2), (3, 3, 6, 10), (2, 5, 28, 28), (130, 12, 4, 8)):
        x = torch.randn(b, c, h, w, device=cuda_device, generator=g)
        rows = K.nchw_to_rows(x)
        out, shape = K.squeeze_rows(rows, b, c, h, w)
        want = SqueezeTransform()(x)[0]
        assert shape == tuple(want.shape[1:])
        assert torch.equal(bits(out), bits(want.permute(0, 2, 3, 1).reshape(-1, 4 * c)))
        back, shape2 = K.squeeze_rows(out, b, 4 * c, h // 2, w // 2, inverse=True)
        assert shape2 == (c, h, w)
        assert torch.equal(bits(back), bits(SqueezeTransform().inverse(want)[0].permute(0, 2, 3, 1).reshape(-1, c)))
        assert torch.equal(bits(back), bits(rows))
    with pytest.raises(ValueError):
        K.squeeze_rows(torch.zeros(3 * 5, 2, device=cuda_device), 1, 2, 3, 5)
    with pytest.raises(ValueError):
        K.squeeze_rows(torch.zeros(4, 6, device=cuda_device), 1, 6, 2, 2, inverse=True)


@torch.no_grad()
def test_fill_and_add_const(cuda_device):
    for n in (1, 7, 1001, more_than_one_round()):
        t = torch.randn(n + 2, device=cuda_device)
        before = t.clone()
        K.fill_(t[1:1 + n], -3.75)
        assert bool((t[1:1 + n] == -3.75).all()) and t[0] == before[0] and t[-1] == before[-1]
        v = torch.randn(n + 2, device=cuda_device)
        want = v.clone()
        want[1:1 + n] += 0.3
        K.add_const_(v[1:1 + n], 0.3)
        assert torch.equal(bits(v), bits(want))
