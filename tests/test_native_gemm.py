"""Dense-layer kernels (FFMA and wgmma split-fp16) against an fp64 matmul: both must be fp32-accurate."""
import pytest
import torch

from conftest import rel_err
from nflows_b200 import kernels as K

pytestmark = pytest.mark.gpu

SHAPES = [(1000, 392, 256), (300, 256, 9016), (257, 32, 128), (129, 784, 784), (5, 256, 736), (128, 8, 16), (4096, 128, 736),
          (260, 72, 40)]


def reference(x, w, b, r, relu_in, relu_out):
    x64 = x.double().clamp_min(0) if relu_in else x.double()
    y = x64 @ w.double().t() + b.double()
    if relu_out:
        y = y.clamp_min(0)
    return y + (r.double() if r is not None else 0)


@torch.no_grad()
@pytest.mark.parametrize("n,k,o", SHAPES)
def test_linear_simt(cuda_device, n, k, o):
    g = torch.Generator(device=cuda_device).manual_seed(n + k + o)
    x = torch.randn(n, k, device=cuda_device, generator=g)
    w = torch.randn(o, k, device=cuda_device, generator=g) / k ** 0.5
    b = torch.randn(o, device=cuda_device, generator=g)
    r = torch.randn(n, o, device=cuda_device, generator=g)
    for relu_in, relu_out, res in ((False, False, None), (True, True, None), (False, False, r)):
        y = K.linear(x, w, b, residual=res, relu_in=relu_in, relu_out=relu_out)
        assert rel_err(y, reference(x, w, b, res, relu_in, relu_out)) <= 8e-6


def fp16_exact(pair, x, relu=False):
    """A Pair16 represents pre(x) to 2^-21 relative of each element (or 2^-24 absolute once the lo part is subnormal)."""
    want = x.double().clamp_min(0) if relu else x.double()
    got = (pair.hi.double() + pair.lo.double()) * 2.0 ** -pair.exp
    tol = want.abs() * 2.0 ** -21 + 2.0 ** (-24 - pair.exp)
    return bool(((got - want).abs() <= tol).all())


@torch.no_grad()
@pytest.mark.parametrize("n,k,o", SHAPES)
def test_linear_f16x3(cuda_device, n, k, o):
    g = torch.Generator(device=cuda_device).manual_seed(n + k + o)
    x = torch.randn(n, k, device=cuda_device, generator=g)
    w = torch.randn(o, k, device=cuda_device, generator=g) / k ** 0.5
    b = torch.randn(o, device=cuda_device, generator=g)
    r = torch.randn(n, o, device=cuda_device, generator=g)
    assert K.f16x3_supported(k, k, k)
    flags = K.new_flags(cuda_device)
    wp = K.split_f16(w, K.weight_exp(w), flags=flags)
    assert fp16_exact(wp, w)
    assert 2 ** 13 <= float(wp.hi.abs().max()) <= 2 ** 14                   # scaled to the top of the fp16 range
    for relu_in, relu_out, res in ((False, False, None), (True, True, None), (False, False, r)):
        xp = K.split_f16(x, 6, relu=relu_in, flags=flags)
        assert fp16_exact(xp, x, relu_in)
        y, pair = K.linear_f16x3(xp, wp, b, residual=res, relu_out=relu_out, want_y=True, want_split=True, split_relu=True,
                                 split_exp=5, flags=flags)
        want = reference(x, w, b, res, relu_in, relu_out)
        assert rel_err(y, want) <= 8e-6, (n, k, o, relu_in, relu_out)
        assert pair.exp == 5 and fp16_exact(pair, y, relu=True)
    assert int(flags.item()) == 0
    # operands far from unit scale: the power-of-two exponents keep the 22-bit precision
    for sx, sw in ((1e-3, 30.0), (40.0, 1e-4)):
        xs, ws = x * sx, w * sw
        y, _ = K.linear_f16x3(K.split_f16(xs, 6 if sx < 1 else 2), K.split_f16(ws, K.weight_exp(ws)), b * sx * sw)
        assert rel_err(y, reference(xs, ws, b * sx * sw, None, False, False)) <= 8e-6, (sx, sw)
    # a strided column block as the A operand (the coupling trunk reads the identity half of a wider pair), pair output
    # limited to the first columns (the affine run in front of a coupling)
    if k % 16 == 0 and o >= 16:
        wide = K.split_f16(torch.cat([x, x.flip(1)], dim=1), 6)
        y2, pair2 = K.linear_f16x3(wide.cols(0, k), wp, b, want_y=True, want_split=True, split_cols=8)
        assert torch.equal(y2, K.linear_f16x3(K.split_f16(x, 6), wp, b)[0])
        assert fp16_exact(pair2.cols(0, 8), y2[:, :8])


@torch.no_grad()
def test_f16_range_flag(cuda_device):
    flags = K.new_flags(cuda_device)
    x = torch.full((4, 8), 2000.0, device=cuda_device)
    K.split_f16(x, 6, flags=flags)                                          # 2000 * 64 > 65000
    assert int(flags.item()) & 4
    with pytest.raises(K.Float16RangeError):
        K.raise_for_flags(flags)
    flags.zero_()
    K.split_f16(x, 4, flags=flags)
    assert int(flags.item()) == 0


@torch.no_grad()
def test_linear_f16x3_unsupported_shapes_are_rejected(cuda_device):
    assert not K.f16x3_supported(12, 12, 12)
    x = torch.randn(10, 8, device=cuda_device)
    w = torch.randn(4, 8, device=cuda_device)
    xp, wp = K.split_f16(x, 6), K.split_f16(w, 10)
    with pytest.raises(RuntimeError):
        K.linear_f16x3(xp.cols(0, 4), wp.cols(0, 4))                       # K = 4, ld = 8: not TMA-addressable
    # ... and the FFMA kernel takes any shape
    x6, w6 = torch.randn(10, 6, device=cuda_device), torch.randn(4, 6, device=cuda_device)
    assert rel_err(K.linear(x6, w6), x6.double() @ w6.double().t()) <= 8e-6
