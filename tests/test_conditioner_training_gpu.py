"""Training a coupling's conditioner on the tensor-core dense layers (config.native_training) on an H100: nfk_linear_f16x3_wgrad
against fp64 across widths, batch sizes and gradient scales, its determinism, nfk_mask_split_f16 at the range flag, the argument
checks, whole-model gradients and an SGD run against fp64 copies, the timeline tags, and nothing launched with the switch off."""
import copy
import ctypes

import pytest
import torch

from nflows_b200 import _native as N
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.distributions import StandardNormal
from nflows_b200.flows import recipes
from nflows_b200.flows.base import Flow
from nflows_b200.nn.nets import MLP
from nflows_b200.utils import torchutils
from test_spline_training_gpu import _cfg2_flow, _grads, _nsf, _sandwich

pytestmark = pytest.mark.gpu

WIDTHS = (8, 40, 128, 256, 736, 1000)


def _pairs(n, out, inp, dev, seed, g_scale=1.0):
    gen = torch.Generator(device=dev).manual_seed(seed)
    g32 = torch.randn(n, out, device=dev, generator=gen) * g_scale
    a32 = torch.relu(torch.randn(n, inp, device=dev, generator=gen))
    g = K.split_f16(g32, K.gradient_exp(K.absmax(g32))) if n else K.Pair16.empty(0, out, 0, dev)
    a = K.split_f16(a32, 6) if n else K.Pair16.empty(0, inp, 6, dev)
    return g, a


def _check(g, a, dw, db):
    vg = (g.hi.double() + g.lo.double()) * 2.0 ** -g.exp
    va = (a.hi.double() + a.lo.double()) * 2.0 ** -a.exp
    ref, mag = vg.t() @ va, vg.abs().t() @ va.abs()
    err = (dw.double() - ref).abs()
    assert bool((err <= 1e-5 * mag + 1e-30).all()), float((err / mag.clamp_min(1e-300)).max())
    bref, bmag = vg.sum(0), vg.abs().sum(0)
    assert bool(((db.double() - bref).abs() <= 1e-5 * bmag + 1e-30).all())


@pytest.mark.parametrize("out", WIDTHS)
@pytest.mark.parametrize("inp", WIDTHS)
def test_wgrad_against_fp64(cuda_device, out, inp):
    for n in (1, 37, 512, 513, 4097):                     # one row, a partial K-slab, one slab, a ragged last slab
        g, a = _pairs(n, out, inp, cuda_device, out * 7 + inp + n)
        _check(g, a, *K.linear_wgrad(g, a))


@pytest.mark.parametrize("shape", [(128, 128), (736, 128), (40, 1000)])
def test_wgrad_large_batches_determinism_and_strides(cuda_device, shape):
    """Up to 2^20 rows (several rounds of (slab, tile) work items), bitwise-identical repeats, and identical bits when the
    same operands sit at another row pitch."""
    out, inp = shape
    for n in (70001, 1 << 20):
        g, a = _pairs(n, out, inp, cuda_device, n + out)
        dw, db = K.linear_wgrad(g, a)
        _check(g, a, dw, db)
        dw2, db2 = K.linear_wgrad(g, a)
        assert torch.equal(dw, dw2) and torch.equal(db, db2)
        if n == 70001:
            wide = K.Pair16(torch.zeros(n, out + 24, dtype=torch.float16, device=cuda_device),
                            torch.zeros(n, out + 24, dtype=torch.float16, device=cuda_device), g.exp)
            wide.hi[:, 8:8 + out] = g.hi
            wide.lo[:, 8:8 + out] = g.lo
            dw3, db3 = K.linear_wgrad(wide.cols(8, 8 + out), a)
            assert torch.equal(dw3, dw) and torch.equal(db3, db)
    none_db = K.linear_wgrad(g, a, want_bias=False)
    assert none_db[1] is None and torch.equal(none_db[0], dw)


@pytest.mark.parametrize("scale", [2.0 ** -30, 2.0 ** -44, 1e3])
def test_wgrad_gradient_scales_and_the_underflow_bound(cuda_device, scale):
    """A mean loss shrinks gradients as 1/B: the pair exponent follows the tensor's absmax, so tiny gradients keep their accuracy.
    Every element is carried within 2^-22 of itself plus 2^-38 of the absmax (kernels.gradient_exp); elements 2^-30 below the
    absmax survive, elements below 2^-39 of it flush to zero."""
    n, out, inp = 3000, 40, 128
    g32 = torch.randn(n, out, device=cuda_device) * scale
    g32[0, 0] = 4.0 * scale
    g32[:, 1::4] = g32[:, 1::4].sign() * 2.0 ** -30 * scale * (1.0 + g32[:, 1::4].abs() / scale)
    g32[:, 3::4] = 2.0 ** -41 * scale
    amax = float(g32.abs().max())
    g = K.split_f16(g32, K.gradient_exp(amax))
    represented = (g.hi.double() + g.lo.double()) * 2.0 ** -g.exp
    assert bool(((represented - g32.double()).abs() <= 2.0 ** -22 * g32.double().abs() + 2.0 ** -38 * amax).all())
    assert bool((represented[:, 1::4] != 0).all()) and not bool(represented[:, 3::4].any())
    a = K.split_f16(torch.relu(torch.randn(n, inp, device=cuda_device)), 6)
    _check(g, a, *K.linear_wgrad(g, a))


def test_wgrad_zero_rows_and_argument_checks(cuda_device):
    g, a = _pairs(0, 16, 24, cuda_device, 0)
    dw, db = K.linear_wgrad(g, a)
    assert not dw.any() and not db.any()
    g, a = _pairs(64, 16, 24, cuda_device, 1)
    dw = torch.empty(16, 24, device=cuda_device)
    ws = torch.empty(int(N.lib().nfk_linear_f16x3_wgrad_workspace(64, 16, 24, 0)) // 4, device=cuda_device)
    call = lambda **kw: N.lib().nfk_linear_f16x3_wgrad(
        g.hi.data_ptr(), g.lo.data_ptr(), kw.get("ldg", 16), kw.get("g_exp", g.exp), a.hi.data_ptr(), a.lo.data_ptr(), 24, a.exp,
        kw.get("dw", dw.data_ptr()), 24, 0, 64, 16, 24, kw.get("ws", ws.data_ptr()), kw.get("ws_bytes", ws.numel() * 4), N.stream())
    before = N.launch_count()
    assert call(ws_bytes=ws.numel() * 4 - 4) == -1                    # workspace too small
    assert call(ldg=8) == -1                                           # pitch below the features
    assert call(g_exp=99) == -1
    assert call(dw=ws.data_ptr()) == -1                                # dW inside the workspace
    assert call(dw=0) == -1
    assert N.launch_count() == before
    assert call() == 0


def test_mask_split_range_flag_mask_skip_and_padding(cuda_device):
    n, c = 300, 21
    da = torch.randn(n, c, device=cuda_device)
    z = torch.randn(n, c, device=cuda_device)
    mask = K.split_f16(torch.relu(z), 6)
    skip = torch.randn(n, c, device=cuda_device)
    flags = torch.zeros(1, dtype=torch.int32, device=cuda_device)
    exp = K.gradient_exp(float((da.abs() + skip.abs()).max()))
    pair, y = K.mask_split(da, exp, mask=mask, skip=skip, cols_pad=24, want_y=True, flags=flags)
    want = da * (z > 0) + skip
    assert torch.equal(y, want) and int(flags.item()) == 0
    got = (pair.hi.double() + pair.lo.double()) * 2.0 ** -exp
    assert float((got[:, :c] - want.double()).abs().max()) <= 2.0 ** -20 * float(want.abs().max())
    assert not pair.hi[:, c:].any() and not pair.lo[:, c:].any()
    _, none = K.mask_split(da, exp, flags=flags)
    assert none is None and int(flags.item()) == 0
    K.mask_split(da * 2.0 ** 20, exp, flags=flags)                       # |v| 2^exp beyond 65000: the range flag
    assert int(flags.item()) & 4
    narrow = K.split_f16(z[:, :8], 6)
    torch.cuda.synchronize()
    before = N.launch_count()
    with pytest.raises(ValueError):
        K.mask_split(da, exp, mask=narrow)
    with pytest.raises(ValueError):
        K.mask_split(da, exp, skip=skip[:, :3])
    assert N.lib().nfk_mask_split_f16(da.data_ptr(), c, 0, 0, 0, 0, 0, c, c - 1, 0, pair.hi.data_ptr(), pair.lo.data_ptr(), 24, 0, 0,
                                      n, 0, N.stream()) == -1      # padding narrower than the columns
    assert N.lib().nfk_mask_split_f16(da.data_ptr(), c, 0, 0, 0, 0, 0, c, c, 0, pair.hi.data_ptr(), pair.lo.data_ptr(), 24,
                                      da.data_ptr(), c, n, 0, N.stream()) == -1     # g aliasing dA
    assert N.launch_count() == before


# ---- whole models ---------------------------------------------------------------------------------------------------------
def _coupling_mlp_flow(kind, d=32):
    torch.manual_seed(11)
    steps = []
    for i in range(2):
        mask = torchutils.create_alternating_binary_mask(d, even=(i % 2 == 0))
        net = lambda a, b: MLP([a], [b], [64, 64])
        steps.append(T.AffineCouplingTransform(mask, net) if kind == "affine" else T.AdditiveCouplingTransform(mask, net))
        steps.append(T.ReversePermutation(d))
    return Flow(T.CompositeTransform(steps), StandardNormal([d]))


MODELS = {
    "cfg2_coupling": (_cfg2_flow, 64, False),
    "nsf_d64": (lambda: _nsf(64), 64, False),
    "nsf_d784": (lambda: _nsf(784, hidden=128), 784, False),
    "affine_mlp": (lambda: _coupling_mlp_flow("affine"), 32, False),
    "additive_mlp": (lambda: _coupling_mlp_flow("additive"), 32, False),
    "sample_and_log_prob": (lambda: _nsf(64, layers=2), 64, True),
}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_model_gradients_against_fp64(cuda_device, name, monkeypatch):
    make, d, sample = MODELS[name]
    model = make().eval().to(cuda_device)
    model64 = copy.deepcopy(model).double()
    torch.manual_seed(1)
    x = (torch.randn(512, d) * 1.2).to(cuda_device)
    g_torch = _grads(model, x, None, False, monkeypatch, sample)
    K.TIMELINE = []
    try:
        g_native = _grads(model, x, None, True, monkeypatch, sample)
        torch.cuda.synchronize()
        tags = {t[0] for t in K.TIMELINE}
    finally:
        K.TIMELINE = None
    assert any(t.startswith("linear_wgrad_") for t in tags) and any(t.startswith("mask_split_") for t in tags), (name, tags)
    g64 = _grads(model64, x.double(), None, False, monkeypatch, sample)
    _sandwich(g_native, g_torch, g64, name)


def test_sgd_run_against_fp64(cuda_device, monkeypatch):
    """20 SGD steps of an affine-coupling flow with MLP conditioners: the parameter changes pass the sandwich against fp64."""
    base = _coupling_mlp_flow("affine").eval()
    runs = {}
    for key, dtype, native in (("native", torch.float32, True), ("torch", torch.float32, False), ("fp64", torch.float64, False)):
        monkeypatch.setattr(config, "native_training", native)
        model = copy.deepcopy(base).to(device=cuda_device, dtype=dtype)
        opt = torch.optim.SGD(model.parameters(), lr=1e-2)
        g = torch.Generator().manual_seed(0)
        for _ in range(20):
            x = torch.randn(512, 32, generator=g).to(device=cuda_device, dtype=dtype)
            opt.zero_grad()
            (-model.log_prob(x).mean()).backward()
            opt.step()
        runs[key] = [p.detach().double().clone() for p in model.parameters()]
    init = [p.detach().double().to(cuda_device) for p in base.parameters()]
    delta = lambda r: [a - b for a, b in zip(r, init)]
    _sandwich(delta(runs["native"]), delta(runs["torch"]), delta(runs["fp64"]), "sgd_affine_mlp")


def test_switch_off_launches_nothing(cuda_device, monkeypatch):
    model = _coupling_mlp_flow("affine").to(cuda_device)
    x = torch.randn(256, 32, device=cuda_device)
    monkeypatch.setattr(config, "native_training", False)
    before = N.launch_count()
    (-model.log_prob(x).mean()).backward()
    torch.cuda.synchronize()
    assert N.launch_count() == before
