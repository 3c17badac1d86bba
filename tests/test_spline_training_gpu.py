"""Training with the spline on the kernels (config.native_training) on an H100: nfk_rqs_rows_backward against fp64 autograd at
every instance, the argument checks, whole-model gradients and an SGD run against fp64 copies of the models, and the evidence that
the kernels ran."""
import copy
import ctypes

import pytest
import torch

import _spline_cases as S
from nflows_b200 import _native as N
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.distributions import StandardNormal
from nflows_b200.flows import recipes
from nflows_b200.flows.base import Flow
from nflows_b200.nn.nets import ResidualNet
from nflows_b200.utils import torchutils
from oracle import flow_oracle as O
from test_spline_training_host import assert_statistically_as_accurate, autograd_vjp, near_knot

pytestmark = pytest.mark.gpu

# every instance branch of nfk_rqs_rows_backward: < 8, 8 exact, < 16, 16 exact, <= 32, <= 64
KERNEL_BINS = (3, 8, 12, 16, 24, 64)


def _case(n_rows, d_t, bins, tails, dev, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    m = 3 * bins - 1 if tails == "linear" else 3 * bins + 1
    uw, uh, ud = S.params(n_rows * d_t, bins, tails, g, scale=1.5)
    params = torch.cat([uw, uh, ud], -1).reshape(n_rows, d_t * m).contiguous()
    x = S.inputs(n_rows * d_t, tails, g).reshape(n_rows, d_t) * 0.999
    gy = torch.randn(n_rows, d_t, generator=g, device=dev)
    gl = torch.randn(n_rows, generator=g, device=dev)
    return x, params, gy, gl, (uw, uh, ud)


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("bins", KERNEL_BINS)
def test_kernel_against_fp64(cuda_device, bins, tails, inverse, monkeypatch):
    monkeypatch.setattr(O, "F32_CUMSUM", True)
    for n_rows, d_t in ((129, 32), (1000, 3), (40, 100)):            # >= 3000 elements: the percentiles are not single elements
        x, params, gy, gl, (uw, uh, ud) = _case(n_rows, d_t, bins, tails, cuda_device, bins * 7 + d_t + inverse)
        desc = S.desc(bins, tails)
        gx, gp = K.rqs_rows_backward(desc, inverse, x, params, gy, gl)
        glx = gl[:, None].expand(n_rows, d_t).reshape(-1)
        args = (x.reshape(-1), uw, uh, ud, gy.reshape(-1), glx, tails, inverse)
        tx, tp = autograd_vjp(*args, torch.float64, S.DIVISOR)
        rx, rp = autograd_vjp(*args, torch.float32, S.DIVISOR)
        what = (bins, tails, inverse, n_rows, d_t)
        skip = near_knot(x.reshape(-1), uw, uh, tails, inverse, S.DIVISOR)
        assert_statistically_as_accurate(gx.reshape(-1).cpu(), rx.cpu(), tx, what + ("g_x",), skip)
        assert_statistically_as_accurate(gp.reshape(n_rows * d_t, -1).cpu(), rp.cpu(), tp, what + ("g_params",), skip)


@pytest.mark.parametrize("d_t", [1, 3, 8, 32, 100, 128, 392, 1000])
def test_kernel_shapes_strides_null_cotangents_and_determinism(cuda_device, d_t):
    """Every feature count, row counts around a chunk and past sm_count * 32 chunks (grid stride), strided x / grad_y /
    grad_x, NULL cotangents and NULL grad_x, bitwise-identical results across runs and across row splits."""
    bins, tails = 8, "linear"
    desc = S.desc(bins, tails)
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    big = (sms * 32 * 128) // d_t + 7
    for n_rows in (0, 1, 127, 129, big if d_t >= 100 else min(big, 40000)):
        x, params, gy, gl, _ = _case(max(n_rows, 1), d_t, bins, tails, cuda_device, d_t + n_rows)
        x, params, gy, gl = x[:n_rows], params[:n_rows], gy[:n_rows], gl[:n_rows]
        gx, gp = K.rqs_rows_backward(desc, False, x, params, gy, gl)
        if n_rows == 0:
            assert gx.shape == (0, d_t) and gp.shape == params.shape
            continue
        gx2, gp2 = K.rqs_rows_backward(desc, False, x, params, gy, gl)
        assert torch.equal(gx, gx2) and torch.equal(gp, gp2)
        # strided x / grad_y, and a row split: identical bits
        xs = torch.zeros(n_rows, d_t + 5, device=cuda_device)[:, 2:2 + d_t]
        xs.copy_(x)
        gys = torch.zeros(n_rows, d_t + 3, device=cuda_device)[:, :d_t]
        gys.copy_(gy)
        h = n_rows // 2
        parts = [K.rqs_rows_backward(desc, False, xs[a:b], params[a:b], gys[a:b], gl[a:b]) for a, b in ((0, h), (h, n_rows))]
        assert torch.equal(torch.cat([p[0] for p in parts]), gx) and torch.equal(torch.cat([p[1] for p in parts]), gp)
        # NULL cotangents: the linear parts of the VJP
        gx_y, gp_y = K.rqs_rows_backward(desc, False, x, params, gy, None)
        gx_l, gp_l = K.rqs_rows_backward(desc, False, x, params, None, gl)
        assert float((gx_y + gx_l - gx).abs().max()) <= 1e-4 * max(1.0, float(gx.abs().max()))
        assert float((gp_y + gp_l - gp).abs().max()) <= 1e-4 * max(1.0, float(gp.abs().max()))
        none_x, gp_n = K.rqs_rows_backward(desc, False, x, params, gy, gl, want_grad_x=False)
        assert none_x is None and torch.equal(gp_n, gp)
        # strided grad_x through the C ABI
        out = torch.full((n_rows, d_t + 4), 7.0, device=cuda_device)
        gp3 = torch.empty_like(params)
        N.check(N.lib().nfk_rqs_rows_backward(ctypes.byref(desc), 0, x.data_ptr(), x.stride(0), params.data_ptr(), gy.data_ptr(),
                                              gy.stride(0), gl.data_ptr(), out.data_ptr(), out.stride(0), gp3.data_ptr(), d_t,
                                              n_rows, N.stream()))
        torch.cuda.synchronize()
        assert torch.equal(out[:, :d_t], gx) and bool((out[:, d_t:] == 7.0).all()) and torch.equal(gp3, gp)


def test_kernel_argument_errors_before_launch(cuda_device):
    desc = S.desc(8, "linear")
    x = torch.zeros(4, 2, device=cuda_device)
    params = torch.zeros(4, 2 * 23, device=cuda_device)
    before = N.launch_count()
    with pytest.raises(ValueError):
        K.rqs_rows_backward(desc, False, x, params, torch.zeros(4, 3, device=cuda_device), None)
    with pytest.raises(ValueError):
        K.rqs_rows_backward(desc, False, x, params.t(), None, None)
    with pytest.raises(RuntimeError, match="alias"):
        N.check(N.lib().nfk_rqs_rows_backward(ctypes.byref(desc), 0, x.data_ptr(), 2, params.data_ptr(), 0, 0, 0, 0, 0,
                                              params.data_ptr(), 2, 4, N.stream()))
    bad = S.desc(8, "linear")
    bad.num_bins = 0
    with pytest.raises(RuntimeError):
        K.rqs_rows_backward(bad, False, x, params, None, None)
    assert N.launch_count() == before


# ---- whole models: gradients against an fp64 copy ------------------------------------------------------------------------
def _nsf(features, layers=3, hidden=64):
    torch.manual_seed(features)
    return recipes.perturb_(recipes.rq_nsf(features=features, hidden_features=hidden, num_layers=layers))


def _maf(features, context=None):
    torch.manual_seed(features + (context or 0))
    steps = []
    for i in range(2):
        steps.append(T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
            features=features, hidden_features=64, context_features=context, num_bins=8, tails="linear", tail_bound=3.0))
        steps.append(T.ReversePermutation(features))
    return Flow(T.CompositeTransform(steps), StandardNormal([features]))


def _context_coupling_flow(features=16, context=4):
    torch.manual_seed(5)
    steps = []
    for i in range(2):
        steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(features, even=(i % 2 == 0)),
            transform_net_create_fn=lambda a, b: ResidualNet(a, b, hidden_features=64, context_features=context, num_blocks=2),
            num_bins=8, tails="linear", tail_bound=3.0))
    return Flow(T.CompositeTransform(steps), StandardNormal([features]))


def _cfg2_flow():
    torch.manual_seed(2)
    return Flow(T.CompositeTransform([recipes.rq_coupling_layer(), T.RandomPermutation(64)]), StandardNormal([64]))


def _loss(model, x, ctx, sample):
    if sample:
        # what sample_and_log_prob computes, with the noise drawn once for the three runs: samples = inverse(z) and
        # log p = base(z) - log|det| of the inverse; the loss reaches both the samples and the log-density
        samples, lad = model._transform.inverse(x, context=ctx)
        return (0.5 * samples.square().sum(1) - (-0.5 * x.square().sum(1) - lad)).mean()
    return -model.log_prob(x, context=ctx).mean()


def _grads(model, x, ctx, native, monkeypatch, sample=False):
    monkeypatch.setattr(config, "native_training", native)
    model.zero_grad()
    _loss(model, x, ctx, sample).backward()
    return [None if p.grad is None else p.grad.detach().double().clone() for p in model.parameters()]


def _sandwich(g32, g_torch, g64, what):
    for i, (a, t, r) in enumerate(zip(g32, g_torch, g64)):
        if r is None:                 # a parameter the loss does not depend on: no gradient in any of the three runs
            assert a is None and t is None, (what, i)
            continue
        n64 = float(r.norm())
        if n64 == 0.0:
            assert float(a.norm()) <= 1e-6, (what, i)
            continue
        e, et = float((a - r).norm()) / n64, float((t - r).norm()) / n64
        assert e <= max(1e-5, 3 * et), (what, i, e, et)


MODELS = {
    "cfg2_coupling": (_cfg2_flow, 64, None, False),
    "nsf_d64": (lambda: _nsf(64), 64, None, False),
    "nsf_d784": (lambda: _nsf(784, hidden=128), 784, None, False),
    "maf_rq_d16": (lambda: _maf(16), 16, None, False),
    "maf_rq_d64": (lambda: _maf(64), 64, None, False),
    "maf_rq_d16_context": (lambda: _maf(16, context=8), 16, 8, False),
    "maf_rq_d64_context": (lambda: _maf(64, context=8), 64, 8, False),
    "coupling_context": (_context_coupling_flow, 16, 4, False),
    "sample_and_log_prob": (lambda: _nsf(64, layers=2), 64, None, True),
}


@pytest.mark.parametrize("name", sorted(MODELS))
def test_model_gradients_against_fp64(cuda_device, name, monkeypatch):
    make, d, c, sample = MODELS[name]
    model = make().eval().to(cuda_device)
    model64 = copy.deepcopy(model).double()
    torch.manual_seed(1)
    n = 512
    x = (torch.randn(n, d) * 1.2).to(cuda_device)
    ctx = None if c is None else torch.randn(n, c).to(cuda_device)
    K._warned_eager[0] = False
    with pytest.warns(RuntimeWarning, match="differentiable PyTorch"):
        g_torch = _grads(model, x, ctx, False, monkeypatch, sample)     # switch off: the torch path and its warning
    before = N.launch_count()
    K.TIMELINE = []
    try:
        g_native = _grads(model, x, ctx, True, monkeypatch, sample)
        torch.cuda.synchronize()
        tags = {t[0] for t in K.TIMELINE}
    finally:
        K.TIMELINE = None
    assert N.launch_count() > before and "rqs_rows_backward" in tags, (name, tags)
    g64 = _grads(model64, x.double(), None if ctx is None else ctx.double(), False, monkeypatch, sample)
    _sandwich(g_native, g_torch, g64, name)


def test_switch_off_launches_nothing(cuda_device, monkeypatch):
    model = _cfg2_flow().to(cuda_device)
    x = torch.randn(256, 64, device=cuda_device)
    monkeypatch.setattr(config, "native_training", False)
    before = N.launch_count()
    (-model.log_prob(x).mean()).backward()
    torch.cuda.synchronize()
    assert N.launch_count() == before


def test_sgd_run_against_fp64(cuda_device, monkeypatch):
    """20 SGD steps from one initialisation on the same batches: the final parameters pass the sandwich against an fp64 run."""
    base = _nsf(64, layers=2).eval()
    runs = {}
    for key, dtype, native in (("native", torch.float32, True), ("torch", torch.float32, False), ("fp64", torch.float64, False)):
        monkeypatch.setattr(config, "native_training", native)
        model = copy.deepcopy(base).to(device=cuda_device, dtype=dtype)
        opt = torch.optim.SGD(model.parameters(), lr=1e-2)
        g = torch.Generator().manual_seed(0)
        for _ in range(20):
            x = (torch.randn(512, 64, generator=g) * 1.2).to(device=cuda_device, dtype=dtype)
            opt.zero_grad()
            (-model.log_prob(x).mean()).backward()
            opt.step()
        runs[key] = [p.detach().double().clone() for p in model.parameters()]
    init = [p.detach().double().to(cuda_device) for p in base.parameters()]
    # compare the parameter CHANGES (the initial values are common to the three runs)
    delta = lambda r: [a - b for a, b in zip(r, init)]
    _sandwich(delta(runs["native"]), delta(runs["torch"]), delta(runs["fp64"]), "sgd")
