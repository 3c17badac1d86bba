"""Training a coupling's conditioner on the tensor-core dense layers (dense.DenseChainTraining, config.native_training) without a
GPU: the autograd Function and its gate with the kernel wrappers replaced by fp64 CPU stand-ins of their contracts
(emulated_kernels plus the three new entry points below), against fp64 autograd through the torch formulation."""
import copy
import types

import pytest
import torch
from torch import nn
from torch.nn import functional as F

import emulated_kernels as E
from nflows_b200 import config
from nflows_b200 import dense as D
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.distributions import StandardNormal
from nflows_b200.flows.base import Flow
from nflows_b200.nn.nets import MLP, ResidualNet
from nflows_b200.transforms.splines import training
from nflows_b200.utils import torchutils


def _install(monkeypatch):
    """emulated_kernels plus stand-ins of nfk_absmax (host reads), nfk_linear_f16x3_wgrad and nfk_mask_split_f16."""
    calls = E.install(monkeypatch)

    def count(name, rows):
        calls[name] = calls.get(name, 0) + 1
        calls.trace.append((name, int(rows)))

    def absmax(x):
        return float(x.abs().max()) if x.numel() else 0.0

    def linear_wgrad(g, a, want_bias=True):
        count("linear_wgrad", g.shape[0])
        vg, va = E._value(g), E._value(a)
        return (vg.t() @ va).float(), vg.sum(0).float() if want_bias else None

    def mask_split(da, exp, mask=None, skip=None, cols_pad=None, want_y=False, flags=None):
        count("mask_split", da.shape[0])
        n, c = da.shape
        v = da.double()
        if mask is not None:
            v = v * (E._value(mask)[:, :c] != 0)
        if skip is not None:
            v = v + skip.double()
        v = v.float()
        pair = K.Pair16(torch.zeros(n, cols_pad or c, dtype=torch.float16), torch.zeros(n, cols_pad or c, dtype=torch.float16), exp)
        E._pair(v, exp, out=pair.cols(0, c))
        return pair, (v.clone() if want_y else None)

    def absmax_start(x):
        v = absmax(x)
        return lambda: v

    for name, fn in dict(absmax=absmax, absmax_start=absmax_start, linear_wgrad=linear_wgrad, mask_split=mask_split).items():
        monkeypatch.setattr(K, name, fn)
    monkeypatch.setattr(training, "_device_ok", lambda t: t.dtype == torch.float32 and t.dim() == 2)
    monkeypatch.setattr(training, "_cuda_fp32", lambda t: t.dtype == torch.float32)
    monkeypatch.setattr(config, "native_training", True)
    return calls


def _resnet(d_in=16, d_out=24, hidden=32, blocks=2, **kw):
    torch.manual_seed(d_in + d_out + hidden + blocks)
    net = ResidualNet(d_in, d_out, hidden_features=hidden, num_blocks=blocks, **kw)
    for p in net.parameters():                       # zero-initialised last layers would hide the blocks' gradients
        p.data.normal_(0.0, 0.3)
    return net


def _mlp(d_in=16, d_out=21, sizes=(32, 40), **kw):
    torch.manual_seed(3)
    return MLP([d_in], [d_out], list(sizes), **kw)


def _check_grads(net, x, w_out):
    """Gradients of sum(net(x) * w_out) through the Function against fp64 autograd and fp32 torch (the yardstick)."""
    net64, x64 = copy.deepcopy(net).double(), x.detach().double().requires_grad_(True)
    (net64(x64) * w_out.double()).sum().backward()
    net32, x32 = copy.deepcopy(net), x.detach().clone().requires_grad_(True)
    (net32(x32) * w_out).sum().backward()
    xn = x.detach().clone().requires_grad_(True)
    out = D.train_chain(net.dense_chain(None), xn)
    assert float((out.detach().double() - net64(x64).detach()).abs().max()) <= 1e-5 * max(1.0, float(out.detach().abs().max()))
    (out * w_out).sum().backward()
    pairs = [(xn.grad, x32.grad, x64.grad)] + [(p.grad, q.grad, r.grad) for p, q, r in zip(net.parameters(), net32.parameters(),
                                                                                             net64.parameters())]
    for i, (a, t, r) in enumerate(pairs):
        n64 = float(r.norm())
        e, et = float((a.double() - r).norm()) / n64, float((t.double() - r).norm()) / n64
        assert e <= max(1e-5, 3 * et), (i, e, et)


@pytest.mark.parametrize("make", [lambda: _resnet(), lambda: _resnet(blocks=1, hidden=40), lambda: _mlp(),
                                  lambda: _mlp(sizes=(24,)), lambda: _resnet(activation=nn.ReLU())],
                         ids=["resnet", "resnet_1block", "mlp", "mlp_1hidden", "resnet_module_relu"])
def test_function_gradients_against_fp64(make, monkeypatch):
    calls = _install(monkeypatch)
    net = make()
    torch.manual_seed(0)
    x = torch.randn(200, 16)
    w_out = torch.randn(200, net.dense_chain(None)[-1][0].shape[0])
    _check_grads(net, x, w_out)
    n_layers = len(net.dense_chain(None))
    assert calls["linear_wgrad"] == n_layers and calls["mask_split"] == n_layers
    assert calls["linear_f16x3"] == 2 * n_layers                                   # forward + input gradient per layer


def test_tiny_gradients_keep_their_relative_accuracy(monkeypatch):
    """A mean loss over a large batch scales every gradient by 1/B: the pair exponents follow each tensor's absmax."""
    _install(monkeypatch)
    net = _resnet()
    x = torch.randn(64, 16)
    _check_grads(net, x, torch.randn(64, 24) * 2.0 ** -30)


def test_gradient_exponent():
    for amax in (1.0, 3.0, 2.0 ** -30, 1e-12, 7e5):
        e = K.gradient_exp(amax)
        assert 2.0 ** 13 <= amax * 2.0 ** e < 2.0 ** 14 or amax * 2.0 ** e == 2.0 ** 14
    assert K.gradient_exp(0.0) == 0 and K.gradient_exp(float("inf")) == 0 and K.gradient_exp(float("nan")) == 0


def test_needs_input_grad_and_none_cotangent(monkeypatch):
    calls = _install(monkeypatch)
    net = _resnet()
    x = torch.randn(32, 16)
    out = D.train_chain(net.dense_chain(None), x)                  # x needs no gradient: the first layer's input gradient is skipped
    out.sum().backward()
    n_layers = len(net.dense_chain(None))
    assert calls["linear_f16x3"] == n_layers + n_layers - 1 and all(p.grad is not None for p in net.parameters())
    for p in net.parameters():
        p.requires_grad_(False)
    net.final_layer.weight.requires_grad_(True)
    before = calls.get("linear_wgrad", 0)
    net.final_layer.weight.grad = None
    D.train_chain(net.dense_chain(None), x).sum().backward()
    assert calls["linear_wgrad"] == before + 1 and net.final_layer.weight.grad is not None
    ctx = types.SimpleNamespace(structure=((0, 0, None),), exp=6, needs_input_grad=(True, False, True, True), saved_tensors=())
    assert D.DenseChainTraining.backward(ctx, None) == (None, None, None, None)


def test_double_backward_is_refused(monkeypatch):
    _install(monkeypatch)
    net = _mlp()
    x = torch.randn(8, 16, requires_grad=True)
    (g,) = torch.autograd.grad(D.train_chain(net.dense_chain(None), x).square().sum(), x, create_graph=True)
    with pytest.raises(RuntimeError, match="once_differentiable|twice"):
        g.sum().backward()


def _coupling_flow(kind, net_fn):
    torch.manual_seed(7)
    steps = []
    for i in range(2):
        mask = torchutils.create_alternating_binary_mask(32, even=(i % 2 == 0))
        if kind == "affine":
            steps.append(T.AffineCouplingTransform(mask, net_fn))
        else:
            steps.append(T.AdditiveCouplingTransform(mask, net_fn))
    return Flow(T.CompositeTransform(steps), StandardNormal([32]))


@pytest.mark.parametrize("kind", ["affine", "additive"])
def test_coupling_flows_route_their_conditioner(kind, monkeypatch):
    """Affine / additive couplings with an MLP: the conditioner runs on the Function, the heads stay torch; the gradients pass
    the fp64 sandwich."""
    net_fn = lambda a, b: MLP([a], [b], [32, 32])
    flow = _coupling_flow(kind, net_fn)
    flow64 = copy.deepcopy(flow).double()
    x = torch.randn(128, 32)
    monkeypatch.setattr(config, "native_training", False)
    flow.zero_grad()
    (-flow.log_prob(x).mean()).backward()
    g_torch = [p.grad.double().clone() for p in flow.parameters()]
    (-flow64.log_prob(x.double()).mean()).backward()
    g64 = [p.grad.clone() for p in flow64.parameters()]
    calls = _install(monkeypatch)
    flow.zero_grad()
    (-flow.log_prob(x).mean()).backward()
    assert calls["linear_wgrad"] == 2 * 3
    for i, (a, t, r) in enumerate(zip([p.grad.double() for p in flow.parameters()], g_torch, g64)):
        n64 = float(r.norm())
        assert float((a - r).norm()) / n64 <= max(1e-5, 3 * float((t - r).norm()) / n64), i


def _refused():
    ctx_net = ResidualNet(16, 24, hidden_features=32, context_features=4)
    bn = ResidualNet(16, 24, hidden_features=32, use_batch_norm=True)
    drop = ResidualNet(16, 24, hidden_features=32, dropout_probability=0.1).train()
    return {
        "tanh": (ResidualNet(16, 24, hidden_features=32, activation=torch.tanh), None),
        "leaky_relu": (_mlp(activation=F.leaky_relu), None),
        "context": (ctx_net, torch.randn(8, 4)),
        "batch_norm": (bn, None),
        "dropout_training": (drop, None),
        "activate_output": (_mlp(activate_output=True), None),
        "in_features_not_8": (ResidualNet(12, 24, hidden_features=32), None),
        "hidden_not_8": (_mlp(sizes=(30,)), None),
        "custom_module": (nn.Sequential(nn.Linear(16, 24)), None),
    }


@pytest.mark.parametrize("case", sorted(_refused()))
def test_refused_conditioners_launch_nothing_and_keep_torch(case, monkeypatch):
    net, ctx = _refused()[case]
    d_in = 12 if case == "in_features_not_8" else 16
    x = torch.randn(8, d_in)
    calls = _install(monkeypatch)
    assert not training.routed_conditioner(net, x, ctx)
    assert not calls


def test_gate(monkeypatch):
    calls = _install(monkeypatch)
    net = _resnet()
    x = torch.randn(8, 16)
    assert training.routed_conditioner(net, x, None)                    # the parameters need gradients
    assert training.routed_conditioner(_mlp(), x, None)
    with torch.no_grad():
        assert not training.routed_conditioner(net, x, None)
    monkeypatch.setattr(config, "native_training", False)
    assert not training.routed_conditioner(net, x, None)
    monkeypatch.setattr(config, "native_training", True)
    assert not training.routed_conditioner(copy.deepcopy(net).double(), x.double(), None)     # fp64
    assert not training.routed_conditioner(net, x[None], None)                                # not 2-D
    frozen = copy.deepcopy(net).requires_grad_(False)
    assert not training.routed_conditioner(frozen, x, None)                                   # nothing to differentiate
    assert training.routed_conditioner(frozen, x.requires_grad_(True), None)
    monkeypatch.setattr(training, "_device_ok", lambda t: t.is_cuda and t.dtype == torch.float32 and t.dim() == 2)
    assert not training.routed_conditioner(net, x, None)                                      # CPU tensors stay torch
    monkeypatch.setenv("NFLOWS_B200_GEMM", "simt")
    monkeypatch.setattr(training, "_device_ok", lambda t: t.dtype == torch.float32 and t.dim() == 2)
    assert not training.routed_conditioner(net, x, None)                                      # the tensor-core layers are off
    assert not calls


def test_switch_off_keeps_the_module_call(monkeypatch):
    """With config.native_training off the coupling calls its conditioner exactly as before: bit-identical gradients, no stand-in."""
    flow = _coupling_flow("affine", lambda a, b: ResidualNet(a, b, hidden_features=32))
    x = torch.randn(64, 32)
    (-flow.log_prob(x).mean()).backward()
    ref = [p.grad.clone() for p in flow.parameters()]
    calls = _install(monkeypatch)
    monkeypatch.setattr(config, "native_training", False)
    flow.zero_grad()
    (-flow.log_prob(x).mean()).backward()
    assert not calls and all(torch.equal(p.grad, r) for p, r in zip(flow.parameters(), ref))


def test_wgrad_wrapper_argument_checks():
    g = K.Pair16(torch.zeros(4, 8, dtype=torch.float16), torch.zeros(4, 8, dtype=torch.float16), 0)
    a = K.Pair16(torch.zeros(5, 8, dtype=torch.float16), torch.zeros(5, 8, dtype=torch.float16), 0)
    with pytest.raises(ValueError, match="same rows"):
        K.linear_wgrad(g, a)
    bad = K.Pair16(torch.zeros(4, 8, dtype=torch.float32), torch.zeros(4, 8, dtype=torch.float32), 0)
    with pytest.raises(ValueError, match="float16"):
        K.linear_wgrad(g, bad)
    with pytest.raises(ValueError):
        K.mask_split(torch.zeros(4, 8), 0)                               # not a CUDA tensor
