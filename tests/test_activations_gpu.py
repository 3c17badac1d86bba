"""Conditioner activations other than relu, and feed-forward MADE blocks, on the H100: the activation codes of the dense-layer
kernels against fp64, the reference's outputs (tests/golden/activation_rows.pt), a sweep of activations x conditioners x widths x
depths x context, batch sizes, row-block splits, the activation rescale and the golden flow's sampling.  Every native case asserts
from the launch timeline that its kernels ran; every out-of-scope case that nothing launched."""
import copy

import pytest
import torch
import torch.nn.functional as F
from torch import nn

from conftest import rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.distributions import MADEMoG
from nflows_b200.nn.nets import MLP, ResidualNet
from test_activations_host import CASES, MASK8, build, outputs, perturb, sandwich_ok, _out_of_scope
from test_conditional_ar_gpu import timeline

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def native_activations(monkeypatch):
    monkeypatch.setattr(config, "native_activations", True)

CODES = [_native.ACT_NONE, _native.ACT_RELU, _native.ACT_TANH, _native.ACT_ELU, _native.ACT_LEAKY_RELU, _native.ACT_GELU,
         _native.ACT_SILU]
ACT64 = {0: lambda t: t, 1: F.relu, 2: torch.tanh, 3: F.elu, 4: F.leaky_relu, 5: F.gelu, 6: F.silu}
ACTIVATIONS = {"relu": nn.ReLU(), "tanh": torch.tanh, "elu": F.elu, "leaky_relu": nn.LeakyReLU(), "gelu": F.gelu, "silu": nn.SiLU()}


def sweep_inputs(device):
    """Dense in [-12, 12], values near 0 of every scale, and large magnitudes, both signs."""
    near0 = torch.logspace(-30, 0, 301, dtype=torch.float64)
    large = torch.logspace(1, 4.3, 101, dtype=torch.float64)
    v = torch.cat([torch.linspace(-12, 12, 4801, dtype=torch.float64), near0, -near0, large, -large, torch.zeros(1, dtype=torch.float64)])
    n = (v.numel() + 7) // 8 * 8
    v = torch.cat([v, torch.zeros(n - v.numel(), dtype=torch.float64)])
    return v.float().reshape(-1, 8).to(device)


@torch.no_grad()
@pytest.mark.parametrize("code", CODES)
def test_split_f16_applies_each_code(cuda_device, code):
    x = sweep_inputs(cuda_device)
    with timeline() as tl:
        pair = K.split_f16(x, 0, relu=code)
    assert tl.launches == 1
    want = ACT64[code](x.double())
    assert rel_err(pair.float().double().cpu(), want.cpu()) <= 1e-6
    zero = K.split_f16(torch.zeros(4, 8, device=cuda_device), 0, relu=code)
    assert torch.equal(zero.hi.float(), torch.zeros_like(zero.hi.float())) and torch.equal(zero.lo.float(), zero.hi.float())


@torch.no_grad()
@pytest.mark.parametrize("code", CODES)
def test_dense_layers_apply_each_code(cuda_device, code):
    """linear_f16x3's output and split activations, and the FFMA layer's input and output activations, against fp64."""
    torch.manual_seed(code)
    x = 3 * torch.randn(600, 32, device=cuda_device)             # large magnitudes: test_split_f16_applies_each_code
    w = torch.randn(96, 32, device=cuda_device) * 0.3
    b = torch.randn(96, device=cuda_device)
    a = K.split_f16(x, 2)
    wp = K.split_f16(w, K.weight_exp(w))
    pre = x.double() @ w.double().t() + b.double()
    with timeline() as tl:
        y, pair = K.linear_f16x3(a, wp, b, relu_out=code, want_split=True, split_relu=code)
    assert tl.launches == 1
    assert rel_err(y.cpu(), ACT64[code](pre).cpu()) <= 1e-5
    assert rel_err(pair.float().cpu(), ACT64[code](ACT64[code](pre)).cpu()) <= 1e-5
    with timeline() as tl:
        y2 = K.linear(x, w, b, relu_in=code, relu_out=code)
    assert tl.launches == 1
    assert rel_err(y2.cpu(), ACT64[code](ACT64[code](x.double()) @ w.double().t() + b.double()).cpu()) <= 1e-5


# the couplings' 4 identity features take the FFMA dense layers (not a multiple of 8), which have no timeline tag (None)
STEP_TAG = {"maf_flow": "affine_ar_step", "maf_rq": "rq_coupling_step", "made_gelu": "affine_ar_step", "rq_elu": None,
            "rq_elu_ctx": None, "affine_leaky": None, "mademog_silu": "mog_made_step",
            "cfg4_tanh": "rq_coupling_step"}


@torch.no_grad()
@pytest.mark.parametrize("case", CASES)
def test_golden_cases(cuda_device, case):
    from conftest import load_golden
    g = load_golden("activation_rows")[case]
    m = build(case, g).to(cuda_device)
    with timeline() as tl:
        got = outputs(case, m, g, cuda_device)
    assert tl.launches > 0 and (STEP_TAG[case] is None or tl.count(STEP_TAG[case]) >= 1), tl.tags
    for key, v in got.items():
        assert sandwich_ok(v, g, key), (key, rel_err(v.cpu(), g[key + "_fp64"]), rel_err(g[key], g[key + "_fp64"]))


def conditioner_ran(tl):
    """A conditioner kernel is on the timeline (the spline of a torch-path MAF-RQ still runs natively: nfk_rqs_elementwise)."""
    return any(t in ("rq_coupling_step", "affine_ar_step", "mog_made_step", "ar_context_terms", "rq_coupling_final",
                     "affine_coupling_final") or t.startswith(("linear_", "trunk_step")) for t in tl.tags)


# ---- the sweep ------------------------------------------------------------------------------------------------------------
def net_case(kind, act, hidden, blocks, context):
    """(module, features, context features) of one sweep point."""
    if kind == "resnet":
        return T.PiecewiseRationalQuadraticCouplingTransform(
            MASK8 * 2, lambda i, o: ResidualNet(i, o, hidden, context_features=context, num_blocks=blocks, activation=act),
            num_bins=8, tails="linear", tail_bound=3.0), 16, context
    if kind == "mlp":
        return T.AffineCouplingTransform(MASK8 * 2, lambda i, o: MLP([i], [o], [hidden] * (blocks + 1), activation=act)), 16, None
    if kind == "made_res":
        return T.MaskedAffineAutoregressiveTransform(16, hidden, context_features=context, num_blocks=blocks, activation=act), 16, context
    if kind == "made_ff":
        return T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
            12, hidden, context_features=context, num_blocks=blocks, use_residual_blocks=False, num_bins=8, tails="linear",
            tail_bound=3.0, activation=act), 12, context
    return MADEMoG(6, hidden, context or 3, num_blocks=blocks, use_residual_blocks=False, num_mixture_components=4,
                   activation=act), 6, context or 3


SHAPES = [(32, 0, None), (50, 1, 16), (96, 2, None), (256, 4, 16)]


@torch.no_grad()
@pytest.mark.parametrize("kind", ["resnet", "mlp", "made_res", "made_ff", "mademog_ff"])
@pytest.mark.parametrize("name", list(ACTIVATIONS))
def test_sweep(cuda_device, kind, name):
    """Forward and inverse (or log_prob and sample) against the fp64 torch formulation, on the native kernels, for widths
    32 / 50 / 96 / 256 with 0 / 1 / 2 / 4 blocks, alternately with a 16-wide context.  Widths that are not a multiple of 32
    run natively where the model pads them (MADEMoG, MAF-affine) or runs the layer-by-layer chain (couplings); MAF-RQ keeps
    the torch path there."""
    for hidden, blocks, context in SHAPES:
        torch.manual_seed(hidden + blocks)
        m, d, cf = net_case(kind, ACTIVATIONS[name], hidden, blocks, context)
        m = perturb(m, 1).eval().to(cuda_device)
        m64 = copy.deepcopy(m).double()
        x = torch.randn(300, d, device=cuda_device)
        c = None if cf is None else torch.randn(300, cf, device=cuda_device)
        c64 = None if c is None else c.double()
        native = not (hidden == 50 and kind == "made_ff")
        label = (kind, name, hidden, blocks, context)
        if kind == "mademog_ff":
            with timeline() as tl:
                lp = m.log_prob(x, context=c)
            assert tl.count("mog_made_step") >= 1, label
            assert rel_err(lp.cpu(), m64.log_prob(x.double(), context=c64).cpu()) <= 1e-4, label
            with timeline() as tl:
                s = m.sample(2, context=c[:50])
            assert tl.count("mog_made_step") >= 6, label
            assert torch.isfinite(s).all()
            continue
        with timeline() as tl:
            y, lad = m(x, context=c)
        assert (tl.launches > 0 if native else not conditioner_ran(tl)), (label, tl.tags)
        y64, lad64 = m64(x.double(), context=c64)
        assert rel_err(y.cpu(), y64.cpu()) <= 1e-4 and rel_err(lad.cpu(), lad64.cpu()) <= 1e-4, label
        with timeline() as tl:
            xi, li = m.inverse(y, context=c)
        assert (tl.launches > 0 if native else not conditioner_ran(tl)), label
        assert rel_err(xi.cpu(), x.cpu()) <= 1e-3 and rel_err(li.cpu(), -lad.cpu()) <= 1e-3, label


# ---- batch sizes, row blocks, rescale, sampling ------------------------------------------------------------------------------
def sbi_maf(device):
    torch.manual_seed(3)
    m = T.MaskedAffineAutoregressiveTransform(5, 50, context_features=7, use_residual_blocks=False, activation=torch.tanh)
    return perturb(m, 4).eval().to(device)


@torch.no_grad()
def test_batch_sizes_and_row_block_splits(cuda_device, monkeypatch):
    """Rows 1 .. 2 * 132 * 128 + 300 on the native kernels; every row's result is bit-identical whatever the row blocks."""
    m = sbi_maf(cuda_device)
    n = 2 * 132 * 128 + 300
    x, c = torch.randn(n, 5, device=cuda_device), torch.randn(n, 7, device=cuda_device)
    monkeypatch.setattr(config, "coupling_block_rows", 1 << 20)
    y_full, lad_full = m(x, context=c)
    monkeypatch.setattr(config, "coupling_block_rows", 128)
    with timeline() as tl:
        y, lad = m(x, context=c)
    assert tl.count("affine_ar_step") == (n + 127) // 128
    assert torch.equal(y, y_full) and torch.equal(lad, lad_full)
    for rows in (1, 127, 128, 129, n):
        with timeline() as tl:
            yr, lr = m(x[:rows], context=c[:rows])
        assert tl.count("affine_ar_step") == (rows + 127) // 128
        assert torch.equal(yr, y_full[:rows]) and torch.equal(lr, lad_full[:rows]), rows
    m64 = copy.deepcopy(m).double()
    assert rel_err(y.cpu(), m64(x.double(), context=c.double())[0].cpu()) <= 1e-5


@torch.no_grad()
def test_activation_rescale_on_large_inputs(cuda_device):
    m = sbi_maf(cuda_device)
    x, c = 1e4 * torch.randn(500, 5, device=cuda_device), torch.randn(500, 7, device=cuda_device)
    with pytest.warns(RuntimeWarning):
        with timeline() as tl:
            y, lad = m(x, context=c)
    assert tl.count("affine_ar_step") >= 2
    y64, lad64 = copy.deepcopy(m).double()(x.double(), context=c.double())
    assert rel_err(y.cpu(), y64.cpu()) <= 1e-5 and rel_err(lad.cpu(), lad64.cpu()) <= 1e-5


@torch.no_grad()
def test_golden_flow_sampling(cuda_device):
    from conftest import load_golden
    g = load_golden("activation_rows")["maf_flow"]
    flow = build("maf_flow", g).to(cuda_device)
    c = g["context"][:20].to(cuda_device)
    with timeline() as tl:
        lp = flow.log_prob(g["x"][:20].to(cuda_device), context=c)
    assert tl.count("affine_ar_step") == 5
    assert rel_err(lp.cpu(), g["log_prob_fp64"][:20]) <= 1e-5
    torch.manual_seed(7)
    with timeline() as tl:
        s = flow.sample(8, context=c)
    assert s.shape == (20, 8, 5) and tl.count("affine_ar_step") >= 5 * 5
    torch.manual_seed(7)
    with timeline() as tl:
        s2, lp2 = flow.sample_and_log_prob(8, context=c)
    assert tl.count("affine_ar_step") >= 5 * 5
    assert rel_err(s2.cpu(), s.cpu()) <= 1e-6
    flow64 = copy.deepcopy(flow).double()
    want = flow64.log_prob(s2.reshape(-1, 5).double(), context=c.double().repeat_interleave(8, dim=0)).reshape(20, 8)
    assert rel_err(lp2.cpu(), want.cpu()) <= 1e-4


@torch.no_grad()
def test_out_of_scope_cases_launch_nothing(cuda_device):
    torch.manual_seed(5)
    for m, d, cf in _out_of_scope():
        m = m.eval().to(cuda_device)
        x, c = torch.randn(100, d, device=cuda_device), None if cf is None else torch.randn(100, cf, device=cuda_device)
        with timeline() as tl:
            if isinstance(m, MADEMoG):
                m.log_prob(x, context=c)
            else:
                m(x, context=c)
                m.inverse(x, context=c)
        assert not conditioner_ran(tl) and (tl.launches == 0 or isinstance(m, T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform)), m
