"""Conditioner activations other than relu, and feed-forward MADE blocks, on the CPU: the torch path against the reference's
outputs (tests/golden/activation_rows.pt, scripts/make_activation_golden.py), the one map from callables to activation codes
(dense.activation_code), the chains, step-plan flag words and context projections built from it, the launch traces of the native
routes on CPU stand-ins that apply the codes, the cases that keep the torch path, and the entry points' checks of the codes."""
import ctypes

import pytest
import torch
import torch.nn.functional as F
from torch import nn

import emulated_kernels as EK
from conftest import load_golden, rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import dense as D
from nflows_b200 import transforms as T
from nflows_b200.distributions import MADEMoG, StandardNormal
from nflows_b200.flows import Flow
from nflows_b200.nn.nde import MixtureOfGaussiansMADE
from nflows_b200.nn.nets import MLP, ConvResidualNet, ResidualNet

MASK8 = [1, 0, 1, 0, 1, 0, 1, 0]
BLOCK = 128             # config.coupling_block_rows of the emulated runs: 160 rows are two row blocks


@pytest.fixture(autouse=True)
def native_activations(monkeypatch):
    """The conditioners of this file run natively only with config.native_activations on (off, they keep the torch path)."""
    monkeypatch.setattr(config, "native_activations", True)


def perturb(module, seed):
    """scripts/make_activation_golden.py: every bias + 0.1 N(0, 1), the residual blocks' second linear + 0.05 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "linear_layers.1" in name:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return module


BUILDERS = {       # the modules of scripts/make_activation_golden.py, built from this package
    "maf_flow": lambda: Flow(T.CompositeTransform(
        [t for _ in range(5) for t in (T.MaskedAffineAutoregressiveTransform(5, 50, context_features=7, use_residual_blocks=False,
                                                                             activation=torch.tanh), T.RandomPermutation(5))]),
        StandardNormal([5])),
    "maf_rq": lambda: T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
        8, 64, context_features=6, num_bins=8, tails="linear", tail_bound=3.0, use_residual_blocks=False, activation=torch.tanh),
    "made_gelu": lambda: T.MaskedAffineAutoregressiveTransform(8, 64, activation=F.gelu),
    "rq_elu": lambda: T.PiecewiseRationalQuadraticCouplingTransform(
        MASK8, lambda i, o: ResidualNet(i, o, 64, num_blocks=2, activation=F.elu), num_bins=8, tails="linear", tail_bound=3.0),
    "rq_elu_ctx": lambda: T.PiecewiseRationalQuadraticCouplingTransform(
        MASK8, lambda i, o: ResidualNet(i, o, 64, context_features=6, num_blocks=2, activation=F.elu), num_bins=8, tails="linear",
        tail_bound=3.0),
    "affine_leaky": lambda: T.AffineCouplingTransform(MASK8, lambda i, o: MLP([i], [o], [64, 64], activation=F.leaky_relu)),
    "mademog_silu": lambda: MADEMoG(5, 50, 7, num_mixture_components=10, use_residual_blocks=False, activation=nn.SiLU()),
    "cfg4_tanh": lambda: T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
        64, 256, num_bins=8, tails="linear", tail_bound=3.0, num_blocks=2, activation=torch.tanh),
}
CASES = list(BUILDERS)


def build(case, g):
    """The fixture's module: its stored reference state_dict, or re-created from its seed and checked against the reference's
    weight checksum."""
    if "state_dict" in g:
        m = BUILDERS[case]().eval()
        m.load_state_dict(g["state_dict"], strict=True)
        return m
    torch.manual_seed(g["seed"])
    m = perturb(BUILDERS[case]().eval(), g["perturb_seed"])
    ck = float(sum(v.double().abs().sum() for v in m.state_dict().values() if v.is_floating_point()))
    if abs(ck - g["checksum"]) > 1e-9 * abs(g["checksum"]):
        pytest.fail("weights re-created from the seed do not match the fixture's checksum: regenerate it with "
                    "scripts/make_activation_golden.py against the reference")
    return m


def outputs(case, m, g, device=None):
    """The outputs the fixture stores for `case`, computed by `m` on the fixture's inputs (moved to `device`)."""
    mv = (lambda t: t) if device is None else (lambda t: None if t is None else t.to(device))
    x, c = mv(g["x"]), mv(g["context"])
    if case == "maf_flow":
        s, lad = m._transform.inverse(mv(g["noise"]), context=c)
        return dict(log_prob=m.log_prob(x, context=c), sample=s, lad_inv=lad)
    if case == "mademog_silu":
        return dict(log_prob=m.log_prob(x, context=c))
    y, lad = m(x, context=c)
    xi, li = m.inverse(x, context=c)
    return dict(y=y, lad=lad, xinv=xi, ladinv=li)


def sandwich_ok(got, g, key):
    """fp64 sandwich (DESIGN section 2): within 3x the reference's own fp32 error of its fp64 result, or the 1e-5 (forward) /
    1e-4 (inverse) bar."""
    floor = 1e-4 if key in ("xinv", "ladinv", "sample", "lad_inv") else 1e-5
    return rel_err(got.cpu(), g[key + "_fp64"]) <= max(floor, 3 * rel_err(g[key], g[key + "_fp64"]))


@torch.no_grad()
@pytest.mark.parametrize("case", CASES)
def test_torch_path_matches_the_reference(case):
    g = load_golden("activation_rows")[case]
    m = build(case, g)
    for key, got in outputs(case, m, g).items():
        assert sandwich_ok(got, g, key), (key, rel_err(got, g[key + "_fp64"]), rel_err(g[key], g[key + "_fp64"]))


# ---- the map from callables to codes ----------------------------------------------------------------------------------------
def test_activation_code_table():
    accepted = {_native.ACT_RELU: [F.relu, torch.relu, nn.ReLU(), nn.ReLU(inplace=True)],
                _native.ACT_TANH: [torch.tanh, F.tanh, nn.Tanh()],
                _native.ACT_ELU: [F.elu, nn.ELU(), nn.ELU(alpha=1.0)],
                _native.ACT_LEAKY_RELU: [F.leaky_relu, nn.LeakyReLU(), nn.LeakyReLU(0.01)],
                _native.ACT_GELU: [F.gelu, nn.GELU(), nn.GELU(approximate="none")],
                _native.ACT_SILU: [F.silu, nn.SiLU()]}
    for code, fns in accepted.items():
        for fn in fns:
            assert D.activation_code(fn) == code, fn
    rejected = [torch.sigmoid, F.sigmoid, nn.Sigmoid(), nn.ELU(alpha=0.5), nn.LeakyReLU(0.2), nn.GELU(approximate="tanh"),
                lambda x: F.relu(x), lambda x: F.gelu(x, approximate="tanh"), F.softplus, nn.Softplus(), nn.Identity(), F.relu6,
                nn.PReLU(), None, "relu", type("MyReLU", (nn.ReLU,), {})()]
    for fn in rejected:
        assert D.activation_code(fn) is None, fn


# ---- chains, flag words, context projections ------------------------------------------------------------------------------
def _codes(chain):
    return [(int(a), int(b), r) for _, _, a, b, r in chain]


def test_chains_carry_the_codes():
    tanh, gelu, elu = _native.ACT_TANH, _native.ACT_GELU, _native.ACT_ELU
    ff = T.MaskedAffineAutoregressiveTransform(8, 64, num_blocks=3, use_residual_blocks=False, activation=torch.tanh).autoregressive_net
    assert _codes(ff.dense_chain()) == [(0, tanh, None)] * 4 + [(0, 0, None)]
    res = T.MaskedAffineAutoregressiveTransform(8, 64, num_blocks=2, activation=F.gelu).autoregressive_net
    assert _codes(res.dense_chain()) == [(0, 0, None)] + [(gelu, gelu, None), (0, 0, "skip")] * 2 + [(0, 0, None)]
    nde_ff = MixtureOfGaussiansMADE(8, 64, num_blocks=2, use_residual_blocks=False, activation=nn.SiLU())
    assert _codes(nde_ff.dense_chain()) == [(0, 0, None)] + [(0, _native.ACT_SILU, None)] * 2 + [(0, 0, None)]
    rn = ResidualNet(4, 16, 64, num_blocks=2, activation=F.elu)
    assert _codes(rn.dense_chain()) == [(0, 0, None)] + [(elu, elu, None), (0, 0, "skip")] * 2 + [(0, 0, None)]
    rnc = ResidualNet(4, 16, 64, context_features=3, num_blocks=1, activation=F.elu)
    assert _codes(rnc.dense_chain(torch.randn(2, 3))) == [(0, 0, "ctx_init"), (elu, elu, None), (0, 0, "glu_skip"), (0, 0, None)]
    mlp = MLP([4], [16], [64, 64], activation=F.leaky_relu, activate_output=True)
    assert _codes(mlp.dense_chain()) == [(0, _native.ACT_LEAKY_RELU, None)] * 3
    relu = T.MaskedAffineAutoregressiveTransform(8, 64).autoregressive_net            # relu: the slots read as they always did
    assert _codes(relu.dense_chain()) == [(0, 0, None)] + [(1, 1, None), (0, 0, "skip")] * 2 + [(0, 0, None)]


def test_step_plan_flag_words():
    shift = _native.STEP_ACT_SHIFT
    relu = T.MaskedAffineAutoregressiveTransform(8, 64).autoregressive_net
    assert D.plan_step_kernel(relu.dense_chain()) == [4 | 8, 1, 2 | 4 | 8, 1, 2]       # the flag words of relu, unchanged
    tanh = T.MaskedAffineAutoregressiveTransform(8, 64, activation=torch.tanh).autoregressive_net
    t = _native.ACT_TANH << shift
    assert D.plan_step_kernel(tanh.dense_chain()) == [4 | 8 | t, 1 | t, 2 | 4 | 8 | t, 1 | t, 2]
    ff = T.MaskedAffineAutoregressiveTransform(8, 64, num_blocks=2, use_residual_blocks=False, activation=F.gelu).autoregressive_net
    g = _native.ACT_GELU << shift
    assert D.plan_step_kernel(ff.dense_chain()) == [1 | g] * 3
    nde = MixtureOfGaussiansMADE(8, 64, num_blocks=1, use_residual_blocks=False, activation=F.silu)
    assert D.plan_step_kernel(nde.dense_chain()) == [0, 1 | (_native.ACT_SILU << shift)]
    # a layer whose output and whose consumer's input take different activations has no flag word
    w, b = torch.zeros(64, 64), torch.zeros(64)
    assert D.plan_step_kernel([(w, b, 0, 2, None), (w, b, 3, 0, None), (w, b, 0, 0, None)]) is None
    assert D.plan_step_kernel([(w, b, 0, 9, None), (w, b, 0, 0, None)]) is None


def test_feed_forward_made_context_layers_and_projection(monkeypatch):
    EK.install(monkeypatch)
    for cls, act in ((T.MaskedAffineAutoregressiveTransform, _native.ACT_TANH), (MADEMoG, 0)):
        m = cls(5, 50, context_features=7, use_residual_blocks=False, activation=torch.tanh, num_blocks=2)
        net = m._made if cls is MADEMoG else m.autoregressive_net
        assert net._has_context_layers()
        proj = net.context_projection()
        assert proj.initial_act == act and proj.num_blocks == 0 and proj.blocks is None
        terms = proj.terms(torch.randn(10, 7))
        assert len(terms) == 1 and terms[0].shape == (10, 50)
    res = T.MaskedAffineAutoregressiveTransform(5, 50, context_features=7, activation=F.gelu, num_blocks=2).autoregressive_net
    proj = res.context_projection()
    assert proj.initial_act == _native.ACT_GELU and proj.num_blocks == 2
    terms = proj.terms(torch.randn(10, 7))
    assert [None if t is None else tuple(t.shape) for t in terms] == [(10, 50), (10, 50), None, (10, 50), None]


# ---- routes on CPU stand-ins that apply the codes ----------------------------------------------------------------------------
@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    monkeypatch.setattr(config, "coupling_block_rows", BLOCK)
    return EK.install(monkeypatch)


STEP_OF = {"maf_flow": "affine_ar_step", "maf_rq": "rq_coupling_step", "made_gelu": "affine_ar_step", "rq_elu": "linear",
           "rq_elu_ctx": "linear", "affine_leaky": "linear", "mademog_silu": "mog_made_step",
           "cfg4_tanh": "rq_coupling_step"}


@torch.no_grad()
@pytest.mark.parametrize("case", CASES)
def test_golden_cases_on_emulated_kernels(emu, case):
    """Every golden case runs its native route on stand-ins that apply the codes, and meets the reference's outputs there."""
    g = load_golden("activation_rows")[case]
    m = build(case, g)
    got = outputs(case, m, g)
    names = [t[0] for t in emu.trace if t is not None]
    assert STEP_OF[case] in names, names
    for key, v in got.items():
        assert sandwich_ok(v, g, key), (key, rel_err(v, g[key + "_fp64"]))


def _out_of_scope():
    """(module, input features, context features or None) that keep the torch path."""
    return [
        (T.MaskedAffineAutoregressiveTransform(8, 64, activation=torch.sigmoid), 8, None),
        (T.MaskedAffineAutoregressiveTransform(8, 64, activation=nn.ELU(alpha=0.5)), 8, None),
        (T.MaskedAffineAutoregressiveTransform(8, 64, activation=nn.GELU(approximate="tanh")), 8, None),
        (T.MaskedAffineAutoregressiveTransform(8, 64, activation=lambda v: torch.tanh(v)), 8, None),
        (T.MaskedAffineAutoregressiveTransform(8, 64, use_residual_blocks=False, random_mask=True, activation=torch.tanh), 8, None),
        (T.MaskedAffineAutoregressiveTransform(8, 64, use_residual_blocks=False, use_batch_norm=True, activation=torch.tanh), 8, None),
        (T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(8, 64, num_bins=8, tails="linear", use_residual_blocks=False,
                                                                  random_mask=True), 8, None),
        (T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(8, 64, context_features=4, num_bins=8, tails="linear",
                                                                  activation=nn.LeakyReLU(0.2)), 8, 4),
        (MADEMoG(5, 64, 7, use_residual_blocks=False, random_mask=True, activation=torch.tanh), 5, 7),
        (MADEMoG(5, 64, 7, activation=torch.sigmoid), 5, 7),
    ]


@torch.no_grad()
def test_out_of_scope_cases_launch_nothing(emu):
    torch.manual_seed(5)
    for m, d, cf in _out_of_scope():
        m.eval()
        x, c = torch.randn(100, d), None if cf is None else torch.randn(100, cf)
        if isinstance(m, MADEMoG):
            m.log_prob(x, context=c)
        else:
            m(x, context=c)
            m.inverse(x, context=c)
        assert emu.trace == [], m
    drop = T.MaskedAffineAutoregressiveTransform(8, 64, use_residual_blocks=False, activation=torch.tanh,
                                                 dropout_probability=0.1).train()
    drop(torch.randn(100, 8))
    assert emu.trace == []
    # conditioners of couplings: no dense chain, so the coupling runs them in torch (its own epilogue stays native)
    assert MLP([4], [8], [64], activation=torch.sigmoid).dense_chain() is None
    assert ResidualNet(4, 8, 64, activation=F.softplus).dense_chain() is None
    assert ResidualNet(4, 8, 64, context_features=3, activation=nn.GELU("tanh")).dense_chain(torch.randn(2, 3)) is None
    with D.image_geometry(1, 4, 4):
        assert ConvResidualNet(4, 8, 16, activation=torch.tanh).eval().dense_chain() is None
        assert ConvResidualNet(4, 8, 16, activation=F.relu).eval().dense_chain() is not None


@torch.no_grad()
def test_switch_off_keeps_the_torch_path(emu, monkeypatch):
    """With config.native_activations off (the default) the new conditioners keep the torch formulation and launch nothing;
    relu under any spelling still runs natively."""
    monkeypatch.setattr(config, "native_activations", False)
    torch.manual_seed(5)
    x, c = torch.randn(100, 16), torch.randn(100, 5)
    for t in [T.MaskedAffineAutoregressiveTransform(16, 64, activation=torch.tanh),
              T.MaskedAffineAutoregressiveTransform(16, 64, use_residual_blocks=False),
              T.MaskedAffineAutoregressiveTransform(16, 50, context_features=5),
              T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(16, 64, context_features=5, num_bins=8, tails="linear",
                                                                      activation=F.gelu)]:
        t.eval()
        ctx = c if t.autoregressive_net._has_context_layers() else None
        y, lad = t(x, context=ctx)
        assert emu.trace == [], t
        want = t._eager(x, ctx, False)
        assert torch.equal(y, want[0]) and torch.equal(lad, want[1])
    assert MixtureOfGaussiansMADE(8, 64, use_residual_blocks=False).dense_chain() is None
    assert ResidualNet(4, 8, 64, activation=F.elu).dense_chain() is None
    assert MLP([4], [8], [64], activation=nn.SiLU()).dense_chain() is None
    for relu in (F.relu, torch.relu, nn.ReLU()):
        t = T.MaskedAffineAutoregressiveTransform(16, 64, activation=relu).eval()
        t(x)
        assert [n for n, _ in emu.trace].count("affine_ar_step") == 1
        del emu.trace[:]


# ---- the entry points' checks of the codes (nothing is launched) -------------------------------------------------------------
@pytest.mark.parametrize("bad", [7, 15, -1])
def test_unknown_activation_codes_are_rejected(bad):
    lib = _native.load()
    rc = lib.nfk_linear(256, 8, 512, 8, 0, 0, 0, 768, 8, 4, 8, 8, bad, 0, None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error()
    rc = lib.nfk_linear(256, 8, 512, 8, 0, 0, 0, 768, 8, 4, 8, 8, 0, bad, None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error()
    rc = lib.nfk_linear_f16x3(256, 256, 8, 0, 512, 512, 8, 0, 0, 0, 0, 768, 8, 0, 0, 0, 0, 0, 0, bad, 0, 4, 8, 8, 0, None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error()
    rc = lib.nfk_linear_f16x3(256, 256, 8, 0, 512, 512, 8, 0, 0, 0, 0, 768, 8, 0, 0, 0, 0, 0, 0, 0, bad, 4, 8, 8, 0, None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error()
    rc = lib.nfk_split_f16(256, 8, 8, bad, 0, 512, 768, 8, 4, 0, None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error()
    rc = lib.nfk_glu_skip_rows(256, 8, 512, 8, 0, 0, 768, 8, 0, 0, 0, 0, bad, 4, 8, 0, None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error()


@pytest.mark.parametrize("field", [7, 15])
def test_unknown_activation_field_of_a_layer_flag_is_rejected(field):
    lib = _native.load()
    d = _native.NfkCouplingStep()
    d.n_rows, d.hidden_features, d.in_features, d.num_square_layers = 10, 64, 16, 1
    d.a_hi = d.a_lo = d.w0_hi = d.w0_lo = d.wt_hi = d.wt_lo = d.bias_trunk = d.workspace = 256
    d.lda, d.ldw0, d.ldwt = 16, 16, 64
    d.wt_exps = (ctypes.c_int32 * 1)(0)
    d.layer_flags = (ctypes.c_int32 * 2)(8, 1 | (field << _native.STEP_ACT_SHIFT))
    d.h_hi = d.h_lo = 512
    d.ldh = 64
    rc = lib.nfk_rq_coupling_step_f16x3(ctypes.byref(d), None)
    assert rc == -1 and b"unknown activation code" in lib.nfk_last_error(), lib.nfk_last_error()
