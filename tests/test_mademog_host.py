"""Mixture-of-Gaussians MADE without a GPU: the torch path and the fp64 oracle (tests/_mademog_oracle.py) against the reference's
outputs (tests/golden/mademog_rows.pt), weights from a seed, constructor errors, the host logic of the native path on the CPU
stand-ins of tests/emulated_kernels.py (route traces included), the argument checks of nfk_mog_made_step_f16x3 and the cases that
stay on the torch path."""
import ctypes

import pytest
import torch

import _mademog_oracle as oracle
import emulated_kernels as EK
from conftest import load_golden, rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.distributions import MADEMoG
from nflows_b200.flows import Flow
from nflows_b200.nn.nde import MixtureOfGaussiansMADE

BLOCK = 128             # config.coupling_block_rows of the emulated runs: 160 rows are two row blocks
CTX_RAW, CTX = 7, 5


def perturb(module, seed):
    """scripts/make_mademog_golden.py: every bias + 0.1 N(0, 1), the residual blocks' second linear + 0.05 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "linear_layers.1" in name:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return module


def checksum(m):
    return float(sum(v.double().abs().sum() for v in m.state_dict().values() if v.is_floating_point()))


def build(case, g):
    """The model of a golden case: its reference state_dict, or (large) re-created from its seed and checked against the
    reference's weight checksum."""
    if case == "sbi":
        m = MADEMoG(5, 50, 7, num_mixture_components=10)
    elif case == "uncond":
        m = MixtureOfGaussiansMADE(8, 64, num_mixture_components=5, custom_initialization=True)
    else:
        torch.manual_seed(g["seed"])
        m = perturb(MADEMoG(64, 256, 16, num_mixture_components=10), g["perturb_seed"])
        assert abs(checksum(m) - g["checksum"]) <= 1e-9 * g["checksum"], "weights from the seed differ from the reference's"
        return m.eval()
    m.load_state_dict(g["state_dict"], strict=True)
    return m.eval()


def golden_flow(g):
    f = g["features"]
    layers = []
    for _ in range(3):
        layers += [T.ReversePermutation(f), T.MaskedAffineAutoregressiveTransform(features=f, hidden_features=64, context_features=CTX)]
    flow = Flow(T.CompositeTransform(layers), MADEMoG(f, 32, CTX, num_mixture_components=3),
                embedding_net=torch.nn.Linear(CTX_RAW, CTX)).eval()
    flow.load_state_dict(g["state_dict"], strict=True)
    return flow


def made_of(m):
    return m._made if isinstance(m, MADEMoG) else m


def call_log_prob(m, x, c):
    return m.log_prob(x, context=c)


CASES = ["sbi", "uncond", "large"]


@torch.no_grad()
@pytest.mark.parametrize("case", CASES)
def test_torch_path_and_oracle_match_the_reference(case):
    g = load_golden("mademog_rows")[case]
    m = build(case, g)
    lp = call_log_prob(m, g["x"], g["context"])
    assert rel_err(lp, g["log_prob"]) <= 1e-6
    sd = made_of(m).state_dict()
    want = oracle.log_prob(sd, g["x"], g["context"], made_of(m).num_mixture_components, prefix="")
    assert rel_err(want, g["log_prob_fp64"]) <= 1e-12
    m.double()
    lp64 = call_log_prob(m, g["x"].double(), None if g["context"] is None else g["context"].double())
    assert rel_err(lp64, g["log_prob_fp64"]) <= 1e-12


@torch.no_grad()
def test_torch_flow_matches_the_reference():
    g = load_golden("mademog_rows")["flow"]
    flow = golden_flow(g)
    assert rel_err(flow.log_prob(g["x"], context=g["context"]), g["log_prob"]) <= 1e-6


@pytest.mark.parametrize("case", ["sbi", "uncond"])
def test_seed_reproduces_the_reference_weights(case):
    g = load_golden("mademog_rows")[case]
    torch.manual_seed(g["seed"])
    m = MADEMoG(5, 50, 7, num_mixture_components=10) if case == "sbi" else MixtureOfGaussiansMADE(8, 64, num_mixture_components=5)
    assert abs(checksum(m) - g["init_checksum"]) <= 1e-9 * g["init_checksum"]
    assert list(m.state_dict()) == list(g["state_dict"])


def test_constructor_errors():
    with pytest.raises(ValueError, match="random masks"):
        MixtureOfGaussiansMADE(4, 32, random_mask=True)
    with pytest.raises(ValueError, match="random masks"):
        MADEMoG(4, 32, 3, random_mask=True)
    m = MixtureOfGaussiansMADE(4, 32, use_residual_blocks=False, random_mask=True)
    assert m.log_prob(torch.randn(3, 4)).shape == (3,)


def test_sample_shape_and_failure_without_context():
    torch.manual_seed(0)
    m = MADEMoG(3, 32, 2, num_mixture_components=2).eval()
    assert m.sample(4, context=torch.randn(5, 2)).shape == (5, 4, 3)
    with pytest.raises(AttributeError):
        m.sample(4)


# ---- host logic on the emulated kernels -------------------------------------------------------------------------------------
@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    monkeypatch.setattr(config, "coupling_block_rows", BLOCK)
    return EK.install(monkeypatch)


def _blocks(n, block=BLOCK):
    return [min(block, n - r0) for r0 in range(0, n, block)]


def expected_log_prob(n, context):
    if not context:
        return [("split_f16", n), ("mog_made_step", n)]
    out = []
    for r in _blocks(n):
        out += [("split_f16", r), ("linear_f16x3", r), ("linear_f16x3", r), ("split_f16", r), ("mog_made_step", r)]
    return out


@torch.no_grad()
@pytest.mark.parametrize("case", ["sbi", "uncond"])
def test_log_prob_on_emulated_kernels(emu, case):
    """One launch per row block; the context terms once per row block; D = 5 and H = 50 run zero padded to 8 and 64."""
    g = load_golden("mademog_rows")[case]
    m = build(case, g)
    call_log_prob(m, g["x"], g["context"])              # the first call also derives the operands
    del emu.trace[:]
    lp = call_log_prob(m, g["x"], g["context"])
    assert rel_err(lp, g["log_prob_fp64"]) <= max(1e-5, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    n = g["x"].shape[0]
    assert emu.trace == expected_log_prob(n, g["context"] is not None)
    if case == "sbi":
        assert set(emu["hidden"]) == {64} and set(emu["in_features"]) == {8}


@torch.no_grad()
def test_flow_on_emulated_kernels(monkeypatch):
    """The flow's MAF-affine layers run on the affine step's stand-in, its base on the mixture step's."""
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    monkeypatch.setattr(config, "coupling_block_rows", BLOCK)
    emu = EK.install(monkeypatch)
    g = load_golden("mademog_rows")["flow"]
    flow = golden_flow(g)
    lp = flow.log_prob(g["x"], context=g["context"])
    assert rel_err(lp, g["log_prob_fp64"]) <= max(1e-5, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    names = [name for name, _ in emu.trace]
    assert names.count("mog_made_step") == len(_blocks(g["x"].shape[0]))


@torch.no_grad()
def test_sample_on_emulated_kernels(emu):
    """D launches per row block on the degree-sorted sub-networks, the context projected once per block; the draws follow the
    oracle's sampler with the same (u, e)."""
    g = load_golden("mademog_rows")["sbi"]
    m = build("sbi", g)
    ctx = g["context"][:40]
    m.sample(1, context=ctx[:2])                        # the first call also derives the operands
    del emu.trace[:]
    torch.manual_seed(3)
    s = m.sample(4, context=ctx)
    assert s.shape == (40, 4, 5)
    rep = ctx.repeat_interleave(4, dim=0)
    torch.manual_seed(3)
    u, e = torch.rand(160, 5), torch.randn(160, 5)
    want, margin = oracle.sample(m._made.state_dict(), u, e, rep, 10, prefix="")
    ok = margin > 1e-5
    assert ok.float().mean() > 0.95
    assert rel_err(s.reshape(160, 5)[ok], want[ok]) <= 1e-5
    per_block = [("split_f16", 128), ("linear_f16x3", 128), ("linear_f16x3", 128)]
    names = [name for name, _ in emu.trace]
    assert names.count("mog_made_step") == 5 * len(_blocks(160))
    assert names.count("linear_f16x3") == 2 * len(_blocks(160))
    assert emu.trace[:3] == per_block
    assert max(emu["hidden"]) == 64


@torch.no_grad()
@pytest.mark.parametrize("features,hidden,num_blocks,components,context", [(1, 32, 0, 1, 3), (8, 96, 1, 16, None), (13, 50, 4, 21, 16)])
def test_shapes_on_emulated_kernels(emu, features, hidden, num_blocks, components, context):
    torch.manual_seed(features + hidden)
    m = perturb(MixtureOfGaussiansMADE(features, hidden, context_features=context, num_blocks=num_blocks,
                                       num_mixture_components=components), 1).eval()
    x = torch.randn(200, features)
    c = None if context is None else torch.randn(200, context)
    want = oracle.log_prob(m.state_dict(), x, c, components, prefix="")
    assert rel_err(m.log_prob(x, context=c), want) <= 1e-5
    assert [n for n, _ in emu.trace].count("mog_made_step") == (len(_blocks(200)) if c is not None else 1)


def _unsupported():
    return [MixtureOfGaussiansMADE(8, 64, activation=torch.tanh), MixtureOfGaussiansMADE(8, 64, use_residual_blocks=False),
            MixtureOfGaussiansMADE(8, 64, use_batch_norm=True), MixtureOfGaussiansMADE(8, 320),
            MixtureOfGaussiansMADE(8, 64, num_blocks=5), MixtureOfGaussiansMADE(8, 64, num_mixture_components=22)]


@torch.no_grad()
def test_unsupported_cases_launch_nothing(emu):
    torch.manual_seed(5)
    x = torch.randn(100, 8)
    for m in _unsupported():
        m.eval()
        lp = m.log_prob(x)
        assert emu.trace == [], m
        assert torch.equal(lp, m._torch_log_prob(x))
    drop = MixtureOfGaussiansMADE(8, 64, dropout_probability=0.1).train()
    drop.log_prob(x)
    assert emu.trace == []
    m = MixtureOfGaussiansMADE(8, 64).eval()
    m.double().log_prob(x.double())
    assert emu.trace == []
    m.float()
    with torch.enable_grad():
        m.log_prob(x)
    assert emu.trace == []
    ctx = MixtureOfGaussiansMADE(8, 64, context_features=CTX).eval()
    ctx.log_prob(x, context=torch.randn(1, CTX))
    assert emu.trace == []


def test_cpu_inputs_take_the_torch_path():
    m = MixtureOfGaussiansMADE(8, 64).eval()
    with torch.no_grad():
        assert not m._native_ready(torch.randn(10, 8), None)


# ---- the C entry point's checks (nothing is launched) -----------------------------------------------------------------------
def _descriptor(n_rows=0, **kw):
    d = _native.NfkCouplingStep()
    d.n_rows, d.hidden_features, d.in_features, d.num_square_layers = n_rows, 64, 16, 4
    d.d_t, d.t_col0, d.ldx, d.ldy, d.x, d.lad_accum = 4, 0, 16, 16, 256, 512
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _mog(**kw):
    g = _native.NfkMogArgs(5, _native.MOG_LOG_PROB, 1e-2)
    for k, v in kw.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("fields,mog,message", [
    (dict(), dict(num_components=0), b"num_components=0"),
    (dict(), dict(num_components=22), b"num_components=22"),
    (dict(), dict(epsilon=0.0), b"epsilon"),
    (dict(), dict(mode=2), b"mode=2"),
    (dict(), dict(u=256, e=256), b"no noise"),
    (dict(y=256), dict(), b"no noise"),
    (dict(lad_accum=0), dict(), b"needs x and lad_accum"),
    (dict(t_col0=14), dict(), b"exceed the row pitch"),
    (dict(t_cols=256), dict(), b"t_cols NULL"),
    (dict(y_hi=256, y_lo=512), dict(), b"fp32 outputs only"),
    (dict(h_hi=256), dict(), b"trunk-only"),
    (dict(y=256), dict(mode=_native.MOG_SAMPLE), b"needs y and the noise"),
    (dict(y=256), dict(mode=_native.MOG_SAMPLE, u=256, e=256, ld_noise=4), b"lad_accum must be NULL"),
    (dict(y=256, lad_accum=0), dict(mode=_native.MOG_SAMPLE, u=256, e=256, ld_noise=2), b"ld_noise=2"),
    (dict(n_rows=-1), dict(), b"bad sizes"),
])
def test_mog_step_arguments_are_checked_before_any_launch(fields, mog, message):
    lib = _native.load()
    rc = lib.nfk_mog_made_step_f16x3(ctypes.byref(_descriptor(**fields)), None, ctypes.byref(_mog(**mog)), None)
    assert rc == -1 and message in lib.nfk_last_error(), lib.nfk_last_error()


def test_mog_step_row_terms_and_shape_are_checked():
    lib = _native.load()
    terms = _native.NfkStepRowTerms()
    terms.layer[5].add, terms.layer[5].ld = 256, 64
    rc = lib.nfk_mog_made_step_f16x3(ctypes.byref(_descriptor()), ctypes.byref(terms), ctypes.byref(_mog()), None)
    assert rc == -1 and b"row term on layer 5" in lib.nfk_last_error()
    assert lib.nfk_mog_made_step_f16x3(ctypes.byref(_descriptor()), None, ctypes.byref(_mog()), None) == 0   # empty batch
    for fields in (dict(hidden_features=48), dict(in_features=5), dict(num_square_layers=9)):
        rc = lib.nfk_mog_made_step_f16x3(ctypes.byref(_descriptor(n_rows=10, **fields)), None, ctypes.byref(_mog()), None)
        assert rc == -1 and b"does not take" in lib.nfk_last_error(), fields


def test_padded_rows_per_component_count():
    got = [K.mog_made_padded_rows(c) for c in range(0, _native.MOG_MAX_COMPONENTS + 2)]
    assert got[0] == 0 and got[-1] == 0
    for c in range(1, _native.MOG_MAX_COMPONENTS + 1):
        assert got[c] >= 3 * c and got[c] % 8 == 0 and got[c] <= 64 and got[c] != 40
