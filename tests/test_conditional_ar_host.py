"""Context-conditioned masked autoregressive spline transforms without a GPU: the package's torch path against the reference's
outputs (tests/golden/conditional_ar_rows.pt), the host logic of the native path on the CPU stand-ins of
tests/emulated_kernels.py, and the argument checks of the C entry point."""
import ctypes

import pytest
import torch

import emulated_kernels as EK
from conftest import load_golden, rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.distributions.normal import StandardNormal
from nflows_b200.flows import Flow, recipes

FEATURES, CTX_RAW, CTX = 16, 7, 5
BLOCK = 128             # config.coupling_block_rows of the emulated runs (its smallest value): 200 rows are two row blocks


def maf(tails, features=FEATURES, hidden=64, context=CTX, num_blocks=2):
    kw = dict(tails="linear", tail_bound=3.0) if tails == "linear" else dict(tails=None)
    return T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=features, hidden_features=hidden,
                                                                    context_features=context, num_bins=8, num_blocks=num_blocks, **kw)


def sharpen(module, seed):
    """Give the residual blocks' zero-initialised second linear some weight, so the block context terms show in the outputs (what
    scripts/make_conditional_ar_golden.py does to the reference's modules)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "linear_layers.1" in name:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return module


def _from_seed(g, build):
    """The fixture's module re-created from its seed (the constructors consume the torch CPU RNG as the reference's do), perturbed
    and sharpened as the generator did, and checked against the reference's weight checksum."""
    torch.manual_seed(g["seed"])
    m = sharpen(recipes.perturb_(build().eval()), g["sharpen_seed"])
    ck = float(sum(v.double().abs().sum() for v in m.state_dict().values() if v.is_floating_point()))
    if abs(ck - g["checksum"]) > 1e-9 * abs(g["checksum"]):
        pytest.fail("weights re-created from the seed do not match the fixture's checksum (torch CPU RNG stream changed?): "
                    "regenerate it with scripts/make_conditional_ar_golden.py against the reference")
    return m


def golden_flow(g):
    return _from_seed(g, lambda: Flow(
        T.CompositeTransform([T.RandomPermutation(FEATURES), maf("linear"), T.RandomPermutation(FEATURES), maf("linear")]),
        StandardNormal([FEATURES]), embedding_net=torch.nn.Linear(CTX_RAW, CTX)))


def golden_transform(g):
    return _from_seed(g, lambda: maf(None))


@torch.no_grad()
def test_torch_path_matches_the_reference():
    g = load_golden("conditional_ar_rows")
    lin = g["linear"]
    flow = golden_flow(lin)
    assert rel_err(flow.log_prob(lin["x"], context=lin["context"]), lin["log_prob"]) <= 1e-6
    e = flow._embedding_net(lin["context"])
    z, lad = flow._transform(lin["x"], context=e)
    assert rel_err(z, lin["z"]) <= 1e-6 and rel_err(lad, lin["lad"]) <= 1e-6
    xs, lad_inv = flow._transform.inverse(lin["noise"], context=e)
    assert rel_err(xs, lin["sample"]) <= 1e-6 and rel_err(lad_inv, lin["lad_inv"]) <= 1e-6
    none = g["none"]
    t = golden_transform(none)
    y, lad = t(none["x"], context=none["context"])
    assert rel_err(y, none["y"]) <= 1e-6 and rel_err(lad, none["lad"]) <= 1e-6
    xi, li = t.inverse(none["x"], context=none["context"])
    assert rel_err(xi, none["xinv"]) <= 1e-6 and rel_err(li, none["ladinv"]) <= 1e-6


# ---- host logic on the emulated kernels -------------------------------------------------------------------------------------
@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    monkeypatch.setattr(config, "coupling_block_rows", BLOCK)
    return EK.install(monkeypatch)


def _traced(emu, fn, *args, **kw):
    fn(*args, **kw)
    del emu.trace[:]
    return fn(*args, **kw), list(emu.trace)


def _blocks(n, block=BLOCK):
    return [min(block, n - r0) for r0 in range(0, n, block)]


def expected_forward(n):
    out = []
    for r in _blocks(n):
        out += [("split_f16", r), ("linear_f16x3", r), ("linear_f16x3", r), ("split_f16", r), ("rq_coupling_step", r)]
    return out


def expected_inverse(n, d):
    out = []
    for r in _blocks(n):
        out += [("split_f16", r), ("linear_f16x3", r), ("linear_f16x3", r)]
        out += [("rq_coupling_step", r), ("split_f16", r)] * (d - 1) + [("rq_coupling_step", r)]
    return out


@torch.no_grad()
def test_conditional_transform_on_emulated_kernels(emu):
    """Forward: per row block the context pair, the two projection GEMMs and one step launch.  Inverse: per row block the same
    two GEMMs, then one launch per feature."""
    g = load_golden("conditional_ar_rows")["none"]
    t = golden_transform(g)
    x, c = g["x"], g["context"]
    (y, lad), fwd = _traced(emu, t, x, context=c)
    assert rel_err(y, g["y_fp64"]) <= max(1e-5, 3 * rel_err(g["y"], g["y_fp64"]))
    # the perturbed, sharpened weights make sharp splines: one row's log|det| carries ~1e-4 of the split-pair conditioner's
    # round-off (fp64 context terms in its place change nothing), hence the floor -- the shape sweep's
    assert rel_err(lad, g["lad_fp64"]) <= max(3e-4, 3 * rel_err(g["lad"], g["lad_fp64"]))
    (xi, li), inv = _traced(emu, t.inverse, x, context=c)
    assert rel_err(xi, g["xinv_fp64"]) <= max(1e-4, 3 * rel_err(g["xinv"], g["xinv_fp64"]))
    assert rel_err(li, g["ladinv_fp64"]) <= max(1e-3, 3 * rel_err(g["ladinv"], g["ladinv_fp64"]))
    assert fwd == expected_forward(x.shape[0])
    assert inv == expected_inverse(x.shape[0], FEATURES)


@torch.no_grad()
def test_conditional_flow_on_emulated_kernels(emu):
    g = load_golden("conditional_ar_rows")["linear"]
    flow = golden_flow(g)
    lp, fwd = _traced(emu, flow.log_prob, g["x"], context=g["context"])
    assert rel_err(lp, g["log_prob_fp64"]) <= max(3e-5, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    e = flow._embedding_net(g["context"])
    (xs, lad_inv), inv = _traced(emu, flow._transform.inverse, g["noise"], context=e)
    assert rel_err(xs, g["sample_fp64"]) <= max(1e-4, 3 * rel_err(g["sample"], g["sample_fp64"]))
    assert rel_err(lad_inv, g["lad_inv_fp64"]) <= max(1e-3, 3 * rel_err(g["lad_inv"], g["lad_inv_fp64"]))
    blocks = len(_blocks(g["x"].shape[0]))
    for trace, steps in ((fwd, 2 * blocks), (inv, 2 * blocks * FEATURES)):
        names = [name for name, _ in trace]
        assert names.count("linear_f16x3") == 2 * 2 * blocks     # two projections per row block of each transform
        assert names.count("rq_coupling_step") == steps


@torch.no_grad()
@pytest.mark.parametrize("features,num_blocks", [(8, 1), (24, 2), (40, 0)])
def test_projection_count_does_not_scale_with_features(emu, features, num_blocks):
    torch.manual_seed(features)
    t = maf("linear", features=features, hidden=96, context=11, num_blocks=num_blocks).eval()
    x, c = torch.randn(200, features), torch.randn(200, 11)
    want = [v.float() for v in t.double()(x.double(), context=c.double())]
    t.float()
    (y, lad), fwd = _traced(emu, t, x, context=c)
    assert rel_err(y, want[0]) <= 1e-4 and rel_err(lad, want[1]) <= 1e-4
    _, inv = _traced(emu, t.inverse, y, context=c)
    gemms = 2 if num_blocks else 1
    for trace, steps in ((fwd, 1), (inv, features)):
        names = [name for name, _ in trace]
        blocks = len(_blocks(200))
        assert names.count("linear_f16x3") == gemms * blocks and names.count("rq_coupling_step") == steps * blocks


@torch.no_grad()
def test_context_net_without_context_runs_the_plain_chain(emu):
    """A MADE with context layers called without a context: the plain chain, no projections (the reference skips the terms)."""
    torch.manual_seed(3)
    t = maf("linear").eval()
    x = torch.randn(100, FEATURES)
    want = [v.float() for v in t.double()(x.double())]
    t.float()
    (y, lad), fwd = _traced(emu, t, x)
    assert rel_err(y, want[0]) <= 1e-4 and rel_err(lad, want[1]) <= 1e-4
    assert fwd == [("split_f16", 100), ("rq_coupling_step", 100)]


@torch.no_grad()
def test_unsupported_context_cases_stay_on_the_torch_path(emu):
    torch.manual_seed(4)
    t = maf("linear").eval()
    x = torch.randn(100, FEATURES)
    t(x, context=torch.randn(1, CTX))                     # broadcasts in the torch formulation
    assert emu.trace == []
    with pytest.raises(RuntimeError):
        t(x, context=torch.randn(99, CTX))
    plain = maf("linear", context=None).eval()            # a context without context layers
    with pytest.raises(AttributeError):
        plain(x, context=torch.randn(100, CTX))
    tanh = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(
        features=FEATURES, hidden_features=64, context_features=CTX, num_bins=8, tails="linear", activation=torch.tanh).eval()
    tanh(x, context=torch.randn(100, CTX))
    assert emu.trace == []


# ---- the C entry point's checks (nothing is launched) -----------------------------------------------------------------------
def _descriptor(n_rows=0, hidden=64, square_layers=4):
    d = _native.NfkCouplingStep()
    d.n_rows, d.hidden_features, d.in_features, d.num_square_layers = n_rows, hidden, 16, square_layers
    return d


@pytest.mark.parametrize("layer,ld,addr,message", [
    (5, 64, 256, b"row term on layer 5"),
    (8, 64, 256, b"row term on layer 8"),
    (0, 32, 256, b"less than the hidden width"),
    (1, 65, 256, b"8-byte aligned"),
    (3, 64, 260, b"8-byte aligned"),
])
def test_row_term_arguments_are_checked_before_any_launch(layer, ld, addr, message):
    lib = _native.load()
    terms = _native.NfkStepRowTerms()
    terms.layer[layer].add, terms.layer[layer].ld = addr, ld
    rc = lib.nfk_rq_coupling_step_terms_f16x3(ctypes.byref(_descriptor()), ctypes.byref(terms), None)
    assert rc == -1 and message in lib.nfk_last_error()


def test_valid_row_terms_on_an_empty_batch_are_a_no_op():
    lib = _native.load()
    terms = _native.NfkStepRowTerms()
    for l in (0, 1, 3):
        terms.layer[l].add, terms.layer[l].ld = 256 * (l + 1), 128
    assert lib.nfk_rq_coupling_step_terms_f16x3(ctypes.byref(_descriptor()), ctypes.byref(terms), None) == 0
    assert lib.nfk_rq_coupling_step_terms_f16x3(ctypes.byref(_descriptor()), None, None) == 0
    d = _descriptor()
    d.h_hi = 256
    rc = lib.nfk_rq_coupling_step_terms_f16x3(ctypes.byref(d), ctypes.byref(terms), None)
    assert rc == -1 and b"trunk-only" in lib.nfk_last_error()
