"""Masked affine autoregressive transforms without a GPU: the torch path against the reference's outputs
(tests/golden/maf_affine_rows.pt), the host logic of the native path on the CPU stand-ins of tests/emulated_kernels.py (route
traces included), the argument checks of nfk_affine_ar_step_f16x3 and the cases that stay on the torch path."""
import ctypes

import pytest
import torch

import emulated_kernels as EK
from conftest import load_golden, rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.distributions.normal import StandardNormal
from nflows_b200.flows import Flow

CTX_RAW, CTX = 7, 5
BLOCK = 128             # config.coupling_block_rows of the emulated runs (its smallest value): 160 rows are two row blocks


def perturb(module, seed):
    """scripts/make_maf_affine_golden.py: every bias + 0.1 N(0, 1), the residual blocks' second linear + 0.05 N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if name.endswith(".bias"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "linear_layers.1" in name:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return module


def maf(features, hidden, context=None, num_blocks=2, **kw):
    return T.MaskedAffineAutoregressiveTransform(features=features, hidden_features=hidden, context_features=context,
                                                 num_blocks=num_blocks, **kw)


def golden_transform(g):
    """The fixture's transform: its stored reference state_dict, or (cfg4) re-created from its seed and checked against the
    reference's weight checksum."""
    if "state_dict" in g:
        t = maf(g["features"], g["hidden"]).eval()
        t.load_state_dict(g["state_dict"], strict=True)
        return t
    torch.manual_seed(g["seed"])
    t = perturb(maf(g["features"], g["hidden"]).eval(), g["perturb_seed"])
    ck = float(sum(v.double().abs().sum() for v in t.state_dict().values() if v.is_floating_point()))
    if abs(ck - g["checksum"]) > 1e-9 * abs(g["checksum"]):
        pytest.fail("weights re-created from the seed do not match the fixture's checksum (torch CPU RNG stream changed?): "
                    "regenerate it with scripts/make_maf_affine_golden.py against the reference")
    return t


def golden_flow(g):
    f = g["features"]
    layers = []
    for _ in range(3):
        layers += [T.ReversePermutation(f), maf(f, 64, context=CTX)]
    flow = Flow(T.CompositeTransform(layers), StandardNormal([f]), embedding_net=torch.nn.Linear(CTX_RAW, CTX)).eval()
    flow.load_state_dict(g["state_dict"], strict=True)
    return flow


TRANSFORM_CASES = ["single", "small", "cfg4"]


@torch.no_grad()
@pytest.mark.parametrize("case", TRANSFORM_CASES)
def test_torch_path_matches_the_reference(case):
    g = load_golden("maf_affine_rows")[case]
    t = golden_transform(g)
    y, lad = t(g["x"])
    assert rel_err(y, g["y"]) <= 1e-6 and rel_err(lad, g["lad"]) <= 1e-6
    xi, li = t.inverse(g["x"])
    assert rel_err(xi, g["xinv"]) <= 1e-6 and rel_err(li, g["ladinv"]) <= 1e-6
    t.double()
    y64, lad64 = t(g["x"].double())
    xi64, li64 = t.inverse(g["x"].double())
    for got, want in ((y64, "y_fp64"), (lad64, "lad_fp64"), (xi64, "xinv_fp64"), (li64, "ladinv_fp64")):
        assert rel_err(got, g[want]) <= 1e-12, want


@torch.no_grad()
def test_torch_flow_matches_the_reference():
    g = load_golden("maf_affine_rows")["flow"]
    flow = golden_flow(g)
    assert rel_err(flow.log_prob(g["x"], context=g["context"]), g["log_prob"]) <= 1e-6
    e = flow._embedding_net(g["context"])
    z, lad = flow._transform(g["x"], context=e)
    assert rel_err(z, g["z"]) <= 1e-6 and rel_err(lad, g["lad"]) <= 1e-6
    xs, lad_inv = flow._transform.inverse(g["noise"], context=e)
    assert rel_err(xs, g["sample"]) <= 1e-6 and rel_err(lad_inv, g["lad_inv"]) <= 1e-6


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


def expected_forward(n, context):
    if not context:
        return [("split_f16", n), ("affine_ar_step", n)]
    out = []
    for r in _blocks(n):
        out += [("split_f16", r), ("linear_f16x3", r), ("linear_f16x3", r), ("split_f16", r), ("affine_ar_step", r)]
    return out


def expected_inverse(n, d, context):
    out = []
    for r in (_blocks(n) if context else [n]):
        if context:
            out += [("split_f16", r), ("linear_f16x3", r), ("linear_f16x3", r)]
        out += [("affine_ar_step", r), ("split_f16", r)] * (d - 1) + [("affine_ar_step", r)]
    return out


def sandwich(got, g, key, floor):
    return rel_err(got, g[key + "_fp64"]) <= max(floor, 3 * rel_err(g[key], g[key + "_fp64"]))


@torch.no_grad()
@pytest.mark.parametrize("case", TRANSFORM_CASES)
def test_transform_on_emulated_kernels(emu, case):
    """Forward: the input pair and one step launch.  Inverse: one launch per feature, a column split between them."""
    g = load_golden("maf_affine_rows")[case]
    t = golden_transform(g)
    x = g["x"]
    (y, lad), fwd = _traced(emu, t, x)
    assert sandwich(y, g, "y", 1e-5) and sandwich(lad, g, "lad", 1e-5)
    (xi, li), inv = _traced(emu, t.inverse, x)
    assert sandwich(xi, g, "xinv", 1e-4) and sandwich(li, g, "ladinv", 1e-4)
    assert fwd == expected_forward(x.shape[0], False)
    assert inv == expected_inverse(x.shape[0], g["features"], False)


@torch.no_grad()
def test_flow_on_emulated_kernels(emu):
    """The conditional flow: per row block of each transform one context projection (two GEMMs), then its launches."""
    g = load_golden("maf_affine_rows")["flow"]
    flow = golden_flow(g)
    d = g["features"]
    lp, fwd = _traced(emu, flow.log_prob, g["x"], context=g["context"])
    assert rel_err(lp, g["log_prob_fp64"]) <= max(1e-5, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    e = flow._embedding_net(g["context"])
    (z, lad), fwd_t = _traced(emu, flow._transform, g["x"], context=e)
    assert sandwich(z, g, "z", 1e-5) and sandwich(lad, g, "lad", 1e-5)
    n = g["x"].shape[0]
    assert fwd_t == ([("gather_cols", n)] + expected_forward(n, True)) * 3            # the permutations are column gathers
    (xs, lad_inv), inv = _traced(emu, flow._transform.inverse, g["noise"], context=e)
    assert sandwich(xs, g, "sample", 1e-4) and sandwich(lad_inv, g, "lad_inv", 1e-4)
    assert inv == (expected_inverse(n, d, True) + [("gather_cols", n)]) * 3
    names = [name for name, _ in fwd]
    assert names.count("affine_ar_step") == 3 * len(_blocks(g["x"].shape[0]))


@torch.no_grad()
@pytest.mark.parametrize("features,hidden,num_blocks,context", [(5, 32, 0, None), (13, 96, 1, 16), (8, 256, 4, 5), (2, 32, 2, 5)])
def test_shapes_on_emulated_kernels(emu, features, hidden, num_blocks, context):
    torch.manual_seed(features + hidden)
    t = perturb(maf(features, hidden, context=context, num_blocks=num_blocks).eval(), 1)
    x = torch.randn(200, features)
    c = None if context is None else torch.randn(200, context)
    t64 = maf(features, hidden, context=context, num_blocks=num_blocks).double().eval()
    t64.load_state_dict(t.state_dict())
    want = t64(x.double(), context=None if c is None else c.double())
    (y, lad), fwd = _traced(emu, t, x, context=c)
    assert rel_err(y, want[0]) <= 1e-5 and rel_err(lad, want[1]) <= 1e-5
    want_inv = t64.inverse(x.double(), context=None if c is None else c.double())
    (xi, li), inv = _traced(emu, t.inverse, x, context=c)
    assert rel_err(xi, want_inv[0]) <= 1e-4 and rel_err(li, want_inv[1]) <= 1e-4
    assert fwd == expected_forward(200, c is not None) if num_blocks else [n for n, _ in fwd].count("affine_ar_step") >= 1
    assert [n for n, _ in inv].count("affine_ar_step") == features * (len(_blocks(200)) if c is not None else 1)


@torch.no_grad()
def test_padded_initial_weight_follows_the_parameters(emu):
    """D = 5: the initial layer's weight is padded to 8 columns once per parameter version."""
    torch.manual_seed(0)
    t = perturb(maf(5, 32).eval(), 2)
    x = torch.randn(50, 5)
    w0 = lambda: t.autoregressive_net._padded_chain[1][0][0]
    t(x)
    first = w0()
    t(x)
    assert w0() is first and first.shape == (32, 8) and torch.equal(first[:, 5:], torch.zeros(32, 3))
    with torch.no_grad():
        t.autoregressive_net.initial_layer.weight.mul_(2.0)
    y, _ = t(x)
    assert w0() is not first
    assert rel_err(y, t._eager(x, None, False)[0]) <= 1e-5


def _unsupported():
    return [maf(16, 64, activation=torch.tanh), maf(16, 64, use_residual_blocks=False), maf(16, 64, use_batch_norm=True),
            maf(16, 48), maf(16, 320), maf(16, 64, num_blocks=5)]


@torch.no_grad()
def test_unsupported_cases_launch_nothing(emu):
    torch.manual_seed(5)
    x = torch.randn(100, 16)
    for t in _unsupported():
        t.eval()
        y, lad = t(x)
        t.inverse(x)
        assert emu.trace == [], type(t)
        want = t._eager(x, None, False)
        assert torch.equal(y, want[0]) and torch.equal(lad, want[1])
    drop = maf(16, 64, dropout_probability=0.1).train()
    drop(x)
    assert emu.trace == []
    t = maf(16, 64).eval()
    t.double()(x.double())                                          # fp64
    assert emu.trace == []
    t.float()
    with torch.enable_grad():                                       # autograd: the parameters need a gradient
        t(x)
    assert emu.trace == []
    ctx = maf(16, 64, context=CTX).eval()
    ctx(x, context=torch.randn(1, CTX))                             # a context of another batch size broadcasts
    assert emu.trace == []


def test_cpu_inputs_take_the_torch_path():
    t = maf(16, 64).eval()
    with torch.no_grad():
        assert not t._native_ready(torch.randn(10, 16), None)


# ---- the C entry point's checks (nothing is launched) -----------------------------------------------------------------------
def _descriptor(n_rows=0, d_t=4, **kw):
    d = _native.NfkCouplingStep()
    d.n_rows, d.hidden_features, d.in_features, d.num_square_layers = n_rows, 64, 16, 4
    d.d_t, d.t_col0, d.ldx, d.ldy, d.y = d_t, 0, 16, 16, 256
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("fields,message", [
    (dict(h_hi=256), b"trunk-only"),
    (dict(d_t=0), b"d_t=0"),
    (dict(t_cols=256), b"t_cols NULL"),
    (dict(t_col0=-1), b"t_cols NULL"),
    (dict(t_col0=14), b"exceed the row pitch"),
    (dict(ldy=3), b"exceed the row pitch"),
    (dict(y=0), b"fp32 outputs only"),
    (dict(y_hi=256, y_lo=512), b"fp32 outputs only"),
    (dict(n_rows=-1), b"bad sizes"),
])
def test_affine_step_arguments_are_checked_before_any_launch(fields, message):
    lib = _native.load()
    rc = lib.nfk_affine_ar_step_f16x3(ctypes.byref(_descriptor(**fields)), None, None)
    assert rc == -1 and message in lib.nfk_last_error()


@pytest.mark.parametrize("layer,ld,message", [(5, 64, b"row term on layer 5"), (0, 32, b"less than the hidden width"),
                                              (1, 65, b"8-byte aligned")])
def test_affine_step_row_terms_are_checked(layer, ld, message):
    lib = _native.load()
    terms = _native.NfkStepRowTerms()
    terms.layer[layer].add, terms.layer[layer].ld = 256, ld
    rc = lib.nfk_affine_ar_step_f16x3(ctypes.byref(_descriptor()), ctypes.byref(terms), None)
    assert rc == -1 and message in lib.nfk_last_error()


def test_affine_step_on_an_empty_batch_is_a_no_op():
    lib = _native.load()
    terms = _native.NfkStepRowTerms()
    terms.layer[0].add, terms.layer[0].ld = 256, 64
    assert lib.nfk_affine_ar_step_f16x3(ctypes.byref(_descriptor()), ctypes.byref(terms), None) == 0
    assert lib.nfk_affine_ar_step_f16x3(ctypes.byref(_descriptor()), None, None) == 0


def test_affine_step_shape_is_checked():
    lib = _native.load()
    for fields in (dict(hidden_features=48), dict(in_features=5), dict(num_square_layers=9)):
        d = _descriptor(n_rows=10, **fields)
        rc = lib.nfk_affine_ar_step_f16x3(ctypes.byref(d), None, None)
        assert rc == -1 and b"does not take" in lib.nfk_last_error(), fields
