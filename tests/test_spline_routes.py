"""Which kernel wrappers every spline-head route runs, in order and on how many rows, with the coupling-step kernel on (the
default): the step route (one launch for conditioner + spline), the final route (trunk, then the fused last layer + spline), the
rows route (trunk, last layer into HBM, `rqs_rows`), the gathered column path, plain-module conditioners, affine couplings and the
autoregressive passes.  Host logic only: the wrappers are the CPU stand-ins of tests/emulated_kernels.py, and every result is
also checked against the fp64 torch formulation."""
import pytest
import torch

import emulated_kernels
from conftest import load_golden, rel_err
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.flows import recipes
from nflows_b200.nn.nets import ResidualNet
from nflows_b200.utils import torchutils

TOL = 1e-5


def calls(spec):
    """'name:rows name:rows ...' -> [(name, rows), ...]"""
    return [(t.split(":")[0], int(t.split(":")[1])) for t in spec.split()]


class _PlainConditioner(torch.nn.Module):
    """A conditioner the dense-chain planner does not know: its output goes to `rqs_rows` as it is."""

    def __init__(self, i, o):
        super().__init__()
        self.layer = torch.nn.Linear(i, o)

    def forward(self, inputs, context=None):
        return self.layer(torch.tanh(inputs))


def _resnet(hidden):
    return lambda i, o: ResidualNet(i, o, hidden_features=hidden, num_blocks=2)


def _coupling(mask, hidden=32, **kw):
    kw = dict(dict(num_bins=8, tails="linear", tail_bound=3.0), **kw)
    return T.PiecewiseRationalQuadraticCouplingTransform(torch.as_tensor(mask), kw.pop("net", None) or _resnet(hidden), **kw)


_alt = torchutils.create_alternating_binary_mask
# name -> () -> (transform, input features); every case runs on 300 rows in row blocks of 128
CASES = {
    "nsf_step": lambda: (recipes.rq_nsf(32, hidden_features=32, num_layers=3)._transform, 32),
    "nsf_final": lambda: (recipes.rq_nsf(32, hidden_features=40, num_layers=3)._transform, 32),
    "nsf_rows": lambda: (recipes.rq_nsf(32, hidden_features=32, num_layers=3, num_bins=6)._transform, 32),
    "gathered_final": lambda: (_coupling([0] * 8 + [1] * 12), 20),
    "rows_ffma": lambda: (_coupling(_alt(20)), 20),
    "unconditional": lambda: (_coupling(_alt(16), apply_unconditional_transform=True), 16),
    "plain_module": lambda: (_coupling(_alt(16), net=_PlainConditioner), 16),
    "affine": lambda: (T.AffineCouplingTransform(_alt(48), _resnet(64)), 48),
    "affine_gathered": lambda: (T.AffineCouplingTransform(torch.tensor([0] * 8 + [1] * 12), _resnet(64)), 20),
    "additive": lambda: (T.AdditiveCouplingTransform(_alt(48), _resnet(64)), 48),
    "additive_user_activation": lambda: (T.AdditiveCouplingTransform(_alt(48), _resnet(64),
                                                                     scale_activation=lambda v: torch.sigmoid(v) + 0.5), 48),
    # 10 identity features: FFMA trunk, last layer into HBM, affine_coupling_rows with the scale and its log|det|
    "affine_rows_general": lambda: (T.AffineCouplingTransform(_alt(20), _resnet(64),
                                                              scale_activation=T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION), 20),
    # a scale activation without a kernel: the torch formulation, no native call
    "affine_user_activation": lambda: (T.AffineCouplingTransform(_alt(48), _resnet(64),
                                                                 scale_activation=lambda v: torch.sigmoid(v) + 0.5), 48),
    "ar_rows": lambda: (T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=8, hidden_features=32, num_bins=6,
                                                                                  tails="linear", tail_bound=3.0), 8),
}


# (forward, inverse) call traces
EXPECTED = {
    "additive": (
        calls("gather_cols:300 split_f16:300") +
        calls("trunk_step:128 affine_coupling_final:128") * 2 +
        calls("trunk_step:44 affine_coupling_final:44 gather_cols:300"),
        calls("gather_cols:300 split_f16:300") +
        calls("trunk_step:128 affine_coupling_final:128") * 2 +
        calls("trunk_step:44 affine_coupling_final:44 gather_cols:300"),
    ),
    "additive_user_activation": (
        calls("gather_cols:300 split_f16:300 trunk_step:300 linear_f16x3:300 affine_coupling_rows:300"),
        calls("gather_cols:300 split_f16:300 trunk_step:300 linear_f16x3:300 affine_coupling_rows:300"),
    ),
    "affine": (
        calls("gather_cols:300 split_f16:300") +
        calls("trunk_step:128 affine_coupling_final:128") * 2 +
        calls("trunk_step:44 affine_coupling_final:44 gather_cols:300"),
        calls("gather_cols:300 split_f16:300") +
        calls("trunk_step:128 affine_coupling_final:128") * 2 +
        calls("trunk_step:44 affine_coupling_final:44 gather_cols:300"),
    ),
    "affine_gathered": (
        calls("gather_cols:300") +
        calls("gather_cols:128 split_f16:128 trunk_step:128 affine_coupling_final:128") * 2 +
        calls("gather_cols:44 split_f16:44 trunk_step:44 affine_coupling_final:44"),
        calls("gather_cols:300") +
        calls("gather_cols:128 split_f16:128 trunk_step:128 affine_coupling_final:128") * 2 +
        calls("gather_cols:44 split_f16:44 trunk_step:44 affine_coupling_final:44"),
    ),
    "affine_rows_general": (
        calls("gather_cols:300") + calls("linear:300") * 6 + calls("affine_coupling_rows:300"),
        calls("gather_cols:300") + calls("linear:300") * 6 + calls("affine_coupling_rows:300"),
    ),
    "affine_user_activation": ([], []),
    "ar_rows": (
        calls("split_f16:300 trunk_step:300 linear_f16x3:300 rqs_rows:300"),
        calls("split_f16:300 trunk_step:300 linear_f16x3:300 rqs_rows:300") * 8,
    ),
    "ar_step": (
        calls("split_f16:96 rq_coupling_step:96"),
        calls("rq_coupling_step:96 split_f16:96") * 63 +
        calls("rq_coupling_step:96"),
    ),
    "context_flow": (
        calls("split_f16:300 linear_f16x3:300") +
        calls("split_f16:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 "
              "glu_skip:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 glu_skip:128 rq_coupling_final:128") * 2 +
        calls("split_f16:44") +
        calls("linear_f16x3:44") * 5 +
        calls("glu_skip:44") +
        calls("linear_f16x3:44") * 3 +
        calls("glu_skip:44 rq_coupling_final:44 linear_f16x3:300") +
        calls("split_f16:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 "
              "glu_skip:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 glu_skip:128 rq_coupling_final:128") * 2 +
        calls("split_f16:44") +
        calls("linear_f16x3:44") * 5 +
        calls("glu_skip:44") +
        calls("linear_f16x3:44") * 3 +
        calls("glu_skip:44 rq_coupling_final:44 linear_f16x3:300") +
        calls("split_f16:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 "
              "glu_skip:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 glu_skip:128 rq_coupling_final:128") * 2 +
        calls("split_f16:44") +
        calls("linear_f16x3:44") * 5 +
        calls("glu_skip:44") +
        calls("linear_f16x3:44") * 3 +
        calls("glu_skip:44 rq_coupling_final:44 gather_cols:300"),
        calls("gather_cols:300 split_f16:300") +
        calls("split_f16:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 "
              "glu_skip:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 glu_skip:128 rq_coupling_final:128") * 2 +
        calls("split_f16:44") +
        calls("linear_f16x3:44") * 5 +
        calls("glu_skip:44") +
        calls("linear_f16x3:44") * 3 +
        calls("glu_skip:44 rq_coupling_final:44 linear_f16x3:300") +
        calls("split_f16:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 "
              "glu_skip:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 glu_skip:128 rq_coupling_final:128") * 2 +
        calls("split_f16:44") +
        calls("linear_f16x3:44") * 5 +
        calls("glu_skip:44") +
        calls("linear_f16x3:44") * 3 +
        calls("glu_skip:44 rq_coupling_final:44 linear_f16x3:300") +
        calls("split_f16:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 "
              "glu_skip:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 glu_skip:128 rq_coupling_final:128") * 2 +
        calls("split_f16:44") +
        calls("linear_f16x3:44") * 5 +
        calls("glu_skip:44") +
        calls("linear_f16x3:44") * 3 +
        calls("glu_skip:44 rq_coupling_final:44 linear_f16x3:300"),
    ),
    "gathered_final": (
        calls("gather_cols:300") +
        calls("gather_cols:128 split_f16:128 trunk_step:128 rq_coupling_final:128") * 2 +
        calls("gather_cols:44 split_f16:44 trunk_step:44 rq_coupling_final:44"),
        calls("gather_cols:300") +
        calls("gather_cols:128 split_f16:128 trunk_step:128 rq_coupling_final:128") * 2 +
        calls("gather_cols:44 split_f16:44 trunk_step:44 rq_coupling_final:44"),
    ),
    "image_flow": (
        calls("nchw_to_rows:1536 squeeze_rows:1536 linear:384 gather_cols:384") +
        calls("gather_cols:128 split_f16:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 "
              "linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 rq_coupling_final:128") * 3 +
        calls("linear:384 gather_cols:384") +
        calls("gather_cols:128 split_f16:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 "
              "linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 rq_coupling_final:128") * 3 +
        calls("segment_sum:384 rows_to_nchw:384 nchw_to_rows:384 squeeze_rows:384 split_f16:96 linear_f16x3:96") +
        calls("gather_cols:96") * 2 +
        calls("split_f16:96") +
        calls("linear_f16x3:96 im2col3x3:96") * 4 +
        calls("linear_f16x3:96 rq_coupling_final:96 split_f16:96 linear_f16x3:96") +
        calls("gather_cols:96") * 2 +
        calls("split_f16:96") +
        calls("linear_f16x3:96 im2col3x3:96") * 4 +
        calls("linear_f16x3:96 rq_coupling_final:96 segment_sum:96 rows_to_nchw:96 nchw_to_rows:96 squeeze_rows:96 "
              "split_f16:24") +
        calls("linear_f16x3:24 linear_f16x3:24 im2col3x3:24 linear_f16x3:24 im2col3x3:24 linear_f16x3:24 "
              "im2col3x3:24 linear_f16x3:24 im2col3x3:24 linear_f16x3:24 rq_coupling_final:24") * 2 +
        calls("gather_cols:24 segment_sum:24 rows_to_nchw:24"),
        calls("nchw_to_rows:24 gather_cols:24 split_f16:24") +
        calls("linear_f16x3:24 im2col3x3:24 linear_f16x3:24 im2col3x3:24 linear_f16x3:24 im2col3x3:24 "
              "linear_f16x3:24 im2col3x3:24 linear_f16x3:24 rq_coupling_final:24 linear_f16x3:24") * 2 +
        calls("segment_sum:24 squeeze_rows:24 rows_to_nchw:96 nchw_to_rows:96") +
        calls("gather_cols:96") * 2 +
        calls("split_f16:96") +
        calls("linear_f16x3:96 im2col3x3:96") * 4 +
        calls("linear_f16x3:96 rq_coupling_final:96 split_f16:96 linear_f16x3:96") +
        calls("gather_cols:96") * 2 +
        calls("split_f16:96") +
        calls("linear_f16x3:96 im2col3x3:96") * 4 +
        calls("linear_f16x3:96 rq_coupling_final:96 split_f16:96 linear_f16x3:96 segment_sum:96 squeeze_rows:96 "
              "rows_to_nchw:384 nchw_to_rows:384 gather_cols:384") +
        calls("gather_cols:128 split_f16:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 "
              "linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 rq_coupling_final:128") * 3 +
        calls("linear:384 gather_cols:384") +
        calls("gather_cols:128 split_f16:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 "
              "linear_f16x3:128 im2col3x3:128 linear_f16x3:128 im2col3x3:128 linear_f16x3:128 rq_coupling_final:128") * 3 +
        calls("linear:384 segment_sum:384 squeeze_rows:384 rows_to_nchw:1536"),
    ),
    "nsf_final": (
        calls("split_f16:300 linear_f16x3:300") +
        calls("linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 rq_coupling_final:128") * 2 +
        calls("linear_f16x3:44") * 5 +
        calls("rq_coupling_final:44 linear_f16x3:300") +
        calls("linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 rq_coupling_final:128") * 2 +
        calls("linear_f16x3:44") * 5 +
        calls("rq_coupling_final:44 linear_f16x3:300") +
        calls("linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 rq_coupling_final:128") * 2 +
        calls("linear_f16x3:44") * 5 +
        calls("rq_coupling_final:44 gather_cols:300"),
        calls("gather_cols:300 split_f16:300") +
        calls("linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 rq_coupling_final:128") * 2 +
        calls("linear_f16x3:44") * 5 +
        calls("rq_coupling_final:44 linear_f16x3:300") +
        calls("linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 rq_coupling_final:128") * 2 +
        calls("linear_f16x3:44") * 5 +
        calls("rq_coupling_final:44 linear_f16x3:300") +
        calls("linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 linear_f16x3:128 rq_coupling_final:128") * 2 +
        calls("linear_f16x3:44") * 5 +
        calls("rq_coupling_final:44 linear_f16x3:300"),
    ),
    "nsf_rows": (
        calls("split_f16:300 linear_f16x3:300 gather_cols:300 split_f16:300 trunk_step:300 linear_f16x3:300 "
              "rqs_rows:300") * 3,
        calls("gather_cols:300 split_f16:300 trunk_step:300 linear_f16x3:300 rqs_rows:300 split_f16:300 "
              "linear_f16x3:300") * 3,
    ),
    "nsf_step": (
        calls("split_f16:300") +
        calls("linear_f16x3:300 rq_coupling_step:128 rq_coupling_step:128 rq_coupling_step:44") * 3 +
        calls("gather_cols:300"),
        calls("gather_cols:300 split_f16:300") +
        calls("rq_coupling_step:128 rq_coupling_step:128 rq_coupling_step:44 linear_f16x3:300") * 3,
    ),
    "plain_module": (
        calls("gather_cols:300 rqs_rows:300"),
        calls("gather_cols:300 rqs_rows:300"),
    ),
    "rows_ffma": (
        calls("gather_cols:300") +
        calls("linear:300") * 6 +
        calls("rqs_rows:300"),
        calls("gather_cols:300") +
        calls("linear:300") * 6 +
        calls("rqs_rows:300"),
    ),
    "unconditional": (
        calls("gather_cols:300") +
        calls("gather_cols:128 split_f16:128 trunk_step:128 rq_coupling_final:128") * 2 +
        calls("gather_cols:44 split_f16:44 trunk_step:44 rq_coupling_final:44 rqs_elementwise:300"),
        calls("rqs_elementwise:300 gather_cols:300") +
        calls("gather_cols:128 split_f16:128 trunk_step:128 rq_coupling_final:128") * 2 +
        calls("gather_cols:44 split_f16:44 trunk_step:44 rq_coupling_final:44"),
    ),
}


@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    monkeypatch.setattr(config, "coupling_block_rows", 128)
    return emulated_kernels.install(monkeypatch)


def _traced(emu, fn, *args):
    """fn(*args) once to fill the derived-weight caches, then again with its calls recorded."""
    fn(*args)
    del emu.trace[:]
    return fn(*args), list(emu.trace)


@torch.no_grad()
@pytest.mark.parametrize("name", sorted(CASES))
def test_route_trace(emu, name):
    torch.manual_seed(0)
    t, features = CASES[name]()
    t = recipes.perturb_(t).eval()
    x = torch.randn(300, features)
    want = [v.float() for v in t.double()(x.double())]
    want_inv = [v.float() for v in t.inverse(want[0].double())]
    t.float()
    with torch.enable_grad():           # parameters that need a gradient: the fp32 torch formulation, whose error sets the bound
        eager, eager_inv = t(x), t.inverse(want[0])
    got, fwd = _traced(emu, t, x)
    back, inv = _traced(emu, t.inverse, want[0])
    for g, e, w, floor in ((got, eager, want, TOL), (back, eager_inv, want_inv, 1e-4)):
        for k in range(2):
            assert rel_err(g[k], w[k]) <= max(floor, 3 * rel_err(e[k].detach(), w[k])), (name, k)
    assert (fwd, inv) == EXPECTED[name]


@torch.no_grad()
def test_route_trace_autoregressive_step(emu):
    """MAF-RQ on the step route: forward is one launch, the inverse one launch per feature on the degree-sorted sub-network."""
    g = load_golden("ar_rq")
    torch.manual_seed(g["seed"])
    ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=64, hidden_features=256, num_bins=8, tails="linear",
                                                                   tail_bound=3.0, num_blocks=2).eval()
    for name, p in ar.named_parameters():
        if "final_layer" in name:
            p.mul_(g["final_scale"])
    x = g["x"][:96]
    (y, lad), fwd = _traced(emu, ar, x)
    assert rel_err(y, g["y_fp64"][:96]) <= max(TOL, 3 * rel_err(g["y"][:96], g["y_fp64"][:96]))
    assert rel_err(lad, g["lad_fp64"][:96]) <= max(3e-5, 3 * rel_err(g["lad"][:96], g["lad_fp64"][:96]))
    (xi, li), inv = _traced(emu, ar.inverse, x)
    assert rel_err(xi, g["xinv_fp64"][:96]) <= max(1e-4, 3 * rel_err(g["xinv"][:96], g["xinv_fp64"][:96]))
    assert rel_err(li, g["ladinv_fp64"][:96]) <= max(1e-3, 3 * rel_err(g["ladinv"][:96], g["ladinv_fp64"][:96]))
    assert (fwd, inv) == EXPECTED["ar_step"]


@torch.no_grad()
def test_route_trace_context_flow(emu):
    """The context-conditioned flow (dense.Chain: the final route with ctx_init / glu_skip layers in the trunk)."""
    from nflows_b200.distributions.normal import StandardNormal
    from nflows_b200.flows import Flow
    g = load_golden("context_rows")["context_flow"]
    features, ctx_raw, ctx = 16, 5, 6
    steps = []
    for i in range(3):
        steps.append(T.ActNorm(features))
        steps.append(T.CompositeTransform([T.RandomPermutation(features), T.LULinear(features, identity_init=True)]))
        steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=_alt(features, even=(i % 2 == 0)),
            transform_net_create_fn=lambda i_, o_: ResidualNet(i_, o_, hidden_features=32, context_features=ctx, num_blocks=2),
            num_bins=8, tails="linear", tail_bound=3.0))
    flow = Flow(T.CompositeTransform(steps), StandardNormal([features]), embedding_net=torch.nn.Linear(ctx_raw, ctx)).eval()
    flow.load_state_dict(g["sd"], strict=True)
    lp, fwd = _traced(emu, flow.log_prob, g["x"], g["context"])
    assert rel_err(lp, g["log_prob_fp64"]) <= max(TOL, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    c = flow._embedding_net(g["context"])
    z = flow._transform(g["x"], c)[0]
    want = [v.float() for v in flow.double()._transform.inverse(z.double(), c.double())]
    flow.float()
    with torch.enable_grad():
        eager = flow._transform.inverse(z, c)
    got, inv = _traced(emu, flow._transform.inverse, z, c)
    for k in range(2):
        assert rel_err(got[k], want[k]) <= max(1e-4, 3 * rel_err(eager[k].detach(), want[k])), k
    assert (fwd, inv) == EXPECTED["context_flow"]


@torch.no_grad()
def test_route_trace_image_flow(emu):
    """The small Glow-style flow on pixel rows (dense.ConvChain: the final route with im2col 3x3 layers in the trunk)."""
    g = load_golden("image_rows")["glow_small"]
    flow = recipes.glow_multiscale(image_shape=(3, 16, 16), levels=3, steps=2, hidden_channels=32).eval()
    flow.load_state_dict(g["sd"], strict=True)
    (z, _), fwd = _traced(emu, flow._transform, g["x"])
    assert rel_err(z, g["z_fp64"]) <= max(TOL, 3 * rel_err(g["z"], g["z_fp64"]))
    (xs, lad_inv), inv = _traced(emu, flow._transform.inverse, g["noise"])
    assert rel_err(xs, g["sample_fp64"]) <= max(1e-4, 3 * rel_err(g["sample"], g["sample_fp64"]))
    assert rel_err(lad_inv, g["lad_inv_fp64"]) <= max(1e-4, 3 * rel_err(g["lad_inv"], g["lad_inv_fp64"]))
    assert (fwd, inv) == EXPECTED["image_flow"]


def test_plain_conditioner_keeps_the_softmax_warning(emu):
    """A conditioner without hidden_features / hidden_channels: the coupling warns that the softmax inputs are not scaled."""
    t = _coupling(_alt(16), net=_PlainConditioner).eval()
    with torch.no_grad(), pytest.warns(UserWarning, match="not scaled down"):
        t(torch.randn(10, 16))
