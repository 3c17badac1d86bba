"""Context-conditioned masked autoregressive spline transforms on the H100: the coupling-step kernel with the context projections as
per-row trunk terms, against the reference's outputs (tests/golden/conditional_ar_rows.pt) and the fp64 torch formulation."""
import copy

import pytest
import torch

from conftest import load_golden, rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.flows import recipes
from test_conditional_ar_host import CTX, FEATURES, golden_flow, golden_transform

pytestmark = pytest.mark.gpu


class timeline:
    """Collects the tagged launches of the block (kernels.TIMELINE) and the native launch count."""

    def __enter__(self):
        self.prev, K.TIMELINE = K.TIMELINE, []
        self.before = _native.launch_count()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.tags = [entry[0] for entry in K.TIMELINE]
        self.launches = _native.launch_count() - self.before
        K.TIMELINE = self.prev

    def count(self, tag):
        return self.tags.count(tag)


def sandwich(got, eager, want, floor, factor=3):
    """got is as close to the fp64 result as `factor` times the fp32 torch formulation's error (or the floor)."""
    return rel_err(got.cpu(), want.cpu()) <= max(floor, factor * rel_err(eager.detach().cpu(), want.cpu()))


def check_against_torch(t, x, c, inverse, floors=None, factor=3):
    """The native fp32 result is held to the fp64 torch formulation by the fp32 torch formulation's error on the same device
    (sandwich); returns the timeline of the native call."""
    with timeline() as tl:
        got = t.inverse(x, context=c) if inverse else t(x, context=c)
    eager = t._eager(x, c, inverse)
    t64 = copy.deepcopy(t).double()
    want = t64.inverse(x.double(), context=c.double()) if inverse else t64(x.double(), context=c.double())
    floors = floors or ((1e-4, 1e-3) if inverse else (1e-5, 3e-5))
    for k in range(2):
        assert sandwich(got[k], eager[k], want[k], floors[k], factor), (inverse, k, rel_err(got[k].cpu(), want[k].cpu()),
                                                                 rel_err(eager[k].cpu(), want[k].cpu()))
    return tl


def sharpen(module, seed=1):
    """Give the residual blocks' zero-initialised second linear some weight, so the block context terms show in the outputs."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            if "linear_layers.1" in name:
                p.add_(0.05 * torch.randn(p.shape, generator=g))
    return module


def make(features=16, hidden=64, context=CTX, num_blocks=2, num_bins=8, tails="linear", seed=0, dev="cuda"):
    torch.manual_seed(seed)
    kw = dict(tails="linear", tail_bound=3.0) if tails == "linear" else dict(tails=None)
    t = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=features, hidden_features=hidden, context_features=context,
                                                                  num_bins=num_bins, num_blocks=num_blocks, **kw)
    return sharpen(recipes.perturb_(t)).eval().to(dev)


def inputs(n, features, tails, context=CTX, dev="cuda", seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, features, generator=g) if tails is None else 1.5 * torch.randn(n, features, generator=g)
    return x.to(dev), torch.randn(n, context, generator=g).to(dev)


@torch.no_grad()
def test_golden_transform(cuda_device):
    g = load_golden("conditional_ar_rows")["none"]
    t = golden_transform(g).to(cuda_device)
    x, c = g["x"].to(cuda_device), g["context"].to(cuda_device)
    with timeline() as tl:
        y, lad = t(x, context=c)
    assert tl.count("rq_coupling_step") == 1 and tl.count("ar_context_terms") == 1
    assert rel_err(y.cpu(), g["y_fp64"]) <= max(1e-5, 3 * rel_err(g["y"], g["y_fp64"]))
    # the perturbed, sharpened weights make sharp splines: one row's log|det| carries ~1e-4 of the split-pair conditioner's
    # round-off (fp64 context terms in its place change nothing), hence the floor -- the shape sweep's
    assert rel_err(lad.cpu(), g["lad_fp64"]) <= max(3e-4, 3 * rel_err(g["lad"], g["lad_fp64"]))
    with timeline() as tl:
        xi, li = t.inverse(x, context=c)
    assert tl.count("rq_coupling_step") == FEATURES and tl.count("ar_context_terms") == 1
    assert rel_err(xi.cpu(), g["xinv_fp64"]) <= max(1e-4, 3 * rel_err(g["xinv"], g["xinv_fp64"]))
    assert rel_err(li.cpu(), g["ladinv_fp64"]) <= max(1e-3, 3 * rel_err(g["ladinv"], g["ladinv_fp64"]))


@torch.no_grad()
def test_golden_flow(cuda_device):
    g = load_golden("conditional_ar_rows")["linear"]
    flow = golden_flow(g).to(cuda_device)
    x, c = g["x"].to(cuda_device), g["context"].to(cuda_device)
    with timeline() as tl:
        lp = flow.log_prob(x, context=c)
    assert tl.count("rq_coupling_step") == 2 and tl.count("ar_context_terms") == 2
    assert rel_err(lp.cpu(), g["log_prob_fp64"]) <= max(3e-5, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    e = flow._embedding_net(c)
    z, lad = flow._transform(x, context=e)
    assert rel_err(z.cpu(), g["z_fp64"]) <= max(1e-5, 3 * rel_err(g["z"], g["z_fp64"]))
    assert rel_err(lad.cpu(), g["lad_fp64"]) <= max(3e-4, 3 * rel_err(g["lad"], g["lad_fp64"]))      # the floor as above
    with timeline() as tl:
        xs, lad_inv = flow._transform.inverse(g["noise"].to(cuda_device), context=e)
    assert tl.count("rq_coupling_step") == 2 * FEATURES and tl.count("ar_context_terms") == 2
    assert rel_err(xs.cpu(), g["sample_fp64"]) <= max(1e-4, 3 * rel_err(g["sample"], g["sample_fp64"]))
    assert rel_err(lad_inv.cpu(), g["lad_inv_fp64"]) <= max(1e-3, 3 * rel_err(g["lad_inv"], g["lad_inv_fp64"]))
    # sample / sample_and_log_prob: the native result against the fp32 torch formulation on the same noise (parameters that need
    # a gradient under enable_grad take the torch path)
    bound = 1e-4 + 4 * rel_err(g["sample"], g["sample_fp64"])
    ctx = c[:20]
    torch.manual_seed(7)
    with timeline() as tl:
        s = flow.sample(15, context=ctx)
    assert tl.count("rq_coupling_step") == 2 * FEATURES and s.shape == (20, 15, FEATURES)
    torch.manual_seed(7)
    with torch.enable_grad():
        s_eager = flow.sample(15, context=ctx)
    assert rel_err(s.cpu(), s_eager.detach().cpu()) <= bound
    torch.manual_seed(8)
    s2, lp2 = flow.sample_and_log_prob(15, context=ctx)
    torch.manual_seed(8)
    with torch.enable_grad():
        s2_eager, lp2_eager = flow.sample_and_log_prob(15, context=ctx)
    assert rel_err(s2.cpu(), s2_eager.detach().cpu()) <= bound
    # (the inverse's log|det| carries the round-off of all D passes: the floor of the autoregressive inverse's log|det| checks)
    assert rel_err(lp2.cpu(), lp2_eager.detach().cpu()) <= 1e-3 + 4 * rel_err(g["lad_inv"], g["lad_inv_fp64"])


SHAPES = [(h, nb, bins, tails) for h in (32, 96, 256) for nb in (0, 1, 2) for bins, tails in
          (((4, "linear"), (10, None), (16, "linear")) if h == 96 else ((8, "linear"), (16, None)))]
SHAPES += [(64, 2, bins, tails) for bins in (4, 8, 10, 16) for tails in ("linear", None)]


@torch.no_grad()
@pytest.mark.parametrize("hidden,num_blocks,num_bins,tails", SHAPES)
def test_shapes(cuda_device, hidden, num_blocks, num_bins, tails):
    t = make(features=16, hidden=hidden, num_blocks=num_blocks, num_bins=num_bins, tails=tails, seed=hidden + num_blocks + num_bins)
    x, c = inputs(300, 16, tails)
    # random weights with the final layer scaled up make sharp splines: an element's log|det| can carry a few 1e-4 of the
    # split-pair conditioner's round-off (the tensor-core arithmetic of every dense layer here), a few 1e-3 after the D passes
    # of the inverse, hence the floors
    tl = check_against_torch(t, x, c, inverse=False, floors=(1e-4, 3e-4))
    assert tl.count("rq_coupling_step") == 1 and tl.count("ar_context_terms") == 1
    assert sum(tag.startswith("linear_8x") for tag in tl.tags) == (2 if num_blocks else 1)
    tl = check_against_torch(t, x, c, inverse=True, floors=(3e-4, 3e-3))
    assert tl.count("rq_coupling_step") == 16 and tl.count("ar_context_terms") == 1


@torch.no_grad()
@pytest.mark.parametrize("batch", [0, 1, 127, 129, 1 << 15])
def test_batch_sizes(cuda_device, batch):
    t = make(features=16, hidden=64, context=16)
    x, c = inputs(batch, 16, "linear", context=16)
    if batch == 0:
        y, lad = t(x, context=c)
        xi, li = t.inverse(x, context=c)
        assert y.shape == (0, 16) and lad.shape == (0,) and xi.shape == (0, 16) and li.shape == (0,)
        return
    check_against_torch(t, x, c, inverse=False)
    check_against_torch(t, x, c, inverse=True)


@torch.no_grad()
def test_row_blocks_give_identical_results(cuda_device, monkeypatch):
    t = make(features=16, hidden=128, context=16)
    x, c = inputs(5000, 16, "linear", context=16)
    y, lad = t(x, context=c)
    xi, li = t.inverse(x, context=c)
    monkeypatch.setattr(config, "coupling_block_rows", 384)
    with timeline() as tl:
        y2, lad2 = t(x, context=c)
    assert tl.count("ar_context_terms") == 14 and tl.count("rq_coupling_step") == 14
    with timeline() as tl:
        xi2, li2 = t.inverse(x, context=c)
    assert tl.count("ar_context_terms") == 14 and tl.count("rq_coupling_step") == 14 * 16
    assert torch.equal(y, y2) and torch.equal(lad, lad2) and torch.equal(xi, xi2) and torch.equal(li, li2)


@torch.no_grad()
@pytest.mark.parametrize("features", [8, 32])
def test_projections_do_not_scale_with_features(cuda_device, features):
    t = make(features=features, hidden=64, context=16)
    x, c = inputs(1000, features, "linear", context=16)
    with timeline() as tl:
        t.inverse(x, context=c)
    assert tl.launches >= features and tl.count("rq_coupling_step") == features
    assert tl.count("ar_context_terms") == 1 and tl.count("linear_16x64") == 1 and tl.count("linear_16x128") == 1


@torch.no_grad()
def test_large_context_takes_the_activation_rescale(cuda_device):
    """|context| ~ 1e4 leaves the fp16 split range at the default activation exponent: the call repeats with a smaller one."""
    t = make(features=16, hidden=64, context=CTX)
    x, c = inputs(500, 16, "linear")
    c = c * 1e4
    # spline logits of magnitude ~1e4: their absolute round-off (fp32's and the split pairs') is amplified by the softmax, so the
    # bound is ten times the fp32 torch formulation's error
    with pytest.warns(RuntimeWarning, match="fp16 split range") if not K._warned_rescale[0] else _nothing():
        tl = check_against_torch(t, x, c, inverse=False, factor=10)
    # the first attempt, then at least one repeat with a smaller exponent
    assert tl.count("rq_coupling_step") >= 2 and tl.count("ar_context_terms") == tl.count("rq_coupling_step"), tl.tags


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


@torch.no_grad()
def test_unsupported_cases_stay_on_the_torch_path(cuda_device):
    x, c = inputs(200, 16, "linear")
    plain = make(features=16, hidden=64, context=None)
    with timeline() as tl, pytest.raises(AttributeError):           # the reference fails the same way: no context layer
        plain(x, context=c)
    assert tl.count("rq_coupling_step") == 0
    t = make(features=16, hidden=64)
    with timeline() as tl, pytest.raises(RuntimeError):             # batch sizes of inputs and context differ
        t(x, context=c[:150])
    assert tl.count("ar_context_terms") == 0
    cases = [make(features=16, hidden=48),                           # not a multiple of 32: no step route
             make(features=12, hidden=64),                           # not a multiple of 8: no tensor-core conditioner
             T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=16, hidden_features=64, context_features=CTX,
                                                                       num_bins=8, tails="linear", activation=torch.tanh),
             T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=16, hidden_features=64, context_features=CTX,
                                                                       num_bins=8, tails="linear", use_residual_blocks=False)]
    for t in cases:
        t = t.eval().to(cuda_device)
        xt = x[:, :t.features]
        with timeline() as tl:
            y, lad = t(xt, context=c)
        assert tl.count("rq_coupling_step") == 0 and tl.count("ar_context_terms") == 0
        want = t._eager(xt, c, False)
        assert torch.equal(y, want[0]) and torch.equal(lad, want[1])
    # a MADE with context layers called without a context: the plain chain on the step kernel, no projections
    t = make(features=16, hidden=64)
    with timeline() as tl:
        y, lad = t(x)
    assert tl.count("rq_coupling_step") == 1 and tl.count("ar_context_terms") == 0
