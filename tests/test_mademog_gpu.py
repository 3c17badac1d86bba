"""Mixture-of-Gaussians MADE on the H100: the coupling-step kernel with its mixture epilogue (nfk_mog_made_step_f16x3) against the
reference's outputs (tests/golden/mademog_rows.pt), the fp64 oracle (tests/_mademog_oracle.py) and the analytic mixture CDF."""
import math

import pytest
import torch

import _mademog_oracle as oracle
from conftest import load_golden, rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.distributions import MADEMoG
from nflows_b200.flows import Flow
from nflows_b200.nn.nde import MixtureOfGaussiansMADE
from test_conditional_ar_gpu import timeline
from test_mademog_host import CASES, build, golden_flow, perturb

pytestmark = pytest.mark.gpu


def sandwich(got, g, floor=1e-5):
    return rel_err(got.cpu(), g["log_prob_fp64"]) <= max(floor, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))


@torch.no_grad()
@pytest.mark.parametrize("case", CASES)
def test_golden_cases(cuda_device, case):
    g = load_golden("mademog_rows")[case]
    m = build(case, g).to(cuda_device)
    x = g["x"].to(cuda_device)
    c = None if g["context"] is None else g["context"].to(cuda_device)
    with timeline() as tl:
        lp = m.log_prob(x, context=c)
    assert tl.count("mog_made_step") == 1
    assert sandwich(lp, g), rel_err(lp.cpu(), g["log_prob_fp64"])


@torch.no_grad()
def test_golden_flow(cuda_device):
    g = load_golden("mademog_rows")["flow"]
    flow = golden_flow(g).to(cuda_device)
    with timeline() as tl:
        lp = flow.log_prob(g["x"].to(cuda_device), context=g["context"].to(cuda_device))
    assert tl.count("mog_made_step") == 1 and tl.count("affine_ar_step") == 3
    assert sandwich(lp, g), rel_err(lp.cpu(), g["log_prob_fp64"])


def make(features, hidden, num_blocks=2, components=5, context=None, seed=0, epsilon=1e-2):
    torch.manual_seed(seed)
    m = MixtureOfGaussiansMADE(features, hidden, context_features=context, num_blocks=num_blocks,
                               num_mixture_components=components, epsilon=epsilon)
    return perturb(m, seed + 1).eval().cuda()


def check(m, n, context, scale=1.0, seed=1):
    gen = torch.Generator().manual_seed(seed)
    x = scale * torch.randn(n, m.features, generator=gen)
    c = None if context is None else torch.randn(n, context, generator=gen)
    xd, cd = x.cuda(), None if c is None else c.cuda()
    with timeline() as tl:
        lp = m.log_prob(xd, context=cd)
    want = oracle.log_prob({k: v.cpu() for k, v in m.state_dict().items()}, x, c, m.num_mixture_components, m.epsilon, prefix="")
    eager = m._torch_log_prob(xd, cd).cpu()
    e_got, e_eager = rel_err(lp.cpu(), want), rel_err(eager, want)
    assert e_got <= max(1e-5, 3 * e_eager), (e_got, e_eager)
    return tl, lp


SWEEP = ([(d, 96, 2, 5, 3) for d in (1, 2, 5, 8, 16, 64, 100)]
         + [(16, h, 2, 5, None) for h in (32, 50, 96, 256)]
         + [(16, 64, b, 5, 16) for b in (0, 1, 2, 3, 4)]
         + [(8, 64, 2, k, 16) for k in (1, 2, 5, 10, 11, 16, 17, _native.MOG_MAX_COMPONENTS)]
         + [(5, 50, 2, 10, ctx) for ctx in (None, 3, 16)]
         + [(100, 256, 4, _native.MOG_MAX_COMPONENTS, 16), (64, 256, 2, 10, 16), (2, 32, 0, 1, None)])
SWEEP = [s + (1e-2,) for s in SWEEP]
# packed rows 24 (C = 6, 8) and the first C of 32 and 64; odd feature counts at one feature per thread (MP >= 48: 12, 17, 21
# components); trunks of two chunks, the second partial (hidden 160, 192, 224); an epsilon other than 1e-2
SWEEP += ([(8, 64, 2, k, 16, 1e-2) for k in (6, 8, 9, 18, 19)]
          + [(7, 96, 2, 12, None, 1e-2), (9, 64, 1, 17, 3, 1e-2), (5, 32, 2, 21, None, 1e-2), (3, 160, 1, 16, None, 1e-2)]
          + [(16, 160, 2, 5, None, 1e-2), (12, 192, 1, 7, 4, 1e-2), (10, 224, 3, 20, None, 1e-2)]
          + [(6, 64, 2, 5, None, 0.5), (6, 64, 2, 9, 3, 1e-4)])


def _sweep_id(s):
    """The entry's values joined by "-" (the default id), with the epsilon appended only where it is not the default."""
    return "-".join(str(v) for v in s[:5]) + ("" if s[5] == 1e-2 else "-eps{}".format(s[5]))


@torch.no_grad()
@pytest.mark.parametrize("features,hidden,num_blocks,components,context,epsilon", SWEEP, ids=[_sweep_id(s) for s in SWEEP])
def test_shape_sweep(cuda_device, features, hidden, num_blocks, components, context, epsilon):
    m = make(features, hidden, num_blocks, components, context, epsilon=epsilon)
    tl, _ = check(m, 300, context)
    assert tl.count("mog_made_step") == 1


@torch.no_grad()
@pytest.mark.parametrize("n", [1, 127, 129, 2 * 132 * 128 + 300])
@pytest.mark.parametrize("context", [None, 16])
def test_batch_sizes(cuda_device, n, context):
    m = make(16, 64, 2, 10, context)
    check(m, n, context)


@torch.no_grad()
def test_row_block_split_is_bit_identical(cuda_device, monkeypatch):
    m = make(5, 50, 2, 10, 7)
    x, c = torch.randn(1000, 5, device="cuda"), torch.randn(1000, 7, device="cuda")
    whole = m.log_prob(x, context=c)
    monkeypatch.setattr(config, "coupling_block_rows", 384)
    with timeline() as tl:
        split = m.log_prob(x, context=c)
    assert tl.count("mog_made_step") == 3
    assert torch.equal(whole, split)


@torch.no_grad()
def test_activation_rescale(cuda_device):
    m = make(8, 64, 2, 5, 3)
    check(m, 500, 3, scale=1e4)


@torch.no_grad()
def test_samples_follow_the_oracle_sampler(cuda_device):
    """The same (u, e) as the native sampler draws: samples equal the oracle's within 1e-5, except rows whose u lies within 1e-5
    of a component's cumulative-weight boundary (fp64), which must be a tiny fraction."""
    g = load_golden("mademog_rows")["sbi"]
    m = build("sbi", g).cuda()
    ctx = torch.randn(2000, 7).cuda()
    torch.manual_seed(11)
    with timeline() as tl:
        s = m.sample(4, context=ctx)
    assert s.shape == (2000, 4, 5) and s.device == ctx.device
    assert tl.count("mog_made_step") == 5 and tl.count("ar_context_terms") == 1
    torch.manual_seed(11)
    u, e = torch.rand(8000, 5, device="cuda"), torch.randn(8000, 5, device="cuda")
    want, margin = oracle.sample({k: v.cpu() for k, v in m._made.state_dict().items()}, u.cpu(), e.cpu(),
                                 ctx.repeat_interleave(4, dim=0).cpu(), 10, prefix="")
    ok = margin > 1e-5
    assert ok.double().mean() >= 0.99, ok.double().mean()
    assert rel_err(s.reshape(8000, 5).cpu()[ok], want[ok]) <= 1e-5


@torch.no_grad()
def test_sample_distribution_ks(cuda_device):
    """2^16 native draws of a D = 1 conditional model for one context row against the analytic mixture CDF."""
    from scipy import stats
    m = make(1, 64, 2, 4, 3, seed=7)
    ctx = torch.randn(1, 3).cuda()
    torch.manual_seed(12)
    s = m.sample(1 << 16, context=ctx).reshape(-1).double().cpu().numpy()
    out = m.double()(torch.zeros(1, 1, dtype=torch.float64, device="cuda"), ctx.double()).reshape(4, 3).cpu()
    w = torch.softmax(out[:, 0], 0).numpy()
    mu, sd = out[:, 1].numpy(), (torch.nn.functional.softplus(out[:, 2]) + m.epsilon).numpy()
    cdf = lambda v: sum(w[c] * stats.norm.cdf((v - mu[c]) / sd[c]) for c in range(4))
    assert stats.kstest(s, cdf).pvalue > 1e-3


@torch.no_grad()
def test_flow_sample_shapes(cuda_device):
    torch.manual_seed(3)
    f = 6
    layers = []
    for _ in range(2):
        layers += [T.ReversePermutation(f), T.MaskedAffineAutoregressiveTransform(features=f, hidden_features=64, context_features=5)]
    flow = Flow(T.CompositeTransform(layers), MADEMoG(f, 50, 5, num_mixture_components=10),
                embedding_net=torch.nn.Linear(7, 5)).eval().cuda()
    c = torch.randn(9, 7).cuda()
    with timeline() as tl:
        s = flow.sample(11, context=c)
    assert s.shape == (9, 11, f) and tl.count("mog_made_step") == f
    s2, lp = flow.sample_and_log_prob(11, context=c)
    assert s2.shape == (9, 11, f) and lp.shape == (9, 11) and bool(torch.isfinite(lp).all())
    assert rel_err(lp.reshape(-1).cpu(), flow.log_prob(s2.reshape(-1, f), context=c.repeat_interleave(11, 0)).cpu()) <= 1e-3
