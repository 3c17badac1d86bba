"""Masked affine autoregressive transforms on the H100: the coupling-step kernel with its affine epilogue (nfk_affine_ar_step_f16x3),
against the reference's outputs (tests/golden/maf_affine_rows.pt) and the fp64 torch formulation, across the shapes it takes."""
import copy

import pytest
import torch

from conftest import load_golden, rel_err
from nflows_b200 import config
from nflows_b200 import kernels as K
from test_conditional_ar_gpu import timeline
from test_maf_affine_host import TRANSFORM_CASES, golden_flow, golden_transform, maf, perturb

pytestmark = pytest.mark.gpu


def sandwich(got, g, key, floor):
    return rel_err(got.cpu(), g[key + "_fp64"]) <= max(floor, 3 * rel_err(g[key], g[key + "_fp64"]))


@torch.no_grad()
@pytest.mark.parametrize("case", TRANSFORM_CASES)
def test_golden_transform(cuda_device, case):
    g = load_golden("maf_affine_rows")[case]
    t = golden_transform(g).to(cuda_device)
    x = g["x"].to(cuda_device)
    with timeline() as tl:
        y, lad = t(x)
    assert tl.count("affine_ar_step") == 1
    assert sandwich(y, g, "y", 1e-5) and sandwich(lad, g, "lad", 1e-5), (rel_err(y.cpu(), g["y_fp64"]), rel_err(lad.cpu(), g["lad_fp64"]))
    with timeline() as tl:
        xi, li = t.inverse(x)
    assert tl.count("affine_ar_step") == g["features"]
    assert sandwich(xi, g, "xinv", 1e-4) and sandwich(li, g, "ladinv", 1e-4), (rel_err(xi.cpu(), g["xinv_fp64"]),
                                                                              rel_err(li.cpu(), g["ladinv_fp64"]))


@torch.no_grad()
def test_golden_flow(cuda_device):
    g = load_golden("maf_affine_rows")["flow"]
    flow = golden_flow(g).to(cuda_device)
    x, c = g["x"].to(cuda_device), g["context"].to(cuda_device)
    with timeline() as tl:
        lp = flow.log_prob(x, context=c)
    assert tl.count("affine_ar_step") == 3 and tl.count("ar_context_terms") == 3
    assert rel_err(lp.cpu(), g["log_prob_fp64"]) <= 1e-5
    e = flow._embedding_net(c)
    z, lad = flow._transform(x, context=e)
    assert sandwich(z, g, "z", 1e-5) and sandwich(lad, g, "lad", 1e-5)
    with timeline() as tl:
        xs, lad_inv = flow._transform.inverse(g["noise"].to(cuda_device), context=e)
    assert tl.count("affine_ar_step") == 3 * g["features"] and tl.count("ar_context_terms") == 3
    assert sandwich(xs, g, "sample", 1e-4) and sandwich(lad_inv, g, "lad_inv", 1e-4)


def make(features, hidden=96, num_blocks=2, context=None, seed=0):
    torch.manual_seed(seed)
    return perturb(maf(features, hidden, context=context, num_blocks=num_blocks), seed + 1).eval().cuda()


def inputs(n, features, context, scale=1.0, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = scale * torch.randn(n, features, generator=g)
    c = None if context is None else torch.randn(n, context, generator=g)
    return x.cuda(), None if c is None else c.cuda()


def check(t, x, c, inverse, floors, factor=3):
    """Native fp32 against the fp64 torch formulation, held to `factor` times the fp32 torch formulation's error (or the floor)."""
    with timeline() as tl:
        got = t.inverse(x, context=c) if inverse else t(x, context=c)
    eager = t._eager(x, c, inverse)
    t64 = copy.deepcopy(t).double()
    c64 = None if c is None else c.double()
    want = t64.inverse(x.double(), context=c64) if inverse else t64(x.double(), context=c64)
    for k in range(2):
        e_got, e_eager = rel_err(got[k].cpu(), want[k].cpu()), rel_err(eager[k].cpu(), want[k].cpu())
        assert e_got <= max(floors[k], factor * e_eager), (inverse, k, e_got, e_eager)
    return tl, got


SHAPES = [(f, 96, 2, None) for f in (2, 5, 8, 16, 64, 100, 392)]
SHAPES += [(16, h, nb, None) for h in (32, 256) for nb in (0, 1, 2, 4)]
SHAPES += [(f, h, 2, ctx) for f in (5, 64) for h in (32, 256) for ctx in (5, 16)]
SHAPES += [(100, 96, nb, 16) for nb in (0, 4)]
# trunks of two chunks, the second partial, and feature counts around one and two column tiles of 64 (the degree-sorted
# sub-networks of the inverse then run every width from 32 up to the hidden one)
SHAPES += [(63, 160, 2, None), (65, 192, 1, 5), (129, 224, 2, None)]


@torch.no_grad()
@pytest.mark.parametrize("features,hidden,num_blocks,context", SHAPES)
def test_shapes(cuda_device, features, hidden, num_blocks, context):
    t = make(features, hidden, num_blocks, context, seed=features + hidden + num_blocks)
    x, c = inputs(300, features, context)
    tl, (y, _) = check(t, x, c, False, (1e-5, 1e-5))
    assert tl.count("affine_ar_step") == 1 and tl.count("ar_context_terms") == (0 if context is None else 1)
    tl, _ = check(t, y, c, True, (1e-4, 1e-4))
    assert tl.count("affine_ar_step") == features


@torch.no_grad()
@pytest.mark.parametrize("batch", [1, 127, 128, 129, 2 * 132 * 128 + 300])
@pytest.mark.parametrize("context", [None, 16])
def test_batch_sizes(cuda_device, batch, context):
    t = make(16, 64, 2, context)
    x, c = inputs(batch, 16, context)
    check(t, x, c, False, (1e-5, 1e-5))
    check(t, x, c, True, (1e-4, 1e-4))


@torch.no_grad()
def test_row_blocks_give_identical_results(cuda_device, monkeypatch):
    t = make(16, 128, 2, 16)
    x, c = inputs(5000, 16, 16)
    y, lad = t(x, context=c)
    xi, li = t.inverse(x, context=c)
    monkeypatch.setattr(config, "coupling_block_rows", 384)
    with timeline() as tl:
        y2, lad2 = t(x, context=c)
    assert tl.count("ar_context_terms") == 14 and tl.count("affine_ar_step") == 14
    with timeline() as tl:
        xi2, li2 = t.inverse(x, context=c)
    assert tl.count("ar_context_terms") == 14 and tl.count("affine_ar_step") == 14 * 16
    assert torch.equal(y, y2) and torch.equal(lad, lad2) and torch.equal(xi, xi2) and torch.equal(li, li2)


@torch.no_grad()
def test_large_inputs_take_the_activation_rescale(cuda_device):
    """|x| ~ 1e4 leaves the fp16 split range at the default activation exponent: the call repeats with a smaller one."""
    t = make(16, 64, 2)
    x, _ = inputs(500, 16, None, scale=1e4)
    # (u, shift) of magnitude ~1e4 carry the absolute round-off of fp32 and of the split pairs at the smaller exponent, so the
    # bound is ten times the fp32 torch formulation's error, as for the RQ twin's large context
    with pytest.warns(RuntimeWarning, match="fp16 split range") if not K._warned_rescale[0] else _nothing():
        tl, _ = check(t, x, None, False, (1e-5, 1e-5), factor=10)
    assert tl.count("affine_ar_step") >= 2


class _nothing:
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False


@torch.no_grad()
@pytest.mark.parametrize("context", [None, 5])
def test_round_trip(cuda_device, context):
    t = make(24, 128, 2, context)
    x, c = inputs(1000, 24, context)
    y, lad = t(x, context=c)
    back, lad_inv = t.inverse(y, context=c)
    assert rel_err(back.cpu(), x.cpu()) <= 1e-4 and rel_err(lad_inv.cpu(), -lad.cpu()) <= 1e-4


@torch.no_grad()
def test_unsupported_cases_stay_on_the_torch_path(cuda_device):
    x, c = inputs(200, 16, 5)
    cases = [maf(16, 64, activation=torch.tanh), maf(16, 64, use_residual_blocks=False), maf(16, 64, use_batch_norm=True),
             maf(16, 48), maf(16, 320), maf(16, 64, num_blocks=5)]
    for t in cases:
        t = t.eval().cuda()
        with timeline() as tl:
            y, lad = t(x)
        assert tl.count("affine_ar_step") == 0 and tl.launches == 0
        want = t._eager(x, None, False)
        assert torch.equal(y, want[0]) and torch.equal(lad, want[1])
    t = make(16, 64, 2, 5)
    with timeline() as tl, pytest.raises(RuntimeError):             # batch sizes of inputs and context differ
        t(x, context=c[:150])
    assert tl.launches == 0
    with timeline() as tl:
        t.double()(x.double(), context=c.double())
        t.float()
        with torch.enable_grad():
            t(x, context=c)
    assert tl.launches == 0
