"""Host logic of the native execution chain -- column layouts, row blocking, context chains, the pixel-row image driver -- run
on the CPU with the kernel wrappers replaced by torch restatements of their contracts (tests/emulated_kernels.py).  What is
under test is everything ABOVE the C ABI; the kernels themselves are checked on hardware by the `-m gpu` tests."""
import pytest
import torch

import emulated_kernels
from conftest import load_golden, rel_err
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.flows import recipes

TOL = 1e-5


@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", False)
    return emulated_kernels.install(monkeypatch)


@torch.no_grad()
def test_small_nsf_flow_through_the_native_chain(emu):
    """The emulation itself: a cfg-3-shaped flow (folded affine runs, packed couplings, pair hand-off) equals the torch path."""
    torch.manual_seed(0)
    flow = recipes.perturb_(recipes.rq_nsf(32, hidden_features=32, num_layers=3)).eval()
    x = torch.randn(300, 32)
    want = [t.float() for t in flow.double()._transform(x.double())]          # fp64 inputs always take the torch formulation
    flow.float()
    config.coupling_block_rows, saved = 128, config.coupling_block_rows
    try:
        got = flow._transform(x)
    finally:
        config.coupling_block_rows = saved
    assert emu.get("rq_coupling_final", 0) == 9 and emu.get("linear_f16x3", 0) > 0            # 3 couplings x 3 row blocks
    assert rel_err(got[0], want[0]) <= TOL and rel_err(got[1], want[1]) <= TOL
    back = flow._transform.inverse(want[0])
    assert rel_err(back[0], x) <= 1e-4


@torch.no_grad()
def test_context_flow_through_the_native_chain(emu):
    """SURVEY row f4: the reference golden of the context-conditioned flow through dense.Chain (ctx_init / glu_skip)."""
    from nflows_b200.distributions.normal import StandardNormal
    from nflows_b200.flows import Flow
    from nflows_b200.nn.nets import ResidualNet
    from nflows_b200.utils import torchutils
    g = load_golden("context_rows")["context_flow"]
    features, ctx_raw, ctx = 16, 5, 6
    steps = []
    for i in range(3):
        steps.append(T.ActNorm(features))
        steps.append(T.CompositeTransform([T.RandomPermutation(features), T.LULinear(features, identity_init=True)]))
        steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(features, even=(i % 2 == 0)),
            transform_net_create_fn=lambda i_, o_: ResidualNet(i_, o_, hidden_features=32, context_features=ctx, num_blocks=2),
            num_bins=8, tails="linear", tail_bound=3.0))
    flow = Flow(T.CompositeTransform(steps), StandardNormal([features]), embedding_net=torch.nn.Linear(ctx_raw, ctx)).eval()
    flow.load_state_dict(g["sd"], strict=True)
    config.coupling_block_rows, saved = 128, config.coupling_block_rows      # 300 rows: three row blocks, context sliced alike
    try:
        lp = flow.log_prob(g["x"], context=g["context"])
    finally:
        config.coupling_block_rows = saved
    assert emu.get("glu_skip", 0) == 3 * 2 * 3                               # 3 couplings x 2 blocks x 3 row blocks
    assert rel_err(lp, g["log_prob_fp64"]) <= max(TOL, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))


@torch.no_grad()
def test_image_flow_through_the_pixel_row_chain(emu):
    """SURVEY row f3: the reference golden of the small Glow-style flow through CompositeTransform._native_apply_image --
    NCHW <-> pixel rows, squeeze on rows, OneByOneConvolution folded into the affine run, ConvChain (padded initial layer, im2col
    3x3 layers) + fused final layer, per-pixel log|det| folded per sample, forward and inverse."""
    g = load_golden("image_rows")["glow_small"]
    flow = recipes.glow_multiscale(image_shape=(3, 16, 16), levels=3, steps=2, hidden_channels=32).eval()
    flow.load_state_dict(g["sd"], strict=True)
    level = flow._transform._transforms[0]
    assert level._native_ready(g["x"], None)
    z, lad = flow._transform(g["x"])
    assert emu.get("nchw_to_rows", 0) == 3 and emu.get("squeeze_rows", 0) == 3 and emu.get("im2col3x3", 0) == 3 * 2 * 4
    # the two 12-channel affine folds (ActNorm + 1x1 convolution of level 1) are 12x12 maps: FFMA dense layer, K is no TMA row
    assert emu.get("rq_coupling_final", 0) == 6 and emu.get("linear", 0) == 2
    assert rel_err(z, g["z_fp64"]) <= max(TOL, 3 * rel_err(g["z"], g["z_fp64"]))
    lp = flow.log_prob(g["x"])
    assert rel_err(lp, g["log_prob_fp64"]) <= max(TOL, 3 * rel_err(g["log_prob"], g["log_prob_fp64"]))
    xs, lad_inv = flow._transform.inverse(g["noise"])
    assert rel_err(xs, g["sample_fp64"]) <= max(1e-4, 3 * rel_err(g["sample"], g["sample_fp64"]))
    assert rel_err(lad_inv, g["lad_inv_fp64"]) <= max(1e-4, 3 * rel_err(g["lad_inv"], g["lad_inv_fp64"]))


@torch.no_grad()
def test_standalone_one_by_one_convolution_through_the_native_chain(emu):
    """OneByOneConvolution called on its own (4-D input, reference golden next_rows.pt): its forward applies the channel
    permutation itself and hands the pixels to the LULinear path -- the folded run must then hold the LU map only (inside an
    image chain the same leaf stands for permutation + LU)."""
    g = load_golden("next_rows")
    for key, channels in (("conv1x1", 3), ("conv1x1_c12", 12)):
        r = g[key]
        conv = T.OneByOneConvolution(channels, identity_init=False).eval()
        conv.load_state_dict(r["sd"], strict=True)
        y, lad = conv(r["x"])
        assert rel_err(y, r["y"]) <= TOL and rel_err(lad, r["lad"]) <= TOL, key
        back, _ = conv.inverse(r["y"])
        assert rel_err(back, r["x"]) <= 1e-4, key


def _affine_cases(g):
    from nflows_b200.nn.nets import ResidualNet
    from nflows_b200.utils import torchutils
    f = lambda i, o: ResidualNet(i, o, hidden_features=64, num_blocks=2)
    alt, mid = torchutils.create_alternating_binary_mask, torchutils.create_mid_split_binary_mask
    yield "default48", T.AffineCouplingTransform(alt(48), f)
    yield "general48", T.AffineCouplingTransform(alt(48), f, scale_activation=T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION)
    yield "default20", T.AffineCouplingTransform(torch.tensor([0] * 8 + [1] * 12), f)
    yield "additive48", T.AdditiveCouplingTransform(alt(48), f)


@torch.no_grad()
def test_affine_couplings_with_the_fused_final_layer(emu):
    """Row ns2: affine / additive couplings whose last conditioner layer is fused with the coupling (interleaved weight rows,
    packed and gathered column paths) against the reference golden affine_rows.pt."""
    g = load_golden("affine_rows")
    for key, t in _affine_cases(g):
        r = g[key]
        t = t.eval()
        t.load_state_dict(r["sd"], strict=True)
        y, lad = t(r["x"])
        assert rel_err(y, r["y"]) <= TOL and rel_err(lad, r["lad"]) <= 3e-5, key
        xi, _ = t.inverse(r["x"])
        assert rel_err(xi, r["xinv"]) <= 1e-4, key
    assert emu.get("affine_coupling_final", 0) == 8 and emu.get("rqs_rows", 0) == 0


@torch.no_grad()
def test_affine_flow_behind_folded_affine_runs(emu):
    """ActNorm + LU runs in front of affine couplings: the coupling asks for the identity-first column layout, the fold emits it."""
    from nflows_b200.distributions.normal import StandardNormal
    from nflows_b200.flows import Flow
    from nflows_b200.nn.nets import ResidualNet
    from nflows_b200.utils import torchutils
    r = load_golden("affine_rows")["flow48"]
    f = lambda i, o: ResidualNet(i, o, hidden_features=64, num_blocks=2)
    steps = []
    for i in range(3):
        steps += [T.ActNorm(48), T.CompositeTransform([T.RandomPermutation(48), T.LULinear(48, identity_init=True)]),
                  T.AffineCouplingTransform(torchutils.create_alternating_binary_mask(48, even=(i % 2 == 0)), f)]
    flow = Flow(T.CompositeTransform(steps), StandardNormal([48])).eval()
    flow.load_state_dict(r["sd"], strict=True)
    lp = flow.log_prob(r["x"])
    assert emu.get("affine_coupling_final", 0) == 3 and emu.get("gather_cols", 0) <= 2
    assert rel_err(lp, r["log_prob_fp64"]) <= max(TOL, 3 * rel_err(r["log_prob"], r["log_prob_fp64"]))


@pytest.fixture
def emu_step(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    return emulated_kernels.install(monkeypatch)


@torch.no_grad()
def test_flow_on_the_one_kernel_coupling_step(emu_step):
    """Row ns1's host side: dense.plan_step_kernel / StepPlan (stacked weight pairs, per-layer exponents, layer flags) and the
    pair hand-off between the affine GEMM and the step kernel, against the fp64 torch formulation."""
    torch.manual_seed(0)
    flow = recipes.perturb_(recipes.rq_nsf(32, hidden_features=32, num_layers=3)).eval()
    x = torch.randn(300, 32)
    want = [t.float() for t in flow.double()._transform(x.double())]
    flow.float()
    config.coupling_block_rows, saved = 128, config.coupling_block_rows
    try:
        got = flow._transform(x)
    finally:
        config.coupling_block_rows = saved
    assert emu_step.get("rq_coupling_step", 0) == 9 and emu_step.get("trunk_step", 0) == 0      # 3 couplings x 3 row blocks
    assert emu_step.get("linear_f16x3", 0) == 3                                                   # only the folded affine runs
    assert rel_err(got[0], want[0]) <= TOL and rel_err(got[1], want[1]) <= TOL


@torch.no_grad()
def test_autoregressive_transform_on_the_step_kernel(emu_step):
    """Row f1's host side (BASELINE cfg 4): forward = one step launch on the masked MADE weights; inverse = one launch per degree
    prefix on the degree-sorted sub-network (MADE.sorted_subnets), against the reference golden ar_rq.pt."""
    g = load_golden("ar_rq")
    torch.manual_seed(g["seed"])
    ar = T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=64, hidden_features=256, num_bins=8, tails="linear",
                                                                   tail_bound=3.0, num_blocks=2).eval()
    for name, p in ar.named_parameters():
        if "final_layer" in name:
            p.mul_(g["final_scale"])
    x = g["x"][:96]
    y, lad = ar(x)
    assert emu_step.get("rq_coupling_step", 0) == 1
    assert rel_err(y, g["y_fp64"][:96]) <= max(TOL, 3 * rel_err(g["y"][:96], g["y_fp64"][:96]))
    assert rel_err(lad, g["lad_fp64"][:96]) <= max(3e-5, 3 * rel_err(g["lad"][:96], g["lad_fp64"][:96]))
    xi, li = ar.inverse(x)
    assert emu_step.get("rq_coupling_step", 0) == 1 + 64                                          # one launch per feature
    assert rel_err(xi, g["xinv_fp64"][:96]) <= max(1e-4, 3 * rel_err(g["xinv"][:96], g["xinv_fp64"][:96]))
    assert rel_err(li, g["ladinv_fp64"][:96]) <= max(1e-3, 3 * rel_err(g["ladinv"][:96], g["ladinv_fp64"][:96]))


@torch.no_grad()
def test_affine_coupling_trunk_as_one_step_launch(emu_step):
    """Row ns2's host side: the conditioner trunk of an affine coupling is the step kernel stopped after its last trunk layer."""
    r = load_golden("affine_rows")["default48"]
    from nflows_b200.nn.nets import ResidualNet
    from nflows_b200.utils import torchutils
    t = T.AffineCouplingTransform(torchutils.create_alternating_binary_mask(48),
                                  lambda i, o: ResidualNet(i, o, hidden_features=64, num_blocks=2)).eval()
    t.load_state_dict(r["sd"], strict=True)
    y, lad = t(r["x"])
    assert emu_step.get("trunk_step", 0) == 1 and emu_step.get("affine_coupling_final", 0) == 1 and emu_step.get("linear_f16x3", 0) == 0
    assert rel_err(y, r["y_fp64"].float()) <= max(TOL, 3 * rel_err(r["y"], r["y_fp64"].float()))
    assert rel_err(lad, r["lad_fp64"].float()) <= max(TOL, 3 * rel_err(r["lad"], r["lad_fp64"].float()))


@torch.no_grad()
@pytest.mark.parametrize("rows", [0, 1, 129])
def test_ragged_and_empty_batches_through_the_native_chain(emu_step, rows):
    """Row blocking with no rows, one row and one row more than a tile: shapes, dtypes and values of the native chain."""
    torch.manual_seed(1)
    flow = recipes.perturb_(recipes.rq_nsf(32, hidden_features=32, num_layers=2)).eval()
    x = torch.randn(rows, 32)
    got = flow.log_prob(x)
    assert got.shape == (rows,) and got.dtype == torch.float32
    if rows:        # (the torch formulation, like the reference, cannot reshape an empty parameter tensor: no comparison for 0 rows)
        want = flow.double().log_prob(x.double()).float()
        flow.float()
        assert rel_err(got, want) <= TOL
        z, lad = flow._transform(x)
        back, lad_back = flow._transform.inverse(z)
        assert rel_err(back, x) <= 1e-4 and rel_err(lad_back, -lad) <= 1e-4
