"""Glow / RealNVP-style image flows with affine and additive couplings (tests/golden/image_affine_rows.pt, reference outputs), on
the CPU: the torch formulation against the golden, the recipe's module tree and RNG order, the pixel-row chain's routes on the
kernel stand-ins of tests/emulated_kernels.py, and the flows the chain refuses."""
import pytest
import torch

import _image_affine_cases as C
import emulated_kernels
from conftest import rel_err
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.flows import recipes
from nflows_b200.nn.nets import ConvResidualNet
from nflows_b200.utils import torchutils

TOL = 1e-5


@pytest.fixture(scope="module")
def g():
    return C.golden()


@pytest.fixture
def emu(monkeypatch):
    # the inverse of the GENERAL_SCALE_ACTIVATION flow divides by scales down to 1e-3 and reaches |x| ~ 1e4: on the GPU the first
    # attempt leaves the fp16 split range and is repeated at smaller exponents (kernels.run_with_activation_rescale); the stand-ins
    # raise no flag, so they start at the exponent the repeats reach
    monkeypatch.setattr(config, "coupling_step_kernel", False)
    monkeypatch.setattr(config, "activation_exp", -4)
    return emulated_kernels.install(monkeypatch)


@pytest.fixture
def conditioner_calls(monkeypatch):
    """Counts forward calls of every ConvResidualNet: a coupling on its torch formulation runs its conditioner as a module."""
    calls = []
    forward = ConvResidualNet.forward

    def counted(self, inputs, context=None):
        calls.append(tuple(inputs.shape))
        return forward(self, inputs, context)
    monkeypatch.setattr(ConvResidualNet, "forward", counted)
    return calls


@torch.no_grad()
@pytest.mark.parametrize("key", C.CASES)
def test_torch_path_against_reference_golden(g, key):
    """The torch formulation (CPU) reproduces the reference's fp32 outputs."""
    r = g[key]
    flow = C.build(key, r)
    z, _ = flow._transform(r["x"])
    assert rel_err(z, r["z"]) <= 1e-6
    assert rel_err(flow.log_prob(r["x"]), r["log_prob"]) <= 1e-6
    xs, lad_inv = flow._transform.inverse(C.noise_input(flow, r))
    assert rel_err(xs, r["sample"]) <= 1e-6 and rel_err(lad_inv, r["lad_inv"]) <= 1e-6


def test_recipe_module_tree_and_seed(g):
    """glow_multiscale(coupling=...) has the reference's state_dict keys and shapes (a reference state_dict loads with strict=True)
    and, from a seed, the reference's weights; the default (RQ) coupling consumes the RNG as before."""
    for key in ("glow_affine", "glow_general", "glow_additive"):
        C.build(key, g[key])                         # keys, shapes and the perturbed weights' checksum from the seed
        reference_shaped = {k: torch.full(tuple(s), 0.5) for k, s in g[key]["shapes"]}
        C.unperturbed(key).load_state_dict(reference_shaped, strict=True)
    torch.manual_seed(g["rq_default_init"]["seed"])
    rq = recipes.glow_multiscale(image_shape=(3, 16, 16), levels=3, steps=2, hidden_channels=32)
    assert abs(C.weight_checksum(rq.state_dict()) - g["rq_default_init"]["checksum"]) <= 1e-9 * g["rq_default_init"]["checksum"]
    kinds = {type(m) for m in recipes.glow_multiscale(levels=1, steps=2, hidden_channels=8, coupling="additive").modules()}
    assert T.AdditiveCouplingTransform in kinds and T.PiecewiseRationalQuadraticCouplingTransform not in kinds
    with pytest.raises(ValueError):
        recipes.glow_multiscale(coupling="spline")


# couplings per case (forward): affine / additive heads and RQ heads
_COUPLINGS = {"glow_affine": (6, 0), "glow_general": (6, 0), "glow_additive": (6, 0), "glow_mixed": (2, 2), "flat_affine": (1, 0)}


@torch.no_grad()
@pytest.mark.parametrize("key", C.CASES)
def test_pixel_row_chain_routes_against_reference_golden(g, emu, conditioner_calls, key):
    """Each golden flow runs as pixel-row chains: NCHW -> rows, ConvChain trunk (im2col of the pair for the 3x3 layers), fused
    final layer + affine coupling, forward and inverse, and no leaf on the torch formulation."""
    r = g[key]
    flow = C.build(key, r)
    level = flow._transform._transforms[0] if isinstance(flow._transform, T.MultiscaleCompositeTransform) else flow._transform
    assert level._image_ready(r["x"], None)
    z, _ = flow._transform(r["x"])
    names = {name for name, _ in emu.trace}
    assert "nchw_to_rows" in names and "im2col3x3" in names and "affine_coupling_final" in names, names
    affine, rq = _COUPLINGS[key]
    assert emu.get("affine_coupling_final", 0) == affine and emu.get("rq_coupling_final", 0) == rq
    assert emu.get("affine_coupling_rows", 0) == 0 and emu.get("rqs_rows", 0) == 0 and not conditioner_calls
    assert rel_err(z, r["z_fp64"]) <= max(TOL, 3 * rel_err(r["z"], r["z_fp64"]))
    lp = flow.log_prob(r["x"])
    assert rel_err(lp, r["log_prob_fp64"]) <= max(TOL, 3 * rel_err(r["log_prob"], r["log_prob_fp64"]))
    emu.trace.clear()
    xs, lad_inv = flow._transform.inverse(C.noise_input(flow, r))
    assert "affine_coupling_final" in {name for name, _ in emu.trace} and not conditioner_calls
    assert rel_err(xs, r["sample_fp64"]) <= max(1e-4, 3 * rel_err(r["sample"], r["sample_fp64"]))
    assert rel_err(lad_inv, r["lad_inv_fp64"]) <= max(1e-4, 3 * rel_err(r["lad_inv"], r["lad_inv_fp64"]))


@torch.no_grad()
def test_gathered_and_packed_paths_and_whole_image_blocks(g, emu, monkeypatch):
    """glow_affine: levels 1 and 2 (6 of 12 and 12 of 24 channels: gathered identity columns, initial layer padded to 8 and 16),
    level 3 (24 of 48: the packed layout behind the folded ActNorm + 1x1 convolution, unpadded); small block sizes split the batch
    into whole-image row blocks without changing the result."""
    r = g["glow_affine"]
    flow = C.build("glow_affine", r)
    want = flow.log_prob(r["x"])
    rows = [n for name, n in emu.trace if name == "affine_coupling_final"]
    assert rows == [4 * 8 * 8] * 2 + [4 * 4 * 4] * 2 + [4 * 2 * 2] * 2, rows
    emu.trace.clear()
    monkeypatch.setattr(config, "coupling_block_rows", 128)
    monkeypatch.setattr(config, "trunk_block_rows", 128)
    got = flow.log_prob(r["x"])
    rows = [n for name, n in emu.trace if name == "affine_coupling_final"]
    # 64 pixels per image at level 1 (two images per 128-row block), 16 and 4 at levels 2 and 3 (all four images in one block)
    assert rows == [128] * 4 + [64] * 2 + [16] * 2, rows
    assert rel_err(got, want) <= 1e-6


@torch.no_grad()
def test_additive_coupling_adds_no_log_det(g, emu):
    """Additive couplings leave the per-pixel log|det| untouched: the flow's log|det| is the ActNorm + 1x1 convolution part."""
    r = g["glow_additive"]
    flow = C.build("glow_additive", r)
    _, lad = flow._transform(r["x"])
    assert rel_err(lad, -r["lad_inv_fp64"]) <= TOL          # the volume change does not depend on the input


def _refused(coupling, c=4):
    return T.CompositeTransform([T.ActNorm(c), coupling]).eval()


def _refusals():
    mask = torchutils.create_mid_split_binary_mask(4)
    own = lambda u: torch.sigmoid(u) + 0.5
    yield "custom scale activation", _refused(T.AffineCouplingTransform(mask, C.conv_net(), scale_activation=own)), None
    yield "unconditional transform", _refused(T.AffineCouplingTransform(mask, C.conv_net(),
                                                                        unconditional_transform=lambda features: T.ActNorm(features))), None
    yield "tanh conditioner", _refused(T.AffineCouplingTransform(mask, C.conv_net(activation=torch.tanh))), None
    yield "batch-norm conditioner", _refused(T.AdditiveCouplingTransform(mask, C.conv_net(use_batch_norm=True))), None
    yield "context conditioner", _refused(T.AffineCouplingTransform(mask, C.conv_net(context_channels=2))), \
        torch.randn(3, 2, 8, 8)
    yield "hidden channels not a multiple of 8", _refused(T.AffineCouplingTransform(mask, C.conv_net(hidden=12))), None
    yield "unknown leaf", T.CompositeTransform([T.ActNorm(4), T.ReversePermutation(4),
                                                T.AffineCouplingTransform(mask, C.conv_net())]).eval(), None


@torch.no_grad()
@pytest.mark.parametrize("case", [name for name, _, _ in _refusals()])
def test_refused_flows_keep_the_torch_path(emu, case):
    """Flows the pixel-row chain does not take are refused as a whole: torch path, no launch, the torch formulation's result."""
    torch.manual_seed(3)
    _, flow, context = next(item for item in _refusals() if item[0] == case)
    recipes.perturb_(flow)
    x = torch.randn(3, 4, 8, 8)
    assert not flow._image_ready(x, None)
    y, lad = flow(x, context)
    assert not emu.trace, emu.trace
    want = [t.float() for t in flow.double()(x.double(), None if context is None else context.double())]
    assert rel_err(y, want[0]) <= TOL and rel_err(lad, want[1]) <= TOL


def test_shapes_without_a_fused_route_are_refused(emu, monkeypatch):
    """No transformed channel (the fused final kernel takes d_t >= 1; the torch formulation cannot run it either), and
    config.fuse_coupling off (the affine head's route is then "rows", which image chains do not run)."""
    x = torch.randn(2, 4, 8, 8)
    assert C.flat_flow()._transform.eval()._image_ready(x, None)
    assert not _refused(T.AffineCouplingTransform(torch.zeros(4), C.conv_net()))._image_ready(x, None)
    monkeypatch.setattr(config, "fuse_coupling", False)
    assert not C.flat_flow()._transform.eval()._image_ready(x, None)
    assert not emu.trace

