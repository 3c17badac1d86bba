"""Glow / RealNVP-style image flows with affine and additive couplings on the H100: the pixel-row chain (nchw_to_rows, folded ActNorm
+ 1x1 convolution, ConvChain trunk with im2col 3x3 layers, nfk_affine_coupling_final_f16x3) against the reference goldens of
tests/golden/image_affine_rows.pt and against the torch formulation in fp64 across channels, sizes, widths and depths."""
import warnings

import pytest
import torch

import _image_affine_cases as C
from conftest import rel_err
from nflows_b200 import _native
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.distributions.normal import StandardNormal
from nflows_b200.flows import Flow
from nflows_b200.nn.nets import ConvResidualNet
from nflows_b200.utils import torchutils

pytestmark = pytest.mark.gpu
TOL = 1e-5


@pytest.fixture
def conditioner_calls(monkeypatch):
    """Forward calls of every ConvResidualNet: a coupling on its torch formulation runs its conditioner as a module."""
    calls = []
    forward = ConvResidualNet.forward

    def counted(self, inputs, context=None):
        calls.append(tuple(inputs.shape))
        return forward(self, inputs, context)
    monkeypatch.setattr(ConvResidualNet, "forward", counted)
    return calls


def traced(fn):
    """(fn(), tags of the tagged launches, native launches) of one call."""
    before = _native.launch_count()
    K.TIMELINE = []
    try:
        out = fn()
        tags = {t[0] for t in K.TIMELINE}
    finally:
        K.TIMELINE = None
    return out, tags, _native.launch_count() - before


@torch.no_grad()
@pytest.mark.parametrize("key", C.CASES)
def test_golden_flows_on_the_pixel_row_chain(cuda_device, conditioner_calls, key):
    """Reference goldens: forward z and log_prob under the fp64 sandwich, inverse / sample / lad_inv at the 1e-4 sandwich; the
    timeline shows the fused affine final kernel and no coupling on the torch formulation."""
    r = C.golden()[key]
    flow = C.build(key, r).to(cuda_device)
    x = r["x"].to(cuda_device)
    (z, _), tags, launches = traced(lambda: flow._transform(x))
    assert launches > 0 and {"nchw_to_rows", "im2col3x3_32", "affine_coupling_final"} <= tags, tags
    assert not conditioner_calls
    assert rel_err(z.cpu(), r["z_fp64"]) <= max(TOL, 3 * rel_err(r["z"], r["z_fp64"]))
    lp = flow.log_prob(x)
    assert rel_err(lp.cpu(), r["log_prob_fp64"]) <= max(TOL, 3 * rel_err(r["log_prob"], r["log_prob_fp64"]))
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)      # the general-scale inverse repeats at a smaller activation exponent
        (xs, lad_inv), tags, _ = traced(lambda: flow._transform.inverse(C.noise_input(flow, r).to(cuda_device)))
    assert "affine_coupling_final" in tags and not conditioner_calls
    assert rel_err(xs.cpu(), r["sample_fp64"]) <= max(1e-4, 3 * rel_err(r["sample"], r["sample_fp64"]))
    assert rel_err(lad_inv.cpu(), r["lad_inv_fp64"]) <= max(1e-4, 3 * rel_err(r["lad_inv"], r["lad_inv_fp64"]))
    if key == "glow_additive":
        _, lad = flow._transform(x)
        assert rel_err(lad.cpu(), -r["lad_inv_fp64"]) <= TOL          # no coupling term: the volume change is input-independent


def _glow(channels, size, hidden, num_blocks, kind, levels=2, steps=2):
    """levels x [squeeze, steps x [ActNorm, 1x1 convolution, affine / general / additive coupling]], perturbed."""
    net = lambda i_, o_: ConvResidualNet(i_, o_, hidden_channels=hidden, num_blocks=num_blocks)
    c, h, w = channels, size, size
    mct = T.MultiscaleCompositeTransform(num_transforms=levels)
    for _ in range(levels):
        squeeze = T.SqueezeTransform()
        c, h, w = squeeze.get_output_shape(c, h, w)
        layers = [squeeze]
        for i in range(steps):
            mask = torchutils.create_mid_split_binary_mask(c)
            if i % 2:
                mask = 1 - mask
            coupling = (T.AdditiveCouplingTransform(mask, net) if kind == "additive" else
                        T.AffineCouplingTransform(mask, net, **(dict(scale_activation=C.GENERAL) if kind == "general" else {})))
            layers.append(T.CompositeTransform([T.ActNorm(c), T.OneByOneConvolution(c), coupling]))
        shape = mct.add_transform(T.CompositeTransform(layers), (c, h, w))
        if shape is not None:
            c, h, w = shape
    return C.perturb(Flow(mct, StandardNormal([channels * size * size])), 7).eval()


@torch.no_grad()
@pytest.mark.parametrize("kind", ["affine", "general", "additive"])
@pytest.mark.parametrize("num_blocks", [1, 2])
@pytest.mark.parametrize("hidden", [32, 64, 96])
@pytest.mark.parametrize("size", [8, 16])
@pytest.mark.parametrize("channels", [3, 4, 6])
def test_sweep_against_the_torch_formulation_in_fp64(cuda_device, conditioner_calls, channels, size, hidden, num_blocks, kind):
    """Channels 3 / 4 / 6 (squeezed 12 / 16 / 24: padded and unpadded initial layers, gathered and packed paths), 8x8 and 16x16
    images, 32 / 64 / 96 hidden channels, 1 or 2 residual blocks: native forward and inverse against fp64 torch on the same weights."""
    torch.manual_seed(channels * 1000 + size * 100 + hidden + num_blocks)
    flow = _glow(channels, size, hidden, num_blocks, kind).to(cuda_device)
    x = torch.randn(5, channels, size, size, device=cuda_device)
    (lp, tags, _) = traced(lambda: flow.log_prob(x))
    assert "affine_coupling_final" in tags and not conditioner_calls, tags
    z = flow.transform_to_noise(x)
    noise = torch.randn(5, channels * size * size, device=cuda_device)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        xs, lad_inv = flow._transform.inverse(noise)
    flow.cpu()                                       # the torch formulation on the CPU: fp32 (inverse sandwich) and fp64
    x, noise = x.cpu(), noise.cpu()
    xs32, lad32 = flow._transform.inverse(noise)
    flow.double()
    want_lp = flow.log_prob(x.double())
    want_z = flow.transform_to_noise(x.double())
    want_xs, want_lad = flow._transform.inverse(noise.double())
    assert rel_err(lp.cpu(), want_lp) <= TOL and rel_err(z.cpu(), want_z) <= 3 * TOL
    # the inverse divides by scales down to 1e-3 and so amplifies the rounding of the conditioner's split-pair operands as it
    # amplifies the torch formulation's own: with GENERAL_SCALE_ACTIVATION (scales near the clamp) the native error was observed
    # at up to 6x the fp32 torch error (1.6e-2 against 2.6e-3 at channels 4, 16x16, hidden 96, 2 blocks)
    k = 10 if kind == "general" else 3
    assert rel_err(xs.cpu(), want_xs) <= max(2e-4, k * rel_err(xs32, want_xs))
    assert rel_err(lad_inv.cpu(), want_lad) <= max(2e-4, k * rel_err(lad32, want_lad))


@torch.no_grad()
def test_batch_split_and_whole_image_blocks(cuda_device, monkeypatch):
    """Images are independent: log_prob of a batch equals that of its halves, and small row blocks (several whole images each)
    give the same result."""
    r = C.golden()["glow_affine"]
    flow = C.build("glow_affine", r).to(cuda_device)
    x = torch.cat([r["x"]] * 6).to(cuda_device)                 # 24 images: 1536 rows at level 1
    lp = flow.log_prob(x)
    halves = torch.cat([flow.log_prob(x[:10]), flow.log_prob(x[10:])])
    assert rel_err(halves, lp) <= 1e-6
    monkeypatch.setattr(config, "coupling_block_rows", 128)
    monkeypatch.setattr(config, "trunk_block_rows", 256)
    blocked = flow.log_prob(x)
    assert rel_err(blocked, lp) <= 1e-6
    xs = flow._transform.inverse(torch.randn(24, 768, device=cuda_device))[0]
    assert torch.isfinite(xs).all()


@torch.no_grad()
@pytest.mark.parametrize("kind", ["affine", "additive"])
def test_activation_rescale_at_large_inputs(cuda_device, kind):
    """|x| ~ 1e4 leaves the fp16 split range at the default activation exponent: the call is repeated at smaller exponents and
    matches fp64."""
    torch.manual_seed(11)
    flow = _glow(4, 8, 32, 2, kind).to(cuda_device)
    x = 1e4 * torch.randn(3, 4, 8, 8, device=cuda_device)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        z, lad = flow._transform(x)
    flow.double()
    want_z, want_lad = flow._transform(x.double())
    assert rel_err(z, want_z) <= 1e-4 and rel_err(lad, want_lad) <= 1e-4


@torch.no_grad()
def test_round_trip_and_flow_sampling(cuda_device):
    """inverse(forward(x)) = x; Flow.sample / sample_and_log_prob shapes."""
    r = C.golden()["glow_mixed"]
    flow = C.build("glow_mixed", r).to(cuda_device)
    x = r["x"].to(cuda_device)
    z, lad = flow._transform(x)
    back, lad_back = flow._transform.inverse(z)
    assert rel_err(back, x) <= 1e-4 and rel_err(lad_back, -lad) <= 1e-4
    assert flow.sample(3).shape == (3, 4, 16, 16)
    s, lp = flow.sample_and_log_prob(4)
    assert s.shape == (4, 4, 16, 16) and lp.shape == (4,) and torch.isfinite(lp).all()
    flat = C.build("flat_affine", C.golden()["flat_affine"]).to(cuda_device)
    assert flat.sample(2).shape == (2, 4, 8, 8)
