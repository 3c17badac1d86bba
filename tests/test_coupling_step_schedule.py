"""The final layer of the coupling-step kernel (nflows_b200/csrc/nfk_coupling_step_tc.cu) at the edges of its schedule: one column
tile (the row-split path), two, an odd number (warpgroup 0 takes one tile more than warpgroup 1) and the 98 of the cfg-3 shape;
1, 127, 129 rows and more rows than one launch round of 132 CTAs x 128 rows; forward and inverse; fp32 outputs and the fp16
pair a folded affine run multiplies; every bin count the kernel is instantiated for, with and without tails.  Each case is
held to the CPU oracle with the tolerances of test_native_parity.py (fp64 sandwich) and to the unfused route."""
import pytest
import torch

from _coupling_checks import step_launches
from conftest import rel_err
from nflows_b200 import config
from nflows_b200 import transforms as T
from nflows_b200.flows import recipes
from nflows_b200.nn.nets import ResidualNet
from oracle import flow_oracle as O

pytestmark = pytest.mark.gpu
TOL = 1e-5
ROWS = (1, 127, 129, 132 * 128 + 1000)
# transformed features per column tile of the final layer (fused_spline.cuh: FusedCfg::TF)
TF = {(4, "linear"): 8, (4, None): 8, (8, "linear"): 4, (8, None): 4, (10, "linear"): 4, (10, None): 4, (16, "linear"): 2,
      (16, None): 2}


def coupling(bins, tails, d_t, hidden, blocks, seed):
    torch.manual_seed(seed)
    mask = torch.cat([-torch.ones(16), torch.ones(d_t)])          # 16 identity features first, d_t transformed
    t = T.PiecewiseRationalQuadraticCouplingTransform(
        mask, lambda i, o: ResidualNet(i, o, hidden_features=hidden, num_blocks=blocks), num_bins=bins, tails=tails,
        tail_bound=2.5).eval()
    with torch.no_grad():
        for name, p in t.named_parameters():
            if "final_layer" in name:
                p.mul_(2.0)
    return t


def check_against_oracle_and_unfused(t, x, dev, monkeypatch, kw):
    sd = {k: v.detach().cpu().clone() for k, v in t.state_dict().items()}
    t = t.to(dev)
    xd = x.to(dev)
    counter = step_launches(monkeypatch)
    for inverse in (False, True):
        want_y, want_l = O.rq_coupling({k: v.clone() for k, v in sd.items()}, "", x, inverse=inverse, **kw)
        truth_y, truth_l = O.rq_coupling({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, "",
                                         x.double(), inverse=inverse, **kw)
        run = (lambda: t.inverse(xd)) if inverse else (lambda: t(xd))
        before = counter.fp32
        y1, l1 = run()
        assert counter.fp32 > before, "the coupling-step kernel did not run"
        config.fuse_coupling = False
        monkeypatch.setenv("NFLOWS_B200_GEMM", "simt")
        try:
            y2, l2 = run()
        finally:
            config.fuse_coupling = True
            monkeypatch.delenv("NFLOWS_B200_GEMM")
        tol_y = max(TOL, 3 * rel_err(want_y, truth_y))
        tol_l = max(3e-5, 5 * rel_err(want_l, truth_l))
        n = x.shape[0]
        assert rel_err(y1.cpu(), truth_y) <= tol_y, (n, inverse, rel_err(y1.cpu(), truth_y), tol_y)
        assert rel_err(l1.cpu(), truth_l) <= tol_l, (n, inverse, rel_err(l1.cpu(), truth_l), tol_l)
        # the unfused route is held to the same bar; the two routes differ by their own round-off only
        assert rel_err(y2.cpu(), truth_y) <= tol_y and rel_err(l2.cpu(), truth_l) <= tol_l, (n, inverse)
        assert rel_err(y1, y2) <= 2 * tol_y and rel_err(l1, l2) <= 2 * tol_l, (n, inverse)
        idf = sd["identity_features"].to(dev)
        assert torch.equal(y1[:, idf], xd[:, idf])


@torch.no_grad()
@pytest.mark.parametrize("d_t", [8, 16, 24])
@pytest.mark.parametrize("bins,tails", sorted(TF, key=lambda k: (k[0], k[1] is None)))
def test_step_final_layer_schedule(cuda_device, bins, tails, d_t, monkeypatch):
    """d_t / TF column tiles: 1, 2 and 3 at K = 4 (one tile takes the row-split path; three leave warpgroup 0 one tile more
    than warpgroup 1), 2, 4 and 6 at K = 8 and 10, 4, 8 and 12 at K = 16 (the step kernel takes 16 identity columns and a
    multiple of 8 transformed ones; the autoregressive inverse, one tile per launch, is test_native_parity.py's cfg-4 case).
    Every row count of ROWS, forward and inverse, against the fp64 oracle and the unfused route."""
    t = coupling(bins, tails, d_t, hidden=64, blocks=1, seed=10 * bins + d_t)
    kw = dict(num_bins=bins, tails=tails, tail_bound=2.5)
    for n in ROWS:
        g = torch.Generator().manual_seed(n)
        x = torch.rand(n, 16 + d_t, generator=g) if tails is None else torch.randn(n, 16 + d_t, generator=g) * 1.3
        check_against_oracle_and_unfused(t, x, cuda_device, monkeypatch, kw)


@torch.no_grad()
def test_step_final_layer_cfg3_shape(cuda_device, monkeypatch):
    """The cfg-3 coupling: H = 256, 2 residual blocks, K = 8 with tails, 392 transformed features = 98 column tiles."""
    torch.manual_seed(98)
    t = recipes.perturb_(recipes.rq_coupling_layer(784, 256, num_bins=8, tail_bound=3.0, num_blocks=2).eval())
    kw = dict(num_bins=8, tails="linear", tail_bound=3.0)
    for n in (129, 132 * 128 + 1000):
        x = torch.randn(n, 784, generator=torch.Generator().manual_seed(n)) * 1.3
        check_against_oracle_and_unfused(t, x, cuda_device, monkeypatch, kw)


@torch.no_grad()
@pytest.mark.parametrize("bins", [4, 8])
def test_step_final_layer_pair_outputs(cuda_device, bins, monkeypatch):
    """Couplings followed by a folded affine run write only the fp16 pair of their outputs.  48 features: 24 transformed = 3
    column tiles at K = 4, 6 at K = 8; the flow's log-density against the CPU oracle, every row count of ROWS."""
    torch.manual_seed(bins)
    flow = recipes.perturb_(recipes.rq_nsf(48, 64, 3, num_bins=bins).eval())
    sd = {k: v.clone() for k, v in flow.state_dict().items()}
    flow = flow.to(cuda_device)
    counter = step_launches(monkeypatch)
    for n in ROWS:
        x = torch.randn(n, 48, generator=torch.Generator().manual_seed(n)) * 1.3
        lp = flow.log_prob(x.to(cuda_device))
        want = O.flow_log_prob(sd, O.nsf_spec(3, num_bins=bins), x)
        assert rel_err(lp.cpu(), want) <= TOL, (n, rel_err(lp.cpu(), want))
    assert counter.pair > 0, "no coupling-step launch wrote the pair outputs"
