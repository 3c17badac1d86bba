"""The coupling-step kernel's final layer around the depth of its weight ring (nflows_b200/csrc/nfk_coupling_step_tc.cu).  At
TILE = 96 (8 or 16 bins with linear tails) the ping-pong streams the final layer's slabs through a ring of its own, 4 slots over
the top of S and the trunk's ring, and reads each column tile's packed bias from shared memory, zero-filled past the last
feature; the TILE = 128 instances keep the trunk's 2-slot ring.

Column-tile counts 1 (the row-split path), 2, 3, 4, 5, 8, 9 and 98, with 2, 3 and 8 K-slabs per tile (fewer slabs than slots,
a ring that wraps inside a tile, every slot filled twice per tile); partial last column tiles; 1, 129 and 17 896 rows, and a
batch that gives every CTA at least two row tiles, so that the final ring's bytes change hands with the trunk repeatedly.
Forward and inverse, fp32 outputs and the fp16 pair.  The kernel is launched through the coupling's own step route on an input
whose identity columns come first, so any number of transformed features is reachable; each case is held to the fp64 oracle
with the sandwich of _coupling_checks.py and asserts from the launch timeline that rq_coupling_step ran."""
import pytest
import torch

import _coupling_checks as C
from conftest import rel_err
from nflows_b200 import dense as D
from nflows_b200 import kernels as K

pytestmark = pytest.mark.gpu

D_ID = 16
ROWS = (1, 129, 132 * 128 + 1000, 2 * 132 * 128 + 300)
TF = {(8, "linear"): 4, (16, "linear"): 2, (8, None): 4}    # transformed features per column tile (FusedCfg::TF)


def _case(bins, tails, d_t, hidden):
    nt = -(-d_t // TF[(bins, tails)])
    name = "k%d%s_t%d_f%d_h%d" % (bins, "t" if tails else "", nt, d_t, hidden)
    return C.Case(name, hidden, "res", 1, D_ID, d_t, bins, tails, "rq", "step", True)


CASES = (
    # TILE = 96, 8 bins: 8 K-slabs per column tile (two fills of every slot per tile)
    [_case(8, "linear", 4 * nt, 256) for nt in (1, 2, 3, 4, 5, 8, 9, 98)]
    # TILE = 96, 16 bins: 3 K-slabs (the ring wraps inside a tile)
    + [_case(16, "linear", 2 * nt, 96) for nt in (1, 2, 3, 4, 5, 8, 9, 98)]
    # partial last column tiles: zero-filled bias past d_t * MP
    + [_case(8, "linear", 33, 64), _case(16, "linear", 9, 256), _case(8, "linear", 390, 256)]
    # TILE = 128 (8 bins without tails): the trunk's 2-slot ring
    + [_case(8, None, 12, 256), _case(8, None, 36, 64), _case(8, None, 10, 96)]
)


def run_step(t, x, inverse, pair_out):
    """The coupling's step route on x ([identity | transformed] columns): (outputs of the transformed block, log|det|, tags)."""
    dev, n = x.device, x.shape[0]
    chain = t.transform_net.dense_chain(None)
    assert t._native_head(chain).route == "step"
    flags = K.new_flags(dev)
    y = x.clone()
    lad = torch.zeros(n, device=dev)
    a = K.Pair16.empty(n, D_ID, D.act_exp(), dev)
    K.split_f16(x[:, :D_ID], a.exp, out=a.cols(0, D_ID), flags=flags)
    y_pair = K.Pair16.empty(n, t.features, D.act_exp(), dev) if pair_out else None
    with C.timeline() as tags:
        t._native_fused(chain, y, a, (D_ID, t.features - D_ID), lad, flags, inverse, y_pair=y_pair)
    torch.cuda.synchronize()
    K.raise_for_flags(flags)
    if pair_out:
        assert torch.equal(y, x)                 # only the pair is written
        scale = 2.0 ** -y_pair.exp
        out = (y_pair.hi[:, D_ID:].float() * scale + y_pair.lo[:, D_ID:].float() * scale)
    else:
        assert torch.equal(y[:, :D_ID], x[:, :D_ID])
        out = y[:, D_ID:]
    return out, lad, tags


@torch.no_grad()
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_step_final_ring_depths_and_partial_tiles(cuda_device, case):
    t = C.build(case, seed=case.d_t + case.hidden + case.bins)
    ref = C.reference(case, t)
    t = t.to(cuda_device)
    for n in ROWS:
        x = C.inputs(case, n, seed=n + case.d_t)
        rows = torch.randperm(n, generator=torch.Generator().manual_seed(n))[:C.SUBSET] if n > C.SUBSET else torch.arange(n)
        xd = x.to(cuda_device)
        for inverse in (False, True):
            want, truth = ref(x[rows], inverse)
            tol_y, tol_l = C.sandwich(want, truth)
            fp32 = None
            for pair_out in (False, True):
                out, lad, tags = run_step(t, xd, inverse, pair_out)
                assert any(tag.startswith("rq_coupling_step") for tag in tags), (case.name, tags)
                assert not any(tag.startswith("rq_coupling_final") for tag in tags), (case.name, tags)
                got_y, got_l = out[rows.to(cuda_device)].cpu(), lad[rows.to(cuda_device)].cpu()
                what = (case.name, n, inverse, pair_out)
                assert rel_err(got_y, truth[0][:, D_ID:]) <= tol_y, what + (rel_err(got_y, truth[0][:, D_ID:]), tol_y)
                assert rel_err(got_l, truth[1]) <= tol_l, what + (rel_err(got_l, truth[1]), tol_l)
                if fp32 is None:
                    fp32 = (out, lad)
                else:                                # the pair is the split of the same fp32 outputs
                    assert torch.equal(lad, fp32[1]), what
                    assert rel_err(out, fp32[0]) <= 2.0 ** -20, what
