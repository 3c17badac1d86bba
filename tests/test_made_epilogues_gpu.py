"""The mixture and affine epilogues of the coupling-step kernel on the H100, called through their wrappers
(kernels.mog_made_step, kernels.affine_ar_step) against fp64: every mixture instance at every tile class in both modes, the affine
tile and group remainders in both directions, the crafted parameter table at every instance and three epsilons, and the C-ABI
contract of both entry points (tests/_made_epilogue_cases.py holds the table)."""
import pytest
import torch

import _made_epilogue_cases as E
from _coupling_checks import timeline

pytestmark = pytest.mark.gpu

EPSILONS = (1e-4, 1e-2, 0.5)


def report(what, e, r, floor=E.FLOOR):
    """The sandwich, with the error's share of its bar printed (pytest -s) for the record."""
    print("sandwich {} {:.3g} (kernel {:.3g}, fp32 {:.3g})".format(what, E.ratio(e, r, floor), e, r))
    return e <= max(floor, 3 * r)


# ---- shape matrix ---------------------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("mode", E.MODES)
@pytest.mark.parametrize("case", E.MOG_CASES, ids=lambda c: c.name)
def test_mixture_shapes(cuda_device, case, mode):
    with timeline() as tags:
        flags, e, r = E.run_mog_case(case, mode, cuda_device)
    assert tags.count("mog_made_step") == 1
    assert flags == 0
    assert report("mp{} {} {}".format(case.mp, mode, case.name), e, r), (e, r)


@torch.no_grad()
@pytest.mark.parametrize("inverse", [False, True], ids=["forward", "inverse"])
@pytest.mark.parametrize("case", E.AFFINE_CASES, ids=lambda c: c.name)
def test_affine_shapes(cuda_device, case, inverse):
    with timeline() as tags:
        (ey, ry), (el, rl), flags = E.run_affine_case(case, inverse, cuda_device)
    assert tags.count("affine_ar_step") == 1
    assert flags == 0
    assert report("affine y {}".format(case.name), ey, ry) and report("affine lad {}".format(case.name), el, rl), (ey, ry, el, rl)


# ---- crafted parameters -----------------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("epsilon", EPSILONS)
@pytest.mark.parametrize("c", E.crafted_components())
def test_mixture_crafted(cuda_device, c, epsilon):
    """Every crafted vector alone (d_t = 1) and all together, in both modes; the boundary draws exactly."""
    with timeline() as tags:
        out, misses = E.run_mog_crafted(c, epsilon, cuda_device)
    assert tags.count("mog_made_step") == len(out)
    assert not misses, misses
    mp = E.K.mog_made_padded_rows(c)
    for what, (flags, e, r) in out.items():
        assert flags == 0, what
        assert report("mp{} crafted c{} eps{} {}".format(mp, c, epsilon, what), e, r), (what, e, r)


@torch.no_grad()
@pytest.mark.parametrize("inverse", [False, True], ids=["forward", "inverse"])
def test_affine_crafted(cuda_device, inverse):
    t, x = E.affine_crafted()
    with timeline() as tags:
        (ey, ry), (el, rl), flags = E.run_affine(t, x, inverse, cuda_device)
    assert tags.count("affine_ar_step") == 1 and flags == 0
    assert report("affine crafted y", ey, ry) and report("affine crafted lad", el, rl), (ey, ry, el, rl)


# ---- the C-ABI contract -------------------------------------------------------------------------------------------------------
SENTINEL = -1234.5
N, BIG, FEATURES, COMPONENTS, C0, DT, PAD = 129, 300, 12, 7, 3, 6, 3    # C = 7: MP = 24, TF = 4; features 3 .. 8: two tiles


def _wide(x, pad, device):
    """x as a column view (columns pad .. pad + width - 1) of a wider sentinel-filled tensor on the device."""
    w = torch.full((x.shape[0], x.shape[1] + 2 * pad - 1), SENTINEL, device=device)
    w[:, pad:pad + x.shape[1]] = x.to(device)
    return w, w[:, pad:pad + x.shape[1]]


def _outside_untouched(buf, rows, col0, col1):
    """Every element of buf outside rows [0, rows) x columns [col0, col1) still holds the sentinel."""
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[:rows, col0:col1] = False
    return bool((buf[keep] == SENTINEL).all())


@torch.no_grad()
@pytest.mark.parametrize("mode", E.MODES)
def test_mixture_wrapper_contract(cuda_device, mode):
    """n = 129 rows into 300-row buffers, features C0 .. C0 + DT - 1 (t_col0 > 0, d_t > 1) of column views of wider tensors;
    log_prob adds to a prefilled lad_accum, sample writes only its columns of a separate y."""
    m = E.mog_model(FEATURES, 160, COMPONENTS, seed=5)
    x = E.inputs(BIG, FEATURES, 7)
    truth = E.MogTruth(m, x[:N])
    m = m.to(cuda_device)
    _, xd = _wide(x, 2, cuda_device)
    prefill = torch.randn(N, generator=torch.Generator().manual_seed(5))
    with timeline() as tags:
        if mode == "log_prob":
            ladbuf = torch.full((BIG,), SENTINEL, device=cuda_device)
            ladbuf[:N] = prefill.to(cuda_device)
            flags = E.mog_launch(m, xd[:N], (C0, DT), mode, lad=ladbuf[:N])
            want, yard = truth.log_prob(C0, DT)
            assert bool((ladbuf[N:] == SENTINEL).all()), "rows past n_rows were written"
            assert report("contract log_prob", *E.within(ladbuf[:N], prefill.double() + want, prefill + yard)[1:])
        else:
            u, e = E.noise(BIG, DT, 9)
            uw, ud = _wide(u, 1, cuda_device)
            ew, ed = _wide(e, 1, cuda_device)
            ybuf, y = _wide(torch.full((BIG, FEATURES), SENTINEL), PAD, cuda_device)
            flags = E.mog_launch(m, xd[:N], (C0, DT), mode, y=y[:N], noise=(ud[:N], ed[:N]))
            y64, y32, margin = truth.sample(u[:N], e[:N], C0, DT)
            keep = margin > E.MARGIN
            got = y[:N, C0:C0 + DT].cpu()
            assert _outside_untouched(ybuf, N, PAD + C0, PAD + C0 + DT), "y was written outside rows < n and its columns"
            assert report("contract sample", *E.within(got[keep], y64[keep], y32[keep])[1:])
    assert int(flags.item()) == 0 and tags.count("mog_made_step") == 1


@torch.no_grad()
@pytest.mark.parametrize("inverse", [False, True], ids=["forward", "inverse"])
def test_affine_wrapper_contract(cuda_device, inverse):
    """As the mixture's, plus in place (y is x): the same bits, the other columns as they were, the same log|det|."""
    t = E.affine_model(FEATURES, 160, seed=5)
    x = E.inputs(BIG, FEATURES, 7)
    (y64, l64), (y32, l32) = E.affine_truth(t, x[:N], inverse)
    t = t.to(cuda_device)
    _, xd = _wide(x, 2, cuda_device)
    prefill = torch.randn(N, generator=torch.Generator().manual_seed(5))
    ybuf, y = _wide(torch.full((BIG, FEATURES), SENTINEL), PAD, cuda_device)
    ladbuf = torch.full((BIG,), SENTINEL, device=cuda_device)
    ladbuf[:N] = prefill.to(cuda_device)
    cols = slice(C0, C0 + DT)
    with timeline() as tags:
        flags = E.affine_launch(t, xd[:N], (C0, DT), y[:N], ladbuf[:N], inverse)
    assert int(flags.item()) == 0 and tags.count("affine_ar_step") == 1
    assert _outside_untouched(ybuf, N, PAD + C0, PAD + C0 + DT), "y was written outside rows < n and its columns"
    assert bool((ladbuf[N:] == SENTINEL).all()), "rows past n_rows were written"
    assert report("contract affine y", *E.within(y[:N, cols], y64[:, cols], y32[:, cols])[1:])
    assert report("contract affine lad", *E.within(ladbuf[:N], prefill.double() + l64[:, cols].sum(-1),
                                                   prefill + l32[:, cols].sum(-1))[1:])
    x_in, lad_in = xd[:N].clone(), prefill.to(cuda_device)
    E.affine_launch(t, x_in, (C0, DT), x_in, lad_in, inverse)
    assert torch.equal(x_in[:, cols], y[:N, cols]) and torch.equal(x_in[:, :C0], xd[:N, :C0])
    assert torch.equal(x_in[:, C0 + DT:], xd[:N, C0 + DT:]) and torch.equal(lad_in, ladbuf[:N])


LARGE = 2 * 132 * 128 + 300          # more row tiles than one launch round of 132 CTAs


@torch.no_grad()
@pytest.mark.parametrize("n", [1, 64, 128, 129, LARGE])
def test_row_counts(cuda_device, n):
    m = E.mog_model(FEATURES, 64, COMPONENTS, seed=6)
    t = E.affine_model(FEATURES, 64, seed=6)
    x = E.inputs(n, FEATURES, n)
    truth = E.MogTruth(m, x)
    aff = [E.affine_truth(t, x, inv) for inv in (False, True)]
    m, t, xd = m.to(cuda_device), t.to(cuda_device), x.to(cuda_device)
    with timeline() as tags:
        lad = torch.zeros(n, device=cuda_device)
        assert int(E.mog_launch(m, xd, (0, FEATURES), "log_prob", lad=lad).item()) == 0
        assert report("rows {} log_prob".format(n), *E.within(lad, *truth.log_prob(0, FEATURES))[1:])
        u, e = E.noise(n, FEATURES, n + 1)
        y = torch.zeros_like(xd)
        assert int(E.mog_launch(m, xd, (0, FEATURES), "sample", y=y, noise=(u.to(cuda_device), e.to(cuda_device))).item()) == 0
        y64, y32, margin = truth.sample(u, e, 0, FEATURES)
        keep = margin > E.MARGIN
        assert report("rows {} sample".format(n), *E.within(y.cpu()[keep], y64[keep], y32[keep])[1:])
        for inverse, ((ya, la), (yb, lb)) in zip((False, True), aff):
            y, lad = torch.zeros_like(xd), torch.zeros(n, device=cuda_device)
            assert int(E.affine_launch(t, xd, (0, FEATURES), y, lad, inverse).item()) == 0
            assert report("rows {} affine y".format(n), *E.within(y, ya, yb)[1:])
            assert report("rows {} affine lad".format(n), *E.within(lad, la.sum(-1), lb.sum(-1))[1:])
    assert tags.count("mog_made_step") == 2 and tags.count("affine_ar_step") == 2


@torch.no_grad()
def test_batch_split_is_bit_identical(cuda_device):
    """Both epilogues sum a row's log|det| in a fixed order and a row's result does not depend on its row tile: rows
    [0, 10001) and [10001, n) in two launches give the bits of one launch."""
    n, cut = LARGE, 10001
    m = E.mog_model(FEATURES, 160, COMPONENTS, seed=8).to(cuda_device)
    t = E.affine_model(65, 96, seed=8).to(cuda_device)
    x = E.inputs(n, FEATURES, 3).to(cuda_device)
    xa = E.inputs(n, 65, 4).to(cuda_device)
    u, e = (v.to(cuda_device) for v in E.noise(n, FEATURES, 5))
    parts = [(0, n)], [(0, cut), (cut, n)]

    def mog(mode):
        outs = []
        for blocks in parts:
            out = torch.zeros(n, device=cuda_device) if mode == "log_prob" else torch.zeros(n, FEATURES, device=cuda_device)
            for r0, r1 in blocks:
                if mode == "log_prob":
                    E.mog_launch(m, x[r0:r1], (0, FEATURES), mode, lad=out[r0:r1])
                else:
                    E.mog_launch(m, x[r0:r1], (0, FEATURES), mode, y=out[r0:r1], noise=(u[r0:r1], e[r0:r1]))
            outs.append(out)
        return outs

    def affine(inverse):
        outs = []
        for blocks in parts:
            y, lad = torch.zeros_like(xa), torch.zeros(n, device=cuda_device)
            for r0, r1 in blocks:
                E.affine_launch(t, xa[r0:r1], (0, 65), y[r0:r1], lad[r0:r1], inverse)
            outs.append((y, lad))
        return outs

    with timeline() as tags:
        for mode in E.MODES:
            whole, split = mog(mode)
            assert torch.equal(whole, split), mode
        for inverse in (False, True):
            (yw, lw), (ys, ls) = affine(inverse)
            assert torch.equal(yw, ys) and torch.equal(lw, ls), inverse
    assert tags.count("mog_made_step") == 6 and tags.count("affine_ar_step") == 6
