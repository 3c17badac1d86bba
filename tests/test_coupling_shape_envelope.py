"""The three fused coupling kernels across the shapes they accept, not only the bench's and the goldens':

  A. nfk_rq_coupling_step_f16x3: trunk widths 32 ... 256 (one 128-column chunk, and two chunks whose second is 32, 64, 96 or
     128 wide), 0 to 8 square layers (ResidualNet and MLP layer flags), conditioner inputs of 8 to 392 columns;
  B. nfk_rq_coupling_final_f16x3: the widths the step kernel refuses (288, 512, 1000, 40, 72), partial last column tiles on the
     gathered route, and the step kernel's own shapes with the step kernel switched off;
  C. nfk_affine_coupling_final_f16x3: several 128-column tiles, odd d_t, additive with an odd column count;
  D. the C-ABI contract of the three wrappers: rows at or past n_rows untouched, lad_accum read-modify-written, in-place and
     separate outputs, tails-free splines at and outside the ends of [0, 1].

Each case is held to an fp64 evaluation on the CPU (oracle/flow_oracle.py; the module's torch path for MLP conditioners) with the
fp64 sandwich of test_native_parity.py, forward and inverse, and proves from the launch timeline that the kernel it targets ran.
Batches of 1 row, 129 rows and more rows than one launch round; of the large batch, 1024 random rows are held to the reference
and the whole batch must equal the same batch run as two splits."""
import pytest
import torch

import _coupling_checks as C
from conftest import rel_err
from nflows_b200 import config
from nflows_b200 import dense as D
from nflows_b200 import kernels as K
from nflows_b200.flows import recipes
from nflows_b200.transforms.base import InputOutsideDomain
from oracle import flow_oracle as O

pytestmark = pytest.mark.gpu


def run_tagged(run, x):
    with C.timeline() as tags:
        y, lad = run(x)
    torch.cuda.synchronize()
    return y, lad, tags


def assert_route(case, tags):
    want, forbid = C.expected_tags(case)
    for w in want:
        assert any(t.startswith(w) for t in tags), (case.name, w, tags)
    for f in forbid:
        assert not any(t.startswith(f) for t in tags), (case.name, f, tags)


def check_case(case, t, ref, x, dev, tags_of=assert_route):
    """t (on dev) against ref on x, forward and inverse; returns the GPU results for further comparison."""
    n = x.shape[0]
    xd = x.to(dev)
    idf = t.identity_features
    rows = torch.randperm(n, generator=torch.Generator().manual_seed(n))[:C.SUBSET] if n > C.SUBSET else torch.arange(n)
    out = {}
    for inverse in (False, True):
        run = t.inverse if inverse else t
        y, lad, tags = run_tagged(run, xd)
        tags_of(case, tags)
        want, truth = ref(x[rows], inverse)
        tol_y, tol_l = C.sandwich(want, truth)
        got_y, got_l = y[rows.to(dev)].cpu(), lad[rows.to(dev)].cpu()
        assert rel_err(got_y, truth[0]) <= tol_y, (case.name, n, inverse, rel_err(got_y, truth[0]), tol_y)
        assert rel_err(got_l, truth[1]) <= tol_l, (case.name, n, inverse, rel_err(got_l, truth[1]), tol_l)
        assert torch.equal(y[:, idf], xd[:, idf]), (case.name, n, inverse)
        if n > C.SUBSET:
            s = 10001
            y1, l1 = run(xd[:s])
            y2, l2 = run(xd[s:])
            assert torch.equal(torch.cat([y1, y2]), y), (case.name, inverse)
            if case.kind == "rq":
                assert torch.equal(torch.cat([l1, l2]), lad), (case.name, inverse)
            else:
                # the affine kernel adds each column tile's log|det| share with atomics: the order of that sum is not fixed
                assert rel_err(torch.cat([l1, l2]), lad) <= 1e-6, (case.name, inverse)
        out[inverse] = (y, lad, tol_y, tol_l, truth)
    return out


def run_case(case, dev, seed, rows=C.ROWS):
    t = C.build(case, seed)
    ref = C.reference(case, t)
    t = t.to(dev)
    for n in rows:
        check_case(case, t, ref, C.inputs(case, n, seed + n), dev)


# ---- A. the coupling-step kernel ----------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("case", C.STEP_CASES, ids=lambda c: c.name)
def test_step_kernel_widths_depths_and_inputs(cuda_device, case):
    run_case(case, cuda_device, seed=case.hidden + case.depth + case.bins)


@torch.no_grad()
def test_step_kernel_pair_outputs_at_a_two_chunk_width(cuda_device, monkeypatch):
    """rq_nsf(48, 192, 3): each coupling is followed by a folded affine run, so the step kernel writes only the fp16 pair of
    its outputs, with a two-chunk trunk."""
    torch.manual_seed(192)
    flow = recipes.perturb_(recipes.rq_nsf(48, 192, 3).eval())
    sd = {k: v.clone() for k, v in flow.state_dict().items()}
    flow = flow.to(cuda_device)
    counter = C.step_launches(monkeypatch)
    for n in C.ROWS:
        x = torch.randn(n, 48, generator=torch.Generator().manual_seed(n)) * 1.3
        lp = flow.log_prob(x.to(cuda_device))
        want = O.flow_log_prob(sd, O.nsf_spec(3), x)
        assert rel_err(lp.cpu(), want) <= C.TOL, (n, rel_err(lp.cpu(), want))
    assert counter.pair > 0, "no coupling-step launch wrote the pair outputs"


# ---- B. the final-layer kernel ------------------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("case", C.FINAL_CASES, ids=lambda c: c.name)
def test_final_kernel_widths_and_partial_column_tiles(cuda_device, case):
    run_case(case, cuda_device, seed=case.hidden + case.d_t + case.bins)


@torch.no_grad()
def test_final_kernel_hidden_512_walks_98_column_tiles(cuda_device):
    run_case(C.WIDE_CASE, cuda_device, seed=512, rows=(129, 132 * 128 + 1000))


@torch.no_grad()
@pytest.mark.parametrize("name", ["h96", "h192a", "h224b"])
def test_final_kernel_agrees_with_the_step_kernel(cuda_device, name):
    """Step-capable shapes with config.coupling_step_kernel off: the trunk layer by layer, then the final-layer kernel.  Both
    routes meet the sandwich and agree with each other within twice of it."""
    case = next(c for c in C.STEP_CASES if c.name == name)

    def layer_by_layer(case, tags):
        assert any(tag.startswith("rq_coupling_final") for tag in tags), tags
        assert not any(tag.startswith(("rq_coupling_step", "trunk_step", "final_linear")) for tag in tags), tags

    t = C.build(case, seed=7)
    ref = C.reference(case, t)
    t = t.to(cuda_device)
    for n in C.ROWS:
        x = C.inputs(case, n, 7 + n)
        on = check_case(case, t, ref, x, cuda_device)
        config.coupling_step_kernel = False
        try:
            fin = check_case(case, t, ref, x, cuda_device, tags_of=layer_by_layer)   # the trunk-only launch is off too
        finally:
            config.coupling_step_kernel = True
        for inverse in (False, True):
            (y1, l1, tol_y, tol_l, _), (y2, l2, _, _, _) = on[inverse], fin[inverse]
            assert rel_err(y1, y2) <= 2 * tol_y and rel_err(l1, l2) <= 2 * tol_l, (name, n, inverse)


@torch.no_grad()
def test_final_kernel_pair_outputs_at_hidden_512(cuda_device, monkeypatch):
    torch.manual_seed(512)
    flow = recipes.perturb_(recipes.rq_nsf(48, 512, 3).eval())
    sd = {k: v.clone() for k, v in flow.state_dict().items()}
    flow = flow.to(cuda_device)
    counter = C.final_launches(monkeypatch)
    for n in C.ROWS:
        x = torch.randn(n, 48, generator=torch.Generator().manual_seed(n)) * 1.3
        lp = flow.log_prob(x.to(cuda_device))
        want = O.flow_log_prob(sd, O.nsf_spec(3), x)
        assert rel_err(lp.cpu(), want) <= C.TOL, (n, rel_err(lp.cpu(), want))
    assert counter.pair > 0, "no final-layer launch wrote the pair outputs"


# ---- C. the affine / additive final kernel ------------------------------------------------------------------------------
@torch.no_grad()
@pytest.mark.parametrize("case", C.AFFINE_CASES, ids=lambda c: c.name)
def test_affine_final_kernel_tiles_odd_columns_and_additive(cuda_device, case):
    run_case(case, cuda_device, seed=case.hidden + case.d_t)


# ---- D. the C-ABI contract of the wrappers ------------------------------------------------------------------------------
CONTRACT = {
    "step": C._rq("contract_step", 64, "res", 1, 16, 16, 8, "linear"),
    "final": C._rq("contract_final", 64, "res", 1, 16, 16, 8, "linear", "final"),
    "affine": C.Case("contract_affine", 64, "res", 1, 16, 16, None, None, "affine", "final", True),
}


def launch(route, t, xd, y, lad, flags, inverse):
    """One direct call of the route's wrapper on the rows of xd (identity columns first, transformed columns after them)."""
    d_id, d_t = t.num_identity_features, t.num_transform_features
    chain = t.transform_net.dense_chain(None)
    a = K.split_f16(xd[:, :d_id], D.act_exp())
    if route == "affine":
        trunk = D.run_trunk(chain, xd, None, True, x_pair=a).pair
        w, b = D.pack_final_affine(chain[-1][0], chain[-1][1], d_t, 2)
        K.affine_coupling_final(trunk, w, b, xd, (d_id, d_t), 2, 0, inverse, y, lad, flags)
        return
    head = D.SplineHead(chain, t, t._softmax_divisor(), d_t, d_id)
    wp, bias, _ = D.spline_operands(chain[-1][0], chain[-1][1], t.num_bins, t.tails, d_t)
    if route == "step":
        K.rq_coupling_step(D.step_plan(chain), a, head.desc, inverse, wp, bias, xd, (d_id, d_t), y, lad, flags)
    else:
        trunk = D.run_trunk(chain, xd, None, True, x_pair=a).pair
        cols = torch.arange(d_id, d_id + d_t, dtype=torch.int32, device=xd.device)
        K.rq_coupling_final(head.desc, inverse, trunk, wp, bias, xd, cols, y, lad, flags)


@torch.no_grad()
@pytest.mark.parametrize("route", ["step", "final", "affine"])
def test_wrapper_contract_rows_past_n_rows_lad_accum_and_in_place(cuda_device, route):
    case = CONTRACT[route]
    t = C.build(case, seed=3)
    ref = C.reference(case, t)
    t = t.to(cuda_device)
    n, big, d = 129, 300, case.d_id + case.d_t
    sentinel = -1234.5
    x = C.inputs(case, big, 11)
    xd = x.to(cuda_device)[:n]
    for inverse in (False, True):
        want, truth = ref(x[:n], inverse)
        tol_y, tol_l = C.sandwich(want, truth)
        ybuf = torch.full((big, d), sentinel, device=cuda_device)
        ladbuf = torch.full((big,), sentinel, device=cuda_device)
        prefill = torch.randn(n, generator=torch.Generator().manual_seed(5)).to(cuda_device)
        ladbuf[:n] = prefill
        flags = torch.zeros(1, dtype=torch.int32, device=cuda_device)
        launch(route, t, xd, ybuf[:n], ladbuf[:n], flags, inverse)
        torch.cuda.synchronize()
        assert int(flags.item()) == 0
        assert bool((ybuf[n:] == sentinel).all()) and bool((ladbuf[n:] == sentinel).all()), "rows past n_rows were written"
        assert bool((ybuf[:n, :case.d_id] == sentinel).all()), "the identity columns of a separate y were written"
        assert rel_err(ybuf[:n, case.d_id:].cpu(), truth[0][:, case.d_id:]) <= tol_y, (route, inverse)
        assert rel_err(ladbuf[:n].cpu(), prefill.cpu().double() + truth[1]) <= tol_l, (route, inverse)
        # in place: y is x; the same values, identity columns as they were
        x_in = xd.clone()
        lad_in = prefill.clone()
        launch(route, t, x_in, x_in, lad_in, flags, inverse)
        assert torch.equal(x_in[:, case.d_id:], ybuf[:n, case.d_id:]) and torch.equal(x_in[:, :case.d_id], xd[:, :case.d_id])
        if route == "affine":            # log|det| shares added with atomics: the order of the sum is not fixed
            assert rel_err(lad_in, ladbuf[:n]) <= 1e-6
        else:
            assert torch.equal(lad_in, ladbuf[:n])


@torch.no_grad()
@pytest.mark.parametrize("route", ["step", "final"])
def test_tails_free_spline_at_and_outside_the_ends_of_the_interval(cuda_device, route):
    """tails=None: inputs of exactly 0 and 1 are inside the domain and match the oracle; an input outside [0, 1] sets
    NFK_FLAG_OUTSIDE_DOMAIN, which raises InputOutsideDomain -- through the wrapper and through the coupling."""
    case = C._rq("ends_" + route, 64, "res", 1, 16, 16, 4, None, route)
    t = C.build(case, seed=4)
    ref = C.reference(case, t)
    t = t.to(cuda_device)
    x = C.inputs(case, 129, 12)
    x[::2, case.d_id::2] = 0.0
    x[1::2, case.d_id::2] = 1.0
    x[::3, case.d_id + 1::2] = 1.0
    xd = x.to(cuda_device)
    for inverse in (False, True):
        want, truth = ref(x, inverse)
        tol_y, tol_l = C.sandwich(want, truth)
        y = xd.clone()
        lad = torch.zeros(129, device=cuda_device)
        flags = torch.zeros(1, dtype=torch.int32, device=cuda_device)
        launch(route, t, xd, y, lad, flags, inverse)
        K.raise_for_flags(flags)
        assert rel_err(y.cpu(), truth[0]) <= tol_y and rel_err(lad.cpu(), truth[1]) <= tol_l, (route, inverse)
        for bad in (-1e-6, 1.0 + 1e-6, 3.0):
            xb = xd.clone()
            xb[64, case.d_id + 3] = bad
            flags.zero_()
            launch(route, t, xb, xb.clone(), torch.zeros(129, device=cuda_device), flags, inverse)
            with pytest.raises(InputOutsideDomain):
                K.raise_for_flags(flags)
        if route == "final":
            config.coupling_step_kernel = False
        try:
            with C.timeline() as tags, pytest.raises(InputOutsideDomain):
                (t.inverse if inverse else t)(xb)
        finally:
            config.coupling_step_kernel = True
        assert any(tag.startswith("rq_coupling_" + route) for tag in tags), tags
