"""The operands the native path derives from parameters (dense.derived) on the CPU stand-ins of tests/emulated_kernels.py: a
repeat call reuses them, a parameter update / a `.data` write followed by invalidate_native_caches() / a train-eval switch
rebuilds them, superseded operands are released and a deleted transform takes its operands with it."""
import gc
import weakref

import pytest
import torch

import emulated_kernels as EK
from conftest import rel_err
from nflows_b200 import config
from nflows_b200 import dense as D
from nflows_b200 import invalidate_native_caches
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.flows import recipes
from nflows_b200.nn.nets import ResidualNet
from nflows_b200.utils import torchutils

#: entries derived from buffers only (index tensors, column layouts): a parameter update keeps them
STRUCTURAL = {"_col_index", "_layout", "_all_cols", "_index", "_inverse_index", "_t_cols"}


@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    monkeypatch.setattr(config, "coupling_block_rows", 128)
    return EK.install(monkeypatch)


def _perturbed(t, seed=3):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in t.parameters():
            p.add_(0.1 * torch.randn(p.shape, generator=g))
    return t.eval()


def _maf_rq(context=None):
    return T.MaskedPiecewiseRationalQuadraticAutoregressiveTransform(features=16, hidden_features=32, context_features=context,
                                                                     num_bins=8, tails="linear", tail_bound=3.0)


def _maf_affine(features, context=None):
    return T.MaskedAffineAutoregressiveTransform(features=features, hidden_features=32, context_features=context)


def _rq_coupling(context=None):
    return T.PiecewiseRationalQuadraticCouplingTransform(
        mask=torchutils.create_alternating_binary_mask(16, even=True),
        transform_net_create_fn=lambda i, o: ResidualNet(i, o, hidden_features=32, context_features=context, num_blocks=2),
        num_bins=8, tails="linear", tail_bound=3.0)


def _affine_run():
    return T.CompositeTransform([T.ActNorm(16), T.RandomPermutation(16), T.LULinear(16, identity_init=False)])


def _image_flow():
    return recipes.perturb_(recipes.glow_multiscale(image_shape=(3, 8, 8), levels=2, steps=1, hidden_channels=32)).eval()._transform


# name: (transform, input shape, context width, entries it must hold, stand-in that must have run)
CASES = {
    "maf_rq": (lambda: _perturbed(_maf_rq()), (100, 16), None,
               {"_masked_weight", "_step_plan", "_pack_spline", "_subnets", "_spline_head"}, "rq_coupling_step"),
    "maf_affine": (lambda: _perturbed(_maf_affine(5)), (100, 5), None,
                   {"_masked_weight", "_padded_chain", "_step_plan", "_ar_affine", "_subnets"}, "affine_ar_step"),
    "maf_affine_context": (lambda: _perturbed(_maf_affine(16, context=5)), (200, 16), 5,
                           {"_masked_weight", "_step_plan", "_ar_affine", "_subnets", "_context_projection",
                            "_sorted_context_projection"}, "affine_ar_step"),
    "rq_coupling": (lambda: _perturbed(_rq_coupling()), (100, 16), None,
                    {"_step_plan", "_pack_spline", "_spline_head", "_layout", "_col_index"}, "rq_coupling_step"),
    "rq_coupling_context": (lambda: _perturbed(_rq_coupling(context=6)), (200, 16), 6,
                            {"_ctx_parts", "_split", "_pack_spline", "_spline_head"}, "rq_coupling_final"),
    "image_flow": (_image_flow, (4, 3, 8, 8), None, {"_dense_mats", "_split", "_pack_spline", "_affine_run", "_inverse_affine_run"},
                   "im2col3x3"),
    "affine_run": (lambda: _perturbed(_affine_run()), (100, 16), None, {"_affine_run", "_inverse_affine_run", "_split"},
                   "linear_f16x3"),
    "permutation": (lambda: T.RandomPermutation(16), (100, 16), None, {"_index", "_inverse_index"}, "gather_cols"),
}


def _objects(v, out):
    """Tensors and plain objects inside a cached value (which may own entries of their own)."""
    if isinstance(v, (tuple, list)):
        for x in v:
            _objects(x, out)
    elif isinstance(v, dict):
        _objects(list(v.values()), out)
    elif isinstance(v, K.Pair16):
        out += [v.hi, v.lo]
    elif torch.is_tensor(v) or (hasattr(v, "__dict__") and not isinstance(v, torch.nn.Module)):
        out.append(v)


def operands(t):
    """{(id(owner), name): value} of every dense.derived entry of t: on its modules and parameters and, transitively, on the
    tensors and objects those entries hold."""
    found, seen = {}, set()
    todo = list(t.modules()) + list(t.parameters())
    while todo:
        o = todo.pop()
        if id(o) in seen:
            continue
        seen.add(id(o))
        table = D._TENSOR_ENTRIES.get(o, {}) if torch.is_tensor(o) else vars(o)
        for name, e in list(table.items()):
            if isinstance(e, tuple) and len(e) == 3 and isinstance(e[0], tuple) and isinstance(e[2], list):
                found[(id(o), name)] = e[1]
                _objects(e[1], todo)
        if not torch.is_tensor(o) and not isinstance(o, torch.nn.Module):
            _objects(list(vars(o).values()), todo)
    return found


def _run(t, x, c, make):
    """Forward, and inverse of its output, native (no grad) against the torch path (grad on: the parameters need a gradient),
    and bit for bit against a new transform with the same state, whose operands are all built afresh."""
    with torch.no_grad():
        y, lad = t(x, context=c)
        got = (y, lad), t.inverse(y, context=c)
        epoch = config.cache_epoch
        fresh = make()                 # its .eval() bumps the cache epoch, which must not rebuild t's operands here
        config.cache_epoch = epoch
        fresh.load_state_dict(t.state_dict())
        same = fresh(x, context=c), fresh.inverse(y, context=c)
    with torch.enable_grad():
        want = t(x, context=c), t.inverse(y, context=c)
    for (out, l), (out_ref, l_ref), (out_new, l_new), tol in zip(got, want, same, (3e-5, 3e-4)):
        assert rel_err(out, out_ref.detach()) <= tol and rel_err(l, l_ref.detach()) <= tol
        assert torch.equal(out, out_new) and torch.equal(l, l_new)


def _new_values(before, after):
    """Names of the entries in `after` whose value is not one of `before`'s (values that are singletons, None or a bool,
    cannot tell)."""
    old = {id(v) for v in before.values()}
    return {name for (_, name), v in after.items() if v is not None and not isinstance(v, bool) and id(v) not in old}


def _mutate_in_place(t):
    with torch.no_grad():
        for p in t.parameters():
            p.add_(1e-3)


def _mutate_data(t):
    for p in t.parameters():
        p.data.add_(1e-3)              # a write through .data does not bump the version counter
    invalidate_native_caches()


def _train_eval(t):
    t.train()
    t.eval()


@pytest.mark.parametrize("case", sorted(CASES))
def test_operands_are_reused_and_rebuilt(emu, case):
    make, shape, ctx, names, kernel = CASES[case]
    torch.manual_seed(0)
    t = make()
    x = torch.randn(*shape)
    c = None if ctx is None else torch.randn(shape[0], ctx)
    _run(t, x, c, make)
    assert emu.get(kernel, 0) > 0
    first = operands(t)
    assert names <= {name for _, name in first}, sorted({name for _, name in first})
    _run(t, x, c, make)
    again = operands(t)
    assert again.keys() == first.keys() and all(again[k] is v for k, v in first.items())
    for mutate, kept in ((_mutate_in_place, STRUCTURAL), (_mutate_data, set()), (_train_eval, set())):
        before = operands(t)
        mutate(t)
        _run(t, x, c, make)
        after = operands(t)
        rebuilt = _new_values(before, after)
        everything = {name for (_, name), v in after.items() if v is not None and not isinstance(v, bool)}
        assert rebuilt == everything - kept, (mutate.__name__, sorted(everything - kept - rebuilt))


def _maf_handles(t, rq):
    """Weakrefs to the forward's StepPlan, the packed final layer's .hi, the inverse's sorted pack .hi and the masked weights."""
    net = t.autoregressive_net
    chain = net.dense_chain(None) if rq else net.padded_chain(None)
    w, b = chain[-1][0], chain[-1][1]
    pack_final = t._pack_final if rq else D.ar_affine_operands
    return [weakref.ref(o) for o in (D.step_plan(chain), pack_final(w, b)[0].hi, net.sorted_subnets(chain, pack_final)[2].hi,
                                     chain[0][0], w)]


@pytest.mark.parametrize("rq", [True, False], ids=["maf_rq", "maf_affine"])
def test_superseded_operands_are_released(emu, rq):
    torch.manual_seed(0)
    t = _perturbed(_maf_rq() if rq else _maf_affine(16))
    x = torch.randn(64, 16)
    with torch.no_grad():
        t(x), t.inverse(x)
        refs = _maf_handles(t, rq)
        for cycle in range(3):
            _mutate_in_place(t)
            t(x), t.inverse(x)
    gc.collect()
    assert [r() is None for r in refs] == [True] * len(refs)


@pytest.mark.parametrize("case", sorted(CASES))
def test_deleting_a_transform_frees_its_operands(emu, case):
    make, shape, ctx, _, _ = CASES[case]
    torch.manual_seed(0)
    t = make()
    x = torch.randn(*shape)
    with torch.no_grad():
        t(x, context=None if ctx is None else torch.randn(shape[0], ctx))
    held = []
    _objects(list(operands(t).values()), held)
    refs = [weakref.ref(o) for o in held]
    assert refs
    del t, held
    gc.collect()
    assert sum(r() is not None for r in refs) == 0
