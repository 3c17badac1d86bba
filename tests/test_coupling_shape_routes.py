"""Without a GPU: the support predicates of the fused coupling kernels at the boundaries test_coupling_shape_envelope.py relies
on, and the route every case of its table takes, decided on CPU-built couplings by the same code that decides it on a GPU --
so a wrong case (a shape that silently lands on another route) fails here first."""
import pytest

import _coupling_checks as C
from nflows_b200 import kernels as K


def test_step_kernel_support_boundaries():
    ok = lambda hidden=64, in_features=16, square=2, bins=8, tails="linear": K.rq_coupling_step_supported(
        bins, tails, hidden, in_features, square)
    assert ok(hidden=32) and ok(hidden=256) and ok(hidden=160) and ok(hidden=224)
    assert not ok(hidden=288) and not ok(hidden=48) and not ok(hidden=0)
    assert ok(in_features=8) and ok(in_features=392) and not ok(in_features=4) and not ok(in_features=12)
    assert ok(square=0) and ok(square=8) and not ok(square=9)
    assert all(ok(bins=b, tails=t) for b in (4, 8, 10, 16) for t in ("linear", None)) and not ok(bins=5)


def test_final_kernel_support_boundaries():
    ok = lambda hidden, bins=8, tails="linear": K.rq_coupling_final_supported(bins, tails, hidden, hidden)
    assert ok(40) and ok(72) and ok(288) and ok(512) and ok(1000) and ok(8)
    assert not ok(36) and not ok(4) and not ok(64, bins=5)


def test_every_spline_instance_meets_a_two_chunk_trunk_and_a_final_only_width():
    two_chunk = {(c.bins, c.tails) for c in C.STEP_CASES if c.hidden > 128}
    final_only = {(c.bins, c.tails) for c in C.FINAL_CASES + [C.WIDE_CASE]
                  if c.hidden > 256 or c.hidden % 32}
    every = {(b, t) for b in (4, 8, 10, 16) for t in ("linear", None)}
    assert two_chunk == every and final_only == every


@pytest.mark.parametrize("case", C.ALL_CASES, ids=lambda c: c.name)
def test_case_takes_its_route(case):
    t = C.build(case, seed=0)
    assert C.head_route(t) == (case.route, case.packed), case
    if case.kind == "rq":
        square = 2 * case.depth if case.net == "res" else case.depth - 1
        assert K.rq_coupling_step_supported(case.bins, case.tails, case.hidden, case.d_id, square) == (case.route == "step"), case
