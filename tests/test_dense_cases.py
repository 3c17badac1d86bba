"""Without a GPU: every branch of the split-fp16 dense layer that _dense_cases.BRANCHES names is reached by a case of the table, on
the H100 SXM (132 SMs) and PCIe (114 SMs), by the launcher's own formulas."""
import pytest

import _dense_cases as D


@pytest.mark.parametrize("sm_count", [132, 114])
def test_every_branch_is_reached(sm_count):
    hit = set().union(*(D.plan(c, sm_count) for c in D.CASES))
    assert D.BRANCHES - hit == set()


def test_case_ids_are_unique_and_shapes_are_launchable():
    assert len({c.id for c in D.CASES}) == len(D.CASES)
    for c in D.CASES:
        assert c.k % 8 == 0 and c.n >= 1 and c.o >= 1, c.id                 # nfk_linear_f16x3_supported
        assert 0 <= c.split_cols <= c.o and 0 <= c.y_first_col < c.o, c.id
        assert not (c.residual and c.out == "pair" and c.relu_out), c.id


def test_plan_follows_the_launcher():
    one = D.case("x", 128 * 132 + 1, 192, 128)
    assert "tiles>ctas" in D.plan(one, 132) and "ring_phase_across_tiles" not in D.plan(one, 132)   # num_k = 6: phase realigns
    assert "tiles>ctas" not in D.plan(D.case("x", 128 * 132, 200, 128), 132)
    assert D.dest_geometry("vec", 7, 4) == (8, 0, 0) and D.dest_geometry("odd_ld", 8, 2) == (9, 0, 0)
    assert D.dest_geometry("odd_col", 7, 2) == (10, 1, 2)
