"""The case table of the mixture and affine epilogues (tests/_made_epilogue_cases.py) on the CPU: each case has the layout it
claims, the cases together cover every mixture instance at every tile class in both modes and the affine remainders, the
crafted boundary draws pick what the kernel's rule picks, and the whole table passes its sandwich on the emulated kernels."""
import itertools

import numpy as np
import pytest
import torch

import _made_epilogue_cases as E
import emulated_kernels as EK
from nflows_b200 import config
from nflows_b200 import kernels as K


def test_each_mixture_case_has_the_layout_it_claims():
    for case in E.MOG_CASES:
        mp = K.mog_made_padded_rows(case.components)
        fpt = 128 // (2 * mp)                         # fused_spline.cuh: FusedCfg, BN = 128
        tiles = -(-case.features // (2 * fpt))
        assert (case.mp, case.tf, case.tiles) == (mp, 2 * fpt, tiles), case
        assert case.path == ("single" if tiles == 1 else "pingpong"), case
        partial = case.features % (2 * fpt) != 0
        assert {"one": tiles == 1 and not partial, "two": tiles == 2 and not partial, "odd": tiles >= 3 and tiles % 2 == 1,
                "partial": partial}[case.cls], case
        assert case.components in (E.components_of(mp)[0], E.components_of(mp)[-1]), case
        assert 2 * fpt * mp <= 128 and 3 * case.components <= mp


def test_the_mixture_cases_cover_every_instance_tile_class_and_mode():
    want = set(itertools.product(E.instances(), E.TILE_CLASSES, E.MODES))
    got = {(c.mp, c.cls, mode) for c in E.MOG_CASES for mode in E.MODES}
    assert got == want, sorted(want - got)
    assert E.instances() == [8, 16, 24, 32, 48, 56, 64]
    for mp in E.instances():
        cases = [c for c in E.MOG_CASES if c.mp == mp]
        assert {c.hidden for c in cases} == set(E.HIDDEN), mp
        assert {c.path for c in cases} == {"single", "pingpong"}, mp
        assert {c.components for c in cases} == {E.components_of(mp)[0], E.components_of(mp)[-1]}, mp
    # at one feature per thread, a partial last tile with an empty second half-row, on an odd feature count
    assert any(c.tf == 2 and c.cls == "partial" and c.features % 2 for c in E.MOG_CASES)


def test_the_affine_cases_cover_the_tile_and_group_remainders():
    for case in E.AFFINE_CASES:
        assert case.tiles == -(-case.features // 64) and case.group_rem == case.features % 8
    got = {(c.tiles, c.features % 64 == 0, c.group_rem, c.hidden) for c in E.AFFINE_CASES}
    for h in E.HIDDEN:
        for tiles in (1, 2, 3):
            assert any(t == tiles and hh == h for t, _, _, hh in got), (tiles, h)
        assert {(full, g) for _, full, g, hh in got if hh == h} >= {(True, 0), (False, 0), (False, 1), (False, 7)}, h


def test_boundary_draws_pick_what_the_rule_says():
    u = E.U_BOUNDARY
    four = E.boundary_logits(4)["quarters"]
    assert torch.equal(four, torch.zeros(4))
    assert [E.pick_fp32(four.numpy(), x) for x in u] == [0, 0, 1, 2, 3, 3]
    five = E.boundary_logits(5)
    assert [E.pick_fp32(five["quarters_zero_middle"].numpy(), x) for x in u] == [0, 0, 1, 3, 4, 4]
    assert [E.pick_fp32(five["quarters"].numpy(), x) for x in u] == [0, 0, 1, 2, 3, 3]      # the zero weight at the end
    # equal logits whose fp32 total stays below nextafter(1, 0): that u takes the C - 1 fallback
    fb = E.fallback_components()
    assert fb and all(K.mog_made_padded_rows(c) > 0 for c in fb)
    for c in fb:
        assert E.pick_fp32(np.zeros(c, np.float32), u[-1]) == c - 1
    assert fb[0] in E.crafted_components()
    # the fp64 rule of the truth agrees wherever the crafted weights are exact
    for c in E.crafted_components():
        for name, logits in E.boundary_logits(c).items():
            if name == "all_equal" and c not in (1, 2, 4):
                continue
            params = (logits.double().expand(len(u), c), torch.zeros(len(u), c, dtype=torch.float64),
                      torch.ones(len(u), c, dtype=torch.float64))
            _, comp, _ = E.mixture_draws(params, torch.tensor(u), torch.zeros(len(u)))
            assert comp.tolist() == [E.pick_fp32(logits.numpy(), x) for x in u], (c, name)


def test_crafted_vectors_are_exactly_what_they_name():
    v = E.mog_vectors(5)
    assert bool((v["uniform"][:, 0] == 0).all()) and float(v["dominant"][0, 0]) == 40.0
    assert float(v["underflow"][-1, 0]) == -200.0 and float(np.exp(np.float32(-200))) == 0.0
    assert torch.equal(v["twins"][0], v["twins"][1])
    assert E.NEAR_T[0] < 20.0 < E.NEAR_T[2] and np.float32(E.NEAR_T[0]) == np.nextafter(np.float32(20), np.float32(0))
    assert bool((v["far+1e3"][:, 1] == 1e3).all() and (v["far+1e3"][:, 2] == -30).all())
    a = E.affine_vectors()
    assert len(a) == len(E.AFFINE_U) * len(E.AFFINE_SHIFT)
    # the crafted model's final layer gives exactly the vector, whatever the input
    t, x = E.affine_crafted()
    with torch.no_grad():
        out = t.autoregressive_net(x)
    for j, vec in enumerate(a.values()):
        assert torch.equal(out[:, 2 * j:2 * j + 2], vec.expand(x.shape[0], 2))


@pytest.fixture
def emu(monkeypatch):
    monkeypatch.setattr(config, "coupling_step_kernel", True)
    return EK.install(monkeypatch)


@torch.no_grad()
@pytest.mark.parametrize("mode", E.MODES)
def test_mixture_shape_table_on_emulated_kernels(emu, mode):
    for case in E.MOG_CASES:
        flags, e, r = E.run_mog_case(case, mode, "cpu")
        assert flags == 0 and e <= max(E.FLOOR, 3 * r), (case.name, mode, e, r)
    assert emu["mog_made_step"] == len(E.MOG_CASES)


@torch.no_grad()
@pytest.mark.parametrize("c", [2, 5, 12])
def test_mixture_crafted_table_on_emulated_kernels(emu, c):
    out, misses = E.run_mog_crafted(c, 1e-2, "cpu")
    assert not misses, misses
    for what, (flags, e, r) in out.items():
        assert flags == 0 and e <= max(E.FLOOR, 3 * r), (c, what, e, r)


@torch.no_grad()
@pytest.mark.parametrize("inverse", [False, True])
def test_affine_tables_on_emulated_kernels(emu, inverse):
    for case in E.AFFINE_CASES[::4]:
        (ey, ry), (el, rl), flags = E.run_affine_case(case, inverse, "cpu")
        assert flags == 0 and ey <= max(E.FLOOR, 3 * ry) and el <= max(E.FLOOR, 3 * rl), (case.name, ey, ry, el, rl)
    t, x = E.affine_crafted()
    (ey, ry), (el, rl), _ = E.run_affine(t, x, inverse, "cpu")
    assert ey <= max(E.FLOOR, 3 * ry) and el <= max(E.FLOOR, 3 * rl), (ey, ry, el, rl)
