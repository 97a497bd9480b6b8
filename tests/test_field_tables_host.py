"""Tables of arbitrary field elements on the CPU: the oracle proves and verifies strategies over them (oracle_custom's
_fr entry points), agrees byte for byte with the u32 entry points when every entry is below 2^32, and its dense MLE of
such a table agrees with Python integers; the Python description accepts (M, 4) tables and rejects bad ones."""
import ctypes
import os

import numpy as np
import pytest

import field_tables as ft
import oracle_custom_fr_lib as oc
import oracle_lib as ol
from test_custom_strategy_host import make_inputs

NGENS = 600


def _lb():
    import lasso_b200 as lb  # the description is pure Python: importing needs no GPU

    return lb


def test_fr_from_ints_is_montgomery_mod_l():
    lb = _lb()
    vals = [0, 1, -1, -5, 2**32, 2**252, ft.L_FR - 1, ft.L_FR, 3 * ft.L_FR + 7, -(2**300)]
    got = lb.fr_from_ints(vals)
    assert got.shape == (len(vals), 4) and got.dtype == np.uint64
    assert ol.fr_ints(got) == [v % ft.L_FR for v in vals]


@pytest.mark.parametrize("name", sorted(ft.INTS))
@pytest.mark.parametrize("C,log_m,degree", [(2, 4, 1), (1, 5, 2), (3, 4, 3)])
def test_oracle_verifies_field_tables(name, C, log_m, degree):
    """proof accepted; rejected with a tampered claimed evaluation or a tampered memory-checking evaluation"""
    S = ft.strategy(None, name, C, log_m, degree, nsub=2)
    assert S.fr_tables and S.num_memories == 2 * C
    idx, r, seed, s = make_inputs(C, log_m, 40, len(name) + C, False)
    gens = ol.generators(NGENS)
    assert oc.prove(S, idx, r, gens, seed, flags=1)["rc"] == 0
    assert oc.prove(S, idx, r, gens, seed, flags=1 | 2)["rc"] == 1
    assert oc.prove(S, idx, r, gens, seed, flags=1 | 4)["rc"] == 1


def test_oracle_u32_and_fr_entry_points_identical_below_2_32():
    lb = _lb()
    rng = np.random.default_rng(3)
    t = rng.integers(0, 2**32, size=1 << 6, dtype=np.uint64)
    t[0], t[1] = 2**32 - 1, 0
    g = ft.g_of_degree(2)
    S_u32 = lb.CustomStrategy(None, 2, 6, [t], g, 2)
    S_fr = lb.CustomStrategy(None, 2, 6, [lb.fr_from_ints(t.tolist())], g, 2)
    assert not S_u32.fr_tables and S_fr.fr_tables
    idx, r, seed, s = make_inputs(2, 6, 50, 9, False)
    gens = ol.generators(NGENS)
    a, b = oc.prove(S_u32, idx, r, gens, seed, flags=1), oc.prove(S_fr, idx, r, gens, seed, flags=1)
    assert a["rc"] == 0 and b["rc"] == 0
    assert a["commitment"] == b["commitment"] and a["proof"] == b["proof"]
    assert (a["challenges"] == b["challenges"]).all()


@pytest.mark.parametrize("name", sorted(ft.INTS))
def test_dense_mle_matches_python_integers(name):
    """evaluate_subtable_mle (point[0] the MSB) = sum_i T[i] eq(bits(i), point) mod l, and T[i] at Boolean points"""
    log_m = 5
    S = ft.strategy(None, name, 1, log_m)
    table = [v % ft.L_FR for v in ft.INTS[name](log_m)]
    rng = np.random.default_rng(len(name))
    for _ in range(3):
        point = ol.rand_fr(rng, log_m)
        x = ol.fr_ints(point)
        want = 0
        for i, v in enumerate(table):
            e = 1
            for b in range(log_m):
                bit = (i >> (log_m - 1 - b)) & 1
                e = e * (x[b] if bit else 1 - x[b]) % ft.L_FR
            want = (want + v * e) % ft.L_FR
        assert ol.fr_ints(oc.evaluate_subtable_mle(S, 0, point)) == [want]
    for i in (0, 7, (1 << log_m) - 1):
        boolean = ol.fr_array([(i >> (log_m - 1 - b)) & 1 for b in range(log_m)])
        assert ol.fr_ints(oc.evaluate_subtable_mle(S, 0, boolean)) == [table[i]]


def test_description_accepts_fr_tables_and_converts_mixed():
    lb = _lb()
    fr = lb.fr_from_ints(ft.ints_differences(4))
    small = np.arange(16, dtype=np.uint32)
    S = lb.CustomStrategy(None, 2, 4, [fr, small], lambda v: v[0] - v[1] * v[2] + v[3], 2)
    assert S.fr_tables and all(t.shape == (16, 4) and t.dtype == np.uint64 for t in S.tables)
    assert ol.fr_ints(S.tables[1]) == list(range(16))
    assert (S.tables[0] == fr).all()
    assert S.program.shape[0] > 0 and S.degree == 2
    # 1-D tables alone keep the u32 description
    S2 = lb.CustomStrategy(None, 2, 4, [small], lambda v: v[0] + v[1], 1)
    assert not S2.fr_tables and S2.tables[0].dtype == np.uint32


def test_description_rejects_bad_fr_tables():
    lb = _lb()
    good = lb.fr_from_ints(range(16))
    bad_l = good.copy()
    bad_l[3] = ol.int_to_limbs(ft.L_FR)           # the value l itself
    bad_max = good.copy()
    bad_max[5] = [2**64 - 1] * 4                   # 2^256 - 1
    for tables in ([bad_l], [bad_max], [good[:, :3]], [good[:8]], [good.astype(np.int64)],
                   [good, np.arange(16) + 2**32]):
        with pytest.raises(lb.LassoError) as e:
            lb.CustomStrategy(None, 1, 4, tables, lambda v: v[0], 1)
        assert e.value.code == 4


def test_create_fr_is_declared_and_exported():
    lb = _lb()
    hdr = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "lasso_b200.h")).read()
    assert "int lasso_strategy_create_fr(" in hdr
    assert hasattr(ctypes.CDLL(lb.library_path()), "lasso_strategy_create_fr")
    for name in ("orc_custom_prove_fr", "orc_custom_sumcheck_round_fr", "orc_custom_evaluate_subtable_mle_fr",
                 "orc_custom_combine_lookups_fr"):
        assert hasattr(oc.lib(), name), name


def test_table_widths():
    """the widths the GPU's row commitments are sized by: full width, 40 bits, and the edges' l - 1"""
    assert ft.width(ft.ints_squares_40(8)) == 40 and ft.width(ft.ints_39bit(8)) == 39
    assert ft.width(ft.ints_edges(6)) == 253 and ft.width(ft.ints_one_top(4)) == 253
    assert ft.width(ft.ints_differences(4)) == 253
