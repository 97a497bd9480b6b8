"""The shape table of the built-in strategies (strategy_shapes.py) against boundary shapes written out by hand, and the
CPU oracle on every whole-proof case of test_gpu_strategy_shapes.py: it proves each one and its verifier accepts."""
import numpy as np
import pytest

import oracle_lib as ol
import strategy_shapes as ss
import test_gpu_prove as tgp

AND, OR, XOR, LT, RANGE = ss.AND, ss.OR, ss.XOR, ss.LT, ss.RANGE_CHECK

# kind, C, log_m, log_r, accepted, provable
BOUNDARY = [
    (AND, 1, 2, 0, True, True),
    (AND, 0, 4, 0, False, False),
    (AND, 16, 4, 0, True, True),         # shift 30
    (AND, 17, 4, 0, False, False),
    (AND, 2, 1, 0, False, False),
    (RANGE, 2, 1, 0, False, False),
    (AND, 1, 24, 0, True, True),
    (AND, 1, 25, 0, False, False),
    (RANGE, 1, 25, 0, False, False),
    (RANGE, 1, 23, 0, True, True),
    (AND, 2, 5, 0, False, False),
    (OR, 2, 7, 0, False, False),
    (XOR, 2, 9, 0, False, False),
    (LT, 2, 5, 0, False, False),
    (RANGE, 2, 5, 0, True, True),
    (AND, 10, 14, 0, True, True),        # shift 63
    (AND, 9, 16, 0, False, False),       # shift 64
    (AND, 8, 18, 0, True, True),         # shift 63
    (XOR, 16, 8, 0, True, True),         # shift 60
    (XOR, 16, 10, 0, False, False),      # shift 75
    (RANGE, 4, 21, 0, True, True),       # shift 63
    (RANGE, 4, 22, 0, False, False),     # shift 66
    (RANGE, 10, 7, 0, True, True),       # shift 63
    (RANGE, 11, 7, 0, False, False),     # shift 70
    (RANGE, 8, 9, 63, True, True),       # shift 63
    (RANGE, 2, 8, -1, False, False),
    (RANGE, 2, 8, 0, True, True),
    (RANGE, 2, 8, 1000, True, True),
    (LT, 16, 24, 0, True, False),        # LT has no weights; 64 circuits
    (LT, 8, 24, 0, True, True),          # 32 circuits
    (LT, 9, 4, 0, True, False),          # 36 circuits
    (5, 2, 4, 0, False, False),
    (-1, 2, 4, 0, False, False),
]


@pytest.mark.parametrize("kind,C,log_m,log_r,acc,prov", BOUNDARY)
def test_shape_table_boundaries(kind, C, log_m, log_r, acc, prov):
    assert ss.accepted(kind, C, log_m, log_r) is acc
    assert ss.provable(kind, C, log_m, log_r) is prov


def test_shape_table_is_consistent():
    """provable() implies accepted(), and the rejected cases of the GPU tests have unique names"""
    for kind in ss.KINDS + (5, -1):
        for C in range(0, 18):
            for log_m in range(1, 26):
                for log_r in (-1, 0, 40):
                    assert not ss.provable(kind, C, log_m, log_r) or ss.accepted(kind, C, log_m, log_r)
    assert len(ss.REJECTED) == len({r[0] for r in ss.REJECTED})


@pytest.mark.parametrize("name,kind,C,log_m,log_r", ss.REJECTED, ids=[r[0] for r in ss.REJECTED])
def test_rejected_case_is_one_step_past_a_boundary(name, kind, C, log_m, log_r):
    """every rejected case of the GPU tests has an accepted neighbour: one of kind, C, log_m or log_r moved by one"""
    shape = [kind, C, log_m, log_r]
    neighbours = [shape[:i] + [shape[i] + d] + shape[i + 1:] for i in range(4) for d in (-1, 1)]
    assert any(ss.accepted(*nb) for nb in neighbours), name


@pytest.mark.parametrize("name,kind,C,log_m,log_r,n,same", ss.PROOFS, ids=[c[0] for c in ss.PROOFS])
def test_oracle_proves_and_verifies(name, kind, C, log_m, log_r, n, same):
    import lasso_b200 as lb

    idx, r, seed, s = tgp.make_inputs(C, log_m, n, ss.seed_of(name), same)
    need = lb.gens_points_needed(C, s, ss.num_memories(kind, C), log_m)
    stream = np.ascontiguousarray(ol.generators(max(need, 300))[:need])
    ref = ol.prove(kind, C, log_m, log_r, idx, r, stream, seed, flags=1)
    assert ref["rc"] == 0, "the oracle's verifier rejected its own proof"
    assert len(ref["proof"]) > 0 and len(ref["commitment"]) > 0
    bad = ol.prove(kind, C, log_m, log_r, idx, r, stream, seed, flags=1 | 2)
    assert bad["rc"] == 1, "a tampered claimed evaluation must be rejected"
