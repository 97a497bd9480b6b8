"""GPU parity, kernel by kernel: every C-ABI entry point against the CPU oracle on the same seeded
inputs — bit-exact (integer arithmetic, canonical residues)."""
import numpy as np
import pytest

import oracle_lib as ol
from oracle_lib import P, lib as orc, sz

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def edge_fr():
    L = ol.L_FR
    return ol.fr_array([0, 1, 2, L - 1, L - 2, (L - 1) // 2, 2**128, 2**252])


@pytest.mark.parametrize("log_n", [1, 2, 5, 10, 16, 20])
def test_bind_top_bot(ctx, log_n):
    import lasso_b200 as lb

    rng = np.random.default_rng(log_n)
    n = 1 << log_n
    Z = ol.rand_fr(rng, n)
    Z[: min(n, 8)] = edge_fr()[: min(n, 8)]
    for r in [ol.rand_fr(rng, 1)[0], ol.fr_array([0])[0], ol.fr_array([1])[0], ol.fr_array([ol.L_FR - 1])[0]]:
        for top, fn in ((1, lb.bind_top), (0, lb.bind_bot)):
            ref = Z.copy()
            orc().orc_bind(top, P(ref), sz(n), P(np.ascontiguousarray(r)))
            got = fn(ctx, Z, r)
            assert (got == ref[: n // 2]).all()


def test_bind_errors(ctx):
    import lasso_b200 as lb

    with pytest.raises(lb.LassoError) as e:
        lb.bind_top(ctx, ol.fr_array([1, 2, 3]), ol.fr_array([5])[0])
    assert e.value.code == 2  # DensePolynomial::new: power of two


@pytest.mark.parametrize("ell", [0, 1, 2, 7, 11, 12, 13, 17, 20, 22, 23, 24])
def test_eq_evals(ctx, ell):
    import lasso_b200 as lb

    rng = np.random.default_rng(100 + ell)
    r = ol.rand_fr(rng, max(ell, 1))[:ell].reshape(ell, 4)
    ref = np.zeros((1 << ell, 4), dtype=np.uint64)
    orc().orc_eq_evals(P(np.ascontiguousarray(r)) if ell else None, sz(ell), P(ref))
    got = lb.eq_evals(ctx, r)
    assert (got == ref).all()


def test_eq_evals_kat(ctx):
    import lasso_b200 as lb

    # dense_mlpoly.rs:436-458 / SURVEY D1: r=(4,3) -> [6,-9,-8,12]
    got = lb.eq_evals(ctx, ol.fr_array([4, 3]))
    assert ol.fr_ints(got) == [6, ol.L_FR - 9, ol.L_FR - 8, 12]


CASES = [(0, 1, 16, 0), (1, 2, 8, 0), (2, 4, 16, 0), (2, 4, 4, 0), (3, 1, 4, 0), (3, 2, 4, 0), (3, 4, 4, 0),
         (3, 8, 4, 0), (4, 3, 8, 40), (4, 4, 16, 40)]


@pytest.mark.parametrize("kind,C,log_m,log_r", CASES)
@pytest.mark.parametrize("log_len", [1, 4, 13])
def test_sumcheck_round_arbitrary(ctx, kind, C, log_m, log_r, log_len):
    import lasso_b200 as lb

    S = lb.Strategy(kind, C, log_m, log_r)
    rng = np.random.default_rng(kind * 100 + C * 10 + log_len)
    n = 1 << log_len
    polys = ol.rand_fr(rng, (S.num_memories + 1) * n).reshape(S.num_memories + 1, n, 4)
    ref = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
    orc().orc_sumcheck_round_arbitrary(kind, sz(C), sz(log_m), sz(log_r), P(np.ascontiguousarray(polys)), sz(n), P(ref))
    got = lb.sumcheck_round_arbitrary(ctx, S, [polys[k] for k in range(S.num_memories + 1)])
    assert (got == ref).all()


@pytest.mark.parametrize("kind,C,log_m,log_r", CASES + [(2, 8, 16, 0), (4, 2, 24, 40), (0, 16, 6, 0)])
@pytest.mark.parametrize("log_len", [2, 5, 14, 17])
def test_sumcheck_bind_round_arbitrary(ctx, kind, C, log_m, log_r, log_len):
    """The bind between two rounds fused with the next round's evaluation (sumcheck.rs:247-253 + 179-237): the bound
    polynomials and the round's evaluations against the oracle's bind followed by its round evaluation."""
    import lasso_b200 as lb

    S = lb.Strategy(kind, C, log_m, log_r)
    rng = np.random.default_rng(kind * 1000 + C * 10 + log_len)
    n = 1 << log_len
    np_ = S.num_memories + 1
    if log_len >= 14:  # any residue below l is a field element in memory format: uniform below 2^252, made by numpy
        polys = rng.integers(0, 1 << 64, size=(np_, n, 4), dtype=np.uint64)
        polys[:, :, 3] &= np.uint64((1 << 60) - 1)
    else:
        polys = ol.rand_fr(rng, np_ * n).reshape(np_, n, 4)
    polys[0][: min(n, 8)] = edge_fr()[: min(n, 8)]
    for r in [ol.rand_fr(rng, 1)[0], ol.fr_array([0])[0], ol.fr_array([ol.L_FR - 1])[0]]:
        bound = np.zeros((np_, n // 2, 4), dtype=np.uint64)
        for k in range(np_):
            z = polys[k].copy()
            orc().orc_bind(1, P(z), sz(n), P(np.ascontiguousarray(r)))
            bound[k] = z[: n // 2]
        ref = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
        orc().orc_sumcheck_round_arbitrary(kind, sz(C), sz(log_m), sz(log_r), P(np.ascontiguousarray(bound)), sz(n // 2), P(ref))
        got_polys, got = lb.sumcheck_bind_round_arbitrary(ctx, S, [polys[k] for k in range(np_)], r)
        assert (got == ref).all()
        for k in range(np_):
            assert (got_polys[k] == bound[k]).all()


@pytest.mark.parametrize("ncirc,log_len", [(1, 1), (2, 3), (8, 10), (16, 14), (32, 6)])
def test_sumcheck_round_cubic(ctx, ncirc, log_len):
    import lasso_b200 as lb

    rng = np.random.default_rng(ncirc + log_len)
    n = 1 << log_len
    A = ol.rand_fr(rng, ncirc * n).reshape(ncirc, n, 4)
    B = ol.rand_fr(rng, ncirc * n).reshape(ncirc, n, 4)
    Cq = ol.rand_fr(rng, n)
    ref = np.zeros((ncirc, 3, 4), dtype=np.uint64)
    orc().orc_sumcheck_round_cubic(P(A), P(B), P(Cq), sz(ncirc), sz(n), P(ref))
    got = lb.sumcheck_round_cubic(ctx, [A[k] for k in range(ncirc)], [B[k] for k in range(ncirc)], Cq)
    assert (got == ref).all()


@pytest.mark.parametrize("kind,C,log_m,log_r", [(0, 4, 16, 0), (1, 4, 16, 0), (2, 4, 16, 0), (3, 4, 16, 0),
                                                (4, 4, 16, 40), (4, 3, 8, 40), (2, 2, 4, 0)])
def test_materialize_and_gather(ctx, kind, C, log_m, log_r):
    import lasso_b200 as lb

    S = lb.Strategy(kind, C, log_m, log_r)
    M = 1 << log_m
    ref = np.zeros((S.num_subtables, M, 4), dtype=np.uint64)
    orc().orc_materialize_subtables(kind, sz(C), sz(log_m), sz(log_r), P(ref))
    got = lb.materialize_subtables(ctx, S)
    for k in range(S.num_subtables):
        assert (got[k] == ref[k]).all()
    rng = np.random.default_rng(kind)
    s = 1 << 9
    nz = rng.integers(0, M, size=(C, s), dtype=np.uint64)
    refE = np.zeros((S.num_memories, s, 4), dtype=np.uint64)
    orc().orc_lookup_polys(kind, sz(C), sz(log_m), sz(log_r), P(nz), sz(s), P(refE))
    gotE = lb.gather_lookup_polys(ctx, S, [nz[d] for d in range(C)])
    for k in range(S.num_memories):
        assert (gotE[k] == refE[k]).all()
    bad = nz.copy()
    bad[0, 3] = M
    with pytest.raises(lb.LassoError) as e:
        lb.gather_lookup_polys(ctx, S, [bad[d] for d in range(C)])
    assert e.value.code == 3


def _affine_of(ext):
    out = np.zeros(8, dtype=np.uint64)
    orc().orc_point_to_affine(P(np.ascontiguousarray(ext)), P(out))
    return out


@pytest.mark.parametrize("n,bits", [(1, 253), (2, 253), (31, 253), (33, 8), (100, 16), (257, 20), (1000, 253),
                                    (5000, 253), (9000, 60), (64, 1)])
def test_msm_vs_oracle(ctx, n, bits):
    import lasso_b200 as lb

    rng = np.random.default_rng(n)
    bases = np.ascontiguousarray(ol.generators(9002)[:n])
    ks = [int.from_bytes(rng.bytes(40), "little") % ol.L_FR % (1 << bits) for _ in range(n)]
    ks[0] = 0
    if n > 3:
        ks[1] = ol.L_FR - 1
        ks[2] = 1
    S = ol.fr_array(ks)
    ref = np.zeros(16, dtype=np.uint64)
    orc().orc_msm(P(bases), P(S), sz(n), 1, P(ref))
    got = lb.msm(ctx, bases, S)
    assert (got[:8] == _affine_of(ref)).all()          # same group element, affine-normalised
    assert orc().orc_point_eq(P(got), P(ref)) == 1
    assert (got[12:16] == ol.to_mont(1, ol.Q_FQ)).all()  # z = 1
    with pytest.raises(lb.LassoError):
        lb.msm(ctx, bases, S[:-1] if n > 1 else np.zeros((0, 4), dtype=np.uint64))  # Err(min_len)


@pytest.mark.parametrize("n,vals", [(3000, [5]), (2000, [1, 2, 3]), (700, [128, 129, 0x8080]), (130, [1]),
                                    (6000, [ol.L_FR - 1, 1])])
def test_msm_skewed_digits(ctx, n, vals):
    """Every digit of a window in one (or a few) buckets: the split-bucket stitch runs all its log steps."""
    import lasso_b200 as lb

    bases = np.ascontiguousarray(ol.generators(9002)[:n])
    S = ol.fr_array([vals[i % len(vals)] for i in range(n)])
    ref = np.zeros(16, dtype=np.uint64)
    orc().orc_msm(P(bases), P(S), sz(n), 1, P(ref))
    got = lb.msm(ctx, bases, S)
    assert (got[:8] == _affine_of(ref)).all()


@pytest.mark.parametrize("L,R,vals", [(8, 2048, [1]), (4, 4096, [0, 1, 255, 256, 65535]), (2, 8192, [7, 1 << 19])])
def test_commit_rows_skewed(ctx, L, R, vals):
    """Many rows over shared bases, skewed small scalars (variable-base path; the fixed-base path is covered end to end)."""
    import lasso_b200 as lb

    gens = np.ascontiguousarray(ol.generators(9002)[: R + 1])
    Z = ol.fr_array([vals[(i * 7 + i // R) % len(vals)] for i in range(L * R)])
    ref = np.zeros((L, 16), dtype=np.uint64)
    orc().orc_commit_rows(P(gens), P(Z), sz(L), sz(R), P(ref))
    got = lb.commit_rows(ctx, gens, Z, L, R)
    for i in range(L):
        assert (got[i][:8] == _affine_of(ref[i])).all()


def test_msm_all_zero_and_identity(ctx):
    import lasso_b200 as lb

    bases = np.ascontiguousarray(ol.generators(66)[:40])
    got = lb.msm(ctx, bases, ol.fr_array([0] * 40))
    assert ol.fq_ints(got.reshape(4, 4)) == [0, 1, 0, 1]  # identity (0, 1)
    # P + (-P): scalars 1 and l-1 on the same base
    two = np.ascontiguousarray(np.stack([bases[0], bases[0]]))
    got = lb.msm(ctx, two, ol.fr_array([1, ol.L_FR - 1]))
    assert ol.fq_ints(got.reshape(4, 4)) == [0, 1, 0, 1]


@pytest.mark.parametrize("L,R,bits", [(4, 8, 253), (32, 64, 16), (16, 512, 8), (8, 64, 1)])
def test_commit_rows_vs_oracle(ctx, L, R, bits):
    import lasso_b200 as lb

    rng = np.random.default_rng(L * R)
    gens = np.ascontiguousarray(ol.generators(9002)[: R + 1])
    Z = ol.fr_array([int.from_bytes(rng.bytes(40), "little") % ol.L_FR % (1 << bits) for _ in range(L * R)])
    ref = np.zeros((L, 16), dtype=np.uint64)
    orc().orc_commit_rows(P(gens), P(Z), sz(L), sz(R), P(ref))
    got = lb.commit_rows(ctx, gens, Z, L, R)
    for i in range(L):
        assert (got[i][:8] == _affine_of(ref[i])).all()
