"""The oracle's SumcheckInstanceProof::prove_cubic_batched with a caller's claim, coefficients and num_rounds
(oracle_dense/ orcd_cubic_prove): its proofs pass the oracle's sumcheck verifier at degree 3 with the final claim
C(r) sum_k coeff_k A_k(r) B_k(r), its finals are the polynomials evaluated at (r || 0..0), and the helpers of
cubic_batched_cases agree with the oracle."""
import numpy as np
import pytest

import cubic_batched_cases as cb
import dense_poly_cases as dc
import oracle_cubic_lib as ocb
import oracle_dense_lib as od
import oracle_lib as ol
import oracle_sumcheck_lib as osc


def _prove(A, B, C, coeffs, claim, rounds, label=b"cubic"):
    t = od.Transcript(label)
    return ocb.cubic_prove(A, B, C, coeffs, claim, rounds, t), t


@pytest.mark.parametrize("n,nv,rounds,ckind", [(1, 1, 1, "random"), (2, 3, 3, "eq"), (3, 5, 2, "random"),
                                                (7, 6, 6, "eq"), (32, 4, 4, "random")])
def test_verifier_accepts_and_finals(n, nv, rounds, ckind):
    A, B, C, coeffs = cb.random_case(n, nv, 100 * n + nv, ckind)
    claim = cb.true_claim(A, B, C, coeffs)
    res, t = _prove(A, B, C, coeffs, claim, rounds)
    assert len(res["proof"]) == 8 + 104 * rounds
    v = od.Transcript(b"cubic")
    rc, e, r = osc.sumcheck_verify(res["proof"], claim, rounds, 3, v)
    assert rc == 0
    assert np.array_equal(r, res["r"])
    assert np.array_equal(v.challenge_scalar(b"after"), t.challenge_scalar(b"after"))
    point = np.concatenate([res["r"], np.zeros((nv - rounds, 4), dtype=np.uint64)])
    want = [od.evaluate(Z, point) for Z in list(A) + list(B) + [C]]
    assert np.array_equal(res["finals"], np.stack(want).reshape(-1, 4))
    if rounds == nv:  # the last round's claim is C(r) sum_k coeff_k A_k(r) B_k(r)
        assert ol.fr_ints(e)[0] == _final_claim(res, coeffs, n)


def _final_claim(res, coeffs, n):
    """C(r) sum_k coeff_k A_k(r) B_k(r) from the finals"""
    fa, fb = ol.fr_ints(res["finals"][:n]), ol.fr_ints(res["finals"][n:2 * n])
    fc = ol.fr_ints(res["finals"][2 * n:])[0]
    return sum(k * a * b for k, a, b in zip(ol.fr_ints(coeffs), fa, fb)) * fc % ol.L_FR


def test_wrong_claim_rejected():
    """the round checks recover the linear term from the verifier's own claim, so a proof from a wrong claim fails the
    final check the caller makes: the verifier's last e is not C(r) sum_k coeff_k A_k(r) B_k(r)"""
    A, B, C, coeffs = cb.random_case(2, 4, 7, "eq")
    claim = cb.true_claim(A, B, C, coeffs)
    bad = ol.fr_array([(ol.fr_ints(claim[None])[0] + 1) % ol.L_FR])[0]
    for c, ok in ((claim, True), (bad, False)):
        res, _ = _prove(A, B, C, coeffs, c, 4)
        rc, e, _ = osc.sumcheck_verify(res["proof"], claim, 4, 3, od.Transcript(b"cubic"))
        assert (rc == 0 and ol.fr_ints(e)[0] == _final_claim(res, coeffs, 2)) == ok


def test_zero_coefficients():
    """a pair with coeff_k = 0 contributes nothing: the proof equals the one without it"""
    A, B, C, coeffs = cb.random_case(3, 5, 11)
    coeffs[1] = 0
    claim = cb.true_claim(A, B, C, coeffs)
    full, _ = _prove(A, B, C, coeffs, claim, 5)
    less, _ = _prove([A[0], A[2]], [B[0], B[2]], C, coeffs[[0, 2]], claim, 5)
    assert full["proof"] == less["proof"] and np.array_equal(full["r"], less["r"])
    rc, _, _ = osc.sumcheck_verify(full["proof"], claim, 5, 3, od.Transcript(b"cubic"))
    assert rc == 0


def test_helpers():
    rng = np.random.default_rng(3)
    tau = ol.rand_fr(rng, 5)
    Z = dc.random_full(rng, 32)
    # <Z, eq(tau)> is Z(tau)
    s = sum(a * b for a, b in zip(ol.fr_ints(Z), ol.fr_ints(cb.eq_table(tau)))) % ol.L_FR
    assert s == ol.fr_ints(od.evaluate(Z, tau))[0]
    A, B, C, coeffs = cb.random_case(2, 3, 5)
    want = sum(ol.fr_ints(coeffs)[k] * a * b * c for k in range(2)
               for a, b, c in zip(ol.fr_ints(A[k]), ol.fr_ints(B[k]), ol.fr_ints(C))) % ol.L_FR
    assert ol.fr_ints(cb.true_claim(A, B, C, coeffs)[None])[0] == want
