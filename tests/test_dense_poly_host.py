"""The host side of the dense-polynomial API, without a GPU: lasso_b200.Transcript and RandomTape against the oracle's
ProofTranscript and RandomTape, PolyCommitment::append_to_transcript, the argument checks of the Python surface, and
the oracle's own commit -> prove -> verify round trip that the GPU tests compare with."""
import numpy as np
import pytest

import oracle_dense_lib as od
import oracle_lib as ol

LABELS = [b"a", b"claim", b"poly_commitment_share", b"protocol-name", b"x" * 40]


def _points(n, seed=0):
    """n valid compressed points (multiples of the sampled generators)"""
    g = ol.generators(max(n, 8) + 2)
    out = []
    for i in range(n):
        ext = np.zeros(16, dtype=np.uint64)
        ol.lib().orc_point_from_affine(ol.P(np.ascontiguousarray(g[(i + seed) % g.shape[0]])), ol.P(ext))
        k = ol.fr_array([i + 3 + seed])[0]
        m = np.zeros(16, dtype=np.uint64)
        ol.lib().orc_point_mul(ol.P(ext), ol.P(k), ol.P(m))
        c = np.zeros(32, dtype=np.uint8)
        ol.lib().orc_point_compress(ol.P(m), ol.P(c))
        out.append(c.tobytes())
    return out


def _random_ops(rng, n_ops):
    """a random sequence of (method, args) over every transcript method"""
    pts = _points(12, int(rng.integers(0, 100)))
    ops = []
    for _ in range(n_ops):
        label = LABELS[int(rng.integers(0, len(LABELS)))]
        k = int(rng.integers(0, 9))
        if k == 0:
            ops.append(("append_message", (label, rng.bytes(int(rng.integers(0, 300))))))
        elif k == 1:
            ops.append(("append_u64", (label, int(rng.integers(0, 2**63)) * 2 + int(rng.integers(0, 2)))))
        elif k == 2:
            ops.append(("append_protocol_name", (label,)))
        elif k == 3:
            ops.append(("append_scalar", (label, ol.rand_fr(rng, 1)[0])))
        elif k == 4:
            ops.append(("append_scalars", (label, ol.rand_fr(rng, int(rng.integers(0, 20))))))
        elif k == 5:
            ops.append(("append_point", (label, pts[int(rng.integers(0, len(pts)))])))
        elif k == 6:
            ops.append(("append_points", (label, pts[: int(rng.integers(0, len(pts) + 1))])))
        elif k == 7:
            ops.append(("challenge_scalar", (label,)))
        else:
            ops.append(("challenge_vector", (label, int(rng.integers(0, 6)))))
    ops.append(("challenge_scalar", (b"final",)))
    return ops


@pytest.mark.parametrize("seed", range(12))
def test_transcript_matches_oracle(seed):
    import lasso_b200 as lb

    rng = np.random.default_rng(seed)
    label = b"example" if seed % 2 else rng.bytes(int(rng.integers(1, 30))).replace(b"\0", b"z")
    t, o = lb.Transcript(label), od.Transcript(label)
    n_chal = 0
    for name, args in _random_ops(rng, 40):
        got, want = getattr(t, name)(*args), getattr(o, name)(*args)
        if name.startswith("challenge"):
            assert np.array_equal(got, want), (seed, name)
            n_chal += 1
    assert n_chal >= 1


def test_transcript_known_values():
    """the library's transcript against the oracle's independent entry points (oracle/capi.cpp's orc_transcript_*)"""
    import lasso_b200 as lb

    L = ol.lib()
    o = ol.C.c_void_p(L.orc_transcript_new(b"example"))
    t = lb.Transcript(b"example")
    s = ol.fr_array([12345678901234567890123])[0]
    L.orc_transcript_append_scalar(o, b"s", ol.P(s))
    t.append_scalar(b"s", s)
    msg = b"hello transcript"
    L.orc_transcript_append_message(o, b"m", msg, ol.sz(len(msg)))
    t.append_message(b"m", msg)
    out = np.zeros(4, dtype=np.uint64)
    L.orc_transcript_challenge_scalar(o, b"c", ol.P(out))
    assert np.array_equal(t.challenge_scalar(b"c"), out)
    L.orc_transcript_free(o)


@pytest.mark.parametrize("seed", range(4))
def test_random_tape_matches_oracle(seed):
    import lasso_b200 as lb

    rng = np.random.default_rng(100 + seed)
    s = ol.rand_fr(rng, 1)[0]
    t, o = lb.RandomTape(b"proof", s), od.RandomTape(b"proof", s)
    for label, n in [(b"d", 1), (b"r_delta", 1), (b"r_delta", 1), (b"blinds_vec_1", 2 * seed), (b"blinds_vec_2", 7)]:
        assert np.array_equal(t.random_vector(label, n), o.random_vector(label, n))
    assert np.array_equal(t.random_scalar(b"x"), o.random_scalar(b"x"))


@pytest.mark.parametrize("n", [0, 1, 5])
def test_append_poly_commitment_is_the_per_point_appends(n):
    import lasso_b200 as lb

    pts = _points(n, 7)
    comm = n.to_bytes(8, "little") + b"".join(pts)
    a, b, o = lb.Transcript(b"t"), lb.Transcript(b"t"), od.Transcript(b"t")
    a.append_poly_commitment(b"comm", comm)
    b.append_message(b"comm", b"poly_commitment_begin")
    for p in pts:
        b.append_point(b"poly_commitment_share", p)
    b.append_message(b"comm", b"poly_commitment_end")
    o.append_poly_commitment(b"comm", comm)
    ca, cb, co = a.challenge_scalar(b"c"), b.challenge_scalar(b"c"), o.challenge_scalar(b"c")
    assert np.array_equal(ca, cb) and np.array_equal(ca, co)


def test_argument_validation():
    import lasso_b200 as lb

    t = lb.Transcript(b"t")
    bad_scalar = ol.int_to_limbs(ol.L_FR)  # l itself: not a canonical residue
    cases = [
        (lambda: lb.Transcript(b"a\0b"), 1),
        (lambda: t.append_message(b"x\0", b""), 1),
        (lambda: t.append_scalar(b"s", np.zeros(3, dtype=np.uint64)), 1),
        (lambda: t.append_scalar(b"s", np.zeros(4, dtype=np.int32)), 1),
        (lambda: t.append_scalar(b"s", bad_scalar), 8),
        (lambda: t.append_scalars(b"s", np.stack([np.zeros(4, dtype=np.uint64), bad_scalar])), 8),
        (lambda: t.append_point(b"p", b"\0" * 31), 1),
        (lambda: t.append_points(b"p", b"\0" * 33), 1),
        (lambda: t.append_poly_commitment(b"c", (2).to_bytes(8, "little") + b"\0" * 32), 1),
        (lambda: t.append_poly_commitment(b"c", b"\0" * 7), 1),
        (lambda: lb.RandomTape(b"proof", bad_scalar), 8),
        (lambda: lb.RandomTape(b"proof", np.zeros(8, dtype=np.uint64)), 1),
        (lambda: lb.DensePolynomial(None, np.zeros((4, 3), dtype=np.uint64)), 1),
        (lambda: lb.DensePolynomial(None, np.zeros(16, dtype=np.uint64)), 1),
        (lambda: lb.DensePolynomial(None, np.zeros((4, 4), dtype=np.float64)), 1),
        (lambda: lb.DensePolynomial(None, np.zeros((4, 4), dtype=np.uint32)), 1),
    ]
    for i, (f, code) in enumerate(cases):
        with pytest.raises(lb.LassoError) as e:
            f()
        assert e.value.code == code, (i, e.value)
    # a failed call leaves the transcript as it was
    u = lb.Transcript(b"t")
    assert np.array_equal(t.challenge_scalar(b"c"), u.challenge_scalar(b"c"))


def test_poly_gens_points_needed():
    import lasso_b200 as lb

    for nv, R in [(0, 1), (1, 2), (2, 2), (3, 4), (20, 1 << 10), (21, 1 << 11), (24, 1 << 12)]:
        assert lb.poly_gens_points_needed(nv) == R + 2


@pytest.mark.parametrize("nv", [0, 1, 2, 5])
def test_oracle_round_trip(nv):
    """the oracle's prove -> verify on serialised bytes accepts, and rejects Zr + 1 and a flipped L point"""
    rng = np.random.default_rng(nv)
    Z = ol.rand_fr(rng, 1 << nv)
    r = ol.rand_fr(rng, nv)
    stream = ol.generators((1 << (nv - nv // 2)) + 2)
    Zr = od.evaluate(Z, r)
    assert ol.fr_ints([Zr]) == [sum(z * w for z, w in zip(ol.fr_ints(Z), _eq(ol.fr_ints(r)))) % ol.L_FR]
    comm = od.commit(Z, stream)
    proof, czr = od.prove(Z, r, Zr, stream, od.Transcript(b"example"), od.RandomTape(b"proof", ol.fr_array([9])[0]))
    assert od.verify(stream, nv, comm, proof, r, Zr, od.Transcript(b"example")) == 0
    Zr1 = ol.fr_array([ol.fr_ints([Zr])[0] + 1])[0]
    assert od.verify(stream, nv, comm, proof, r, Zr1, od.Transcript(b"example")) == 1
    if nv >= 2:  # L_vec is empty below R = 2
        bad = bytearray(proof)
        bad[8:40] = _points(1, 3)[0]
        assert od.verify(stream, nv, comm, bytes(bad), r, Zr, od.Transcript(b"example")) == 1


def _eq(r):
    """eq(r, x) over the hypercube, r[0] the MSB (eq_poly.rs:21-38), as Python integers"""
    ev = [1]
    for rj in r:
        ev = [v for e in ev for v in (e * (1 - rj) % ol.L_FR, e * rj % ol.L_FR)]
    return ev
