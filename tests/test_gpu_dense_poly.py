"""Dense polynomials of a caller on the GPU: PolyCommitmentGens, DensePolynomial.commit / evaluate and
PolyEvalProof.prove on a caller-held Transcript and RandomTape, bit for bit against the CPU oracle (oracle_dense/).
Covers the integer (u32 mirror, 16-bit tables) and the full-width (8-bit windows) forms, host and device input, the
path without digit-multiples tables, every error of the C ABI, composition on one transcript, and the sizes of
tests/golden/dense_poly.json."""
import ctypes
import hashlib
import json
import os

import numpy as np
import pytest

import dense_poly_cases as dc
import oracle_dense_lib as od
import oracle_lib as ol

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ERR_LENGTH, ERR_NOT_POW2, ERR_STRATEGY, ERR_GENS, ERR_POINTER, ERR_VALUE = 1, 2, 4, 5, 7, 8
L_MINUS_1 = ol.L_FR - 1


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


_gens_cache = {}


def _gens(ctx, nv):
    import lasso_b200 as lb

    if nv not in _gens_cache:
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
        _gens_cache[nv] = (lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream), stream)
    return _gens_cache[nv]


def _values(kind, nv, seed):
    """2^nv evaluations of one value class, Montgomery limbs"""
    rng = np.random.default_rng(seed)
    n = 1 << nv
    if kind == "zero":
        return np.zeros((n, 4), dtype=np.uint64)
    if kind == "full":
        return dc.random_full(rng, n)
    if kind == "l-1":  # every third entry l - 1 (the full width as an integer), the others small
        Z = dc.fr_from_u64(rng.integers(0, 256, size=n, dtype=np.uint64))
        Z[::3] = ol.fr_array([L_MINUS_1])[0]
        return Z
    bits = {"u8": 8, "u32": 32, "2^32": 32, "40-bit": 40}[kind]
    v = rng.integers(0, 1 << bits, size=n, dtype=np.uint64)
    if kind == "u32":
        v[-1] = 2**32 - 1  # the widest value the u32 path takes
    if kind == "2^32":
        v[n // 2] = 2**32  # one value past it: the Fr path with 33-bit values
    return dc.fr_from_u64(v)


KINDS = ["zero", "u8", "u32", "2^32", "40-bit", "full", "l-1"]
NVS = [0, 1, 2, 3, 5, 8, 11, 16, 20]


@pytest.mark.parametrize("nv", NVS)
@pytest.mark.parametrize("kind", KINDS)
def test_commitment_bytes(ctx, kind, nv):
    import lasso_b200 as lb

    if nv == 20 and kind in ("zero", "u8", "40-bit"):
        pytest.skip("covered by the other value classes at this size and by every class below it")
    Z = _values(kind, nv, 1000 * nv + KINDS.index(kind))
    gens, stream = _gens(ctx, nv)
    before = ctx.launches
    p = lb.DensePolynomial(ctx, Z)
    integer = kind in ("zero", "u8", "u32")
    assert ctx.launches - before == (3 if integer else 2)  # ingest + verdict (+ the u32 mirror)
    assert p.num_vars == nv
    got = p.commit(gens)
    assert len(got) == 8 + 32 * (1 << (nv // 2))
    assert got == od.commit(Z, stream)


@pytest.mark.parametrize("nv,kind", [(0, "full"), (1, "u8"), (4, "u32"), (7, "2^32"), (10, "full"), (13, "l-1"),
                                     (18, "u32"), (20, "full")])
def test_evaluate(ctx, nv, kind):
    import lasso_b200 as lb

    Z = _values(kind, nv, 7 * nv + 1)
    r = dc.random_full(np.random.default_rng(nv), nv)
    p = lb.DensePolynomial(ctx, Z)
    assert np.array_equal(p.evaluate(r), od.evaluate(Z, r))


def _prove_both(ctx, Z, nv, seed):
    """-> (gpu proof, oracle proof bytes, oracle C_Zr, r, Zr, stream, commitment, both after-challenges)"""
    import lasso_b200 as lb

    rng = np.random.default_rng(seed)
    r = dc.random_full(rng, nv)
    tape_seed = dc.random_full(rng, 1)[0]
    gens, stream = _gens(ctx, nv)
    p = lb.DensePolynomial(ctx, Z)
    comm = p.commit(gens)
    Zr = p.evaluate(r)
    t, tape = lb.Transcript(b"example"), lb.RandomTape(b"proof", tape_seed)
    t.append_poly_commitment(b"poly", comm)
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, tape)
    o = od.Transcript(b"example")
    o.append_poly_commitment(b"poly", comm)
    want, czr = od.prove(Z, r, Zr, stream, o, od.RandomTape(b"proof", tape_seed))
    return proof, want, czr, r, Zr, stream, comm, t.challenge_scalar(b"after"), o.challenge_scalar(b"after")


@pytest.mark.parametrize("nv", [0, 1, 2, 3, 5, 8, 11, 16])
@pytest.mark.parametrize("kind", ["u32", "full"])
def test_proof_bytes_and_verifier(ctx, nv, kind):
    Z = _values(kind, nv, 31 * nv + len(kind))
    proof, want, czr, r, Zr, stream, comm, after, after_o = _prove_both(ctx, Z, nv, nv + 500)
    assert proof.bytes == want
    assert proof.C_Zr == czr
    assert np.array_equal(after, after_o)

    def verify(pb, zr):
        v = od.Transcript(b"example")
        v.append_poly_commitment(b"poly", comm)
        return od.verify(stream, nv, comm, pb, r, zr, v)

    assert verify(proof.bytes, Zr) == 0
    assert verify(proof.bytes, ol.fr_array([ol.fr_ints([Zr])[0] + 1])[0]) == 1
    if nv >= 2:  # L_vec is empty below R = 2: flip its first point to another valid point
        bad = bytearray(proof.bytes)
        bad[8:40] = comm[8:40] if comm[8:40] != proof.bytes[8:40] else comm[40:72]
        assert verify(bytes(bad), Zr) == 1


def test_composition_on_one_transcript(ctx):
    """commit two polynomials, absorb both commitments, draw r, evaluate, absorb the claims, prove both openings in
    sequence on one transcript and one tape: every byte and the final challenge equal the oracle's replay"""
    import lasso_b200 as lb

    nv = 9
    A, B = _values("u32", nv, 1), _values("full", nv, 2)
    gens, stream = _gens(ctx, nv)
    seed = ol.fr_array([77])[0]
    pa, pb = lb.DensePolynomial(ctx, A), lb.DensePolynomial(ctx, B)
    ca, cb = pa.commit(gens), pb.commit(gens)
    t, tape = lb.Transcript(b"composed"), lb.RandomTape(b"proof", seed)
    o, otape = od.Transcript(b"composed"), od.RandomTape(b"proof", seed)
    for x in (t, o):
        x.append_protocol_name(b"two witness columns")
        x.append_poly_commitment(b"comm_a", ca)
        x.append_poly_commitment(b"comm_b", cb)
        x.append_u64(b"num_vars", nv)
    r = t.challenge_vector(b"r", nv)
    assert np.array_equal(r, o.challenge_vector(b"r", nv))
    ea, eb = pa.evaluate(r), pb.evaluate(r)
    assert np.array_equal(ea, od.evaluate(A, r)) and np.array_equal(eb, od.evaluate(B, r))
    for x in (t, o):
        x.append_scalars(b"claims", np.stack([ea, eb]))
    pra = lb.PolyEvalProof.prove(ctx, pa, r, ea, gens, t, tape)
    prb = lb.PolyEvalProof.prove(ctx, pb, r, eb, gens, t, tape)
    wa, _ = od.prove(A, r, ea, stream, o, otape)
    wb, _ = od.prove(B, r, eb, stream, o, otape)
    assert pra.bytes == wa and prb.bytes == wb
    assert np.array_equal(t.challenge_scalar(b"final"), o.challenge_scalar(b"final"))


def _tensor_views(torch, Z):
    n = Z.shape[0]
    t64 = torch.from_numpy(Z.view(np.int64)).cuda()
    wide = torch.zeros((n, 7), dtype=torch.int64, device="cuda")
    wide[:, 1:5] = t64  # rows 56 bytes apart, each starting 8 bytes into its row
    rows = torch.zeros((2 * n, 4), dtype=torch.int64, device="cuda")
    rows[::2] = t64
    views = [("contiguous_int64", t64), ("row_stride_7", wide[:, 1:5]), ("every_other_row", rows[::2])]
    if hasattr(torch, "uint64"):
        views.append(("contiguous_uint64", t64.view(torch.uint64)))
    return views


@pytest.mark.parametrize("nv,kind", [(0, "u32"), (6, "u32"), (6, "full"), (12, "2^32"), (12, "l-1"), (17, "full")])
def test_device_input(ctx, nv, kind):
    import torch

    import lasso_b200 as lb

    Z = _values(kind, nv, 3 * nv + 11)
    gens, _ = _gens(ctx, nv)
    r = dc.random_full(np.random.default_rng(5), nv)
    host = lb.DensePolynomial(ctx, Z)
    want = (host.commit(gens), host.evaluate(r).tobytes())
    for name, view in _tensor_views(torch, Z):
        if name in ("row_stride_7", "every_other_row") and nv > 0:
            assert not view.is_contiguous()
        p = lb.DensePolynomial(ctx, view)
        del view  # the library keeps its own copy
        torch.cuda.synchronize()
        assert (p.commit(gens), p.evaluate(r).tobytes()) == want, name


def test_device_input_pointer_errors(ctx):
    import torch

    import lasso_b200 as lb

    Z = _values("u32", 4, 9)
    pinned = torch.from_numpy(Z.view(np.int64)).pin_memory()
    out = ctypes.c_void_p()
    for name, ptr in [("host", Z.ctypes.data), ("pinned", pinned.data_ptr()), ("null", None)]:
        before = ctx.launches
        rc = lb.lib().lasso_poly_create_device(ctx._h, ctypes.c_void_p(ptr), ctypes.c_size_t(16), ctypes.c_size_t(4),
                                               None, ctypes.byref(out))
        assert rc == ERR_POINTER, name
        assert ctx.launches == before and not out.value, name
    # a CPU tensor, pinned or not, takes the host path through the Python surface
    assert lb.DensePolynomial(ctx, pinned).commit(_gens(ctx, 4)[0]) == lb.DensePolynomial(ctx, Z).commit(_gens(ctx, 4)[0])
    _assert_usable(ctx)


def test_no_multiples_tables(ctx, monkeypatch):
    """with LASSO_B200_NO_MULTIPLES=1 the generators carry no digit tables: the bucket paths give the same bytes"""
    import lasso_b200 as lb

    for nv, kind in [(8, "u32"), (11, "full"), (11, "u8"), (5, "2^32")]:
        Z = _values(kind, nv, 99 + nv)
        want = _prove_both(ctx, Z, nv, 40 + nv)
        monkeypatch.setenv("LASSO_B200_NO_MULTIPLES", "1")
        stream = np.ascontiguousarray(ol.generators(dc.n_generators(nv)))
        g = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
        monkeypatch.delenv("LASSO_B200_NO_MULTIPLES")
        rng = np.random.default_rng(40 + nv)
        r = dc.random_full(rng, nv)
        tape_seed = dc.random_full(rng, 1)[0]
        p = lb.DensePolynomial(ctx, Z)
        comm = p.commit(g)
        assert comm == want[6]
        t = lb.Transcript(b"example")
        t.append_poly_commitment(b"poly", comm)
        proof = lb.PolyEvalProof.prove(ctx, p, r, p.evaluate(r), g, t, lb.RandomTape(b"proof", tape_seed))
        assert proof.bytes == want[1] and proof.C_Zr == want[2]


def _assert_usable(ctx):
    """a correct proof on the same context after an error"""
    Z = _values("full", 6, 123)
    proof, want, czr, *_ = _prove_both(ctx, Z, 6, 321)
    assert proof.bytes == want and proof.C_Zr == czr


def test_errors(ctx):
    """every error of the dense-polynomial C ABI, each returned before any launch (the non-canonical entry: after the
    ingest pass, with no polynomial made), each followed by a correct proof on the same context"""
    import lasso_b200 as lb

    L = lb.lib()
    c_sz = ctypes.c_size_t
    nv = 6
    gens, stream = _gens(ctx, nv)
    other, _ = _gens(ctx, 8)  # R = 16 != 8
    same_R, _ = _gens(ctx, 5)  # R = 8 == 8: accepted (commitments.rs:85 compares R only)
    Z = _values("u32", nv, 5)
    p = lb.DensePolynomial(ctx, Z)
    r = dc.random_full(np.random.default_rng(1), nv)
    Zr = p.evaluate(r)
    small = np.zeros((4, 4), dtype=np.uint64)
    h = ctypes.c_void_p()
    buf = np.zeros(1 << 16, dtype=np.uint8)
    n = c_sz(0)
    czr = np.zeros(32, dtype=np.uint8)
    t, tape = lb.Transcript(b"e"), lb.RandomTape(b"proof", ol.fr_array([1])[0])

    def prove_rc(g, rr, r_len):
        return L.lasso_poly_eval_prove(ctx._h, p._h, g._h, lb.api._p(rr), c_sz(r_len), lb.api._p(Zr), t._h, tape._h,
                                       lb.api._p(buf), c_sz(buf.shape[0]), ctypes.byref(n), lb.api._p(czr))

    cases = [
        ("len 0", ERR_NOT_POW2, lambda: L.lasso_poly_create(ctx._h, lb.api._p(small), c_sz(0), ctypes.byref(h))),
        ("len 3", ERR_NOT_POW2, lambda: L.lasso_poly_create(ctx._h, lb.api._p(small), c_sz(3), ctypes.byref(h))),
        ("len 2^29", ERR_LENGTH, lambda: L.lasso_poly_create(ctx._h, lb.api._p(small), c_sz(1 << 29), ctypes.byref(h))),
        ("device len 2^29", ERR_LENGTH,
         lambda: L.lasso_poly_create_device(ctx._h, None, c_sz(1 << 29), c_sz(4), None, ctypes.byref(h))),
        ("row_stride 3", ERR_LENGTH,
         lambda: L.lasso_poly_create_device(ctx._h, None, c_sz(4), c_sz(3), None, ctypes.byref(h))),
        ("device host pointer", ERR_POINTER,
         lambda: L.lasso_poly_create_device(ctx._h, lb.api._p(small), c_sz(4), c_sz(4), None, ctypes.byref(h))),
        ("gens n_points < R + 2", ERR_GENS,
         lambda: L.lasso_poly_gens_create(ctx._h, lb.api._p(stream), c_sz(stream.shape[0] - 1), c_sz(nv), ctypes.byref(h))),
        ("gens num_vars 29", ERR_LENGTH,
         lambda: L.lasso_poly_gens_create(ctx._h, lb.api._p(stream), c_sz(stream.shape[0]), c_sz(29), ctypes.byref(h))),
        ("commit with another R", ERR_GENS,
         lambda: L.lasso_poly_commit(ctx._h, p._h, other._h, lb.api._p(buf), c_sz(buf.shape[0]), ctypes.byref(n))),
        ("commit cap too small", ERR_LENGTH,
         lambda: L.lasso_poly_commit(ctx._h, p._h, gens._h, lb.api._p(buf), c_sz(8), ctypes.byref(n))),
        ("evaluate r_len", ERR_LENGTH,
         lambda: L.lasso_poly_evaluate(ctx._h, p._h, lb.api._p(r), c_sz(nv - 1), lb.api._p(czr))),
        ("prove r_len", ERR_LENGTH, lambda: prove_rc(gens, r, nv + 1)),
        ("prove with another R", ERR_GENS, lambda: prove_rc(other, r, nv)),
        ("prove non-canonical r", ERR_VALUE,
         lambda: prove_rc(gens, np.concatenate([r[:-1], ol.int_to_limbs(ol.L_FR)[None]]), nv)),
    ]
    for name, code, f in cases:
        h.value = None
        before = ctx.launches
        assert f() == code, (name, L.lasso_last_error())
        assert ctx.launches == before, name
        assert not h.value, name
        _assert_usable(ctx)
    # the transcript and tape the failed calls were given are untouched: a proof on them equals a fresh one's
    proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, tape)
    fresh = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, lb.Transcript(b"e"), lb.RandomTape(b"proof", ol.fr_array([1])[0]))
    assert proof.bytes == fresh.bytes
    # generators of the same R are accepted
    assert lb.DensePolynomial(ctx, Z).commit(same_R) == p.commit(gens)
    # non-canonical entries, first / middle / last, host and device: no polynomial is made, the context stays usable
    import torch

    for at in (0, 31, 63):
        bad = Z.copy()
        bad[at] = ol.int_to_limbs(ol.L_FR + at)
        for src in (bad, torch.from_numpy(bad.view(np.int64)).cuda()):
            with pytest.raises(lb.LassoError) as e:
                lb.DensePolynomial(ctx, src)
            assert e.value.code == ERR_VALUE, at
        all_ones = Z.copy()
        all_ones[at] = np.uint64(2**64 - 1)
        with pytest.raises(lb.LassoError) as e:
            lb.DensePolynomial(ctx, all_ones)
        assert e.value.code == ERR_VALUE
    _assert_usable(ctx)


GOLD = json.load(open(os.path.join(HERE, "golden", "dense_poly.json")))["cases"]


@pytest.mark.parametrize("name", ["full_nv22", "u16_nv22", "full_nv24", "u16_nv24"])
def test_at_size_against_golden(ctx, name):
    import torch

    import lasso_b200 as lb

    gold = GOLD[name]
    nv, Z, r, seed = dc.inputs(name)
    assert hashlib.sha256(Z.tobytes()).hexdigest() == gold["Z_sha256"]
    stream = np.ascontiguousarray(ol.generators(gold["n_generators"]))
    assert hashlib.sha256(stream.tobytes()).hexdigest() == gold["generators_sha256"]
    gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv, stream=stream)
    for src in (Z, torch.from_numpy(Z.view(np.int64)).cuda()):
        p = lb.DensePolynomial(ctx, src)
        comm = p.commit(gens)
        assert hashlib.sha256(comm).hexdigest() == gold["commitment_sha256"]
        Zr = p.evaluate(r)
        assert Zr.tobytes().hex() == gold["Zr_hex"]
        t = lb.Transcript(dc.TRANSCRIPT_LABEL)
        t.append_poly_commitment(dc.COMMIT_LABEL, comm)
        proof = lb.PolyEvalProof.prove(ctx, p, r, Zr, gens, t, lb.RandomTape(dc.TAPE_LABEL, seed))
        assert hashlib.sha256(proof.bytes).hexdigest() == gold["proof_sha256"]
        assert proof.C_Zr.hex() == gold["C_Zr_hex"]
        assert t.challenge_scalar(b"after").tobytes().hex() == gold["after_challenge_hex"]
        del p
