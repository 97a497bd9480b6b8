"""Deriving polynomials from a caller's and reading them back, on the GPU: DensePolynomial.bound_top / bound_bot (k
variables in passes of up to 8), split, new_padded, to_numpy / to_tensor / copy_to.  Every result is compared with
Python integers (tests/pyref.py through poly_transform_cases.py) and the oracle, at num_vars 1..12 for every k, on
16-bit polynomials (u32 mirror), full-width ones, eq tables and comb results; then the golden hashes at 2^22 and 2^24,
commitments of the results against the oracle's, two-phase sumchecks, the inputs left unchanged, and every error code
with the launch count unchanged.  The sharded forms are in test_gpu_sharded_poly_transforms.py."""
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import dense_poly_cases as dc  # noqa: E402
import oracle_dense_lib as od  # noqa: E402
import oracle_lib as ol  # noqa: E402
import poly_transform_cases as pt  # noqa: E402
import pyref  # noqa: E402

pytestmark = pytest.mark.gpu
ERR_LENGTH, ERR_STRATEGY, ERR_POINTER, ERR_VALUE = 1, 4, 7, 8


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _u16(rng, n):
    return dc.fr_from_u64(rng.integers(0, 1 << 16, size=n, dtype=np.uint64))


def _inputs(ctx, nv, rng):
    """-> [(name, polynomial, its evaluations)]: 16-bit, full width, eq, comb"""
    import lasso_b200 as lb

    out = []
    for name, Z in (("u16", _u16(rng, 1 << nv)), ("full", dc.random_full(rng, 1 << nv))):
        out.append((name, lb.DensePolynomial(ctx, Z), Z))
    tau = dc.random_full(rng, nv)
    eq = lb.DensePolynomial.eq(ctx, tau)
    want = ol.fr_array(pyref.eq_evals(ol.fr_ints(tau)))
    assert (eq.to_numpy() == want).all()
    out.append(("eq", eq, want))
    a, b = out[0][1], out[1][1]
    q = lb.DensePolynomial.from_comb(ctx, lb.Comb(lambda v: v[0] * v[1] + v[0], 2), [a, b])
    A, B = ol.fr_ints(out[0][2]), ol.fr_ints(out[1][2])
    out.append(("comb", q, ol.fr_array([(x * y + x) % pyref.L for x, y in zip(A, B)])))
    return out


@pytest.mark.parametrize("nv", list(range(1, 13)))
def test_binds_every_k(ctx, nv):
    rng = np.random.default_rng(500 + nv)
    r = dc.random_full(rng, nv)
    for name, p, Z in _inputs(ctx, nv, rng):
        for k in range(1, nv + 1):
            for top in (True, False):
                q = p.bound_top(r[:k]) if top else p.bound_bot(r[:k])
                assert q.num_vars == nv - k
                got = q.to_numpy()
                assert (got == pt.py_bind(Z, r[:k], top)).all(), (name, k, top)
        assert (p.to_numpy() == Z).all(), name  # the input is unchanged
    # a single challenge as a (4,) array
    p = _inputs(ctx, nv, rng)[1]
    assert (p[1].bound_top(r[0]).to_numpy() == pt.bind(p[2], r[:1], True)).all()


@pytest.mark.parametrize("nv", [1, 2, 5, 12])
def test_split(ctx, nv):
    rng = np.random.default_rng(600 + nv)
    for name, p, Z in _inputs(ctx, nv, rng)[:2]:
        idx = 1
        while 2 * idx <= Z.shape[0]:
            lo, hi = p.split(idx)
            assert (lo.to_numpy() == Z[:idx]).all() and (hi.to_numpy() == Z[idx:2 * idx]).all(), (name, idx)
            idx *= 2
        lo, hi = p.split()
        assert lo.num_vars == nv - 1 and (hi.to_numpy() == Z[Z.shape[0] // 2:]).all()


@pytest.mark.parametrize("n", [0, 1, 2, 3, 5, 1000, (1 << 20) + 1])
def test_new_padded(ctx, n):
    import torch

    import lasso_b200 as lb

    rng = np.random.default_rng(n)
    Z = dc.random_full(rng, n) if n != 1000 else _u16(rng, n)
    want = pt.new_padded(Z)
    t = torch.from_numpy(Z.view(np.int64)).cuda()
    wide = torch.zeros((n, 9), dtype=torch.int64, device="cuda")
    wide[:, 3:7] = t
    for src in (Z, t, wide[:, 3:7]) if n else (Z,):  # an empty tensor has no row layout to pass
        p = lb.DensePolynomial.new_padded(ctx, src)
        assert p.num_vars == int(want.shape[0]).bit_length() - 1
        assert (p.to_numpy() == want).all()
    # a padded integer polynomial commits through the 16-bit tables, with the oracle's bytes
    if n == 1000:
        gens = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", 10, stream=_stream(10))
        assert lb.DensePolynomial.new_padded(ctx, Z).commit(gens) == od.commit(want, _stream(10))


def test_read_back(ctx):
    import torch

    import lasso_b200 as lb

    rng = np.random.default_rng(9)
    for Z in (_u16(rng, 1 << 10), dc.random_full(rng, 1 << 13)):
        p = lb.DensePolynomial(ctx, Z)
        assert (p.to_tensor().cpu().numpy().view(np.uint64) == Z).all()
        wide = torch.full((Z.shape[0], 6), -1, dtype=torch.int64, device="cuda")
        side = torch.cuda.Stream()
        with torch.cuda.stream(side):
            p.copy_to(wide[:, 1:5])
        side.synchronize()
        w = wide.cpu().numpy()
        assert (w[:, 1:5].view(np.uint64) == Z).all() and (w[:, 0] == -1).all() and (w[:, 5] == -1).all()
        out = np.zeros((Z.shape[0] + 3, 4), dtype=np.uint64)
        assert lb.lib().lasso_poly_read(ctx._h, p._h, lb.api._p(out), lb.api.C.c_size_t(out.shape[0])) == 0
        assert (out[: Z.shape[0]] == Z).all() and not out[Z.shape[0]:].any()


_STREAMS = {}


def _stream(nv):
    if nv not in _STREAMS:
        import lasso_b200 as lb

        _STREAMS[nv] = np.ascontiguousarray(ol.generators(lb.poly_gens_points_needed(nv), b"gens_sparse_poly"))
    return _STREAMS[nv]


def test_commitments_of_results(ctx):
    """bound, split and padded polynomials commit to the oracle's bytes of the same values"""
    import lasso_b200 as lb

    rng = np.random.default_rng(11)
    nv = 14
    r = dc.random_full(rng, 9)
    for name, p, Z in _inputs(ctx, nv, rng)[:2]:
        for k in (1, 5, 9):
            for top in (True, False):
                q = p.bound_top(r[:k]) if top else p.bound_bot(r[:k])
                g = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv - k, stream=_stream(nv - k))
                assert q.commit(g) == od.commit(pt.bind(Z, r[:k], top), _stream(nv - k)), (name, k, top)
        for idx in (1 << (nv - 1), 1 << (nv - 3)):
            g = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", idx.bit_length() - 1, stream=_stream(idx.bit_length() - 1))
            lo, hi = p.split(idx)
            assert lo.commit(g) == od.commit(Z[:idx], _stream(idx.bit_length() - 1))
            assert hi.commit(g) == od.commit(Z[idx:2 * idx], _stream(idx.bit_length() - 1))


@pytest.mark.parametrize("nv", pt.GOLDEN_NV)
def test_golden(ctx, nv):
    import lasso_b200 as lb

    g = json.load(open(os.path.join(HERE, "golden", "poly_transforms.json")))["cases"]
    Z, r = pt.golden_inputs(nv)
    p = lb.DensePolynomial(ctx, Z)
    bad = []
    for k in pt.GOLDEN_K:
        for d, top in (("top", True), ("bot", False)):
            q = p.bound_top(r[:k]) if top else p.bound_bot(r[:k])
            if pt.sha(q.to_numpy()) != g["%s_nv%d_k%d" % (d, nv, k)]:
                bad.append((d, k))
            del q
    for div in pt.SPLIT_DIV:
        lo, hi = p.split(Z.shape[0] // div)
        if [pt.sha(lo.to_numpy()), pt.sha(hi.to_numpy())] != g["split_nv%d_div%d" % (nv, div)]:
            bad.append(("split", div))
    if nv == pt.GOLDEN_NV[0]:
        if pt.sha(lb.DensePolynomial.new_padded(ctx, pt.padded_input()).to_numpy()) != g["padded_%d" % pt.PADDED_LEN]:
            bad.append("padded")
    assert not bad, bad


def _prod(v):
    return v[0] * v[1] + v[2]


@pytest.mark.parametrize("nv,k", [(6, 2), (10, 3), (12, 9)])
def test_two_phase_sumcheck(ctx, nv, k):
    """prove_arbitrary for k rounds, bound_top(r) on every input, prove_arbitrary on the results: together the single
    nv-round proof, challenges, finals and transcript state; the same for prove_cubic_batched"""
    import lasso_b200 as lb

    rng = np.random.default_rng(70 + nv)
    arrays = [_u16(rng, 1 << nv), dc.random_full(rng, 1 << nv), dc.random_full(rng, 1 << nv)]
    polys = [lb.DensePolynomial(ctx, a) for a in arrays]
    comb = lb.Comb(_prod, 3)
    t1 = lb.Transcript(b"two_phase")
    full = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, t1)
    t2 = lb.Transcript(b"two_phase")
    a = lb.SumcheckInstanceProof.prove_arbitrary(ctx, polys, comb, t2, num_rounds=k)
    bound = [p.bound_top(a.r) for p in polys]
    b = lb.SumcheckInstanceProof.prove_arbitrary(ctx, bound, comb, t2)
    assert full.bytes[8:] == a.bytes[8:] + b.bytes[8:]
    assert (np.concatenate([a.r, b.r]) == full.r).all() and (b.final_evals == full.final_evals).all()
    assert (t1.challenge_scalar(b"next") == t2.challenge_scalar(b"next")).all()
    for p, z in zip(polys, arrays):
        assert (p.to_numpy() == z).all()
    # the cubic form: claim = sum_x C(x) (c0 A0 B0 + c1 A1 B1)
    A, B, Cp = [polys[0], polys[1]], [polys[2], polys[0]], lb.DensePolynomial.eq(ctx, dc.random_full(rng, nv))
    coeffs = dc.random_full(rng, 2)

    def claim_of(As, Bs, C_):
        va, vb, vc = ([ol.fr_ints(p.to_numpy()) for p in X] for X in (As, Bs, [C_]))
        cf = ol.fr_ints(coeffs)
        s = sum(vc[0][x] * (cf[0] * va[0][x] * vb[0][x] + cf[1] * va[1][x] * vb[1][x]) for x in range(len(vc[0])))
        return ol.fr_array([s % pyref.L])[0]

    claim = claim_of(A, B, Cp)
    t1, t2 = lb.Transcript(b"two_phase_cubic"), lb.Transcript(b"two_phase_cubic")
    full = lb.SumcheckInstanceProof.prove_cubic_batched(ctx, A, B, Cp, coeffs, claim, t1)
    a = lb.SumcheckInstanceProof.prove_cubic_batched(ctx, A, B, Cp, coeffs, claim, t2, num_rounds=k)
    A2, B2, C2 = [p.bound_top(a.r) for p in A], [p.bound_top(a.r) for p in B], Cp.bound_top(a.r)
    b = lb.SumcheckInstanceProof.prove_cubic_batched(ctx, A2, B2, C2, coeffs, claim_of(A2, B2, C2), t2)
    assert full.bytes[8:] == a.bytes[8:] + b.bytes[8:]
    assert (np.concatenate([a.r, b.r]) == full.r).all() and (b.final_evals == full.final_evals).all()
    assert (t1.challenge_scalar(b"next") == t2.challenge_scalar(b"next")).all()


def test_grand_product_after_transforms(ctx):
    """a circuit over P, proven after P was bound, split and read, gives the bytes of a circuit over an untouched copy"""
    import lasso_b200 as lb

    rng = np.random.default_rng(12)
    Z = dc.random_full(rng, 1 << 9)
    P, Q = lb.DensePolynomial(ctx, Z), lb.DensePolynomial(ctx, Z)
    cp, cq = lb.GrandProductCircuit(ctx, P), lb.GrandProductCircuit(ctx, Q)
    P.bound_top(dc.random_full(rng, 3))
    P.bound_bot(dc.random_full(rng, 9))
    P.split(64)
    P.to_numpy()
    a = lb.BatchedGrandProductArgument.prove(ctx, [cp], lb.Transcript(b"gp"))
    b = lb.BatchedGrandProductArgument.prove(ctx, [cq], lb.Transcript(b"gp"))
    assert a.bytes == b.bytes and (a.claims == b.claims).all()
    assert (P.to_numpy() == Z).all()


def test_errors(ctx):
    import torch

    import lasso_b200 as lb
    from lasso_b200.api import C, _p

    L = lb.lib()
    rng = np.random.default_rng(13)
    Z = dc.random_full(rng, 1 << 6)
    p = lb.DensePolynomial(ctx, Z)
    other = lb.Context(0)
    po = lb.DensePolynomial(other, Z)
    r = dc.random_full(rng, 7)
    bad_r = r.copy()
    bad_r[1, 3] = np.uint64(2**64 - 1)
    h = C.c_void_p()
    h2 = C.c_void_p()
    out = np.zeros((64, 4), dtype=np.uint64)
    calls = {
        "top_k0": (lambda: L.lasso_poly_bind_top(ctx._h, p._h, _p(r), C.c_size_t(0), C.byref(h)), ERR_LENGTH),
        "top_k7": (lambda: L.lasso_poly_bind_top(ctx._h, p._h, _p(r), C.c_size_t(7), C.byref(h)), ERR_LENGTH),
        "bot_k7": (lambda: L.lasso_poly_bind_bot(ctx._h, p._h, _p(r), C.c_size_t(7), C.byref(h)), ERR_LENGTH),
        "top_null_r": (lambda: L.lasso_poly_bind_top(ctx._h, p._h, None, C.c_size_t(2), C.byref(h)), ERR_LENGTH),
        "bot_null_out": (lambda: L.lasso_poly_bind_bot(ctx._h, p._h, _p(r), C.c_size_t(2), None), ERR_LENGTH),
        "top_value": (lambda: L.lasso_poly_bind_top(ctx._h, p._h, _p(bad_r), C.c_size_t(3), C.byref(h)), ERR_VALUE),
        "bot_value": (lambda: L.lasso_poly_bind_bot(ctx._h, p._h, _p(bad_r), C.c_size_t(3), C.byref(h)), ERR_VALUE),
        "top_other": (lambda: L.lasso_poly_bind_top(ctx._h, po._h, _p(r), C.c_size_t(1), C.byref(h)), ERR_STRATEGY),
        "split_3": (lambda: L.lasso_poly_split(ctx._h, p._h, C.c_size_t(3), C.byref(h), C.byref(h2)), ERR_LENGTH),
        "split_0": (lambda: L.lasso_poly_split(ctx._h, p._h, C.c_size_t(0), C.byref(h), C.byref(h2)), ERR_LENGTH),
        "split_64": (lambda: L.lasso_poly_split(ctx._h, p._h, C.c_size_t(64), C.byref(h), C.byref(h2)), ERR_LENGTH),
        "split_null": (lambda: L.lasso_poly_split(ctx._h, p._h, C.c_size_t(2), None, C.byref(h2)), ERR_LENGTH),
        "split_other": (lambda: L.lasso_poly_split(ctx._h, po._h, C.c_size_t(2), C.byref(h), C.byref(h2)), ERR_STRATEGY),
        "padded_long": (lambda: L.lasso_poly_create_padded(ctx._h, _p(Z), C.c_size_t((1 << 28) + 1), C.byref(h)), ERR_LENGTH),
        "padded_null": (lambda: L.lasso_poly_create_padded(ctx._h, None, C.c_size_t(3), C.byref(h)), ERR_LENGTH),
        "padded_host_as_device": (lambda: L.lasso_poly_create_padded_device(ctx._h, _p(Z), C.c_size_t(5), C.c_size_t(4), None,
                                                                            C.byref(h)), ERR_POINTER),
        "padded_stride": (lambda: L.lasso_poly_create_padded_device(ctx._h, _p(Z), C.c_size_t(5), C.c_size_t(3), None,
                                                                    C.byref(h)), ERR_LENGTH),
        "read_cap": (lambda: L.lasso_poly_read(ctx._h, p._h, _p(out), C.c_size_t(63)), ERR_LENGTH),
        "read_null": (lambda: L.lasso_poly_read(ctx._h, p._h, None, C.c_size_t(64)), ERR_LENGTH),
        "read_other": (lambda: L.lasso_poly_read(ctx._h, po._h, _p(out), C.c_size_t(64)), ERR_STRATEGY),
        "read_dev_host": (lambda: L.lasso_poly_read_device(ctx._h, p._h, _p(out), C.c_size_t(4), None), ERR_POINTER),
        "read_dev_stride": (lambda: L.lasso_poly_read_device(ctx._h, p._h, _p(out), C.c_size_t(2), None), ERR_LENGTH),
    }
    t = lb.Transcript(b"errors")
    before = lb.Transcript(b"errors").challenge_scalar(b"c")
    for name, (fn, want) in calls.items():
        n0 = ctx.launches
        assert fn() == want, name
        assert ctx.launches == n0, name
    assert (t.challenge_scalar(b"c") == before).all()
    if torch.cuda.device_count() > 1:  # device memory of another GPU
        z1 = torch.zeros((64, 4), dtype=torch.int64, device="cuda:1")
        assert L.lasso_poly_read_device(ctx._h, p._h, C.c_void_p(z1.data_ptr()), C.c_size_t(4), None) == ERR_POINTER
    # a non-canonical evaluation is found by the ingest pass, from the host and from a tensor
    badZ = Z[:5].copy()
    badZ[4, 3] = np.uint64(2**64 - 1)
    for src in (badZ, torch.from_numpy(badZ.view(np.int64)).cuda()):
        with pytest.raises(lb.LassoError) as e:
            lb.DensePolynomial.new_padded(ctx, src)
        assert e.value.code == ERR_VALUE
    assert (p.to_numpy() == Z).all()
    del po
    other.close()
