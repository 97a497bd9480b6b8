"""Σ-protocols of committed scalars without a GPU: the oracle's KnowledgeProof, EqualityProof and ProductProof provers
against its verifiers (restated from subprotocols/zk.rs).  Every proof field and every commitment is load-bearing, other
generators are rejected, and so are proofs of false statements."""
import numpy as np
import pytest

import oracle_dense_lib as od
import oracle_lib as ol
import oracle_sigma_lib as osg
import oracle_zk_lib as oz

L = ol.L_FR
SEED = ol.fr_array([5151])[0]
OTHER_FR = (12345).to_bytes(32, "little")


def _gens(label=b"sigma_gens"):
    return oz.mc_gens(ol.generators(2, label), 1)


def _fr(v):
    return ol.fr_array([v % L])[0]


def _io():
    return od.Transcript(b"sigma"), od.RandomTape(b"tape", SEED)


def _other_pt(g):
    return oz.commit(g, _fr(7), _fr(0))


def _swapped(proof, off, other):
    return proof[:off] + other + proof[off + 32:]


VALUES = [  # (x, r) as integers: random, and the edges 0, 1 and p - 1 with zero blinds
    (None, None), (0, 0), (1, 0), (L - 1, 0), (0, 5), (L - 1, L - 1),
]


def _vals(rng, pair):
    return [ol.rand_fr(rng, 1)[0] if v is None else _fr(v) for v in pair]


@pytest.mark.parametrize("pair", VALUES)
def test_knowledge(pair):
    rng = np.random.default_rng(1)
    g = _gens()
    x, r = _vals(rng, pair)
    proof, C = osg.knowledge_prove(g, *_io(), x, r)
    assert len(proof) == 96 and C == oz.commit(g, x, r)
    assert osg.knowledge_verify(g, proof, C, _io()[0]) == 0
    assert osg.knowledge_verify(g, _swapped(proof, 0, _other_pt(g)), C, _io()[0]) == 1
    for off in (32, 64):
        assert osg.knowledge_verify(g, _swapped(proof, off, OTHER_FR), C, _io()[0]) == 1, off
    assert osg.knowledge_verify(g, proof, _other_pt(g), _io()[0]) == 1
    assert osg.knowledge_verify(_gens(b"other"), proof, C, _io()[0]) == 1
    assert osg.knowledge_verify(g, proof[:95], C, _io()[0]) == 2


@pytest.mark.parametrize("pair", VALUES)
def test_equality(pair):
    rng = np.random.default_rng(2)
    g = _gens()
    v, s1 = _vals(rng, pair)
    s2 = ol.rand_fr(rng, 1)[0]  # the same value under different blinds is a true statement
    proof, C1, C2 = osg.equality_prove(g, *_io(), v, s1, v, s2)
    assert len(proof) == 64 and C1 == oz.commit(g, v, s1) and C2 == oz.commit(g, v, s2)
    assert osg.equality_verify(g, proof, C1, C2, _io()[0]) == 0
    assert osg.equality_verify(g, _swapped(proof, 0, _other_pt(g)), C1, C2, _io()[0]) == 1
    assert osg.equality_verify(g, _swapped(proof, 32, OTHER_FR), C1, C2, _io()[0]) == 1
    assert osg.equality_verify(g, proof, _other_pt(g), C2, _io()[0]) == 1
    assert osg.equality_verify(g, proof, C1, _other_pt(g), _io()[0]) == 1
    assert osg.equality_verify(_gens(b"other"), proof, C1, C2, _io()[0]) == 1
    # v1 != v2: the proof does not convince
    v2 = _fr(ol.fr_ints(v)[0] + 1)
    proof, C1, C2 = osg.equality_prove(g, *_io(), v, s1, v2, s2)
    assert osg.equality_verify(g, proof, C1, C2, _io()[0]) == 1


PRODUCTS = [  # (x, y) as integers, or None for random; blinds random unless the pair is an edge case
    (None, None), (0, 0), (1, 1), (L - 1, L - 1), (0, 9), (1, L - 1),
]


@pytest.mark.parametrize("pair", PRODUCTS)
def test_product(pair):
    rng = np.random.default_rng(3)
    g = _gens()
    x, y = _vals(rng, pair)
    edge = pair[0] is not None
    rX, rY, rZ = (_fr(0),) * 3 if edge else ol.rand_fr(rng, 3)
    z = _fr(ol.fr_ints(x)[0] * ol.fr_ints(y)[0])
    proof, X, Y, Z = osg.product_prove(g, *_io(), x, rX, y, rY, z, rZ)
    assert len(proof) == 256
    assert (X, Y, Z) == (oz.commit(g, x, rX), oz.commit(g, y, rY), oz.commit(g, z, rZ))
    assert osg.product_verify(g, proof, X, Y, Z, _io()[0]) == 0
    for off in (0, 32, 64):
        assert osg.product_verify(g, _swapped(proof, off, _other_pt(g)), X, Y, Z, _io()[0]) == 1, off
    for off in range(96, 256, 32):
        assert osg.product_verify(g, _swapped(proof, off, OTHER_FR), X, Y, Z, _io()[0]) == 1, off
    for k in range(3):
        pts = [X, Y, Z]
        pts[k] = _other_pt(g)
        assert osg.product_verify(g, proof, *pts, _io()[0]) == 1, k
    assert osg.product_verify(_gens(b"other"), proof, X, Y, Z, _io()[0]) == 1
    assert osg.product_verify(g, proof + bytes(8), X, Y, Z, _io()[0]) == 2
    # z != x y: the proof does not convince
    bad = _fr(ol.fr_ints(z)[0] + 1)
    proof, X, Y, Z = osg.product_prove(g, *_io(), x, rX, y, rY, bad, rZ)
    assert osg.product_verify(g, proof, X, Y, Z, _io()[0]) == 1


def test_point_lincomb():
    """sum a_i C_i of commitments is the commitment to sum a_i v_i with blind sum a_i s_i"""
    rng = np.random.default_rng(4)
    g = _gens()
    v, s, a = ol.rand_fr(rng, 3), ol.rand_fr(rng, 3), ol.rand_fr(rng, 3)
    C = [oz.commit(g, v[i], s[i]) for i in range(3)]
    dot = lambda p, q: _fr(sum(i * j for i, j in zip(ol.fr_ints(p), ol.fr_ints(q))))  # noqa: E731
    assert osg.point_lincomb(C, a) == oz.commit(g, dot(a, v), dot(a, s))
