"""The generator tables every commitment and opening reads, built as a proof builds them (gens_build_tables, prover.cu;
tests/kernel_harness: kh_tables_build, harness_setup.cu) and read back entry by entry, against the CPU oracle's group
law on generators from orc_sample_generators:

  T[w][j]        = 2^(8w) G_j                  launch_build_table, every window, over n_points generators
  M[w][j][d-1]   = d 2^(8w) G_j,  d = 1..128   launch_build_multiples over the first nd generators (stride n_points)
  M16[jl][d-1]   = d G_j, d = 1..32768         launch_build_multiples16, j = jl col_mul + col_add (npts8 = nd)
  K16[k]         = 2^15 sum_{jl < 2^k} G_j     launch_centre_constant, every 2^k <= ncols16

Shapes: n_points 130 (a partial CTA of 128), 2050 (the 2^20-lookup configuration) and 4098; nd = n_points and the
prover's nd < n_points; ncols16 1, 2, 64 and 256; the column maps of G = 1, 2, 4 and 8 ranks at every rank.  Entries
come back as arkworks affine (x, y) with the niels entries' t2d (checked against 2 d x y) or the extended K16's T / Z
(checked against x y).  Every window and digit of the columns {0, 1, 127, 128, 129, last} and a random sample of the
rest; all 32768 entries of the first, a middle and the last local column of M16, and a sample of the others that hits
each of its 128 blocks of 256 entries at each of the 16 positions of a batch inversion."""
import ctypes as C
import random

import numpy as np
import pytest

import kernel_harness_lib as kh
import oracle_lib as ol
from oracle_lib import P, lib as orc
from test_gpu_launchers import raw_ints

pytestmark = pytest.mark.gpu

Q, L = ol.Q_FQ, ol.L_FR
RM = 2**256 % Q  # the Montgomery factor of Fq
D2 = 2 * (-121665 * pow(121666, -1, Q)) % Q
NGENS = 4098
TABLE_T, TABLE_M, TABLE_M16, TABLE_K16 = range(4)


@pytest.fixture(scope="module")
def gens():
    return np.ascontiguousarray(ol.generators(NGENS))


# ---------------------------------------------------------------- the oracle's points (projective Montgomery limbs)
_proj = {}


def gen_point(gens, j):
    if j not in _proj:
        out = np.zeros(16, dtype=np.uint64)
        orc().orc_point_from_affine(P(np.ascontiguousarray(gens[j])), P(out))
        _proj[j] = out
    return _proj[j]


def point_mul(pt, k):
    out = np.zeros(16, dtype=np.uint64)
    orc().orc_point_mul(P(pt), P(ol.to_mont(k % L, L)), P(out))
    return out


def chain(start, step, count):
    """start, start + step, ..., start + (count - 1) step: (count, 16) limbs"""
    out = np.zeros((count, 16), dtype=np.uint64)
    out[0] = start
    add, base, sp = orc().orc_point_add, out.ctypes.data, P(step)
    for i in range(1, count):
        add(C.c_void_p(base + 128 * (i - 1)), sp, C.c_void_p(base + 128 * i))
    return out


def projective(points):
    """(count, 16) limbs -> [(X, Y, Z)] Montgomery integers"""
    v = raw_ints(points.reshape(-1, 4))
    return [(v[4 * i], v[4 * i + 1], v[4 * i + 3]) for i in range(points.shape[0])]


_windows, _digits, _m16 = {}, {}, {}


def windows(gens, j):
    """2^(8w) G_j, w = 0..31, by doubling"""
    if j not in _windows:
        out = np.zeros((32, 16), dtype=np.uint64)
        out[0] = gen_point(gens, j)
        for w in range(1, 32):
            out[w] = out[w - 1]
            for _ in range(8):
                orc().orc_point_dbl(P(out[w]), P(out[w]))
        _windows[j] = out
    return _windows[j]


def digits(gens, j):
    """d 2^(8w) G_j, (w, d) -> index w * 128 + d - 1, by repeated addition"""
    if j not in _digits:
        ws = windows(gens, j)
        _digits[j] = projective(np.concatenate([chain(ws[w], np.ascontiguousarray(ws[w]), 128) for w in range(32)]))
    return _digits[j]


def multiples16(gens, j):
    """d G_j, d = 1..32768, by repeated addition"""
    if j not in _m16:
        g = gen_point(gens, j)
        _m16[j] = projective(chain(g, g, 32768))
    return _m16[j]


# ---------------------------------------------------------------- device entries
def entries(t, which, idx):
    idx = np.ascontiguousarray(np.asarray(idx, dtype=np.uint64))
    out = np.zeros((idx.shape[0], 12), dtype=np.uint64)
    kh.call("kh_table_entries", t.h, which, idx.ctypes.data, idx.shape[0], out.ctypes.data)
    v = raw_ints(out.reshape(-1, 4))
    return [tuple(v[3 * i:3 * i + 3]) for i in range(idx.shape[0])]


def check(what, got, want, labels, ext=False):
    """device (x, y, t) against the oracle's (X, Y, Z), all Montgomery: x Z = X R, y Z = Y R, and t R = 2d x y (niels)
    or t R = x y (extended)"""
    for (x, y, t), (X, Y, Z), lab in zip(got, want, labels):
        assert (x * Z - X * RM) % Q == 0 and (y * Z - Y * RM) % Q == 0, "%s: entry %s differs" % (what, lab)
        rhs = x * y if ext else D2 * x * y
        assert (t * RM - rhs) % Q == 0, "%s: entry %s: %s" % (what, lab, "T / Z != x y" if ext else "t2d != 2 d x y")
    assert len(got) == len(want)


def named_columns(count):
    return sorted({c for c in (0, 1, 127, 128, 129, count - 1) if c < count})


# ---------------------------------------------------------------- the tables of one build
def check_T(t, gens, n_points, rng, what):
    cols = named_columns(n_points)
    idx = [w * n_points + j for j in cols for w in range(32)]
    want = [p for j in cols for p in projective(windows(gens, j))]
    check(what + " T", entries(t, TABLE_T, idx), want, [(w, j) for j in cols for w in range(32)])
    sample = [(rng.randrange(32), rng.randrange(n_points)) for _ in range(256)]
    want = projective(np.stack([point_mul(gen_point(gens, j), 1 << (8 * w)) for w, j in sample]))
    check(what + " T sample", entries(t, TABLE_T, [w * n_points + j for w, j in sample]), want, sample)


def check_M(t, gens, nd, rng, what):
    cols = named_columns(nd)
    idx = [(w * nd + j) * 128 + d - 1 for j in cols for w in range(32) for d in range(1, 129)]
    want = [p for j in cols for p in digits(gens, j)]
    check(what + " M", entries(t, TABLE_M, idx), want, [(w, j, d) for j in cols for w in range(32) for d in range(1, 129)])
    sample = [(rng.randrange(32), rng.randrange(nd), rng.randrange(1, 129)) for _ in range(256)]
    want = projective(np.stack([point_mul(gen_point(gens, j), d << (8 * w)) for w, j, d in sample]))
    check(what + " M sample", entries(t, TABLE_M, [(w * nd + j) * 128 + d - 1 for w, j, d in sample]), want, sample)


def check_M16(t, gens, ncols16, col_mul, col_add, rng, what):
    full = sorted({0, ncols16 // 2, ncols16 - 1})
    for jl in full:
        j = jl * col_mul + col_add
        check("%s M16 local column %d (generator %d)" % (what, jl, j), entries(t, TABLE_M16, range(jl * 32768, (jl + 1) * 32768)),
              multiples16(gens, j), ["d=%d" % d for d in range(1, 32769)])
    # every (block b, batch position k): entry 256 b + 16 grp + k of a random column, grp random
    others = [c for c in range(ncols16) if c not in full] or full
    sample = [(rng.choice(others), 256 * b + 16 * rng.randrange(16) + k) for b in range(128) for k in range(16)]
    want = projective(np.stack([point_mul(gen_point(gens, jl * col_mul + col_add), e + 1) for jl, e in sample]))
    check(what + " M16 sample", entries(t, TABLE_M16, [jl * 32768 + e for jl, e in sample]), want,
          ["column %d d=%d" % (jl, e + 1) for jl, e in sample])


def check_K16(t, gens, ncols16, col_mul, col_add, what):
    ks = [k for k in range(32) if 1 << k <= ncols16]
    acc, want = None, []
    for jl in range(ncols16):
        g = gen_point(gens, jl * col_mul + col_add)
        if acc is None:
            acc = g.copy()
        else:
            orc().orc_point_add(P(acc), P(g), P(acc))
        if (jl + 1) in [1 << k for k in ks]:
            want.append(point_mul(acc, 1 << 15))
    check(what + " K16", entries(t, TABLE_K16, ks), projective(np.stack(want)), ["k=%d" % k for k in ks], ext=True)


# (n_points, nd, ncols16, G): rank g of G builds M16 over its columns jl G + g, every g.  nd - 2 = ncols16 G is the
# prover's own choice (the openings' R_size + 2 generators; ncols16 = (nd - 2) / G)
CASES = [(130, 130, 1, 1), (130, 66, 64, 1), (130, 130, 2, 2), (2050, 2050, 256, 8), (2050, 1026, 256, 4),
         (4098, 4098, 64, 1), (4098, 2050, 2, 2)]


@pytest.mark.parametrize("n_points,nd,ncols16,G", CASES, ids=["n%d-nd%d-c%d-G%d" % c for c in CASES])
def test_tables(gens, n_points, nd, ncols16, G):
    rng = random.Random(repr((n_points, nd, ncols16, G)))
    for g in range(G):
        what = "tables n_points=%d nd=%d ncols16=%d, rank %d of %d" % (n_points, nd, ncols16, g, G)
        t = kh.Tables.as_prover(gens[:n_points], nd, ncols16, G, g)
        try:
            if g == 0:  # T and M do not depend on the rank
                check_T(t, gens, n_points, rng, what)
                check_M(t, gens, nd, rng, what)
            check_M16(t, gens, ncols16, G, g, rng, what)
            check_K16(t, gens, ncols16, G, g, what)
        finally:
            t.close()


def test_arguments_refused(gens):
    """M16 may only read columns of M: a column map past nd, or nd past n_points, is refused before any launch"""
    g = np.ascontiguousarray(gens[:130])
    h = C.c_void_p()
    for nd, ncols16, mul, add in ((131, 0, 1, 0), (0, 0, 1, 0), (130, 17, 8, 2), (66, 66, 1, 1)):
        assert kh.lib().kh_tables_build(g.ctypes.data, 130, nd, ncols16, mul, add, C.byref(h)) == -4, (nd, ncols16, mul, add)
