"""Edge grids, plain-integer references and checks for the field and group primitives of the op table in
tests/kernel_harness/arith_ops.cuh (fr.cuh, fq.cuh, ed25519.cuh, quad.cuh).  Shared by test_gpu_arith.py (the sm_90a
build, in both compilations of fq_mul) and test_arith_host.py (the same table compiled with g++).

Fr inputs are Montgomery limbs of residues below l; Fq inputs are any integer below 2^256 (the kernels' loose
reduction).  Points are handed over as several projective representatives of each affine point: Z = 1 or a random
lambda, and coordinates replaced by x + q (still below 2^256).  Every result is checked against Python integers:
exact limbs for Fr and for the canonical Fq outputs, the residue mod q for the loose ones, and projectively (X/Z, Y/Z
against the affine result, T Z = X Y) for points."""
import functools
import random

import numpy as np

import oracle_lib as ol
import pyref
from test_gpu_launchers import raw, raw_ints

L = ol.L_FR
Q = ol.Q_FQ
D = pyref.D
R = 2**256 % L
R2 = R * R % L
RINV = pow(2**256, -1, L)
INV38 = pow(38, -1, Q)
SQRT_M1 = pow(2, (Q - 1) // 4, Q)
N_RANDOM = 1 << 16  # random structured inputs per operation, on top of the grid

LIMB_PATTERNS = (0, 1, 2, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF, None)  # None: a random limb

FQ_SPECIALS = [0, 1, 2, 37, 38, 39, Q - 1, Q, Q + 1, 2**255 - 1, 2**255, 2**255 + 18, 2**255 + 19, 2**256 - 1,
               2**256 - 19, 2**256 - 37, 2**256 - 38, 2**256 - 39]
FR_SPECIALS = ([0, 1, 2, L - 1, L - 2, (L - 1) // 2, (L + 1) // 2, 2**252 - 1, 2**252, R, R2]
               + [L - 2**j for j in (0, 1, 2, 31, 32, 33, 63, 64, 95, 96, 124, 125, 126, 127, 128, 159, 160, 191, 192,
                                     223, 224, 250, 251)])
GRID = 100  # values per grid: every ordered pair of it goes through each binary operation


# ---------------------------------------------------------------- scalar inputs
def structured(rng):
    """a 256-bit value built limb by limb from LIMB_PATTERNS; a quarter of them repeat one pattern in every limb"""
    if rng.random() < 0.25:
        p = rng.choice(LIMB_PATTERNS)
        limbs = [rng.getrandbits(32) if p is None else p for _ in range(8)]
    else:
        limbs = [rng.getrandbits(32) if p is None else p for p in (rng.choice(LIMB_PATTERNS) for _ in range(8))]
    return sum(v << (32 * i) for i, v in enumerate(limbs))


def structured_fr(rng):
    """a structured value below l: one at or above l keeps its low 252 bits"""
    x = structured(rng)
    return x if x < L else x & (2**252 - 1)


@functools.lru_cache(maxsize=None)
def grid(field):
    rng = random.Random("grid-" + field)
    vals = list(FR_SPECIALS if field == "fr" else FQ_SPECIALS)
    gen = structured_fr if field == "fr" else structured
    while len(vals) < GRID:
        vals.append(gen(rng))
    return vals


@functools.lru_cache(maxsize=None)
def randoms(field, count, salt=""):
    rng = random.Random("rand-%s-%s" % (field, salt))
    gen = structured_fr if field == "fr" else structured
    return [gen(rng) for _ in range(count)]


# ---------------------------------------------------------------- points
def fq_sqrt(a):
    a %= Q
    r = pow(a, (Q + 3) // 8, Q)
    if r * r % Q != a:
        r = r * SQRT_M1 % Q
    return r if r * r % Q == a else None


def on_curve(P):
    x, y = P
    return (-x * x + y * y - 1 - D * x * x * y * y) % Q == 0


def te_neg(P):
    return ((-P[0]) % Q, P[1])


def torsion_points():
    """the seven non-identity points of the 8-torsion: (0, -1), (+-sqrt(-1), 0) and the four of order 8 (2P has
    y = 0: y^2 = -x^2 and d x^4 - 2 x^2 - 1 = 0)"""
    pts = [(0, Q - 1), (SQRT_M1, 0), (Q - SQRT_M1, 0)]
    s = fq_sqrt(1 + D)
    for u in ((1 + s) * pow(D, -1, Q) % Q, (1 - s) * pow(D, -1, Q) % Q):
        x, y = fq_sqrt(u), fq_sqrt(-u)
        if x is not None and y is not None:
            pts += [(x, y), (x, Q - y), (Q - x, y), (Q - x, Q - y)]
    assert len(pts) == 7 and all(on_curve(P) for P in pts)
    assert [order(P) for P in pts] == [2, 4, 4, 8, 8, 8, 8]
    return pts


def order(P):
    k, S = 1, P
    while S != (0, 1):
        S = pyref.te_add(S, P)
        k += 1
    return k


@functools.lru_cache(maxsize=None)
def points():
    """the identity, generators and their negatives, the 8-torsion, generators plus torsion, random multiples"""
    g = ol.generators(8)
    gens = list(zip(ol.fq_ints(g[:, :4]), ol.fq_ints(g[:, 4:])))[:4] + [(pyref.BX, pyref.BY)]
    tors = torsion_points()
    rng = random.Random("points")
    pts = [(0, 1)] + gens + [te_neg(P) for P in gens[:2]] + tors
    pts += [pyref.te_add(gens[0], tors[3]), pyref.te_add(gens[1], tors[1]), pyref.te_add(gens[2], tors[0])]
    pts += [pyref.te_mul(gens[k % 5], rng.randrange(1, L)) for k in range(6)]
    assert all(on_curve(P) for P in pts)
    return pts


NREPS = 4


def ext_rep(P, r, lam):
    """projective representative r of affine P: 0 = (x, y, 1, xy); 1 = times a random lambda; 2 = as 1, every
    coordinate + q; 3 = lambda = -1 with X and Z + q"""
    x, y = P
    if r == 0:
        return (x, y, 1, x * y % Q)
    lam = lam if r in (1, 2) else Q - 1
    c = [lam * x % Q, lam * y % Q, lam, lam * x * y % Q]
    if r == 2:
        c = [v + Q for v in c]
    if r == 3:
        c[0] += Q
        c[2] += Q
    return tuple(c)


def niels(P):
    x, y = P
    return ((y + x) % Q, (y - x) % Q, 2 * D * x * y % Q)


def niels_rep(P, r):
    """0 = canonical, 1 = every coordinate + q, 2 = y+x + q, 3 = y-x and 2dxy + q"""
    add = ((0, 0, 0), (Q, Q, Q), (Q, 0, 0), (0, Q, Q))[r]
    return tuple(v + a for v, a in zip(niels(P), add))


def affine_rep(P, r):
    return (P[0] + (Q if r & 1 else 0), P[1] + (Q if r & 2 else 0))


def _point_inputs(kind):
    """(a, b, k, meta) rows for the point kinds; meta holds the affine points the reference works on"""
    pts = points()
    rng = random.Random("reps-" + kind)
    rows = []
    if kind in ("ext1", "niels1", "aff", "ark_aff"):
        for P in pts:
            for r in range(NREPS):
                if kind == "ext1":
                    a = ext_rep(P, r, rng.randrange(2, Q))
                elif kind == "niels1":
                    a = niels_rep(P, r)
                elif kind == "aff":
                    a = affine_rep(P, r)
                else:  # arkworks Montgomery limbs 38 x mod q, loose as well
                    a = affine_rep((38 * P[0] % Q, 38 * P[1] % Q), r)
                rows.append((a, (), 0, (P,)))
    elif kind in ("ext2", "ext_niels"):
        for i, P in enumerate(pts):
            for j, P2 in enumerate(pts):
                for ra, rb in (((i + j) % 4, (i + 2 * j + 1) % 4), ((i + j + 2) % 4, (i + 2 * j + 3) % 4)):
                    a = ext_rep(P, ra, rng.randrange(2, Q))
                    b = ext_rep(P2, rb, rng.randrange(2, Q)) if kind == "ext2" else niels_rep(P2, rb)
                    rows.append((a, b, 0, (P, P2)))
    elif kind == "xy":  # canonical affine coordinates for compression: every point, and x at the sign boundary
        for P in pts:
            rows.append((P, (), 0, (P,)))
        for x in (0, 1, (Q - 3) // 2, (Q - 1) // 2, (Q + 1) // 2, Q - 1):
            for y in (0, 1, Q - 1, rng.randrange(Q)):
                rows.append(((x, y), (), 0, ((x, y),)))
    else:
        raise KeyError(kind)
    return rows


def _scalar_inputs(kind):
    if kind in ("fr1", "fq1", "raw256"):
        f = "fr" if kind == "fr1" else "fq"
        vals = grid(f) + randoms(f, N_RANDOM)
        return [((a,), (), 0, (a, None, 0)) for a in vals]
    if kind in ("fr2", "fq2"):
        f = kind[:2]
        g = grid(f)
        pairs = [(a, b) for a in g for b in g] + list(zip(randoms(f, N_RANDOM, "a"), randoms(f, N_RANDOM, "b")))
        return [((a,), (b,), 0, (a, b, 0)) for a, b in pairs]
    if kind == "fr_pow2":
        rng = random.Random(kind)
        ak = [(a, k) for a in grid("fr") for k in range(32)] + [(a, rng.randrange(32)) for a in randoms("fr", N_RANDOM)]
        return [((a,), (), k, (a, None, k)) for a, k in ak]
    if kind == "fq_small":
        ks = (1, 38, 2**26 - 1)
        ak = [(a, k) for a in grid("fq") for k in ks] + [(a, ks[i % 3]) for i, a in enumerate(randoms("fq", N_RANDOM))]
        return [((a,), (), k, (a, None, k)) for a, k in ak]
    if kind == "u64":
        ks = sorted({0, 1, 2, 2**32 - 1, 2**32, 2**63, 2**64 - 1, L % 2**64} | {v % 2**64 for v in grid("fq")}
                    | {v % 2**64 for v in randoms("fq", N_RANDOM)})
        return [((), (), k, (None, None, k)) for k in ks]
    raise KeyError(kind)


@functools.lru_cache(maxsize=None)
def inputs(kind):
    """-> (A, B, K, rows): A, B (n, 16) u64 element arrays, K (n,) u64, rows [(a, b, k, meta)]"""
    rows = _scalar_inputs(kind) if kind in SCALAR_KINDS else _point_inputs(kind)
    return pack([r[0] for r in rows]), pack([r[1] for r in rows]), np.array([r[2] for r in rows], dtype=np.uint64), rows


SCALAR_KINDS = ("fr1", "fr2", "fq1", "fq2", "raw256", "fr_pow2", "fq_small", "u64")


def pack(rows):
    """rows of up to four 256-bit coordinates -> (n, 16) u64, the element layout of arith_ops.cuh"""
    out = np.zeros((len(rows), 16), dtype=np.uint64)
    width = max((len(r) for r in rows), default=0)
    for j in range(width):
        out[:, 4 * j:4 * j + 4] = raw([r[j] if j < len(r) else 0 for r in rows])
    return out


def unpack(out, ncoords):
    cols = [raw_ints(out[:, 4 * j:4 * j + 4]) for j in range(ncoords)]
    return list(zip(*cols))


# ---------------------------------------------------------------- operations: input kind, reference, check, coords out
def _fr_inv(a):
    return R2 * pow(a, -1, L) % L if a else 0


def _add(m):
    return pyref.te_add(m[0], m[1])


OPS = {
    # Fr, Montgomery limbs in and out, every output the canonical residue
    "fr_add": ("fr2", lambda m: ((m[0] + m[1]) % L,), "exact", 1),
    "fr_sub": ("fr2", lambda m: ((m[0] - m[1]) % L,), "exact", 1),
    "fr_neg": ("fr1", lambda m: (-m[0] % L,), "exact", 1),
    "fr_dbl": ("fr1", lambda m: (2 * m[0] % L,), "exact", 1),
    "fr_mul": ("fr2", lambda m: (m[0] * m[1] * RINV % L,), "exact", 1),
    "fr_mul_chain": ("fr2", lambda m: (m[0] * m[1] * RINV % L,), "exact", 1),
    "fr_sqr": ("fr1", lambda m: (m[0] * m[0] * RINV % L,), "exact", 1),
    "fr_mul_pow2": ("fr_pow2", lambda m: ((m[0] << m[2]) % L,), "exact", 1),
    "fr_from_u64": ("u64", lambda m: (m[2] * R % L,), "exact", 1),
    "fr_to_canonical": ("fr1", lambda m: (m[0] * RINV % L,), "exact", 1),
    "fr_eq": ("fr2", lambda m: (int(m[0] == m[1]),), "exact", 1),
    "fr_is_zero": ("fr1", lambda m: (int(m[0] == 0),), "exact", 1),
    "fr_from_raw_int": ("raw256", lambda m: (m[0] * R % L,), "exact", 1),
    "fr_inv": ("fr1", lambda m: (_fr_inv(m[0]),), "exact", 1),
    # Fq, internal integers: loose outputs need the right residue, canonical ones the exact value below q
    "fq_add": ("fq2", lambda m: ((m[0] + m[1]) % Q,), "loose", 1),
    "fq_sub": ("fq2", lambda m: ((m[0] - m[1]) % Q,), "loose", 1),
    "fq_neg": ("fq1", lambda m: (-m[0] % Q,), "loose", 1),
    "fq_dbl": ("fq1", lambda m: (2 * m[0] % Q,), "loose", 1),
    "fq_mul": ("fq2", lambda m: (m[0] * m[1] % Q,), "loose", 1),
    "fq_sqr": ("fq1", lambda m: (m[0] * m[0] % Q,), "loose", 1),
    "fq_mul_small": ("fq_small", lambda m: (m[0] * m[2] % Q,), "loose", 1),
    "fq_canonical": ("fq1", lambda m: (m[0] % Q,), "exact", 1),
    "fq_is_zero": ("fq1", lambda m: (int(m[0] % Q == 0),), "exact", 1),
    "fq_equal": ("fq2", lambda m: (int((m[0] - m[1]) % Q == 0),), "exact", 1),
    "fq_inv": ("fq1", lambda m: (pow(m[0], Q - 2, Q),), "loose", 1),
    "fq_from_ark": ("fq1", lambda m: (m[0] * INV38 % Q,), "loose", 1),
    "fq_to_ark": ("fq1", lambda m: (38 * m[0] % Q,), "exact", 1),
    # group
    "niels_from_affine": ("aff", lambda m: niels(m[0]), "loose", 3),
    "niels_from_ark_affine": ("ark_aff", lambda m: niels(m[0]), "loose", 3),
    "niels_neg": ("niels1", lambda m: niels(te_neg(m[0])), "loose", 3),
    "pt_madd": ("ext_niels", _add, "proj", 4),
    "pt_msub": ("ext_niels", lambda m: pyref.te_add(m[0], te_neg(m[1])), "proj", 4),
    "pt_add": ("ext2", _add, "proj", 4),
    "pt_dbl": ("ext1", lambda m: pyref.te_add(m[0], m[0]), "proj", 4),
    "pt_neg": ("ext1", lambda m: te_neg(m[0]), "proj", 4),
    "pt_from_niels": ("niels1", lambda m: m[0], "proj", 4),
    "pt_to_affine_canonical": ("ext1", lambda m: m[0], "exact", 2),
    "pt_compress_canonical": ("xy", lambda m: (int.from_bytes(pyref.ark_encode(m[0]), "little"),), "exact", 1),
    # quad-lane forms (device only): the same group law on four lanes
    "quad_add": ("ext2", _add, "proj", 4),
    "quad_madd": ("ext_niels", _add, "proj", 4),
    "quad_dbl": ("ext1", lambda m: pyref.te_add(m[0], m[0]), "proj", 4),
}
QUAD_OPS = ("quad_add", "quad_madd", "quad_dbl")
THREAD_OPS = tuple(k for k in OPS if k not in QUAD_OPS)


def _ok(how, got, want):
    if how == "exact":
        return tuple(got) == tuple(want)
    if how == "loose":
        return all(g % Q == w for g, w in zip(got, want))
    X, Y, Z, T = got  # proj
    if Z % Q == 0:
        return False
    zi = pow(Z, -1, Q)
    return X * zi % Q == want[0] and Y * zi % Q == want[1] and T * Z % Q == X * Y % Q


@functools.lru_cache(maxsize=None)
def wants(name):
    kind, ref, _, _ = OPS[name]
    return [ref(r[3]) for r in inputs(kind)[3]]


def hexs(t):
    return "(" + ", ".join("%#x" % v for v in t) + ")"


def check_op(run, variant, name):
    """run(name, A, B, K) -> (n, 16) u64 outputs; every element against its reference, the first mismatch named"""
    kind, _, how, nout = OPS[name]
    A, B, K, rows = inputs(kind)
    got = unpack(run(name, A, B, K), nout)
    want = wants(name)
    bad = [i for i in range(len(rows)) if not _ok(how, got[i], want[i])]
    if bad:
        i = bad[0]
        a, b, k, _ = rows[i]
        raise AssertionError("%s [%s]: %d of %d elements wrong, first [%d]: a = %s, b = %s, k = %d: got %s, want %s (%s)"
                             % (name, variant, len(bad), len(rows), i, hexs(a), hexs(b), k, hexs(got[i]), hexs(want[i]),
                                {"exact": "exact limbs", "loose": "residue mod q",
                                 "proj": "affine x, y of X/Z, Y/Z and T Z = X Y"}[how]))
