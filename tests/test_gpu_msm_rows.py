"""The row-MSM family of msm_kernels.cu one launch at a time, against the CPU oracle (tests/kernel_harness:
harness_msm.cu).  Every Hyrax commitment with at most 8 rows, every commitment without the multiples tables, the
variable-base lasso_msm / lasso_commit_rows below 2^14 terms and every commitment of a proof sharded over several GPUs
goes through these launchers; the whole-proof tests reach them only at a few shapes.

a. launch_msm_rows (msm_bucket_kernel<1> / <8>, one launch per 65535 rows, msm_finish_kernel) in the three forms the
   library runs: fixed-base u32 (shifted = 1, nw = 1..5), fixed-base 256-bit (nw = 32) and variable-base 256-bit
   (shifted = 0, nw from the data).  The shapes reach every branch of msm_geometry: one or two rows, whose columns are
   split so that about one CTA runs per SM (up to 128 partials per row in the finish), >= 132 rows (chunk = min(ncols,
   cap)), one column, a chunk plus one, and 65535 .. 131071 rows.  Scalar sets per row: uniform, zero, a zero chunk
   inside a row (a CTA with no entry), one value repeated (every digit of a window in one bucket), digits -128 and
   +127 only, {0, 1, the widest value msm_windows_for_bits allows}, and exactly 127 / 128 / 129 entries in one CTA.
b. launch_sum_raw_points: 1..8 loosely reduced projective sources per row, with the identity, P + (-P) and P + P.
c. launch_canonicalize: bit-exact canonical limbs and the atomic maximum of the bit length over limbs, warps, CTAs and
   the grid-stride loop; chained into (a) as lasso_msm chains them: the window count it implies is enough.
d. Sharded commitments as a proof over G = 2, 4, 8 GPUs computes them, in one process: each rank's launch over its
   columns (col_mul = G, col_add = rank) with out_raw, the ranks' points stacked, one launch_sum_raw_points.  The
   three commit paths: the bucket MSM, msm_rows_direct_u32 (with and without the 16-bit table) and msm_rows_direct_fr.

Points are compared bit-exact: out_comp with the oracle's compressed bytes, out_ext with (x, y, x y, 1) in arkworks
Montgomery limbs, out_raw as X / Z, Y / Z with T Z = X Y, in Python integers mod q."""
import random

import numpy as np
import pytest

import kernel_harness_lib as kh
import oracle_lib as ol
from oracle_lib import P, lib as orc, sz
from test_gpu_launchers import mont, ptr, raw, raw_ints

pytestmark = pytest.mark.gpu

L, Q = ol.L_FR, ol.Q_FQ
R256 = 2**256
RQ_INV = pow(R256, -1, Q)
NUM_SMS = 132  # kNumSMs (common.cuh)
NGENS = 4098


@pytest.fixture(scope="module")
def gens():
    return np.ascontiguousarray(ol.generators(NGENS))


@pytest.fixture(scope="module")
def tables(gens):
    t = kh.Tables(gens)
    yield t
    t.close()


# ---------------------------------------------------------------- restated launch arithmetic
def windows_for_bits(bits):
    """msm_windows_for_bits (msm.cuh)"""
    return max(1, (bits + 2 + 7) // 8)


def geometry(nrows, ncols, nw, shifted):
    """msm_geometry (msm_kernels.cu): (window groups, columns per chunk, chunks per row)"""
    wpc = nw if shifted else 1
    ngroups = -(-nw // wpc)
    cap = max(1, 8192 // wpc)
    ctas = nrows * ngroups
    want = -(-NUM_SMS // ctas)
    chunk = -(-ncols // want) if want > 1 else ncols
    chunk = max(chunk, max(8, 1024 // wpc))
    chunk = max(1, min(chunk, cap, ncols))
    return ngroups, chunk, -(-ncols // chunk)


def widest(limbs, nw):
    """the widest scalar nw windows take: 2^(8 nw - 2) - 1, clamped to the scalar type"""
    return min((1 << (8 * nw - 2)) - 1, (1 << 32) - 1 if limbs == 1 else L - 1)


# ---------------------------------------------------------------- references
class Ref:
    """the oracle's points: compressed bytes (n, 32), out_ext limbs (n, 16) and affine integers"""

    def __init__(self, points):
        n = points.shape[0]
        self.comp = np.zeros((n, 32), dtype=np.uint8)
        aff = np.zeros((n, 8), dtype=np.uint64)
        for i in range(n):
            orc().orc_point_compress(P(points[i]), P(self.comp[i]))
            orc().orc_point_to_affine(P(points[i]), P(aff[i]))
        xy = raw_ints(aff)
        self.xy = [(xy[2 * i] * RQ_INV % Q, xy[2 * i + 1] * RQ_INV % Q) for i in range(n)]
        self.ext = raw([v for x, y in self.xy for v in (x * R256 % Q, y * R256 % Q, x * y * R256 % Q, R256 % Q)]
                       ).reshape(n, 16)


def oracle_rows(gens, rows, col_map=(1, 0)):
    """the oracle's Hyrax row commitments (blind zero) of `rows` (lists of integers) over gens[c * col_mul + col_add]"""
    nrows, ncols = len(rows), len(rows[0])
    col_mul, col_add = col_map
    gsel = np.ascontiguousarray(np.concatenate([gens[[c * col_mul + col_add for c in range(ncols)]], gens[:1]]))
    out = np.zeros((nrows, 16), dtype=np.uint64)
    orc().orc_commit_rows(P(gsel), P(mont([v for r in rows for v in r])), sz(nrows), sz(ncols), P(out))
    return Ref(out)


def check_points(what, ref, ext=None, comp=None, out_raw=None, row_of=None):
    """output row i against reference row row_of[i] (default i); names the first differing row"""
    n = next(a.shape[0] for a in (ext, comp, out_raw) if a is not None)
    idx = np.arange(n) if row_of is None else row_of
    for name, got, want in (("out_comp", comp, ref.comp), ("out_ext", ext, ref.ext)):
        if got is not None:
            bad = np.nonzero((got != want[idx]).any(axis=1))[0]
            assert not len(bad), "%s: %s: %d of %d rows differ, first row %d" % (what, name, len(bad), n, bad[0])
    if out_raw is not None:
        v = raw_ints(out_raw.view(np.uint64).reshape(-1, 4))
        for i in range(n):
            X, Y, Z, T = v[4 * i:4 * i + 4]
            x, y = ref.xy[idx[i]]
            assert Z % Q and (T * Z - X * Y) % Q == 0 and (X - x * Z) % Q == 0 and (Y - y * Z) % Q == 0, \
                "%s: out_raw: row %d differs (or Z = 0, or T Z != X Y)" % (what, i)


def outputs(nrows, ext=True, comp=True, out_raw=True):
    return (np.zeros((nrows, 16), dtype=np.uint64) if ext else None,
            np.zeros((nrows, 32), dtype=np.uint8) if comp else None,
            np.zeros((nrows, 32), dtype=np.uint32) if out_raw else None)


def optr(a):
    return None if a is None else ptr(a)


def device_scalars(rows, limbs):
    """rows of integers -> compact u32 words (limbs 1: one word each, 8: canonical 256-bit)"""
    flat = [v for r in rows for v in r]
    if limbs == 1:
        return np.ascontiguousarray(np.array(flat, dtype=np.uint64).astype(np.uint32))
    return np.ascontiguousarray(raw(flat).view(np.uint32).reshape(-1))


def msm_rows(tables, shifted, rows, limbs, nw, col_map=(1, 0), pad=0, nrows=None, outs=(True, True, True)):
    """one kh_msm_rows launch over `rows` (repeated to nrows rows when given), row stride ncols + pad"""
    nrows = nrows or len(rows)
    ncols = len(rows[0])
    sc = device_scalars(rows, limbs)
    if nrows > len(rows):
        sc = np.ascontiguousarray(np.tile(sc.reshape(len(rows), -1), (-(-nrows // len(rows)), 1))[:nrows].reshape(-1))
    ext, comp, out_raw = outputs(nrows, *outs)
    kh.call("kh_msm_rows", tables.h, shifted, ptr(sc), limbs, ncols + pad, nrows, ncols, nw, col_map[0], col_map[1],
            optr(ext), optr(comp), optr(out_raw))
    return ext, comp, out_raw


# ---------------------------------------------------------------- (a) scalar sets
KINDS = ["uniform", "zero", "zero_chunk", "repeated", "digits", "edges", "count127", "count128", "count129"]


def digit_value(digits):
    """the scalar whose signed 8-bit digits (offset trick) are `digits`, low window first (top digit >= 0)"""
    return sum(d << (8 * w) for w, d in enumerate(digits))


def row_values(kind, ncols, limbs, nw, shifted, chunk, rng):
    top = widest(limbs, nw)
    if kind == "uniform":
        return [rng.randrange(top + 1) for _ in range(ncols)]
    if kind == "zero":
        return [0] * ncols
    if kind == "zero_chunk":  # the second chunk (or the first half of a one-chunk row) is all zero
        v = [rng.randrange(1, top + 1) for _ in range(ncols)]
        lo, hi = (chunk, 2 * chunk) if ncols > chunk else (0, ncols // 2)
        return [0 if lo <= c < hi else x for c, x in enumerate(v)]
    if kind == "repeated":
        return [rng.randrange(top // 2, top + 1)] * ncols
    if kind == "digits":  # every digit below the top window is -128 (bucket 128) or +127; the top one 0 or 1
        out = []
        for _ in range(ncols):
            if nw == 1:
                out.append(rng.randrange(top + 1))
                continue
            low = digit_value([rng.choice((-128, 127)) for _ in range(nw - 1)])
            out.append(low if low >= 0 else low + (1 << (8 * (nw - 1))))
        return out
    if kind == "edges":
        return [(0, 1, top)[rng.randrange(3)] for _ in range(ncols)]
    # countK: exactly K non-zero digits in the first CTA of the row, the rest of the row zero.  Over a shifted table a
    # CTA takes every window: columns of m = nw - 1 random non-zero digits (fewer in the last one), the top one
    # positive, so that each value stays below 2^(8 (nw - 1)).  Variable-base: window 0 only, one digit per column.
    want, m = int(kind[5:]), digits_per_column(nw, shifted)
    v = [0] * ncols
    c = 0
    while want > 0:
        k = min(m, want)
        if m == 1:
            v[c] = rng.randrange(1, min(top, 127) + 1)
        else:
            ds = [rng.choice(NONZERO_DIGITS) for _ in range(k)]
            ds[-1] = abs(ds[-1])
            v[c] = digit_value(ds)
        c += 1
        want -= k
    windows = range(nw) if shifted else range(1)
    assert sum(signed_digits(x, nw)[w] != 0 for x in v[:chunk] for w in windows) == int(kind[5:])
    return v


def signed_digits(v, nw):
    """the nw digits the kernels take from v: byte w of v + sum_w 128 * 2^(8w), minus 128"""
    b = v + sum(128 << (8 * w) for w in range(nw))
    return [((b >> (8 * w)) & 0xff) - 128 for w in range(nw)]


NONZERO_DIGITS = [d for d in range(-127, 128) if d]


def digits_per_column(nw, shifted):
    return max(1, nw - 1) if shifted else 1


def scalar_rows(kinds, ncols, limbs, nw, shifted, chunk, rng, nrows):
    """nrows rows, the scalar sets cycling over the rows; the countK sets only where one CTA can hold 129 entries"""
    kinds = [k for k in kinds if not k.startswith("count") or chunk * digits_per_column(nw, shifted) >= 129]
    if not kinds:
        return None, kinds
    return [row_values(kinds[r % len(kinds)], ncols, limbs, nw, shifted, chunk, rng) for r in range(nrows)], kinds


# (nrows, ncols, pad, column map); pad > 0: row stride ncols + pad with a poisoned gap
U32_SHAPES = [(1, 1, 0, (1, 0)), (1, 205, 0, (1, 0)), (1, 4096, 0, (1, 0)), (2, 4096, 3, (1, 0)), (2, 205, 0, (8, 7)),
              (132, 1639, 0, (2, 1)), (140, 300, 5, (1, 0)), (133, 1, 0, (1, 0))]
FULL_SHAPES = [(1, 1, 0, (1, 0)), (1, 33, 0, (8, 7)), (1, 4096, 0, (1, 0)), (2, 4096, 1, (1, 0)), (3, 300, 0, (1, 0)),
               (132, 4096, 0, (1, 0)), (133, 257, 2, (1, 0)), (140, 1, 0, (1, 0))]
VAR_SHAPES = [(1, 1, 0, (1, 0)), (1, 1025, 0, (1, 0)), (2, 4096, 0, (1, 0)), (3, 700, 2, (3, 2)), (132, 600, 0, (1, 0)),
              (140, 1, 1, (1, 0))]
CASES = ([("u32", 1, 1, 5, s) for s in U32_SHAPES] + [("u32", 1, 1, nw, s) for nw in (1, 2, 3, 4) for s in U32_SHAPES[1:6:2]]
         + [("full", 1, 8, 32, s) for s in FULL_SHAPES]
         + [("var", 0, 8, nw, s) for nw in (1, 2, 5, 17, 32) for s in VAR_SHAPES])


@pytest.mark.parametrize("form,shifted,limbs,nw,shape", CASES,
                         ids=["%s-nw%d-%dx%d%s%s" % (c[0], c[3], c[4][0], c[4][1], "-pad" if c[4][2] else "",
                                                     "-map%d.%d" % c[4][3] if c[4][3] != (1, 0) else "") for c in CASES])
def test_msm_rows(tables, gens, form, shifted, limbs, nw, shape):
    """nw: the windows of a fixed-base launch; variable-base: the width of the data (nw is then taken from it)"""
    nrows, ncols, pad, col_map = shape
    rng = random.Random(repr((form, nw, shape)))
    # few rows: one launch per scalar set; many: the sets cycle over the rows of one launch
    layouts = [[k] for k in KINDS] if nrows < len(KINDS) else [KINDS]
    for kinds in layouts:
        rows, used = scalar_rows(kinds, ncols, limbs, nw, shifted, geometry(nrows, ncols, nw, shifted)[1], rng, nrows)
        if not used:
            continue
        # variable-base: nw from the data, as lasso_msm takes it from launch_canonicalize
        nwl = nw if shifted else windows_for_bits(max(v.bit_length() for r in rows for v in r))
        ngroups, chunk, nchunks = geometry(nrows, ncols, nwl, shifted)
        what = ("msm_rows %s shifted=%d nw=%d %dx%d stride %d col_map %d*c+%d, %d partials/row (chunk %d), sets %s"
                % (form, shifted, nwl, nrows, ncols, ncols + pad, col_map[0], col_map[1], ngroups * nchunks, chunk, used))
        ext, comp, out_raw = msm_rows(tables, shifted, rows, limbs, nwl, col_map, pad)
        check_points(what, oracle_rows(gens, rows, col_map), ext, comp, out_raw)


@pytest.mark.parametrize("nrows", [65535, 65536, 65537, 131071])
def test_msm_rows_split(tables, gens, nrows):
    """more rows than one launch's gridDim.y: rows of period 251, every row compared"""
    period, ncols, nw = 251, 2, 5
    rng = random.Random(nrows)
    rows, used = scalar_rows(KINDS, ncols, 1, nw, 1, ncols, rng, period)
    ext, comp, out_raw = msm_rows(tables, 1, rows, 1, nw, nrows=nrows)
    what = "msm_rows u32 shifted=1 nw=%d %dx%d (rows of period %d) sets %s" % (nw, nrows, ncols, period, used)
    check_points(what, oracle_rows(gens, rows), ext, comp, out_raw, row_of=np.arange(nrows) % period)


def test_msm_rows_outputs_alone(tables, gens):
    """each output requested on its own gives what it gives next to the others"""
    rng = random.Random(5)
    for shifted, limbs, nw, nrows, ncols in ((1, 1, 5, 3, 300), (1, 8, 32, 2, 100), (0, 8, 32, 2, 100)):
        rows = [[rng.randrange(widest(limbs, nw) + 1) for _ in range(ncols)] for _ in range(nrows)]
        ref = oracle_rows(gens, rows)
        for outs in ((True, False, False), (False, True, False), (False, False, True)):
            what = "msm_rows shifted=%d limbs=%d nw=%d %dx%d outputs (ext, comp, raw) = %s" % (shifted, limbs, nw, nrows,
                                                                                              ncols, outs)
            check_points(what, ref, *msm_rows(tables, shifted, rows, limbs, nw, outs=outs))


# ---------------------------------------------------------------- (b) gather-then-add
def loose(v, rng):
    """v mod q as the device may hold it: v or v + q (both below 2^256)"""
    return v + Q if rng.randrange(3) == 0 else v


def projective(xy, rng):
    """(λx, λy, λ, λxy), loosely reduced, as 32 u32 words"""
    x, y = xy
    lam = rng.randrange(1, Q)
    coords = [lam * x % Q, lam * y % Q, lam, lam * x * y % Q]
    return np.frombuffer(b"".join(loose(c, rng).to_bytes(32, "little") for c in coords), dtype=np.uint32)


def oracle_sum(points):
    """the oracle's sum of affine points (x, y integers)"""
    bases = np.ascontiguousarray(np.concatenate([np.concatenate([ol.to_mont(x, Q), ol.to_mont(y, Q)]) for x, y in points]))
    out = np.zeros(16, dtype=np.uint64)
    orc().orc_msm(P(bases), P(mont([1] * len(points))), sz(len(points)), 2, P(out))
    return out


@pytest.mark.parametrize("nrows", [1, 63, 64, 65, 1000])
@pytest.mark.parametrize("nsrc", [1, 2, 3, 4, 8])
def test_sum_raw_points(gens, nsrc, nrows):
    rng = random.Random(nsrc * 10007 + nrows)
    pool = raw_ints(gens[:256].reshape(-1, 4))
    pool = [(pool[2 * i] * RQ_INV % Q, pool[2 * i + 1] * RQ_INV % Q) for i in range(256)]
    ident = (0, 1)
    pts = [[rng.choice(pool) for _ in range(nsrc)] for _ in range(nrows)]
    for r in range(nrows):
        kind = ("random", "random", "random", "identity", "P,-P", "P,P", "random")[r % 7]
        if kind == "identity":
            pts[r] = [ident] * nsrc
        elif kind == "P,-P":
            x, y = pts[r][0]
            pts[r][1:2] = [((Q - x) % Q, y)][:nsrc - 1]
        elif kind == "P,P":
            pts[r][1:2] = [pts[r][0]][:nsrc - 1]
    src = np.zeros((nsrc, nrows, 32), dtype=np.uint32)
    for r in range(nrows):
        for k in range(nsrc):
            src[k, r] = projective(pts[r][k], rng)
    src = np.ascontiguousarray(src.reshape(-1))
    ref = Ref(np.ascontiguousarray(np.stack([oracle_sum(pts[r]) for r in range(nrows)])))
    for outs in ((True, True, True), (True, False, False), (False, True, False), (False, False, True)):
        ext, comp, out_raw = outputs(nrows, *outs)
        kh.call("kh_sum_raw_points", ptr(src), nsrc, nrows, optr(out_raw), optr(comp), optr(ext))
        what = "sum_raw_points nsrc=%d nrows=%d outputs (ext, comp, raw) = %s" % (nsrc, nrows, outs)
        check_points(what, ref, ext, comp, out_raw)


# ---------------------------------------------------------------- (c) canonicalize
EDGES = [1, L - 1] + [v for k in (31, 32, 63, 64, 223, 224, 252) for v in ((1 << k) - 1, 1 << k)]
GRID = NUM_SMS * 8 * 256  # launch_canonicalize's grid in threads


def canonicalize(vals_mont, preset):
    n = vals_mont.shape[0]
    out = np.zeros((n, 4), dtype=np.uint64)
    mb = np.zeros(1, dtype=np.uint32)
    kh.call("kh_canonicalize", ptr(vals_mont), n, preset, ptr(out), ptr(mb))
    return out, int(mb[0])


@pytest.mark.parametrize("n", [1, 255, 256, 257, GRID, GRID + 1, 1 << 20])
def test_canonicalize(n):
    rng = random.Random(n)
    nrng = np.random.default_rng(n)
    for wide in [0] + EDGES:
        below = [0] if wide <= 1 else [0, 1] + [rng.randrange(1 << rng.randrange(wide.bit_length() - 1)) for _ in range(62)]
        below = [v for v in below if v.bit_length() < wide.bit_length()] or [0]
        pool_m, pool_c = mont(below + [wide]), raw(below + [wide])
        idx = nrng.integers(0, len(below), size=n)
        for pos in ((0, n - 1) if n > 1 else (0,)):
            i = idx.copy()
            i[pos] = len(below)
            for preset in ((0, 7) if wide == 0 else (0, wide.bit_length() + 1)):
                out, mb = canonicalize(np.ascontiguousarray(pool_m[i]), preset)
                what = "canonicalize n=%d widest %#x at [%d], preset %d" % (n, wide, pos, preset)
                bad = np.nonzero((out != pool_c[i]).any(axis=1))[0]
                assert not len(bad), "%s: %d elements differ, first at [%d]" % (what, len(bad), bad[0])
                assert mb == max(preset, wide.bit_length()), "%s: max_bits %d" % (what, mb)


def test_canonicalize_sizes_variable_base_windows(tables, gens):
    """lasso_msm's chain: canonicalize, nw = msm_windows_for_bits(max_bits), the variable-base MSM over nw windows"""
    rng = random.Random(3)
    for bits in [b for k in range(1, 32) for b in range(8 * k - 3, 8 * k + 1)] + list(range(249, 254)):
        top = (1 << bits) - 1 if bits < 253 else L - 1
        row = [top, 1 << (bits - 1)] + [rng.randrange(top + 1) for _ in range(14)]
        canon, mb = canonicalize(mont(row), 0)
        assert mb == bits, "canonicalize: max_bits %d for %d-bit values" % (mb, bits)
        nw = windows_for_bits(mb)
        ext, comp, out_raw = outputs(1)
        kh.call("kh_msm_rows", tables.h, 0, ptr(np.ascontiguousarray(canon.view(np.uint32).reshape(-1))), 8, 16, 1, 16, nw,
                1, 0, ptr(ext), ptr(comp), ptr(out_raw))
        check_points("msm_rows shifted=0 nw=%d over canonicalize's %d-bit output" % (nw, bits), oracle_rows(gens, [row]),
                     ext, comp, out_raw)


# ---------------------------------------------------------------- (d) sharded commitments
def u32_matrix(rng, nrows, ncols):
    edges = [0, 1, 0x7fff, 0x8000, 0x8001, 0xffff, 0x10000, 2**24 - 1, 2**32 - 1]
    return [[rng.choice(edges) if rng.randrange(4) == 0 else rng.randrange(1 << rng.choice((8, 16, 24, 32)))
             for _ in range(ncols)] for _ in range(nrows)]


def rank_launch(tables, path, rows, G, g, nw):
    """rank g's launch over its columns rows[:, g::G]: (raw (nrows, 32) u32, compressed (nrows, 32))"""
    loc = [r[g::G] for r in rows]
    nrows, ncols = len(loc), len(loc[0])
    comp, out_raw = np.zeros((nrows, 32), dtype=np.uint8), np.zeros((nrows, 32), dtype=np.uint32)
    if path in ("bucket_u32", "bucket_full"):
        limbs = 1 if path == "bucket_u32" else 8
        kh.call("kh_msm_rows", tables.h, 1, ptr(device_scalars(loc, limbs)), limbs, ncols, nrows, ncols, nw, G, g, None,
                ptr(comp), ptr(out_raw))
    elif path == "direct_fr":
        kh.call("kh_msm_rows_direct_raw", tables.h, 1, ptr(mont([v for r in loc for v in r])), nrows, ncols, nw, G, g, 0,
                ptr(out_raw), ptr(comp))
    else:
        kh.call("kh_msm_rows_direct_raw", tables.h, 0, ptr(device_scalars(loc, 1)), nrows, ncols, nw, G, g,
                int(path == "direct_u32_m16"), ptr(out_raw), ptr(comp))
    return out_raw, comp


SHARD_CASES = ([(G, p, nrows, 1024) for G in (2, 4, 8) for p in ("bucket_u32", "bucket_full", "direct_u32", "direct_fr")
                for nrows in (3, 33)] + [(G, "direct_u32_m16", 9, 64) for G in (2, 8)])


@pytest.mark.parametrize("G,path,nrows,ncols", SHARD_CASES)
def test_sharded_commitment(tables, gens, G, path, nrows, ncols):
    rng = random.Random(repr((G, path, nrows)))
    if path in ("bucket_u32", "direct_u32", "direct_u32_m16"):
        rows = u32_matrix(rng, nrows, ncols)
    else:
        rows = [[(0, 1, L - 1)[rng.randrange(3)] if rng.randrange(8) == 0 else rng.randrange(L) for _ in range(ncols)]
                for _ in range(nrows)]
    nw = 32 if path == "bucket_full" else windows_for_bits(max(v.bit_length() for r in rows for v in r))
    raws = []
    for g in range(G):
        t = kh.Tables(gens[: ncols + 2], ncols16=ncols // G, col_mul=G, col_add=g) if path == "direct_u32_m16" else tables
        try:
            out_raw, comp = rank_launch(t, path, rows, G, g, nw)
        finally:
            if t is not tables:
                t.close()
        what = "%s rank %d of %d, %dx%d local columns, col_map %d*c+%d, nw=%d" % (path, g, G, nrows, ncols // G, G, g, nw)
        check_points(what, oracle_rows(gens, [r[g::G] for r in rows], (G, g)), comp=comp, out_raw=out_raw)
        raws.append(out_raw)
    stacked = np.ascontiguousarray(np.stack(raws).reshape(-1))
    comp = np.zeros((nrows, 32), dtype=np.uint8)
    kh.call("kh_sum_raw_points", ptr(stacked), G, nrows, None, ptr(comp), None)
    check_points("%s: gather-then-add over %d ranks, %dx%d, nw=%d" % (path, G, nrows, ncols, nw), oracle_rows(gens, rows),
                 comp=comp)
