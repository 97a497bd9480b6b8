"""launch_densify (densify_kernels.cu) one launch at a time (tests/kernel_harness: harness_setup.cu), against the CPU
oracle's sequential timestamp scan (orc_densify) or, where its 2^log_m-entry tables would be too large, the same
definition in numpy: a stable argsort by address, read = sorted position - first position of the address, final = the
number of accesses of each address.

The shapes reach what the whole-proof tests do not: one to four radix passes (log_m 1 .. 28, each digit boundary crossed
in both directions), partial radix tiles (s not a multiple of 2048), padding with address 0 (n < s), both exclusive
scans with one tile, 2 .. 1024 tiles and more than 1024 tiles (the carried loop of dz_scan_sums_kernel: s = 2^26 for the
histogram scan, log_m >= 23 for the count scan), C = 1, 3 and 16 dimensions of different distributions, this rank's
shards for G = 1, 2, 4, 8 at every rank, u32 / u64 entries in row-major, column-major and padded layouts, and the range
check.  Every word of every output is compared; the output buffers are longer than the shards and their gaps hold a
poison word that must survive the launch."""
import numpy as np
import pytest

import kernel_harness_lib as kh
from oracle_lib import P, lib as orc, sz

POISON = 0xDEADBEEF  # above any address (< 2^28), read or count (<= s <= 2^26) a test writes
KINDS = ["uniform", "one", "top", "alternating", "ascending", "descending", "low_byte", "top_digit", "run"]


# ---------------------------------------------------------------- inputs
def addresses(kind, n, log_m, rng):
    """n addresses below 2^log_m of one distribution"""
    m = 1 << log_m
    uni = rng.integers(0, m, size=n, dtype=np.uint64)
    if kind == "uniform":
        return uni
    if kind == "one":  # every access to one address: its count is s (with the padding, when that address is 0)
        return np.full(n, rng.integers(0, m), dtype=np.uint64)
    if kind == "top":
        return np.full(n, m - 1, dtype=np.uint64)
    if kind == "alternating":
        a, b = rng.choice(m, size=2, replace=False)
        return np.where(np.arange(n) % 2 == 0, a, b).astype(np.uint64)
    if kind == "ascending":
        return np.sort(uni)
    if kind == "descending":
        return np.sort(uni)[::-1].copy()
    if kind == "low_byte":  # every key has the same digit in the first pass
        return (uni & np.uint64(~0xff & (m - 1))) | np.uint64(int(rng.integers(0, 256)) & (m - 1))
    if kind == "top_digit":  # the addresses differ only in the top digit
        lo_bits = 8 * ((log_m - 1) // 8)
        low = np.uint64(int(rng.integers(0, 1 << lo_bits)) if lo_bits else 0)
        return (uni >> np.uint64(lo_bits) << np.uint64(lo_bits)) | low
    assert kind == "run"  # a long run of one address inside uniform data
    uni[n // 4:n // 4 + n // 2] = rng.integers(0, m)
    return uni


def matrix(n, C, log_m, seed, shift=0):
    """(n, C) u64 addresses; dimension i of distribution KINDS[(i + shift) % 9]"""
    rng = np.random.default_rng(seed)
    return np.stack([addresses(KINDS[(i + shift) % len(KINDS)], n, log_m, rng) for i in range(C)], axis=1)


# ---------------------------------------------------------------- references
def reference(mat, s, log_m):
    """per dimension (dim, read, (addresses, counts)) of the matrix padded to s rows with address 0; the nonzero
    entries of final as (addresses, counts)"""
    n, C = mat.shape
    padded = np.zeros((s, C), dtype=np.uint64)
    padded[:n] = mat
    if s & (s - 1) == 0 and log_m <= 24 and s * C <= 1 << 26:
        m = 1 << log_m
        dim, read = np.zeros((C, s), dtype=np.uint64), np.zeros((C, s), dtype=np.uint64)
        fin = np.zeros((C, m), dtype=np.uint64)
        orc().orc_densify(P(padded), sz(s), sz(C), sz(log_m), P(dim), P(read), P(fin))
        out = []
        for i in range(C):
            nz = np.flatnonzero(fin[i])
            out.append((dim[i], read[i], (nz.astype(np.uint64), fin[i][nz])))
        return out
    return [numpy_reference(padded[:, i]) for i in range(C)]


def numpy_reference(a):
    order = np.argsort(a, kind="stable")
    srt = a[order]
    read = np.empty(a.shape[0], dtype=np.uint64)
    read[order] = np.arange(a.shape[0], dtype=np.uint64) - np.searchsorted(srt, srt, side="left").astype(np.uint64)
    addr, cnt = np.unique(a, return_counts=True)
    return a, read, (addr, cnt.astype(np.uint64))


# ---------------------------------------------------------------- one launch
FORMS = [(eb, lay) for eb in (4, 8) for lay in ("row", "col", "padded")]


def index_buffer(mat, elem_bytes, layout):
    """(buffer, row_stride, col_stride) holding the (n, C) matrix; entries as unsigned integers of elem_bytes (-1 as
    all ones).  The padding columns of the padded layout hold m-sized garbage: read, it would change an output."""
    n, C = mat.shape
    dt = np.uint32 if elem_bytes == 4 else np.uint64
    v = mat.astype(np.uint64).astype(dt)
    if layout == "row":
        return np.ascontiguousarray(v.reshape(-1)), C, 1
    if layout == "col":
        return np.ascontiguousarray(v.T.reshape(-1)), 1, n
    buf = np.full((n, C + 3), np.iinfo(dt).max, dtype=dt)
    buf[:, :C] = v
    return np.ascontiguousarray(buf.reshape(-1)), C + 3, 1


def shard_len(total, G, g):
    return len(range(g, total, G))


def launch(mat, s, log_m, G=1, g=0, form=(8, "row"), check=1):
    """kh_densify: (dims, reads, finals, flag), each a list of this rank's C shards; the poison gaps are checked"""
    n, C = mat.shape
    buf, rs, cs = index_buffer(mat, *form)
    ls, lm = shard_len(s, G, g), shard_len(1 << log_m, G, g)
    strides = (ls + 3 + g, ls + 5, lm + 7)
    outs = [np.full(C * st, POISON, dtype=np.uint32) for st in strides]
    flag = np.zeros(1, dtype=np.uint32)
    kh.call("kh_densify", buf.ctypes.data, form[0], rs, cs, n, s, C, log_m, G, g, check, outs[0].ctypes.data, strides[0],
            outs[1].ctypes.data, strides[1], outs[2].ctypes.data, strides[2], flag.ctypes.data)
    shards = []
    for name, o, st, ln in zip(("dim", "read", "final"), outs, strides, (ls, ls, lm)):
        o = o.reshape(C, st)
        bad = np.nonzero((o[:, ln:] != POISON).any(axis=1))[0]
        assert not len(bad), "%s: a write outside the shard of dimension %d (rank %d of %d)" % (name, bad[0], g, G)
        shards.append([o[i, :ln] for i in range(C)])
    return shards[0], shards[1], shards[2], int(flag[0])


def compare(what, got, ref, G=1, g=0):
    dims, reads, fins = got[:3]
    for i, (dim, read, (addr, cnt)) in enumerate(ref):
        for name, a, b in (("dim", dims[i], dim[g::G]), ("read", reads[i], read[g::G])):
            assert a.shape == b.shape, "%s: %s of dimension %d: shard length %d, want %d" % (what, name, i, a.shape[0],
                                                                                           b.shape[0])
            bad = np.flatnonzero(a != b)
            assert not len(bad), "%s: %s of dimension %d: %d words differ, first at %d (%d, want %d)" % (
                what, name, i, len(bad), bad[0], a[bad[0]], b[bad[0]])
        assert int(cnt.sum()) == read.shape[0]
        sel = addr % np.uint64(G) == np.uint64(g)
        nz = np.flatnonzero(fins[i])
        assert np.array_equal(nz.astype(np.uint64) * np.uint64(G) + np.uint64(g), addr[sel]), \
            "%s: final of dimension %d: the nonzero addresses differ" % (what, i)
        assert np.array_equal(fins[i][nz], cnt[sel]), "%s: final of dimension %d: the counts differ" % (what, i)


def run(s, n, C, log_m, seed, shift=0, G=1, form=(8, "row"), check=1):
    mat = matrix(n, C, log_m, seed, shift)
    ref = reference(mat, s, log_m)
    for g in range(G):
        what = "densify s=%d n=%d C=%d log_m=%d G=%d g=%d form=%s kinds %s" % (
            s, n, C, log_m, G, g, form, [KINDS[(i + shift) % len(KINDS)] for i in range(C)])
        got = launch(mat, s, log_m, G, g, form, check)
        assert got[3] == 0, what + ": the range flag is raised for a valid matrix"
        compare(what, got, ref, G, g)


# ---------------------------------------------------------------- the numpy reference itself
@pytest.mark.parametrize("log_m", [1, 5, 12])
def test_numpy_reference_matches_oracle(log_m):
    """the reference of the shapes orc_densify cannot take is the oracle's scan wherever both apply"""
    for shift in range(len(KINDS)):
        mat = matrix(700, 2, log_m, 100 + shift, shift)
        want = reference(mat, 1024, log_m)
        padded = np.zeros((1024, 2), dtype=np.uint64)
        padded[:700] = mat
        for i in range(2):
            got = numpy_reference(padded[:, i])
            assert np.array_equal(got[0], want[i][0]) and np.array_equal(got[1], want[i][1])
            assert np.array_equal(got[2][0], want[i][2][0]) and np.array_equal(got[2][1], want[i][2][1])


# ---------------------------------------------------------------- GPU
LOG_MS = [1, 7, 8, 9, 15, 16, 17, 23, 24, 25, 28]


@pytest.mark.gpu
@pytest.mark.parametrize("log_m", LOG_MS)
def test_radix_passes(log_m):
    """one to four passes; the count scan with one tile (log_m <= 12), 2 .. 1024 tiles and > 1024 tiles (>= 23)"""
    C = 3 if log_m <= 24 else 1
    for shift in range(0, len(KINDS), 3):
        run(4096, 2049, C, log_m, log_m * 100 + shift, shift, check=shift % 2)
    run(6000, 6000, 1, log_m, log_m, 8)


S_CASES = sorted({(s, n) for s in (1, 2, 2048, 4096, 2**15, 2**16, 2047, 2049, 6000) for n in (1, s // 2 + 1, s)})


@pytest.mark.gpu
@pytest.mark.parametrize("s,n", S_CASES)
def test_lengths(s, n):
    """partial radix tiles, padding with address 0, one radix tile and several; the histogram scan's 1 and 2 tiles"""
    for log_m in (9, 16):
        run(s, n, 3, log_m, s * 7 + n + log_m, s + n, check=n % 2)


@pytest.mark.gpu
@pytest.mark.parametrize("n,log_m,shift", [(2**26, 17, 0), (2**25 + 1, 9, 8)])
def test_histogram_scan_over_1024_tiles(n, log_m, shift):
    """s = 2^26: 32768 radix tiles, a histogram scan of 2048 tiles, carried across two blocks of 1024"""
    run(2**26, n, 1, log_m, n, shift)


@pytest.mark.gpu
@pytest.mark.parametrize("s,log_m", [(6000, 17), (2**16, 9)])
def test_sixteen_dimensions(s, log_m):
    """every distribution in one launch, each in more than one dimension (blockIdx.y): a mix-up shows"""
    run(s, s - 17, 16, log_m, s + log_m, 0)
    run(s, s, 16, log_m, s + log_m + 1, 4)


SHARD_CASES = [(2049, 2049, 3, 9), (2**16, 2**15 + 1, 3, 17), (4096, 4096, 2, 1), (6000, 4000, 2, 23)]


@pytest.mark.gpu
@pytest.mark.parametrize("G", [2, 4, 8])
@pytest.mark.parametrize("s,n,C,log_m", SHARD_CASES)
def test_shards(G, s, n, C, log_m):
    """rank g of G stores accesses k = i G + g at i and addresses a = i G + g at i, every g"""
    run(s, n, C, log_m, s + G, G, G=G)


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS, ids=["u%d-%s" % (8 * f[0], f[1]) for f in FORMS])
def test_index_forms(form):
    for check in (0, 1):
        run(6000, 4001, 3, 16, 11, 2, G=2, form=form, check=check)
        run(2049, 2049, 16, 9, 12, 5, form=form, check=check)


def bad_values(elem_bytes, m):
    vals = [("m", m), ("2^32-1", 2**32 - 1), ("-1", -1)]
    return vals + [("2^32+5", 2**32 + 5)] if elem_bytes == 8 else vals


@pytest.mark.gpu
@pytest.mark.parametrize("form", FORMS, ids=["u%d-%s" % (8 * f[0], f[1]) for f in FORMS])
def test_range_check(form):
    """an entry >= m raises the flag and is used as address 0: every other output is that of the matrix with the
    entry replaced by 0"""
    n, C, log_m, s = 3000, 3, 8, 4096
    mat = matrix(n, C, log_m, 13, 3).astype(np.int64)
    for label, value in bad_values(form[0], 1 << log_m):
        for place, (row, col) in (("first", (0, 0)), ("middle", (n // 2, 1)), ("last", (n - 1, C - 1))):
            bad = mat.copy()
            bad[row, col] = value
            clean = mat.copy().astype(np.uint64)
            clean[row, col] = 0
            ref = reference(clean, s, log_m)
            for G, g in ((1, 0), (2, 1)):
                what = "densify range check: %s at the %s entry, form %s, rank %d of %d" % (label, place, form, g, G)
                got = launch(bad.view(np.uint64), s, log_m, G, g, form, 1)
                assert got[3] == 1, what + ": the flag is not raised"
                compare(what, got, ref, G, g)
