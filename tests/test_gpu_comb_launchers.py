"""The launchers of the caller-polynomial paths (kernels.cuh), one launch at a time, against plain Python integers mod l:
the combining-function interpreter (a sumcheck round, the fused bind + round, the bind, the final evaluations, the
pointwise map), layer 0 of a caller's grand product, the ingest of a caller's dense polynomial and eq tables of 2^23 to
2^28 entries.  The launches go through tests/kernel_harness (harness_comb.cu: the library's own kernel objects, its
own program checker and slot allocator).  Every comparison is bit-exact on Montgomery limbs, and a failure names the
launch, the shape and the first element that differs.

The reference interprets the SSA program as the caller wrote it, so it depends on neither the slot allocation nor any
other interpreter.  Large launches use periodic inputs, array k being B_k[j mod p] for a prime p: the pair at i then
depends only on i mod p, a round's sums are sum_a count(a) f(a), and a bound array is ref[arange(n) % p]."""
import ctypes as C
import os

import numpy as np
import pytest

import kernel_harness_lib as kh
from test_gpu_launchers import L, RINV, mont, ptr, raw, raw_ints, rvals

PERIOD = 251
ADD, SUB, MUL, MULK, ADDK = range(5)
NUM_SMS, CUSTOM_THREADS = 132, 128
I32, U64 = np.int32, np.uint64


# ---------------------------------------------------------------- the reference
class Prog:
    """a combining function in lasso_comb_create's format: ins = [(op, a, b)], operands < n_inputs are inputs, n_inputs + j
    the result of instruction j; b indexes consts for MULK and ADDK"""

    def __init__(self, name, n_inputs, ins, consts, degree, n_slots):
        self.name, self.n_inputs, self.ins, self.consts, self.degree = name, n_inputs, ins, consts, degree
        self.n_slots = n_slots  # what the library's allocator must give (test_program_allocation)
        self.n_ops, self.n_consts = len(ins), len(consts)
        self.h_ins = np.ascontiguousarray(np.array(ins, dtype=I32).reshape(-1, 3))
        self.h_consts = mont(consts) if consts else np.zeros((1, 4), dtype=U64)

    def run(self, xs):
        vals = list(xs)
        for op, a, b in self.ins:
            x = vals[a]
            if op == MULK:
                v = x * self.consts[b]
            elif op == ADDK:
                v = x + self.consts[b]
            else:
                y = vals[b]
                v = x + y if op == ADD else (x - y if op == SUB else x * y)
            vals.append(v % L)
        return vals[-1]

    def traced_degree(self):
        deg = [1] * self.n_inputs
        for op, a, b in self.ins:
            deg.append(deg[a] + deg[b] if op == MUL else (deg[a] if op in (MULK, ADDK) else max(deg[a], deg[b])))
        return deg[-1]

    def args(self):
        return (self.n_inputs, ptr(self.h_ins), self.n_ops, ptr(self.h_consts), self.n_consts, self.degree)


def round_sums(g, classes):
    """sum over the pair classes (count, lo, hi) of count * g(lo + t (hi - lo)), t = 0..degree"""
    out = [0] * (g.degree + 1)
    for cnt, lo, hi in classes:
        if cnt:
            d = [h - x for x, h in zip(lo, hi)]
            for t in range(g.degree + 1):
                out[t] += cnt * g.run([(x + t * dd) % L for x, dd in zip(lo, d)])
    return [x % L for x in out]


def pair_classes(B, half):
    """the pairs (i, half + i), i < half, of the arrays B_k[j mod p] by i mod p: (count, lo, hi)"""
    p = len(B[0])
    return [(len(range(a, half, p)), [b[a] for b in B], [b[(half + a) % p] for b in B]) for a in range(min(p, half))]


def bind_periodic(B, half, r):
    """element a of Z[i] + r (Z[half + i] - Z[i]) for Z = B[j mod p], a < p (the bound array is that at i mod p)"""
    p = len(B)
    return [(B[a] + r * (B[(half + a) % p] - B[a])) % L for a in range(p)]


def eq_ref(r, idx):
    """eq(r, i) = prod_j (bit_{ell-1-j}(i) ? r_j : 1 - r_j), r_0 <-> the MSB; the product is split at bit 8 so that each
    of its two factors is computed once per distinct high or low part"""
    ell = len(r)
    lo_bits = min(8, ell)

    def part(v, js):
        acc = 1
        for pos, j in enumerate(js):
            bit = (v >> (len(js) - 1 - pos)) & 1
            acc = acc * (r[j] if bit else 1 - r[j]) % L
        return acc

    hi_js, lo_js = list(range(ell - lo_bits)), list(range(ell - lo_bits, ell))
    hi_c, lo_c = {}, {}
    out = []
    for i in idx:
        h, l_ = i >> lo_bits, i & ((1 << lo_bits) - 1)
        if h not in hi_c:
            hi_c[h] = part(h, hi_js)
        if l_ not in lo_c:
            lo_c[l_] = part(l_, lo_js)
        out.append(hi_c[h] * lo_c[l_] % L)
    return out


def fail_at(what, got, want_vals, bad, montgomery=True):
    i = int(bad[0])
    g = raw_ints(got[i:i + 1])[0]
    raise AssertionError("%s: %d of %d elements differ, first at [%d]: got limbs %#x (value %d), want value %d"
                         % (what, len(bad), got.shape[0], i, g, g * RINV % L if montgomery else g, want_vals(i)))


def check_periodic(what, got, vals):
    """got (n, 4) must be the Montgomery limbs of vals[i mod len(vals)] (vals as long as got: plain elementwise)"""
    got = np.ascontiguousarray(got, dtype=U64).reshape(-1, 4)
    want = mont(vals)[np.arange(got.shape[0]) % len(vals)]
    bad = np.nonzero((got != want).any(axis=1))[0]
    if len(bad):
        fail_at(what, got, lambda i: vals[i % len(vals)], bad)


def check_same(what, got, want):
    """got must equal the limbs want, unchanged (no field interpretation: sentinels may be non-canonical)"""
    got = np.ascontiguousarray(got, dtype=U64).reshape(-1, 4)
    want = np.ascontiguousarray(want, dtype=U64).reshape(-1, 4)
    bad = np.nonzero((got != want).any(axis=1))[0]
    if len(bad):
        fail_at(what + " (must be unchanged)", got, lambda i: raw_ints(want[i:i + 1])[0], bad, montgomery=False)


def tiled(B, n):
    """(k, n, 4) Montgomery limbs of the arrays B_k[j mod p]"""
    idx = np.arange(n) % len(B[0])
    return np.ascontiguousarray(np.stack([mont(b)[idx] for b in B]))


def sentinel(k, n):
    """limbs no launch writes: 2^256 - 1 - i (not canonical, so a store of any residue changes them)"""
    s = np.full((k, n, 4), np.iinfo(np.uint64).max, dtype=U64)
    s[:, :, 0] -= np.arange(n, dtype=U64)
    return s


# ---------------------------------------------------------------- programs
def _limit_program():
    """128 instructions, 64 constants, 16 values live at once, 16 inputs, degree 16, every opcode"""
    rng = np.random.default_rng(7)
    # 0, 1 and l - 1 where they cannot cancel g: x_0 + 0, w_1 * 1, w_2 * (l - 1), w_3 + (l - 1)
    consts = rvals(rng, 64, edges=False)
    consts[0], consts[17], consts[50], consts[35] = 0, 1, L - 1, L - 1
    ins, slot = [], list(range(16))  # slot[j]: the SSA value currently standing for w_j

    def emit(op, a, b):
        ins.append((op, a, b))
        return 16 + len(ins) - 1

    for j in range(16):  # 16 live values
        slot[j] = emit(ADDK, j, j)
    for base, op in ((16, MULK), (32, ADDK), (48, MULK)):  # each rewrites w_j from its own last use
        for j in range(16):
            slot[j] = emit(op, slot[j], base + j)
    for j in range(15):  # linear mixing with the next value, which stays live
        slot[j] = emit(ADD if j % 2 == 0 else SUB, slot[j], slot[j + 1])
    p = emit(MUL, slot[0], slot[1])
    for j in range(2, 16):
        p = emit(MUL, p, slot[j])
    for j in range(17):  # p <- p - c p, degree stays 16
        p = emit(SUB, p, emit(MULK, p, j))
    assert len(ins) == 128
    return Prog("limit", 16, ins, consts, 16, 16)


LIMIT = _limit_program()
MINIMAL = Prog("minimal", 1, [(MULK, 0, 0)], [5], 1, 0)
PROGRAMS = [
    LIMIT,
    MINIMAL,
    # x0 x1 declared as degree 5: six evaluation points of a quadratic
    Prog("declared_above", 2, [(MUL, 0, 1)], [], 5, 0),
    # (x0 + x1) * (x1 - x2) * 7 + 3 - x0 x0
    Prog("every_opcode", 3, [(ADD, 0, 1), (SUB, 1, 2), (MUL, 3, 4), (MULK, 5, 0), (ADDK, 6, 1), (MUL, 0, 0), (SUB, 7, 8)],
         [7, 3], 3, 2),
    # x0 x0 (a = b on an input), then (x0 x0)^2 (a = b on a slot)
    Prog("square", 1, [(MUL, 0, 0), (MUL, 1, 1)], [], 4, 1),
    # t = x0 + x1; t <- t * c (same slot); t <- t + x1 (same slot); t * t
    Prog("slot_reuse", 2, [(ADD, 0, 1), (MULK, 2, 0), (ADD, 3, 1), (MUL, 4, 4)], [L - 2], 2, 1),
    # two dead values between live ones
    Prog("dead_values", 2, [(MUL, 0, 1), (ADDK, 0, 0), (SUB, 1, 0), (MULK, 2, 0), (ADD, 5, 1)], [11], 2, 2),
    # g = x0 + 0: the program returns an input
    Prog("returns_input", 1, [(ADDK, 0, 0)], [0], 1, 0),
]
BY_NAME = {g.name: g for g in PROGRAMS}


def allocated(g):
    ins = np.zeros((g.n_ops, 4), dtype=I32)
    n_slots = C.c_int(-1)
    kh.call("kh_comb_program", *g.args(), ptr(ins), C.byref(n_slots))
    return ins, n_slots.value


def wave(g, npts):
    """threads of one full grid of the interpreter kernels at npts accumulators (custom_grid, poly_kernels.cu)"""
    smem = 16 * g.n_ops + 32 * g.n_consts + (g.n_slots + npts) * 32 * CUSTOM_THREADS
    per_sm = max(1, min(8, (200 << 10) // (smem + 1024)))
    return NUM_SMS * per_sm * CUSTOM_THREADS


def sizes(g, npts, big=True):
    """1 and 2, one CTA and one more, a full wave and one either side, a non-power of two past it, and 2^20 (grid-stride
    trips); `big`: the limit and minimal programs, the others stop at one wave + 1"""
    w = wave(g, npts)
    if not big:
        return [1, 2, 129, 1000, w + 1]
    return [1, 2, 128, 129, w - 1, w, w + 1, 3 * w + 77, 1 << 20]


def period(g, n_pairs):
    """fully random inputs while the direct reference stays cheap, else period PERIOD"""
    return PERIOD if n_pairs * (g.degree + 1) * g.n_ops > 500_000 else None


def inputs(g, rng, length, share=False):
    """the k arrays B (values, period p or the whole length), the map of shared sources, and the per-input arrays"""
    p = period(g, length // 2) or length
    B = [rvals(rng, p) for _ in range(g.n_inputs)]
    src_of = list(range(g.n_inputs))
    if share:  # input 1 reads input 0's array; the last input reads the array of the one before it
        src_of[1] = 0
        src_of[-1] = src_of[-2]
    return B, src_of, [B[s] for s in src_of]


def publish_out(n):
    return np.zeros((n, 4), dtype=U64)


# ---------------------------------------------------------------- the reference alone
def test_reference_periodic_round_equals_direct():
    """round_sums over the classes of periodic arrays equals the sum over every pair"""
    rng = np.random.default_rng(5)
    g = BY_NAME["every_opcode"]
    B = [rvals(rng, 7) for _ in range(3)]
    for half in (1, 6, 7, 8, 23):
        A = [[b[j % 7] for j in range(2 * half)] for b in B]
        direct = round_sums(g, [(1, [a[i] for a in A], [a[half + i] for a in A]) for i in range(half)])
        assert round_sums(g, pair_classes(B, half)) == direct, half
        assert bind_periodic(B[0], half, 9)[:1] == [(A[0][0] + 9 * (A[0][half] - A[0][0])) % L]


def test_reference_eq_is_the_product():
    rng = np.random.default_rng(6)
    r = rvals(rng, 10)
    for i in (0, 1, 255, 256, 1023, 777):
        want = 1
        for j in range(10):
            want = want * (r[j] if (i >> (9 - j)) & 1 else 1 - r[j]) % L
        assert eq_ref(r, [i]) == [want]


@pytest.mark.parametrize("name", [g.name for g in PROGRAMS])
def test_reference_program_is_not_degenerate(name):
    """along a random line every program has its traced degree exactly (its last finite difference is not zero), so
    no test program is constant or cancels to zero"""
    g = BY_NAME[name]
    rng = np.random.default_rng(8)
    a, d = rvals(rng, g.n_inputs, edges=False), rvals(rng, g.n_inputs, edges=False)
    ys = [g.run([(x + t * dx) % L for x, dx in zip(a, d)]) for t in range(g.traced_degree() + 1)]
    for _ in range(g.traced_degree()):
        ys = [(y1 - y0) % L for y0, y1 in zip(ys, ys[1:])]
    assert ys[0] != 0


def test_reference_program_degrees():
    assert LIMIT.traced_degree() == 16 and LIMIT.n_consts == 64 and LIMIT.n_ops == 128
    assert {op for op, _, _ in LIMIT.ins} == {ADD, SUB, MUL, MULK, ADDK}
    assert BY_NAME["declared_above"].traced_degree() == 2
    assert BY_NAME["returns_input"].run([12345]) == 12345


# ---------------------------------------------------------------- slot allocation
@pytest.mark.gpu
@pytest.mark.parametrize("name", [g.name for g in PROGRAMS])
def test_program_allocation(name):
    """the library's checker accepts every program and its allocator gives the slot count the sizes above assume: 16 for
    the limit program; the last instruction stores nothing; slot_reuse's results take their operand's slot"""
    g = BY_NAME[name]
    ins, n_slots = allocated(g)
    assert n_slots == g.n_slots, "%s: %d slots, want %d" % (name, n_slots, g.n_slots)
    assert ins[-1][1] == -1
    if name == "slot_reuse":
        assert ins[1][1] == ins[1][2] == ins[2][1] == ins[2][2]


# ---------------------------------------------------------------- one round
EVAL_CASES = [(g.name, n) for g in PROGRAMS for n in sizes(g, g.degree + 1, g in (LIMIT, MINIMAL))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,half", EVAL_CASES)
def test_comb_eval(name, half):
    """launch_sumcheck_eval_comb: the degree + 1 published sums (twice on one Finalize), inputs unchanged"""
    g = BY_NAME[name]
    rng = np.random.default_rng(half + 31 * g.n_ops)
    share = g.n_inputs > 1 and half % 2 == 1
    B, src_of, Bin = inputs(g, rng, 2 * half, share)
    arr = tiled(B, 2 * half)
    before = arr.copy()
    out = publish_out(g.degree + 1)
    kh.call("kh_comb_eval", *g.args(), ptr(np.array(src_of, dtype=I32)), ptr(arr), half, 1, ptr(out))
    what = "eval_comb %s half=%d%s" % (name, half, " shared" if share else "")
    check_periodic(what + " published sums", out, round_sums(g, pair_classes(Bin, half)))
    for k in range(g.n_inputs):
        if src_of[k] == k:
            check_same(what + " input %d" % k, arr[k], before[k])


# ---------------------------------------------------------------- fused bind + round
def fused_cases():
    out = []
    for g in PROGRAMS:
        big = g in (LIMIT, MINIMAL)
        for q in sizes(g, g.degree + 1, big):
            if q == 1 << 20 and g is LIMIT:
                out += [(g.name, q, 1, 0)]  # 2 GiB of inputs: in place only; out of place at 2^18 below
                continue
            out += [(g.name, q, 1, 0), (g.name, q, 0, 0)] + ([(g.name, q, 0, 1)] if g.n_inputs > 1 else [])
    return out + [(LIMIT.name, 1 << 18, 0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,q,in_place,share", fused_cases())
def test_comb_bind_eval(name, q, in_place, share):
    """launch_sumcheck_bind_eval_comb with min_q = 1: arrays of 4q bound with r to 2q, then the round over the bound
    values.  In place: the bound halves and the untouched upper halves.  Out of place: src unchanged, dst bound below 2q
    and unwritten from 2q up.  Small rounds run r = 0, 1, l - 1 too."""
    g = BY_NAME[name]
    rng = np.random.default_rng(q + 17 * g.n_ops + 2 * in_place + share)
    rs = [rvals(rng, 1, edges=False)[0]] + ([0, 1, L - 1] if q <= 129 else [])
    B, src_of, Bin = inputs(g, rng, 4 * q, bool(share))
    for r in rs:
        what = "bind_eval_comb %s q=%d %s%s r=%s" % (name, q, "in place" if in_place else "out of place",
                                                   " shared" if share else "", "random" if r == rs[0] else r)
        src = tiled(B, 4 * q)
        before = src.copy()
        dst = None if in_place else sentinel(g.n_inputs, 4 * q)
        dst_before = None if in_place else dst.copy()
        out = publish_out(g.degree + 1)
        launched = C.c_int(-1)
        kh.call("kh_comb_bind_eval", *g.args(), ptr(np.array(src_of, dtype=I32)), ptr(src), q, ptr(mont([r])[0]), 1,
                in_place, 1, None if in_place else ptr(dst), ptr(out), C.byref(launched))
        assert launched.value == 1, what + ": not launched with min_q = 1"
        D = [bind_periodic(b, 2 * q, r) for b in Bin]
        check_periodic(what + " published sums", out, round_sums(g, pair_classes(D, q)))
        bound = src if in_place else dst
        for k in range(g.n_inputs):
            check_periodic(what + " input %d bound" % k, bound[k][:2 * q], D[k])
            if in_place:
                check_same(what + " input %d upper half" % k, src[k][2 * q:], before[k][2 * q:])
            else:
                check_same(what + " input %d dst from 2q" % k, dst[k][2 * q:], dst_before[k][2 * q:])
                if src_of[k] == k:
                    check_same(what + " input %d src" % k, src[k], before[k])


@pytest.mark.gpu
@pytest.mark.parametrize("q,min_q", [(1, 2), (5, 5), (5, 6), (129, 130), (129, 2), ((1 << 15) - 1, 0), (1 << 15, 0)])
def test_comb_bind_eval_threshold(q, min_q):
    """launch_sumcheck_bind_eval_comb launches exactly when q >= min_q (0: the default threshold, 2^15 pairs).  Below
    it nothing is published and neither src nor dst is written; at or above it the round is the reference's."""
    if min_q == 0 and "LASSO_B200_FUSED_MIN_Q" in os.environ:
        pytest.skip("the default threshold is overridden in this environment")
    g = BY_NAME["every_opcode"]
    rng = np.random.default_rng(q + min_q)
    B, src_of, Bin = inputs(g, rng, 4 * q)
    r = rvals(rng, 1, edges=False)[0]
    src = tiled(B, 4 * q)
    before = src.copy()
    dst = sentinel(g.n_inputs, 4 * q)
    dst_before = dst.copy()
    out = publish_out(g.degree + 1)
    launched = C.c_int(-1)
    kh.call("kh_comb_bind_eval", *g.args(), ptr(np.array(src_of, dtype=I32)), ptr(src), q, ptr(mont([r])[0]), min_q,
            0, 1, ptr(dst), ptr(out), C.byref(launched))
    what = "bind_eval_comb q=%d min_q=%d" % (q, min_q)
    want = q >= (min_q or 1 << 15)
    assert launched.value == int(want), "%s: launched = %d, want %d" % (what, launched.value, want)
    check_same(what + " src", src, before)
    if not want:
        check_same(what + " dst", dst, dst_before)
        return
    D = [bind_periodic(b, 2 * q, r) for b in Bin]
    check_periodic(what + " published sums", out, round_sums(g, pair_classes(D, q)))
    for k in range(g.n_inputs):
        check_periodic(what + " input %d bound" % k, dst[k][:2 * q], D[k])
        check_same(what + " input %d dst from 2q" % k, dst[k][2 * q:], dst_before[k][2 * q:])


# ---------------------------------------------------------------- pointwise map
MAP_CASES = [(g.name, n) for g in PROGRAMS for n in sizes(g, 0, g in (LIMIT, MINIMAL))]


@pytest.mark.gpu
@pytest.mark.parametrize("name,n", MAP_CASES)
def test_comb_map(name, n):
    """launch_comb_map: out[i] = g(x_0[i], ..), nothing written past n, inputs unchanged"""
    g = BY_NAME[name]
    rng = np.random.default_rng(n + 13 * g.n_ops)
    p = PERIOD if n * g.n_ops > 500_000 else n
    B = [rvals(rng, p) for _ in range(g.n_inputs)]
    src_of = list(range(g.n_inputs))
    if g.n_inputs > 1 and n % 2:
        src_of[1] = 0
    Bin = [B[s] for s in src_of]
    arr = tiled(B, n)
    before = arr.copy()
    guard = 64
    out = sentinel(1, n + guard)[0]
    kh.call("kh_comb_map", *g.args(), ptr(np.array(src_of, dtype=I32)), ptr(arr), n, ptr(out), guard)
    what = "comb_map %s n=%d" % (name, n)
    check_periodic(what, out[:n], [g.run([b[a] for b in Bin]) for a in range(p)])
    check_same(what + " guard", out[n:], sentinel(1, n + guard)[0][n:])
    for k in range(g.n_inputs):
        if src_of[k] == k:
            check_same(what + " input %d" % k, arr[k], before[k])


# ---------------------------------------------------------------- bind, final evaluations
def edge_arrays(n, p):
    """n arrays of p < 4 values drawn from 0, 1 and l - 1, rotated between arrays (rvals places these edges only from 4
    values up)"""
    return [[(0, 1, L - 1)[(k + j) % 3] for j in range(p)] for k in range(n)]


R_KINDS = ["random", 0, 1, "l-1"]


def r_of(kind, rng):
    return {"random": None, 0: 0, 1: 1, "l-1": L - 1}[kind] if kind != "random" else rvals(rng, 1, edges=False)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("r_kind", R_KINDS)
@pytest.mark.parametrize("n,half,in_place", [(1, 1, 1), (1, 1, 0), (2, 3, 0), (3, 129, 1), (5, 1000, 0), (8, 4097, 1),
                                             (15, 1, 0), (16, 1, 1), (16, 33000, 0), (16, 1 << 17, 1), (4, 1 << 20, 0)])
def test_bind_comb(n, half, in_place, r_kind):
    """launch_bind_comb: every bound array; in place the upper halves unchanged, out of place src unchanged and dst
    unwritten from half up; out of place with n > 1 input 1 shares input 0's array"""
    rng = np.random.default_rng(n * 7 + half + in_place)
    r = r_of(r_kind, rng)
    p = PERIOD if half > 4096 else 2 * half
    B = [rvals(rng, p) for _ in range(n)] if p >= 4 else edge_arrays(n, p)
    src_of = list(range(n))
    if not in_place and n > 1:
        src_of[1] = 0
    src = tiled(B, 2 * half)
    before = src.copy()
    dst = None if in_place else sentinel(n, 2 * half)
    dst_before = None if in_place else dst.copy()
    kh.call("kh_bind_comb", n, ptr(np.array(src_of, dtype=I32)), ptr(src), half, ptr(mont([r])[0]), in_place,
            None if in_place else ptr(dst))
    what = "bind_comb n=%d half=%d %s r=%s" % (n, half, "in place" if in_place else "out of place", r_kind)
    bound = src if in_place else dst
    for k in range(n):
        check_periodic(what + " array %d" % k, bound[k][:half], bind_periodic(B[src_of[k]], half, r))
        if in_place:
            check_same(what + " array %d upper half" % k, src[k][half:], before[k][half:])
        else:
            check_same(what + " array %d dst upper half" % k, dst[k][half:], dst_before[k][half:])
            check_same(what + " array %d src" % k, src[k], before[k])


@pytest.mark.gpu
@pytest.mark.parametrize("r_kind", R_KINDS)
@pytest.mark.parametrize("n", list(range(1, 17)))
def test_final_comb(n, r_kind):
    """launch_final_comb: the n values src_k[0] + r (src_k[half] - src_k[0]), published twice on one Finalize"""
    rng = np.random.default_rng(100 + n)
    r = r_of(r_kind, rng)
    for half in (1, 2, 1000):
        B = [rvals(rng, 2 * half) for _ in range(n)]
        if half == 1:
            B = [[(0, 1, L - 1)[k % 3], (1, L - 1, 0)[k % 3]] for k in range(n)]
        src = tiled(B, 2 * half)
        before = src.copy()
        out = publish_out(n)
        kh.call("kh_final_comb", n, ptr(src), half, ptr(mont([r])[0]), 1, ptr(out))
        what = "final_comb n=%d half=%d r=%s" % (n, half, r_kind)
        check_periodic(what, out, [(b[0] + r * (b[half] - b[0])) % L for b in B])
        check_same(what + " src", src, before)


# ---------------------------------------------------------------- layer 1, bind over pointer tables
@pytest.mark.gpu
@pytest.mark.parametrize("half", [1, 2, 255, 256, 257, 135169, 1 << 22])
def test_product_layer1(half):
    """launch_product_layer1: out[i] = P[i] P[half + i]; P unchanged, nothing written past half"""
    rng = np.random.default_rng(half)
    p = PERIOD if half > 4096 else 2 * half
    B = rvals(rng, p) if p >= 4 else [L - 1, L - 1]
    P = tiled([B], 2 * half)[0]
    before = P.copy()
    guard = 64
    out = sentinel(1, half + guard)[0]
    kh.call("kh_product_layer1", ptr(P), half, ptr(out), guard)
    what = "product_layer1 half=%d" % half
    check_periodic(what, out[:half], [B[a] * B[(a + half) % p] % L for a in range(p)])
    check_same(what + " guard", out[half:], sentinel(1, half + guard)[0][half:])
    check_same(what + " P", P, before)


@pytest.mark.gpu
@pytest.mark.parametrize("r_kind", R_KINDS)
@pytest.mark.parametrize("n,half", [(1, 1), (2, 1), (65, 1), (65, 1000), (33, 4097), (2, 1 << 22)])
def test_bind_ptrs(n, half, r_kind):
    """launch_bind_ptrs: dst_k = src_k bound with r, out of place, with shared sources; src unchanged, dst unwritten
    from half up"""
    rng = np.random.default_rng(n + half)
    r = r_of(r_kind, rng)
    p = PERIOD if half > 4096 else 2 * half
    B = [rvals(rng, p) for _ in range(n)] if p >= 4 else edge_arrays(n, p)
    src_of = [k if k % 3 else max(k - 1, 0) for k in range(n)]  # inputs 3, 6, ... read the array before them
    src_of = [s if src_of[s] == s else src_of[s] for s in src_of]
    src = tiled(B, 2 * half)
    before = src.copy()
    dst = sentinel(n, 2 * half)
    kh.call("kh_bind_ptrs", n, ptr(np.array(src_of, dtype=I32)), ptr(src), half, ptr(mont([r])[0]), ptr(dst))
    what = "bind_ptrs n=%d half=%d r=%s" % (n, half, r_kind)
    untouched = sentinel(1, 2 * half)[0][half:]
    for k in range(n):
        check_periodic(what + " dst %d" % k, dst[k][:half], bind_periodic(B[src_of[k]], half, r))
        check_same(what + " dst %d upper half" % k, dst[k][half:], untouched)
    check_same(what + " src", src, before)


# ---------------------------------------------------------------- ingest
INGEST_BLOCKS, INGEST_THREADS = NUM_SMS * 8, 256
NONCANON = [L, L + 1, 2**256 - 1]


def ingest_positions(n):
    """index 0, the last index, a non-zero lane of a non-zero warp of a non-zero CTA, and a position in the last
    grid-stride trip other than the last index"""
    stride = INGEST_BLOCKS * INGEST_THREADS
    pos = {0, n - 1}
    inner = 3 * INGEST_THREADS + 5 * 32 + 17
    if inner < n:
        pos.add(inner)
    last_trip = (n - 1) // stride * stride + 6 * 32 + 9
    if last_trip < n:
        pos.add(last_trip)
    return sorted(pos)


def ingest_planted(base, row_stride, positions, row):
    """for each position in turn: base with `row` there (limbs), rows row_stride u64 apart (the padding 0x5A bytes);
    yields (pos, dst, flags) of one launch each"""
    n = base.shape[0]
    src = np.full((n, row_stride), 0x5A5A5A5A5A5A5A5A, dtype=U64)
    src[:, :4] = base
    flat = src.reshape(-1)
    size = (n - 1) * row_stride + 4
    for pos in positions:
        flat[pos * row_stride:pos * row_stride + 4] = row
        dst = np.zeros((n, 4), dtype=U64)
        flags = np.zeros(2, dtype=np.uint32)
        kh.call("kh_poly_ingest", ptr(flat[:size]), row_stride, n, ptr(dst), ptr(flags))
        flat[pos * row_stride:pos * row_stride + 4] = base[pos]
        yield pos, dst, flags


def check_ingest_dst(what, dst, base, pos, row):
    check_same(what + " dst[%d]" % pos, dst[pos], row)
    dst[pos] = base[pos]
    check_same(what + " dst", dst, base)


def background(rng, width, count):
    """count values of fewer than `width` bits (0 when width <= 1), with 0 and the largest such value among them"""
    if width <= 1:
        return [0] * count
    top = (1 << (width - 1)) - 1
    out = [int.from_bytes(rng.bytes(32), "little") & top for _ in range(count)]
    out[0], out[-1] = 0, top
    return out


def wide_value(rng, width):
    """a value of exactly `width` bits, below l"""
    if width <= 1:
        return width
    if width == 253:
        return L - 1 - int.from_bytes(rng.bytes(8), "little")
    return (1 << (width - 1)) | (int.from_bytes(rng.bytes(32), "little") % (1 << (width - 1)))


ONE_WAVE = INGEST_BLOCKS * INGEST_THREADS
# row stride 4 at every size; 5..7 (rows 8-byte but mostly not 32-byte aligned) at a few
INGEST_SHAPES = [(n, 4) for n in (1, 2, 255, 257, 8193, ONE_WAVE + 1, 1 << 22)] + \
    [(257, 5), (ONE_WAVE + 1, 5), (257, 6), (8193, 6), (257, 7), (1 << 22, 7)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,row_stride", INGEST_SHAPES)
@pytest.mark.parametrize("width", [0, 1, 31, 32, 33, 64, 252, 253])
def test_poly_ingest_width(width, n, row_stride):
    """launch_poly_ingest: dst equals the rows; flags[0] = 0; flags[1] = the exact widest canonical bit length, with the
    single widest value planted at each position in turn (every other value narrower)"""
    rng = np.random.default_rng(width * 1000 + n % 997 + row_stride)
    p = min(PERIOD, n)
    base = mont(background(rng, width, p))[np.arange(n) % p]
    wide = mont([wide_value(rng, width)])[0]
    for pos, dst, flags in ingest_planted(base, row_stride, ingest_positions(n) if width else [0], wide):
        what = "poly_ingest width=%d n=%d stride=%d planted at %d" % (width, n, row_stride, pos)
        check_ingest_dst(what, dst, base, pos, wide)
        assert flags[0] == 0, what + ": a canonical input flagged non-canonical"
        assert flags[1] == width, "%s: flags[1] = %d, want %d" % (what, flags[1], width)


@pytest.mark.gpu
@pytest.mark.parametrize("n,row_stride", [(1, 4), (300, 4), (ONE_WAVE + 1, 7), (1 << 22, 4)])
@pytest.mark.parametrize("bad", NONCANON)
def test_poly_ingest_noncanonical(bad, n, row_stride):
    """one row of limbs >= l at each position: flags[0] = 1, dst still equals the rows, flags[1] the width of the
    canonical rest (33 bits; nothing left for n = 1)"""
    rng = np.random.default_rng(n + row_stride)
    p = min(PERIOD, n)
    base = mont(background(rng, 34, p))[np.arange(n) % p]
    row = raw([bad])[0]
    for pos, dst, flags in ingest_planted(base, row_stride, ingest_positions(n), row):
        what = "poly_ingest non-canonical %#x n=%d stride=%d at %d" % (bad, n, row_stride, pos)
        check_ingest_dst(what, dst, base, pos, row)
        assert flags[0] == 1, what + ": not flagged"
        want = 0 if n == 1 else 33
        assert flags[1] == want, "%s: flags[1] = %d, want %d" % (what, flags[1], want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 257, 1 << 20])
def test_poly_mirror_u32(n):
    """launch_poly_mirror_u32: the integer values, 0 and 2^32 - 1 among them"""
    rng = np.random.default_rng(n)
    vals = [int(v) for v in rng.integers(0, 1 << 32, size=min(n, PERIOD), dtype=np.uint64)]
    vals[0] = 0
    if len(vals) > 1:
        vals[-1] = 2**32 - 1
    src = mont(vals)[np.arange(n) % len(vals)]
    out = np.zeros(n, dtype=np.uint32)
    kh.call("kh_poly_mirror_u32", ptr(np.ascontiguousarray(src)), n, ptr(out))
    want = np.array(vals, dtype=np.uint32)[np.arange(n) % len(vals)]
    bad = np.nonzero(out != want)[0]
    assert not len(bad), "poly_mirror_u32 n=%d: %d differ, first at [%d]: got %d, want %d" % (
        n, len(bad), bad[0], out[bad[0]], want[bad[0]])


# ---------------------------------------------------------------- eq tables
@pytest.mark.gpu
@pytest.mark.parametrize("ell", [23, 24, 25, 26, 27, 28])
def test_eq_evals_large(ell):
    """launch_eq_evals at 2^23 .. 2^28 entries (the high table built in the output's tail and staged in the scratch):
    the first and last 4096 entries, the whole tail the high table was built in, random samples; neither the output's
    guard nor the guard after a scratch of exactly kEqScratchElems is written"""
    rng = np.random.default_rng(ell)
    # no 0 or 1 among the coordinates: either would make half of the table zero, and with it whole checked regions
    # (the first 4096 entries, the staged tail) that an unwritten or wrongly staged entry could then match; l - 1 on
    # the last coordinate keeps an edge value without zeroing anything
    r = rvals(rng, ell, edges=False)
    r[-1] = L - 1
    n = 1 << ell
    tail = 1 << (ell - 11)
    samples = sorted(set(int(x) for x in rng.integers(0, n, size=2000)))
    ranges = [(0, 4096), (n - tail, tail)] + [(s, 1) for s in samples]
    idx = [i for a, c in ranges for i in range(a, a + c)]
    out = np.zeros((len(idx), 4), dtype=U64)
    guards = np.zeros(2, dtype=np.int32)
    kh.call("kh_eq_evals", ell, ptr(mont(r)), ptr(np.array(ranges, dtype=U64)), len(ranges), ptr(out), ptr(guards))
    want = eq_ref(r, idx)
    assert all(want), "eq_evals ell=%d: the reference has a zero entry, which an unwritten entry could match" % ell
    got = np.ascontiguousarray(out)
    bad = np.nonzero((got != mont(want)).any(axis=1))[0]
    if len(bad):
        fail_at("eq_evals ell=%d (entry %d)" % (ell, idx[int(bad[0])]), got, lambda i: want[i], bad)
    assert guards[0] == 0, "eq_evals ell=%d wrote past 2^ell entries" % ell
    assert guards[1] == 0, "eq_evals ell=%d wrote past the scratch" % ell
