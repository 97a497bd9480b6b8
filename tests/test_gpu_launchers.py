"""The prover's internal launchers (kernels.cuh, msm.cuh), one launch at a time, against plain references: Python
integers mod l for the scalar side, the CPU oracle's MSM for points.  Every comparison is bit-exact, on Montgomery
limbs or on normalised points, and a failure names the launch, the shape and the first element that differs.  The
launches go through tests/kernel_harness (the library's own kernel objects behind one C wrapper each).

Also: whole proofs on the commitment path a GPU without room for the 16-bit multiples table takes (the 8-bit table
only, msm_rows_direct_u32 with M16 = nullptr), against the oracle."""
import ctypes as C

import numpy as np
import pytest

import custom_builtins as cb
import kernel_harness_lib as kh
import oracle_custom_lib as oc
import oracle_lib as ol
import test_gpu_prove as tgp
from oracle_lib import P, lib as orc, sz

pytestmark = pytest.mark.gpu

L = ol.L_FR
Q = ol.Q_FQ
R256 = 2**256
RINV = pow(R256, -1, L)
U32MAX = 2**32 - 1


# ---------------------------------------------------------------- conversions (vectorised through bytes)
def mont(ints):
    """field elements -> (n, 4) Montgomery limbs"""
    b = b"".join((x % L * R256 % L).to_bytes(32, "little") for x in ints)
    return np.frombuffer(b, dtype=np.uint64).reshape(-1, 4).copy()


def raw(ints):
    """integers < 2^256 -> (n, 4) limbs, as they are (Montgomery limbs given directly, or canonical integers)"""
    b = b"".join(int(x).to_bytes(32, "little") for x in ints)
    return np.frombuffer(b, dtype=np.uint64).reshape(-1, 4).copy()


def raw_ints(arr):
    b = np.ascontiguousarray(arr, dtype=np.uint64).tobytes()
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def one(x):
    return np.ascontiguousarray(mont([x])[0])


def ptr(a):
    """pointer argument that keeps the array alive through the call (arguments are often temporaries)"""
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def rvals(rng, n, edges=True):
    """n uniform field elements; with edges and n >= 4, 0, 1 and l-1 among them (shorter vectors stay random: a zero
    in a one-element weight vector would hide every error that only scales it)"""
    b = rng.bytes(40 * n)
    out = [int.from_bytes(b[40 * i:40 * i + 40], "little") % L for i in range(n)]
    if edges and n >= 4:
        for j, e in enumerate((0, 1, L - 1)):
            out[(7 * j + 1) % n] = e
    return out


def check(what, got_limbs, want, montgomery=True):
    """bit-exact: got_limbs (n, 4) must equal the limbs of want (field elements as Montgomery, or raw integers)"""
    want_limbs = mont(want) if montgomery else raw(want)
    got_limbs = np.ascontiguousarray(got_limbs, dtype=np.uint64).reshape(-1, 4)
    assert got_limbs.shape == want_limbs.shape, "%s: %d elements, want %d" % (what, got_limbs.shape[0], want_limbs.shape[0])
    bad = np.nonzero((got_limbs != want_limbs).any(axis=1))[0]
    if len(bad):
        i = int(bad[0])
        g = raw_ints(got_limbs[i:i + 1])[0]
        raise AssertionError("%s: %d of %d elements differ, first at [%d]: got limbs %#x (value %d), want value %d"
                             % (what, len(bad), len(want), i, g, g * RINV % L if montgomery else g, want[i]))


@pytest.fixture(scope="module")
def gens():
    return np.ascontiguousarray(ol.generators(4098))


@pytest.fixture(scope="module")
def tables(gens):
    t = kh.Tables(gens)
    yield t
    t.close()


# ---------------------------------------------------------------- K3: batched cubic rounds
def cubic_eval_ref(A, B, Cq, cf, scale):
    """sum_k coeff_k (e0, e2, e3)_k of sumcheck.rs:49-93 with the batching of sumcheck.rs:95-97; A_k already scaled in
    memory when scale == 0"""
    half = len(Cq) // 2
    e = [0, 0, 0]
    for i in range(half):
        s0 = s2 = s3 = 0
        for k in range(len(A)):
            a0, a1 = A[k][i], A[k][half + i]
            if scale:
                a0, a1 = a0 * cf[k] % L, a1 * cf[k] % L
            b0, b1 = B[k][i], B[k][half + i]
            da, db = a1 - a0, b1 - b0
            s0 += a0 * b0
            s2 += (a1 + da) * (b1 + db)
            s3 += (a1 + 2 * da) * (b1 + 2 * db)
        c0, c1 = Cq[i], Cq[half + i]
        dc = c1 - c0
        e[0] += s0 % L * c0
        e[1] += s2 % L * (c1 + dc)
        e[2] += s3 % L * (c1 + 2 * dc)
    return [x % L for x in e]


def bind_top_ref(Z, r):
    h = len(Z) // 2
    return [(Z[i] + r * (Z[i + h] - Z[i])) % L for i in range(h)]


# (ncirc, q): q = pairs per array in the evaluated round.  Both sides of the single-CTA limit 4 ncirc q <= 1024 and of
# kQuadMaxQ = 2048 (quad-lane kernel up to it, thread-per-pair kernels beyond), circuits strided over blockIdx.y.
CUBIC_SHAPES = [(1, 1), (2, 2), (3, 4), (8, 4), (31, 4), (32, 8), (32, 16), (1, 256), (2, 256), (3, 2048), (31, 2048),
                (1, 4096), (8, 4096), (32, 4096), (2, 1 << 15)]


def _cubic_inputs(rng, ncirc, length):
    A = [rvals(rng, length) for _ in range(ncirc)]
    B = [rvals(rng, length) for _ in range(ncirc)]
    Cq = rvals(rng, length)
    cf = rvals(rng, ncirc, edges=False)
    for k, e in enumerate((0, 1, L - 1)[: ncirc]):
        cf[(k + 1) % ncirc] = e
    return A, B, Cq, cf


@pytest.mark.parametrize("scale", [0, 1])
@pytest.mark.parametrize("ncirc,q", CUBIC_SHAPES)
def test_cubic_eval(ncirc, q, scale):
    """launch_sumcheck_eval_cubic_comb: the three published values; A, B, C unchanged"""
    rng = np.random.default_rng(1000 * ncirc + q + scale)
    n = 2 * q
    A, B, Cq, cf = _cubic_inputs(rng, ncirc, n)
    dA, dB, dC = mont([x for a in A for x in a]), mont([x for b in B for x in b]), mont(Cq)
    inA, inB = dA.copy(), dB.copy()
    out = np.zeros((3, 4), dtype=np.uint64)
    kh.call("kh_cubic", 0, ncirc, n, ptr(dA), ptr(dB), ptr(dC), None, ptr(one(0)), ptr(mont(cf)), scale, ptr(out))
    what = "eval_cubic ncirc=%d half=%d scale=%d" % (ncirc, q, scale)
    check(what + " published (e0, e2, e3)", out, cubic_eval_ref(A, B, Cq, cf, scale))
    assert (dA == inA).all() and (dB == inB).all(), what + ": A or B written"
    check(what + " Ceq", dC, Cq)


@pytest.mark.parametrize("scale", [0, 1])
@pytest.mark.parametrize("ncirc,q", CUBIC_SHAPES)
def test_cubic_bind_eval(ncirc, q, scale):
    """launch_sumcheck_bind_eval_cubic_comb: arrays of 4q bound with r to 2q (A_k stored scaled when scale = 1), then the
    round over the bound values.  Every bound A_k, B_k and Cout, the untouched upper halves, Cin unchanged, and the
    published values.  The small shapes run r = random, 0, 1, l-1."""
    rng = np.random.default_rng(2000 * ncirc + q + scale)
    h = 2 * q
    n = 2 * h
    rs = [rvals(rng, 1, edges=False)[0]] + ([0, 1, L - 1] if ncirc * q <= 256 else [])
    A, B, Cq, cf = _cubic_inputs(rng, ncirc, n)
    for r in rs:
        what = "bind_eval_cubic ncirc=%d h=%d scale=%d r=%s" % (ncirc, h, scale, "random" if r == rs[0] else r)
        dA, dB, dC = mont([x for a in A for x in a]), mont([x for b in B for x in b]), mont(Cq)
        dCout = np.zeros((h, 4), dtype=np.uint64)
        out = np.zeros((3, 4), dtype=np.uint64)
        kh.call("kh_cubic", 1, ncirc, n, ptr(dA), ptr(dB), ptr(dC), ptr(dCout), ptr(one(r)), ptr(mont(cf)), scale, ptr(out))
        Ab = [bind_top_ref(a, r) for a in A]
        if scale:
            Ab = [[x * cf[k] % L for x in a] for k, a in enumerate(Ab)]
        Bb = [bind_top_ref(b, r) for b in B]
        Cb = bind_top_ref(Cq, r)
        gA, gB = dA.reshape(ncirc, n, 4), dB.reshape(ncirc, n, 4)
        for k in range(ncirc):
            check(what + " A_%d bound" % k, gA[k][:h], Ab[k])
            check(what + " B_%d bound" % k, gB[k][:h], Bb[k])
            check(what + " A_%d upper half" % k, gA[k][h:], A[k][h:])
            check(what + " B_%d upper half" % k, gB[k][h:], B[k][h:])
        check(what + " Cout", dCout, Cb)
        check(what + " Cin", dC, Cq)
        check(what + " published (e0, e2, e3)", out, cubic_eval_ref(Ab, Bb, Cb, cf, 0))


# ---------------------------------------------------------------- product trees, bind heads
# (N, ntrees, slot0, stop_len): both sides of the 4096-element layer threshold (layer launches above it, the one-CTA
# walk below), whole trees (stop_len 2) and low-bit shards (stop_len 1)
TREE_CASES = [(2, 1, 0, 2), (4, 5, 3, 2), (4096, 32, 0, 2), (8192, 5, 7, 2), (1 << 14, 32, 1, 2), (2, 5, 0, 1),
              (4, 1, 200, 1), (4096, 1, 0, 1), (8192, 32, 2, 1), (1 << 14, 5, 9, 1)]


@pytest.mark.parametrize("N,ntrees,slot0,stop_len", TREE_CASES)
def test_product_trees(N, ntrees, slot0, stop_len):
    rng = np.random.default_rng(N + ntrees + stop_len)
    sentinel = 0x1234567
    trees, layers = [], []
    for t in range(ntrees):
        leaves = rvals(rng, N)
        if t == 1:
            leaves = [0] * N            # an all-zero tree
        elif t == 2:
            leaves = [L - 1] * N        # (-1)^N
        elif t == 0:
            leaves[N - 1] = 0           # one zero leaf
        lay = [leaves]
        while len(lay[-1]) > stop_len:
            x = lay[-1]
            hh = len(x) // 2
            lay.append([x[i] * x[i + hh] % L for i in range(hh)])
        flat = [v for l_ in lay for v in l_]
        trees.append(flat + [sentinel] * (2 * N - len(flat)))
        layers.append(lay)
    d = mont([v for t in trees for v in t])
    tops = np.zeros((ntrees * stop_len, 4), dtype=np.uint64)
    kh.call("kh_product_trees", ntrees, N, slot0, stop_len, ptr(d), ptr(tops))
    d = d.reshape(ntrees, 2 * N, 4)
    what = "product_trees N=%d ntrees=%d slot0=%d stop_len=%d" % (N, ntrees, slot0, stop_len)
    for t in range(ntrees):
        check(what + " tree %d (all layers + untouched tail)" % t, d[t], trees[t])
    check(what + " published tops", tops, [layers[t][-1][j] for t in range(ntrees) for j in range(stop_len)])


@pytest.mark.parametrize("n", [1, 31, 32, 33, 64])
def test_bind_heads(n):
    rng = np.random.default_rng(n)
    heads = [rvals(rng, 2) for _ in range(n)]
    for r in [rvals(rng, 1, edges=False)[0], 0, 1, L - 1]:
        d = mont([x for hd in heads for x in hd])
        out = np.zeros((n, 4), dtype=np.uint64)
        kh.call("kh_bind_heads", n, ptr(d), ptr(one(r)), ptr(out))
        want = [(hd[0] + r * (hd[1] - hd[0])) % L for hd in heads]
        what = "bind_heads n=%d r=%d" % (n, r)
        check(what + " x[0]", d.reshape(n, 2, 4)[:, 0], want)
        check(what + " x[1]", d.reshape(n, 2, 4)[:, 1], [hd[1] for hd in heads])
        check(what + " published", out, want)


# ---------------------------------------------------------------- u32-mirror reductions (320-bit accumulator)
# The kernels multiply the Montgomery LIMBS of a field element by a u32 and reduce the integer sum once, so the
# reference works on limbs: result limbs = sum_j limbs(L_j) * z_j mod l.  The largest limbs are l - 1, the largest z
# 2^32 - 1: 17 such terms pass 2^288 (the top accumulator word).
def _u32_sets(rng, nL, nz):
    """(name, L limbs, z values): adversarial maximum, the field element l-1 (small limbs), random with edges"""
    Lr = [int.from_bytes(rng.bytes(40), "little") % L for _ in range(nL)]
    for j, e in enumerate((0, 1, L - 1)):
        if nL > j:
            Lr[(5 * j) % nL] = e
    zr = rng.integers(0, 2**32, size=nz, dtype=np.uint64).astype(np.uint32)
    zr[: min(nz, 2)] = [0, U32MAX][: min(nz, 2)]
    return [("max", [L - 1] * nL, np.full(nz, U32MAX, dtype=np.uint32)),
            ("value_l-1", [(L - 1) * R256 % L] * nL, np.full(nz, U32MAX, dtype=np.uint32)),
            ("random", Lr, zr)]


@pytest.mark.parametrize("L_size", [1, 2, 63, 64, 65, 4097])
@pytest.mark.parametrize("R_size", [1, 255, 256, 257])
def test_bound_u32(L_size, R_size):
    rng = np.random.default_rng(L_size * 1000 + R_size)
    for name, Ll, Z in _u32_sets(rng, L_size, L_size * R_size):
        out = np.zeros((R_size, 4), dtype=np.uint64)
        kh.call("kh_bound_u32", ptr(Z), ptr(raw(Ll)), L_size, R_size, ptr(out))
        if name == "random":
            Zi = [int(z) for z in Z]
            want = [sum(Ll[j] * Zi[j * R_size + i] for j in range(L_size)) % L for i in range(R_size)]
        else:
            want = [Ll[0] * U32MAX * L_size % L] * R_size
        check("bound_u32 L_size=%d R_size=%d %s" % (L_size, R_size, name), out, want, montgomery=False)


# (npolys, n): n = 2^22 / 2^19 give every thread of the grid-stride loop ~31 terms
@pytest.mark.parametrize("npolys,n", [(1, 1), (1, 1000), (3, 200000), (8, 4097), (1, 1 << 22), (8, 1 << 19)])
def test_multi_dot_u32(npolys, n):
    rng = np.random.default_rng(npolys * 7 + n)
    stride = n + 3 if npolys > 1 else n  # rows of a strided batch; the padding must not be read
    sets = _u32_sets(rng, n, n) if n <= 200000 else [("max", [L - 1] * n, np.full(n, U32MAX, dtype=np.uint32))]
    for name, Ll, z in sets:
        base = np.full((npolys, stride), U32MAX, dtype=np.uint32)
        zs = [np.roll(z, k) for k in range(npolys)]
        for k in range(npolys):
            base[k, :n] = zs[k]
        eq = np.ascontiguousarray(np.tile(raw([Ll[0]]), (n, 1))) if name != "random" else raw(Ll)
        out = np.zeros((npolys, 4), dtype=np.uint64)
        kh.call("kh_multi_dot_u32", ptr(base), stride, npolys, ptr(eq), n, ptr(out))
        if name == "random":
            want = [sum(a * int(b) for a, b in zip(Ll, zs[k])) % L for k in range(npolys)]
        else:
            want = [Ll[0] * U32MAX * n % L] * npolys
        check("multi_dot_u32 npolys=%d n=%d %s" % (npolys, n, name), out, want, montgomery=False)


# ---------------------------------------------------------------- fingerprints (memory_checking.rs:249-252)
@pytest.mark.parametrize("G,g", [(1, 0), (2, 1), (4, 3)])
def test_fingerprints_mem(G, g):
    """init = v gamma + a - tau (t = 0), final = init + t gamma^2, for local cell i = address i G + g"""
    rng = np.random.default_rng(G)
    M_local = 150001  # more cells than one pass of the grid
    table = rvals(rng, M_local * G)
    fin = [int(x) for x in rng.integers(0, 1 << 20, size=M_local)]
    fin[3] = L - 1
    d_table, d_fin = mont(table), mont(fin)
    for gamma, tau in [tuple(rvals(rng, 2, edges=False)), (L - 1, 0), (1, L - 1)]:
        oi = np.zeros((M_local, 4), dtype=np.uint64)
        of = np.zeros((M_local, 4), dtype=np.uint64)
        kh.call("kh_fingerprints_mem", ptr(d_table), ptr(d_fin), M_local, G, g, ptr(one(gamma)), ptr(one(tau)),
                ptr(oi), ptr(of))
        init = [(table[i * G + g] * gamma + i * G + g - tau) % L for i in range(M_local)]
        g2 = gamma * gamma % L
        what = "gp_fingerprints_mem G=%d g=%d gamma=%d tau=%d" % (G, g, gamma, tau)
        check(what + " init", oi, init)
        check(what + " final", of, [(init[i] + fin[i] * g2) % L for i in range(M_local)])


def test_fingerprints_ops():
    """read = E gamma + dim - tau + read_ts gamma^2, write = read + gamma^2"""
    rng = np.random.default_rng(5)
    s = 150001
    dim, E, rd = rvals(rng, s), rvals(rng, s), rvals(rng, s)
    for gamma, tau in [tuple(rvals(rng, 2, edges=False)), (L - 1, 1)]:
        orr = np.zeros((s, 4), dtype=np.uint64)
        ow = np.zeros((s, 4), dtype=np.uint64)
        kh.call("kh_fingerprints_ops", ptr(mont(dim)), ptr(mont(E)), ptr(mont(rd)), s, ptr(one(gamma)), ptr(one(tau)),
                ptr(orr), ptr(ow))
        g2 = gamma * gamma % L
        want = [(E[i] * gamma + dim[i] - tau + rd[i] * g2) % L for i in range(s)]
        check("gp_fingerprints_ops gamma=%d tau=%d read" % (gamma, tau), orr, want)
        check("gp_fingerprints_ops gamma=%d tau=%d write" % (gamma, tau), ow, [(x + g2) % L for x in want])


# ---------------------------------------------------------------- Bulletproofs scalar helpers (bullet.rs:73-134)
H_SIZES = [1, 2, 255, 4096, 1 << 16]


def _challenges(rng):
    u = rvals(rng, 1, edges=False)[0] or 1
    return [(u, pow(u, -1, L)), (1, 1), (L - 1, L - 1)]


@pytest.mark.parametrize("h", H_SIZES)
def test_fold_ab(h):
    rng = np.random.default_rng(h)
    a, b = rvals(rng, 2 * h), rvals(rng, 2 * h)
    for u, ui in _challenges(rng)[: 3 if h <= 4096 else 1]:
        da, db = mont(a), mont(b)
        kh.call("kh_fold_ab", ptr(da), ptr(db), h, ptr(one(u)), ptr(one(ui)))
        what = "fold_ab h=%d u=%s" % (h, u if u in (1, L - 1) else "random")
        check(what + " a", da, [(a[i] * u + ui * a[h + i]) % L for i in range(h)] + a[h:])
        check(what + " b", db, [(b[i] * ui + u * b[h + i]) % L for i in range(h)] + b[h:])


@pytest.mark.parametrize("h", H_SIZES)
def test_cross_inner_products(h):
    rng = np.random.default_rng(h + 1)
    a, b = rvals(rng, 2 * h), rvals(rng, 2 * h)
    out = np.zeros((2, 4), dtype=np.uint64)
    kh.call("kh_cross_inner_products", ptr(mont(a)), ptr(mont(b)), h, ptr(out))
    want = [sum(a[i] * b[h + i] for i in range(h)) % L, sum(a[h + i] * b[i] for i in range(h)) % L]
    check("cross_inner_products h=%d (c_L, c_R)" % h, out, want)


@pytest.mark.parametrize("n_in", H_SIZES)
def test_expand_weights(n_in):
    rng = np.random.default_rng(n_in + 2)
    w = rvals(rng, n_in)
    for u, ui in _challenges(rng)[: 3 if n_in <= 4096 else 1]:
        out = np.zeros((2 * n_in, 4), dtype=np.uint64)
        kh.call("kh_expand_weights", ptr(mont(w)), n_in, ptr(one(u)), ptr(one(ui)), ptr(out))
        want = [x for t in range(n_in) for x in (w[t] * ui % L, w[t] * u % L)]
        check("expand_weights n_in=%d u=%s" % (n_in, u if u in (1, L - 1) else "random"), out, want)


def bullet_scalars_ref(a, w, n, m, G, g):
    """columns j = jl G + g: sL[j] = a[pos - h] w[t] for pos >= h, sR[j] = a[h + pos] w[t] for pos < h (t = j / m)"""
    h = m // 2
    sL, sR = [], []
    for jl in range(n // G):
        j = jl * G + g
        t, pos = divmod(j, m)
        if pos >= h:
            sL.append(a[pos - h] * w[t] % L)
            sR.append(0)
        else:
            sL.append(0)
            sR.append(a[h + pos] * w[t] % L)
    return sL, sR


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("a_rep", [0, 1])
def test_bullet_scalars(G, a_rep):
    """every round m = n .. 2 of n = 1024 columns; a_rep = 0 (the rank's low-bit shard of a) while m >= 2G"""
    rng = np.random.default_rng(G * 10 + a_rep)
    n = 1024
    m = n
    while m >= 2:
        if a_rep == 0 and m < 2 * G:
            break
        a, w = rvals(rng, m), rvals(rng, n // m)
        for g in sorted({0, G - 1}):
            a_dev = a if a_rep else a[g::G]
            sL = np.zeros((n // G, 4), dtype=np.uint64)
            sR = np.zeros((n // G, 4), dtype=np.uint64)
            kh.call("kh_bullet_scalars", ptr(mont(a_dev)), len(a_dev), ptr(mont(w)), len(w), n // G, m, G, g, a_rep,
                    ptr(sL), ptr(sR))
            wL, wR = bullet_scalars_ref(a, w, n, m, G, g)
            what = "bullet_scalars n=%d m=%d G=%d g=%d a_rep=%d" % (n, m, G, g, a_rep)
            check(what + " sL", sL, wL)
            check(what + " sR", sR, wR)
        m //= 2


def test_bullet_scalars_grid_stride():
    rng = np.random.default_rng(3)
    n, m = 1 << 18, 1 << 9
    a, w = rvals(rng, m), rvals(rng, n // m)
    sL = np.zeros((n, 4), dtype=np.uint64)
    sR = np.zeros((n, 4), dtype=np.uint64)
    kh.call("kh_bullet_scalars", ptr(mont(a)), m, ptr(mont(w)), len(w), n, m, 1, 0, 1, ptr(sL), ptr(sR))
    wL, wR = bullet_scalars_ref(a, w, n, m, 1, 0)
    check("bullet_scalars n=%d m=%d sL" % (n, m), sL, wL)
    check("bullet_scalars n=%d m=%d sR" % (n, m), sR, wR)


@pytest.mark.parametrize("scale", [0, 1])
@pytest.mark.parametrize("n", [1, 255, 1 << 16])
def test_two_row_scalars(n, scale):
    """row 0 = (k v, t00, t01), row 1 = (0 .., t10, t11), canonical integers"""
    rng = np.random.default_rng(n + scale)
    v = rvals(rng, n)
    for k, ts in [(rvals(rng, 1, edges=False)[0], rvals(rng, 4, edges=False)), (L - 1, [0, 1, L - 1, 2])]:
        out = np.zeros((2 * (n + 2), 4), dtype=np.uint64)
        kh.call("kh_two_row_scalars", ptr(mont(v)), scale, ptr(one(k)), ptr(mont(ts)), n, ptr(out))
        row0 = [x * k % L if scale else x for x in v] + ts[:2]
        row1 = [0] * n + ts[2:]
        check("two_row_scalars n=%d scale=%d k=%d" % (n, scale, k), out, row0 + row1, montgomery=False)


# ---------------------------------------------------------------- MSMs over the digit-multiples table
def oracle_affine(bases, scalars):
    """sum_i scalars[i] * bases[i] by the oracle -> affine (x, y) integers"""
    ref = np.zeros(16, dtype=np.uint64)
    b = np.ascontiguousarray(bases)
    orc().orc_msm(P(b), P(mont(scalars)), sz(len(scalars)), 1, P(ref))
    aff = np.zeros(8, dtype=np.uint64)
    orc().orc_point_to_affine(P(ref), P(aff))
    return ol.fq_ints(aff.reshape(2, 4))


def published_affine(xyz):
    """canonical projective (X, Y, Z) as published -> affine (x, y) integers"""
    X, Y, Z = raw_ints(xyz)
    assert max(X, Y, Z) < Q, "published coordinate not canonical"
    zi = pow(Z, -1, Q)
    return [X * zi % Q, Y * zi % Q]


def canon_u32(ints):
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in ints), dtype=np.uint32).copy()


@pytest.mark.parametrize("length", [3, 4, 130, 2050])
def test_msm_direct(tables, gens, length):
    rng = np.random.default_rng(length)
    rows = {"zero": [0] * length, "equal": [rvals(rng, 1, edges=False)[0]] * length, "edges": rvals(rng, length),
            "ones": [1, L - 1] * (length // 2) + [1] * (length % 2), "random": rvals(rng, length, edges=False)}
    for r0, r1 in [("zero", "edges"), ("equal", "random"), ("ones", "zero")]:
        out = np.zeros((6, 4), dtype=np.uint64)
        kh.call("kh_msm_direct", tables.h, ptr(canon_u32(rows[r0] + rows[r1])), length, ptr(out))
        for row, name in enumerate((r0, r1)):
            got = published_affine(out[3 * row:3 * row + 3])
            assert got == oracle_affine(gens[:length], rows[name]), "msm_direct len=%d row %d (%s) differs" % (length, row, name)


def bullet_round_ref(a_in, b_in, w_in, n, m, fold, u, ui):
    """bullet.rs:73-134 with the generators kept unfolded: the current G_i = sum_t w[t] G_orig[t m + i]"""
    if fold:
        a = [(a_in[i] * u + ui * a_in[m + i]) % L for i in range(m)]   # bullet.rs:127-128
        b = [(b_in[i] * ui + u * b_in[m + i]) % L for i in range(m)]   # bullet.rs:129-130
        w = [x for t in w_in for x in (t * ui % L, t * u % L)]          # bullet.rs:131 G_L ui + G_R u
    else:
        a, b, w = a_in, b_in, w_in
    h = m // 2
    c_L = sum(a[i] * b[h + i] for i in range(h)) % L
    c_R = sum(a[h + i] * b[i] for i in range(h)) % L
    sL, sR = [0] * n, [0] * n
    for t in range(n // m):
        for p in range(h):
            sL[t * m + h + p] = a[p] * w[t] % L       # a_L on G_R
            sR[t * m + p] = a[h + p] * w[t] % L       # a_R on G_L
    return a, b, w, sL, sR, c_L, c_R


@pytest.mark.parametrize("n", [4, 64, 2048, 4096])
def test_bullet_fused(tables, gens, n):
    """one Bulletproofs round in one launch, every m = n .. 2 and fold 0 / 1: the published L and R against the oracle
    MSM of the restated scalars plus c Q + blind h (which checks c_L and c_R), and the folded a', b' and w'"""
    rng = np.random.default_rng(n)
    m = n
    while m >= 2:
        for fold in ([0, 1] if 2 * m <= n else [0]):
            ab_len, w_len = (2 * m, n // (2 * m)) if fold else (m, n // m)
            a_in, b_in, w_in = rvals(rng, ab_len), rvals(rng, ab_len), rvals(rng, w_len)
            u = rvals(rng, 1, edges=False)[0] or 1
            ui = pow(u, -1, L)
            bl, br = rvals(rng, 2, edges=False)
            if m == 2:
                bl = 0
            a_o = np.zeros((m, 4), dtype=np.uint64)
            b_o = np.zeros((m, 4), dtype=np.uint64)
            w_o = np.zeros((n // m, 4), dtype=np.uint64)
            out = np.zeros((6, 4), dtype=np.uint64)
            kh.call("kh_bullet_fused", tables.h, ptr(mont(a_in)), ptr(mont(b_in)), ptr(mont(w_in)), n, m, fold, ptr(one(u)),
                    ptr(one(ui)), ptr(one(bl)), ptr(one(br)), ptr(a_o), ptr(b_o), ptr(w_o), ptr(out))
            a, b, w, sL, sR, c_L, c_R = bullet_round_ref(a_in, b_in, w_in, n, m, fold, u, ui)
            what = "bullet_fused n=%d m=%d fold=%d" % (n, m, fold)
            if fold:
                check(what + " a'", a_o, a)
                check(what + " b'", b_o, b)
                check(what + " w'", w_o, w)
            assert published_affine(out[0:3]) == oracle_affine(gens[: n + 2], sL + [c_L, bl]), what + ": L differs"
            assert published_affine(out[3:6]) == oracle_affine(gens[: n + 2], sR + [c_R, br]), what + ": R differs"
        m //= 2


# ---------------------------------------------------------------- Hyrax rows of u32 scalars over the multiples tables
U32_EDGES = [0, 1, 0x7fff, 0x8000, 0x8001, 0xffff, 0x10000, 2**24 - 1, U32MAX]


def _u32_rows(rng, nrows, ncols, bits):
    """edge values below 2^bits and random values of that width"""
    edges = [v for v in U32_EDGES if v < 2**bits]
    z = rng.integers(0, 2**bits, size=nrows * ncols, dtype=np.uint64)
    for i in range(min(len(z), 3 * len(edges))):
        z[(i * 7) % len(z)] = edges[i % len(edges)]
    if nrows > 1:
        z[:ncols] = 0                                    # an all-zero row
        z[ncols:2 * ncols] = edges[-1]                   # an all-equal row
    return z.astype(np.uint32)


def _rows_check(tables, gens, ncols, col_mul, col_add, use16):
    rng = np.random.default_rng(ncols * 4 + use16 + col_mul)
    gsel = np.ascontiguousarray(np.concatenate([gens[[c * col_mul + col_add for c in range(ncols)]], gens[:1]]))
    for nrows in (1, 9, 64):
        for bits in (15, 16, 24, 32):
            z = _u32_rows(rng, nrows, ncols, bits)
            nw = (int(z.max()).bit_length() + 2 + 7) // 8  # msm_windows_for_bits of the data
            out = np.zeros((nrows, 16), dtype=np.uint64)
            kh.call("kh_msm_rows_direct_u32", tables.h, ptr(z), nrows, ncols, nw, col_mul, col_add, use16, ptr(out))
            ref = np.zeros((nrows, 16), dtype=np.uint64)
            orc().orc_commit_rows(P(gsel), P(mont([int(x) for x in z])), sz(nrows), sz(ncols), P(ref))
            for i in range(nrows):
                aff = np.zeros(8, dtype=np.uint64)
                orc().orc_point_to_affine(P(np.ascontiguousarray(ref[i])), P(aff))
                assert (out[i][:8] == aff).all(), ("msm_rows_direct_u32 %s ncols=%d nrows=%d nw=%d bits=%d col_map=%d*c+%d: "
                                                   "row %d differs" % ("M16" if use16 else "8-bit only", ncols, nrows, nw,
                                                                       bits, col_mul, col_add, i))


@pytest.mark.parametrize("use16", [0, 1])
@pytest.mark.parametrize("ncols", [1, 4, 200, 256])
def test_msm_rows_direct_u32(tables, gens, ncols, use16):
    """with M16 + K16 (built for exactly this ncols) and with M16 = nullptr (the 5-window 8-bit path)"""
    if not use16:
        _rows_check(tables, gens, ncols, 1, 0, 0)
        return
    t16 = kh.Tables(gens[: ncols + 2], ncols16=ncols)
    try:
        _rows_check(t16, gens, ncols, 1, 0, 1)
    finally:
        t16.close()


@pytest.mark.parametrize("use16", [0, 1])
def test_msm_rows_direct_u32_sharded_columns(gens, use16):
    """one rank of a proof sharded over two GPUs: local column c <-> generator 2c + 1, M16 built for that rank"""
    ncols = 128
    t = kh.Tables(gens[: 2 * ncols + 2], ncols16=ncols if use16 else 0, col_mul=2, col_add=1)
    try:
        _rows_check(t, gens, ncols, 2, 1, use16)
    finally:
        t.close()


# ---------------------------------------------------------------- whole proofs without the 16-bit multiples table
FALLBACK_CASES = [c for c in tgp.CASES if c[0] in ("prove_4d_lt_big_s", "range_c4", "or_c2_ragged")]


def _nv_max(C_, s, num_memories, log_m):
    lg = lambda x: (x - 1).bit_length()  # log2 of the next power of two
    return max(lg(2 * C_ * s), lg(C_) + log_m, lg(num_memories * s))


def _fallback_prove(monkeypatch, make_strategy, C_, log_m, idx, r, seed, s):
    """prove once with the default tables and once with LASSO_B200_TABLE_GB=0; returns the fallback's bytes and the
    difference in launches of the two generator setups"""
    import lasso_b200 as lb

    out = {}
    for mode in ("default", "fallback"):
        if mode == "fallback":
            monkeypatch.setenv("LASSO_B200_TABLE_GB", "0")
        else:
            monkeypatch.delenv("LASSO_B200_TABLE_GB", raising=False)
        ctx = lb.Context(0)
        S = make_strategy(ctx)
        need = lb.gens_points_needed(C_, s, S.num_memories, log_m)
        stream = np.ascontiguousarray(ol.generators(max(need, 300))[:need])
        before = ctx.launches
        gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C_, s, S.num_memories, log_m, stream=stream)
        launches = ctx.launches - before
        dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
        com = dense.commit(gens)
        proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=seed)
        out[mode] = (launches, com, proof.bytes, S.num_memories, stream)
        del gens, dense
        if hasattr(S, "close"):
            S.close()
        ctx.close()
    nv = _nv_max(C_, s, out["default"][3], log_m)
    # multiples16 once + one centre constant per power-of-two row length up to the 2^(nv - nv/2) columns
    assert out["default"][0] - out["fallback"][0] == 1 + (nv - nv // 2 + 1), "the 16-bit table was not skipped"
    return out


@pytest.mark.parametrize("name,kind,C,log_m,log_r,n,same", FALLBACK_CASES, ids=[c[0] for c in FALLBACK_CASES])
def test_prove_without_16bit_table(monkeypatch, name, kind, C, log_m, log_r, n, same):
    """LASSO_B200_TABLE_GB=0: the 8-bit multiples table only; the commitments take msm_rows_direct_u32 with M16 = nullptr.
    Commitment and proof bytes must equal the oracle's."""
    import lasso_b200 as lb

    idx, r, seed, s = tgp.make_inputs(C, log_m, n, len(name), same)
    out = _fallback_prove(monkeypatch, lambda ctx: lb.Strategy(kind, C, log_m, log_r), C, log_m, idx, r, seed, s)
    ref = ol.prove(kind, C, log_m, log_r, idx, r, out["fallback"][4], seed, flags=1)
    assert ref["rc"] == 0
    assert out["fallback"][1] == ref["commitment"]
    assert out["fallback"][2] == ref["proof"]


def test_prove_custom_wide_entries_without_16bit_table(monkeypatch):
    """a caller-defined table with entries near 2^32 - 1: five 8-bit windows per committed table value"""
    import lasso_b200 as lb

    probe = lb.Context(0)
    S0 = cb.NEW_TABLES["wide_entries"](probe)
    C_, log_m = S0.C, S0.log_m
    S0.close()
    probe.close()
    idx, r, seed, s = tgp.make_inputs(C_, log_m, 1 << 12, 7, False)
    out = _fallback_prove(monkeypatch, cb.NEW_TABLES["wide_entries"], C_, log_m, idx, r, seed, s)
    ctx = lb.Context(0)
    S = cb.NEW_TABLES["wide_entries"](ctx)
    ref = oc.prove(S, idx, r, out["fallback"][4], seed, flags=1)
    S.close()
    ctx.close()
    assert ref["rc"] == 0
    assert out["fallback"][1] == ref["commitment"]
    assert out["fallback"][2] == ref["proof"]
