"""The large MSM (msm_large.cu, msm_final.cu) at every window width it can run, not only the ones its size rule picks
for the sizes the other tests use.

Forced widths (msm_large_plan's c_force, through tests/kernel_harness: kh_msm_large) against the CPU oracle at 4100
terms over a pool of 4096 bases: c = 8..17 with full-width scalars (nw = 32 windows at c = 8, every lane of
msm_final_kernel, down to 15 at c = 17), c = 2..7 with scalars of at most 32 c - 2 bits (nw <= 32).  Each width runs
uniform scalars, a mix of {0, 1, the widest value}, one value repeated (each window has one bucket holding every term,
split into units; more than 32 of them from c = 9 on), all zeros (every bucket empty, the identity; the plan's
small-scalar clamp takes c down to 2) and a single term.  Both outputs are checked: the normalised arkworks point and
the raw internal (X, Y, Z, T), normalised here.

The product's own plans at the sizes the benchmark times and no other test checks, against the independent GPU sum
(MsmJob.naive: per-term double-and-add, no digits or buckets; its primitives are checked on their own by
test_gpu_arith.py): 2^20 terms (c = 15, reduction levels 16, 16, 16, 4), 2^21 (c = 16, levels 16, 16, 16, 8) and
2^24 (c = 17, 15 windows)."""
import ctypes as C
import random

import numpy as np
import pytest

import kernel_harness_lib as kh
import oracle_lib as ol
from test_gpu_launchers import mont, raw_ints
from test_gpu_msm_large import full_width, oracle_msm, same, small

pytestmark = pytest.mark.gpu

L, Q = ol.L_FR, ol.Q_FQ
N, POOL = 4100, 4096


@pytest.fixture(scope="module")
def pool():
    return np.ascontiguousarray(ol.generators(POOL))


def scalar_ints(kind, c, n, rng):
    """the scalars of one case: full width for c >= 8, else below 2^(32 c - 2) so that nw <= 32"""
    top = L - 1 if c >= 8 else (1 << (32 * c - 2)) - 1
    if kind == "uniform":
        return [rng.randrange(top + 1) for _ in range(n)]
    if kind == "edges":
        return [(0, 1, top)[rng.randrange(3)] for _ in range(n)]
    if kind == "repeated":
        return [rng.randrange(top // 2, top + 1)] * n
    if kind == "zeros":
        return [0] * n
    return [rng.randrange(top // 2, top + 1)]  # single


def expected_plan(c, ints):
    nbits = max(1, max(s.bit_length() for s in ints))
    ce = min(c, max(2, nbits + 1))
    return ce, -(-(nbits + 2) // ce)


@pytest.mark.parametrize("kind", ["uniform", "edges", "repeated", "zeros", "single"])
@pytest.mark.parametrize("c", list(range(2, 18)))
def test_forced_window_width_vs_oracle(pool, c, kind):
    rng = random.Random("%d-%s" % (c, kind))
    ints = scalar_ints(kind, c, N, rng)
    n = len(ints)
    n_pool = min(n, POOL)
    sc = mont(ints)
    out_ext = np.zeros(16, dtype=np.uint64)
    out_raw = np.zeros(32, dtype=np.uint32)
    info = (C.c_int * 14)()
    kh.call("kh_msm_large", pool.ctypes.data, n_pool, sc.ctypes.data, n, c, out_ext.ctypes.data, out_raw.ctypes.data,
            info)
    ce, nw = expected_plan(c, ints)
    what = "c_force %d, %s, %d terms: plan c %d nw %d nbits %d S %d levels %s" % (
        c, kind, n, info[0], info[1], info[2], info[4], list(info[6:6 + info[5]]))
    assert (info[0], info[1]) == (ce, nw), what
    bases = np.ascontiguousarray(np.tile(pool, ((n + POOL - 1) // POOL, 1))[:n])
    ref = oracle_msm(bases, sc)
    assert same(out_ext, ref), "out_ext: " + what
    X, Y, Z, T = raw_ints(out_raw.view(np.uint64).reshape(4, 4))
    rx, ry, _, rz = ol.fq_ints(ref.reshape(4, 4))
    rzi = pow(rz, -1, Q)
    assert Z % Q != 0, "out_raw: Z = 0: " + what
    zi = pow(Z, -1, Q)
    assert (X * zi % Q, Y * zi % Q) == (rx * rzi % Q, ry * rzi % Q), "out_raw: " + what
    assert T * Z % Q == X * Y % Q, "out_raw: T Z != X Y: " + what


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("log_n,kind,c,nw", [(20, "full", 15, 17), (20, "small16", 15, 2), (20, "small20", 15, 2),
                                             (21, "full", 16, 16), (21, "small16", 16, 2), (21, "small20", 16, 2),
                                             (24, "full", 17, 15)])
def test_product_plan_vs_independent_gpu_sum(ctx, log_n, kind, c, nw):
    import lasso_b200 as lb

    n = 1 << log_n
    rng = np.random.default_rng(log_n * 31 + len(kind))
    gens = np.ascontiguousarray(ol.generators(8194)[:8192])
    sc = full_width(rng, n) if kind == "full" else small(rng, n, int(kind[5:]))
    job = lb.MsmJob(ctx, gens, sc)
    pt, ms, info = job.run(1)
    assert (info["c"], info["windows"], info["T2"]) == (c, nw, 4), info
    assert same(pt, job.naive()), info
    job.close()
