"""The five built-in strategies (subtables/{and,or,xor,lt,range_check}.rs) re-expressed as caller-defined strategies,
and a few tables that are not built in.  Shared by the CPU and GPU tests of lasso_b200.CustomStrategy."""
import numpy as np

AND, OR, XOR, LT, RANGE_CHECK = 0, 1, 2, 3, 4


def builtin_tables(kind, C, log_m, log_r=0):
    """materialize_subtables() as u32 arrays"""
    M = 1 << log_m
    idx = np.arange(M, dtype=np.uint64)
    if kind == RANGE_CHECK:
        rem = np.where(idx < (1 << (log_r % log_m)), idx, 0)
        return [idx.astype(np.uint32), rem.astype(np.uint32), np.zeros(M, dtype=np.uint32)]
    bits = log_m // 2
    mask = (1 << bits) - 1
    lhs, rhs = (idx >> bits) & mask, idx & mask
    if kind == LT:
        return [(lhs < rhs).astype(np.uint32), (lhs == rhs).astype(np.uint32)]
    op = {AND: np.bitwise_and, OR: np.bitwise_or, XOR: np.bitwise_xor}[kind]
    return [op(lhs, rhs).astype(np.uint32)]


def builtin_maps(kind, C, log_m, log_r=0):
    """memory_to_subtable_index / memory_to_dimension_index; None = the trait's defaults"""
    if kind != RANGE_CHECK:
        return None, None
    sub = [2 if i * log_m > log_r else (1 if (i + 1) * log_m > log_r else 0) for i in range(C)]
    return sub, list(range(C))


def builtin_g(kind, C, log_m):
    """combine_lookups as a Horner chain: sum_i 2^(i inc) v_i (and.rs:45-53, range_check.rs:78-86) or
    sum_i LT_i prod_{j<i} EQ_j (lt.rs:60-69)"""
    if kind == LT:
        def g(v):
            h = v[2 * (C - 1)]
            for k in range(C - 2, -1, -1):
                h = v[2 * k] + v[2 * k + 1] * h
            return h
        return g, C
    inc = log_m if kind == RANGE_CHECK else log_m // 2

    def g(v):
        acc = v[-1]
        for x in reversed(v[:-1]):
            acc = acc * (1 << inc) + x
        return acc
    return g, 1


def as_custom(ctx, kind, C, log_m, log_r=0):
    """The built-in strategy as a CustomStrategy.  RangeCheck with C < 3 has more subtables (3) than memories: the
    tables no memory reads are left out (a custom strategy needs num_subtables <= num_memories), which changes no
    proof byte."""
    import lasso_b200 as lb

    g, deg = builtin_g(kind, C, log_m)
    sub, dim = builtin_maps(kind, C, log_m, log_r)
    tables = builtin_tables(kind, C, log_m, log_r)
    if sub is not None:
        used = sorted(set(sub))
        tables = [tables[k] for k in used]
        sub = [used.index(k) for k in sub]
    return lb.CustomStrategy(ctx, C, log_m, tables, g, deg, sub, dim)


# ---- tables that are not built in: name -> constructor (ctx -> CustomStrategy)
def _product(ctx):
    """degree 2: a product of two memories over two tables, non-default, non-monotone maps"""
    import lasso_b200 as lb

    log_m = 6
    idx = np.arange(1 << log_m, dtype=np.uint64)
    t0 = (idx * 7 + 3) % 61
    t1 = idx * idx
    return lb.CustomStrategy(ctx, 3, log_m, [t0, t1], lambda v: v[0] * v[3] + 5 * v[1] - v[2], 2,
                             memory_to_subtable=[1, 0, 1, 0], memory_to_dimension=[2, 0, 1, 2])


def _wide(ctx):
    """entries near 2^32 - 1 (the widest commitment path), odd log_m, one memory per dimension"""
    import lasso_b200 as lb

    log_m = 5
    t = (2**32 - 1) - np.arange(1 << log_m, dtype=np.uint64) * 977
    return lb.CustomStrategy(ctx, 2, log_m, [t], lambda v: v[0] + v[1] * (2**32), 1)


def _constants(ctx):
    """non-power-of-two and negative constants, a SUB from a constant, an unused memory, a declared degree above the
    program's"""
    import lasso_b200 as lb

    log_m = 4
    idx = np.arange(1 << log_m, dtype=np.uint64)
    return lb.CustomStrategy(ctx, 2, log_m, [idx ^ 5, (idx * 3) % 11, idx & 9],
                             lambda v: (-3) * v[0] + 1000003 * v[4] - (v[2] - 12345) * v[1] - 7, 3,
                             memory_to_subtable=[2, 0, 1, 2, 1, 0], memory_to_dimension=[1, 1, 0, 0, 1, 0])


def _cubic(ctx):
    """degree 3 in one memory, C = 1"""
    import lasso_b200 as lb

    log_m = 8
    idx = np.arange(1 << log_m, dtype=np.uint64)
    return lb.CustomStrategy(ctx, 1, log_m, [(idx * 2654435761) % (2**32)], lambda v: v[0] * v[0] * v[0] + v[0] - 1, 3)


NEW_TABLES = {"product_deg2": _product, "wide_entries": _wide, "constants": _constants, "cubic": _cubic}
