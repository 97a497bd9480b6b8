"""Caller-defined strategies over tables of arbitrary field elements (lasso_strategy_create_fr), shared by the CPU and
GPU tests: each builder takes (ctx, C, log_m, degree) and returns a lasso_b200.CustomStrategy whose tables are (M, 4)
Montgomery arrays.  ctx=None builds only the host description (for the oracle)."""
import numpy as np

L_FR = 2**252 + 27742317777372353535851937790883648493


def g_of_degree(degree):
    """combine_lookups of exactly `degree`: the sum of the memory values, plus a product of `degree` of them"""
    def g(v):
        acc = v[0]
        for x in v[1:]:
            acc = acc + x
        if degree > 1:
            p = v[0]
            for j in range(1, degree):
                p = p * v[j % len(v)]
            acc = acc + p * 3
        return acc
    return g


def _rng(name, log_m):
    return np.random.default_rng(sum(map(ord, name)) * 64 + log_m)


def ints_random_full(log_m):
    rng = _rng("random", log_m)
    return [int.from_bytes(rng.bytes(32), "little") % L_FR for _ in range(1 << log_m)]


def ints_differences(log_m):
    """a signed difference table: entry (a, b) = a - b, so half the entries are l - k"""
    h = log_m // 2
    lo_bits = log_m - h
    return [(i >> lo_bits) - (i & ((1 << lo_bits) - 1)) for i in range(1 << log_m)]


def ints_squares_40(log_m):
    """squares of 20-bit values: every entry has 40 bits"""
    return [(i + 0xC0000) ** 2 for i in range(1 << log_m)]


def ints_39bit(log_m):
    """entries up to 2^39 - 1: a width one below a multiple of 8, where the signed digits need a sixth window"""
    return [2**39 - 1 - 977 * i for i in range(1 << log_m)]


def ints_one_top(log_m):
    """small entries with a single l - 1"""
    t = [i * 3 + 1 for i in range(1 << log_m)]
    t[(1 << log_m) // 3] = L_FR - 1
    return t


EDGE_VALUES = [0, 1, 2**32 - 1, 2**32, 2**252, L_FR - 1]


def ints_edges(log_m):
    """2^32, 2^252 and l - 1 among small values and zeros"""
    rng = _rng("edges", log_m)
    t = [int(x) for x in rng.integers(0, 1 << 20, size=1 << log_m)]
    for k, v in enumerate(EDGE_VALUES):
        t[(k * 5 + 1) % len(t)] = v
    return t


INTS = {
    "random_full": ints_random_full,
    "differences": ints_differences,
    "squares_40bit": ints_squares_40,
    "max_39bit": ints_39bit,
    "one_top_entry": ints_one_top,
    "edges": ints_edges,
}


def strategy(ctx, name, C, log_m, degree=1, nsub=1):
    """a strategy over nsub copies of table `name` (the k-th rotated by k), default maps, g of the given degree"""
    import lasso_b200 as lb

    base = INTS[name](log_m)
    tables = [lb.fr_from_ints(base[k:] + base[:k]) for k in range(nsub)]
    return lb.CustomStrategy(ctx, C, log_m, tables, g_of_degree(degree), degree)


def width(values):
    return max(max(int(v) % L_FR for v in values).bit_length(), 1)
