"""The shapes the C ABI accepts for the built-in strategies, restated in Python, and the case lists the shape tests
(test_gpu_strategy_shapes.py, test_strategy_shapes_host.py) derive from them."""
import zlib

AND, OR, XOR, LT, RANGE_CHECK = 0, 1, 2, 3, 4
KINDS = (AND, OR, XOR, LT, RANGE_CHECK)
NAMES = {AND: "and", OR: "or", XOR: "xor", LT: "lt", RANGE_CHECK: "range"}

# Strategy::valid() (lasso_b200/csrc/kernels.cuh): the boundaries of every list below
C_MIN, C_MAX = 1, 16
LOG_M_MIN, LOG_M_MAX = 2, 24
SHIFT_LIMIT = 64          # combine_lookups weights are F::from(1u64 << shift): the widest shift must stay below 64
MAX_CIRCUITS = 32         # grand-product circuits in one batch (prove_gpa): 2 per memory


def num_memories(kind, C):
    return 2 * C if kind == LT else C


def inc(kind, log_m):
    """the weight step of combine_lookups (and.rs:45-53, range_check.rs:78-86)"""
    return log_m if kind == RANGE_CHECK else log_m // 2


def widest_shift(kind, C, log_m):
    """the largest weight shift, (alpha - 1) * inc; LT has no weights"""
    return None if kind == LT else (num_memories(kind, C) - 1) * inc(kind, log_m)


def accepted(kind, C, log_m, log_r=0):
    """Strategy::valid(): what the round, materialize, gather and prove entry points accept"""
    if kind not in KINDS or not C_MIN <= C <= C_MAX or not LOG_M_MIN <= log_m <= LOG_M_MAX:
        return False
    if log_m % 2 and kind != RANGE_CHECK:
        return False
    if kind != LT and widest_shift(kind, C, log_m) >= SHIFT_LIMIT:
        return False
    return kind != RANGE_CHECK or log_r >= 0


def provable(kind, C, log_m, log_r=0):
    """accepted() and a batched grand product that fits: LT with C <= 8"""
    return accepted(kind, C, log_m, log_r) and 2 * num_memories(kind, C) <= MAX_CIRCUITS


def seed_of(*parts):
    """a stable seed for a case"""
    return zlib.crc32(repr(parts).encode())


def _checked(cases, pred=accepted):
    for c in cases:
        assert pred(*c[:4]), c
    return cases


# ---- round messages: (kind, C, log_m, log_r), lengths
LT_ROUNDS = _checked([(LT, C, 4, 0) for C in range(C_MIN, C_MAX + 1)])
LT_ROUND_LENGTHS = [2, 16, 1 << 12, 1 << 13]  # at C = 8, 2^12 and 2^13 straddle the switch to the two-lane kernel
LT_GRID_STRIDE = _checked([(LT, 5, 4, 0), (LT, C_MAX, 4, 0)])  # 2^16: more pairs than threads in the grid
# 2^14: the bind round then evaluates 2^12 pairs, so it also reaches the two-lane C = 8 kernel
LT_TWO_LANE_BIND = _checked([(LT, 8, 4, 0)])
# inc = log_m / 2 odd (log_m = 6) and even (log_m = 8); RangeCheck: inc = log_m, odd 3 and even 4
LINEAR_ROUNDS = _checked([(k, C, log_m, 0) for k in (AND, OR, XOR) for C in (1, 2, 3, 7, 16) for log_m in (6, 8)] +
                         [(RANGE_CHECK, C, log_m, 5) for C in (1, 2, 3, 5, 16) for log_m in (3, 4)])
# the widest weights the ABI accepts: shift 63 (and 60 for XOR with C = 16)
WEIGHT_BOUNDARY = _checked([(AND, 10, 14, 0), (RANGE_CHECK, 4, 21, 0), (RANGE_CHECK, 10, 7, 0), (XOR, 16, 8, 0)])
for _c in WEIGHT_BOUNDARY:
    assert widest_shift(*_c[:3]) in (60, SHIFT_LIMIT - 1), _c
LINEAR_ROUND_LENGTHS = [4, 16, 1 << 13]

# ---- subtables and gather
TABLES_SMALLEST = _checked([(k, 2, LOG_M_MIN, 1) for k in KINDS])
TABLES_RANGE = _checked(sorted({(RANGE_CHECK, 4, log_m, log_r) for log_m in (3, 5, 7, 13)
                                for log_r in (0, 1, log_m - 1, log_m, 2 * log_m, 4 * log_m + 3)}))
TABLES_LARGE = _checked([(AND, 2, 20, 0), (OR, 2, 20, 0), (XOR, 2, 20, 0), (LT, 2, 20, 0), (RANGE_CHECK, 3, 20, 45)])
GATHER_ALL_MEMORIES = _checked([(LT, C_MAX, 4, 0)])  # 32 memories

# ---- whole proofs: name, kind, C, log_m, log_r, lookups, same_index
PROOFS = [
    ("lt_c3_m4_same", LT, 3, 4, 0, 37, True),
    ("lt_c5_m6", LT, 5, 6, 0, 200, False),
    ("lt_c6_m8_same", LT, 6, 8, 0, 300, True),
    ("lt_c7_m6", LT, 7, 6, 0, 129, False),
    ("range_c3_m5_r13", RANGE_CHECK, 3, 5, 13, 100, False),
    ("range_c1_m7_r3", RANGE_CHECK, 1, 7, 3, 50, False),
    ("range_c4_m9_r0", RANGE_CHECK, 4, 9, 0, 70, True),
    ("range_c3_m6_r12", RANGE_CHECK, 3, 6, 12, 64, False),
    ("range_c2_m8_r40", RANGE_CHECK, 2, 8, 40, 33, False),
    ("range_c8_m9_r63", RANGE_CHECK, 8, 9, 63, 40, False),      # shift 63
    ("xor_c16_m8", XOR, 16, 8, 0, 60, False),                      # shift 60, 32 circuits
    ("and_c10_m14", AND, 10, 14, 0, 20, False),                    # shift 63
    ("and_c4_m2", AND, 4, LOG_M_MIN, 0, 12, False),
    ("lt_c2_m2_same", LT, 2, LOG_M_MIN, 0, 9, True),
]
_checked([c[1:] for c in PROOFS], provable)
assert any(num_memories(c[1], c[2]) * 2 == MAX_CIRCUITS for c in PROOFS)
# the proofs also checked through the interpreter, without the digit-multiples tables and sharded
PROOF_SUBSET = ["lt_c5_m6", "range_c3_m5_r13"]

# ---- just past each boundary: every built-in entry point must return LASSO_ERR_STRATEGY
REJECTED = [
    ("C_0", AND, C_MIN - 1, 4, 0),
    ("C_17", AND, C_MAX + 1, 4, 0),
    ("log_m_1", RANGE_CHECK, 2, LOG_M_MIN - 1, 0),
    ("log_m_25", AND, 1, LOG_M_MAX + 1, 0),
    ("odd_log_m_and", AND, 2, 5, 0),
    ("odd_log_m_or", OR, 2, 7, 0),
    ("odd_log_m_xor", XOR, 2, 9, 0),
    ("odd_log_m_lt", LT, 2, 5, 0),
    ("shift_64", AND, 9, 16, 0),
    ("shift_66", RANGE_CHECK, 4, 22, 0),
    ("log_r_neg", RANGE_CHECK, 2, 8, -1),
    ("kind_5", 5, 2, 4, 0),
    ("kind_neg", -1, 2, 4, 0),
]
for _r in REJECTED:
    assert not accepted(*_r[1:]), _r
_rejected = {r[0]: r[1:] for r in REJECTED}
assert widest_shift(*_rejected["shift_64"][:3]) == SHIFT_LIMIT and widest_shift(*_rejected["shift_66"][:3]) == 66
# accepted but not provable: the round entry points take them, lasso_prove refuses them up front
UNPROVABLE = [(LT, 9, 4, 0), (LT, C_MAX, 4, 0)]
for _u in UNPROVABLE:
    assert accepted(*_u) and not provable(*_u)
