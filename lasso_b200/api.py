"""ctypes binding of liblasso_b200.so (include/lasso_b200.h) + the reference-shaped Python surface.

Field elements are numpy uint64 arrays (..., 4): ark-ff Montgomery limbs.  Affine points (..., 8),
extended points (..., 16)."""
import ctypes as C
import os
import sys

import numpy as np

AND, OR, XOR, LT, RANGE_CHECK = 0, 1, 2, 3, 4
_HERE = os.path.dirname(os.path.abspath(__file__))


class LassoError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("lasso_b200 error %d: %s" % (code, msg))
        self.code = code


def library_path():
    return os.path.join(_HERE, "liblasso_b200.so")


_lib = None


def lib():
    """Load the CUDA extension.  Fails loudly if it has not been built — there is no other code path."""
    global _lib
    if _lib is None:
        p = library_path()
        if not os.path.exists(p):
            raise RuntimeError("liblasso_b200.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(nvcc, sm_90a).  lasso_b200 has no CPU fallback.")
        L = C.CDLL(p)
        L.lasso_last_error.restype = C.c_char_p
        L.lasso_gens_points_needed.restype = C.c_size_t
        L.lasso_gens_points_needed.argtypes = [C.c_size_t] * 4
        L.lasso_dense_s.restype = C.c_size_t
        L.lasso_dense_read.restype = C.c_size_t
        L.lasso_launch_count.restype = C.c_ulonglong
        L.lasso_spans.restype = C.c_size_t
        L.lasso_poly_gens_points_needed.restype = C.c_size_t
        L.lasso_poly_gens_points_needed.argtypes = [C.c_size_t]
        L.lasso_poly_num_vars.restype = C.c_size_t
        L.lasso_gp_circuit_num_vars.restype = C.c_size_t
        L.lasso_transcript_append_u64.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
        # the zero-knowledge calls, declared so that a pointer passed as a Python int keeps its 64 bits (an undeclared
        # int argument goes over as a C int)
        V, S = C.c_void_p, C.c_size_t
        L.lasso_mc_commit.argtypes = [V, V, V, S, V, V]
        L.lasso_dot_product_prove.argtypes = [V] * 8 + [S, V, V, V, S, V, V, V]
        L.lasso_zk_sumcheck_prove.argtypes = [V, V, V, S, S] + [V] * 6 + [S] + [V] * 6
        L.lasso_knowledge_prove.argtypes = [V] * 8
        L.lasso_equality_prove.argtypes = [V] * 11
        L.lasso_product_prove.argtypes = [V] * 14
        _lib = L
    return _lib


def _chk(rc):
    if rc != 0:
        raise LassoError(rc, lib().lasso_last_error().decode())


def _p(a):
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.c_void_p)


def _fr(a, shape_last=4):
    a = np.ascontiguousarray(a, dtype=np.uint64)
    assert a.shape[-1] == shape_last
    return a


def _ptr_array(arrays):
    arr = (C.c_void_p * len(arrays))()
    for i, a in enumerate(arrays):
        arr[i] = a.ctypes.data
    return arr


class Strategy:
    """SubtableStrategy<F, C, M> (src/subtables/mod.rs:31-93) as runtime parameters."""

    def __init__(self, kind, C_, log_m, log_r=0):
        self.kind, self.C, self.log_m, self.log_r = int(kind), int(C_), int(log_m), int(log_r)

    @property
    def num_subtables(self):
        return {LT: 2, RANGE_CHECK: 3}.get(self.kind, 1)

    @property
    def num_memories(self):
        return 2 * self.C if self.kind == LT else self.C

    @property
    def sumcheck_poly_degree(self):
        return (self.C if self.kind == LT else 1) + 1


# ------------------------------------------------------------------ caller-defined strategies
OP_ADD, OP_SUB, OP_MUL, OP_MULK, OP_ADDK = 0, 1, 2, 3, 4
LASSO_ERR_LENGTH, LASSO_ERR_NOT_POW2, LASSO_ERR_GENS, LASSO_ERR_VALUE = 1, 2, 5, 8
LASSO_ERR_INDEX_RANGE, LASSO_ERR_STRATEGY, LASSO_ERR_POINTER = 3, 4, 7
FR_MODULUS = 2**252 + 27742317777372353535851937790883648493
MAX_MEMORIES, MAX_OPS, MAX_CONSTANTS, MAX_DEGREE = 16, 128, 64, 16


class _Value:
    """A value of the traced combine_lookups: an SSA slot and its degree in the memory values."""

    __slots__ = ("tr", "slot", "degree")

    def __init__(self, tr, slot, degree):
        self.tr, self.slot, self.degree = tr, slot, degree

    def __add__(self, o):
        return self.tr.binary(OP_ADD, self, o)

    __radd__ = __add__

    def __sub__(self, o):
        if isinstance(o, (int, np.integer)):
            return self.tr.binary(OP_ADD, self, -int(o))
        return self.tr.binary(OP_SUB, self, o)

    def __rsub__(self, o):  # o - self, o an int
        return self.tr.binary(OP_ADD, self.tr.binary(OP_MUL, self, -1), o)

    def __mul__(self, o):
        return self.tr.binary(OP_MUL, self, o)

    __rmul__ = __mul__

    def __neg__(self):
        return self.tr.binary(OP_MUL, self, -1)


class _Tracer:
    def __init__(self, num_memories):
        self.alpha = num_memories
        self.program, self.constants, self._kidx = [], [], {}

    def _const(self, x):
        x %= FR_MODULUS
        if x not in self._kidx:
            self._kidx[x] = len(self.constants)
            self.constants.append(x)
        return self._kidx[x]

    def _emit(self, op, a, b, degree):
        self.program.append((op, a, b))
        return _Value(self, self.alpha + len(self.program) - 1, degree)

    def binary(self, op, a, b):
        if isinstance(b, _Value):
            if b.tr is not self:
                raise ValueError("combine_lookups mixes values of two traces")
            deg = a.degree + b.degree if op == OP_MUL else max(a.degree, b.degree)
            return self._emit(op, a.slot, b.slot, deg)
        if not isinstance(b, (int, np.integer)):
            return NotImplemented
        return self._emit(OP_MULK if op == OP_MUL else OP_ADDK, a.slot, self._const(int(b)), a.degree)


def trace_combine_lookups(combine_lookups, num_memories):
    """Trace combine_lookups(vals), vals a list of num_memories symbolic values, through + - * (Python ints are constants
    mod l, negatives allowed) into the SSA program of lasso_strategy_create.  -> (program (n, 3) int32, constants
    (k, 4) uint64 Montgomery limbs, degree of g)."""
    tr = _Tracer(num_memories)
    g = combine_lookups([_Value(tr, k, 1) for k in range(num_memories)])
    if not isinstance(g, _Value) or g.tr is not tr:
        raise LassoError(LASSO_ERR_STRATEGY, "combine_lookups must return an expression of the memory values")
    if not tr.program or g.slot != num_memories + len(tr.program) - 1:  # g is an input or an earlier value
        g = tr._emit(OP_ADDK, g.slot, tr._const(0), g.degree)
    prog = np.array(tr.program, dtype=np.int32).reshape(-1, 3)
    consts = np.zeros((len(tr.constants), 4), dtype=np.uint64)
    for k, x in enumerate(tr.constants):
        m = x * 2**256 % FR_MODULUS
        consts[k] = [(m >> (64 * i)) & (2**64 - 1) for i in range(4)]
    return prog, consts, g.degree


def fr_from_ints(values):
    """Python integers (any sign, any size) -> (n, 4) uint64 Montgomery limbs of their residues mod l: the Fr layout of
    the binding, e.g. a CustomStrategy table of differences fr_from_ints([a - b for ...])."""
    vals = [int(v) % FR_MODULUS * 2**256 % FR_MODULUS for v in values]
    out = np.zeros((len(vals), 4), dtype=np.uint64)
    for i in range(4):
        out[:, i] = [(v >> (64 * i)) & (2**64 - 1) for v in vals]
    return out


def _is_canonical(limbs):
    """per row of (n, 4) uint64 limbs: the 256-bit integer they hold is below l"""
    below = np.zeros(limbs.shape[0], dtype=bool)
    equal = np.ones(limbs.shape[0], dtype=bool)
    for i in range(3, -1, -1):
        li = np.uint64((FR_MODULUS >> (64 * i)) & (2**64 - 1))
        below |= equal & (limbs[:, i] < li)
        equal &= limbs[:, i] == li
    return below


class CustomStrategy:
    """A caller-defined SubtableStrategy<F, C, M> (src/subtables/mod.rs:31-93):
    - tables: materialize_subtables(), num_subtables tables of M = 2^log_m entries, each either a 1-D array of integers
      below 2^32 or an (M, 4) uint64 array of Fr in Montgomery limbs (any field element; see fr_from_ints).  When any
      table is (M, 4) all of them are kept in that form (fr_tables) and the strategy is made by
      lasso_strategy_create_fr;
    - combine_lookups: a Python function of a list of num_memories values, written as the trait's method with + - *;
    - g_poly_degree: declared as in the trait; at least the degree of combine_lookups;
    - memory_to_subtable / memory_to_dimension: the trait's maps as lists (default i % num_subtables and
      i // num_subtables over num_memories = C * num_subtables memories).
    With ctx=None only the host description is built (tracing and checks); otherwise it is uploaded to ctx's device."""

    def __init__(self, ctx, C_, log_m, tables, combine_lookups, g_poly_degree, memory_to_subtable=None,
                 memory_to_dimension=None):
        self.C, self.log_m, self.g_poly_degree = int(C_), int(log_m), int(g_poly_degree)
        self.tables = []
        raw = [np.asarray(t) for t in tables]
        self.fr_tables = any(t.ndim == 2 for t in raw)
        for t in raw:
            if t.ndim == 2:
                if t.shape != (1 << self.log_m, 4) or t.dtype != np.uint64:
                    raise LassoError(LASSO_ERR_STRATEGY, "a field-element table is a (2^log_m, 4) uint64 array")
                if not _is_canonical(t).all():
                    raise LassoError(LASSO_ERR_STRATEGY, "a table entry is not a canonical Montgomery residue")
                self.tables.append(np.ascontiguousarray(t))
                continue
            if t.shape != (1 << self.log_m,):
                raise LassoError(LASSO_ERR_STRATEGY, "every table needs 2^log_m entries")
            if t.size and (int(t.min()) < 0 or int(t.max()) >= 1 << 32):
                raise LassoError(LASSO_ERR_STRATEGY, "table entries must be integers in [0, 2^32)")
            t = np.ascontiguousarray(t, dtype=np.uint32)
            self.tables.append(fr_from_ints(t.tolist()) if self.fr_tables else t)
        nsub = len(self.tables)
        if memory_to_subtable is None and memory_to_dimension is None:
            alpha = self.C * nsub
            memory_to_subtable = [i % nsub for i in range(alpha)]
            memory_to_dimension = [i // nsub for i in range(alpha)]
        if memory_to_subtable is None or memory_to_dimension is None or len(memory_to_subtable) != len(memory_to_dimension):
            raise LassoError(LASSO_ERR_STRATEGY, "memory_to_subtable and memory_to_dimension need the same length")
        self.memory_to_subtable = np.ascontiguousarray(memory_to_subtable, dtype=np.int32)
        self.memory_to_dimension = np.ascontiguousarray(memory_to_dimension, dtype=np.int32)
        if not 1 <= self.num_memories <= MAX_MEMORIES:
            raise LassoError(LASSO_ERR_STRATEGY, "num_memories must be in 1..16")
        self.program, self.constants, self.degree = trace_combine_lookups(combine_lookups, self.num_memories)
        if self.g_poly_degree < self.degree:
            raise LassoError(LASSO_ERR_STRATEGY, "declared g_poly_degree %d is below the degree %d of combine_lookups"
                             % (self.g_poly_degree, self.degree))
        self.ctx, self._h = ctx, None
        if ctx is not None:
            h = C.c_void_p()
            create = lib().lasso_strategy_create_fr if self.fr_tables else lib().lasso_strategy_create
            _chk(create(
                ctx._h, self.C, self.log_m, nsub, _ptr_array(self.tables), self.num_memories, _p(self.memory_to_subtable),
                _p(self.memory_to_dimension), _p(self.program), int(self.program.shape[0]), _p(self.constants),
                int(self.constants.shape[0]), self.g_poly_degree, C.byref(h)))
            self._h = h

    @property
    def num_subtables(self):
        return len(self.tables)

    @property
    def num_memories(self):
        return int(self.memory_to_subtable.shape[0])

    @property
    def sumcheck_poly_degree(self):
        return self.g_poly_degree + 1

    def close(self):
        if self._h:
            lib().lasso_strategy_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                self.close()
        except Exception:
            pass


class Context:
    """One per GPU: device, stream, memory pool, scratch."""

    def __init__(self, device=0):
        h = C.c_void_p()
        _chk(lib().lasso_ctx_create(C.byref(h), int(device)))
        self._h = h
        self._scratch = {}

    def _buf(self, name, shape, dtype):
        """Output staging reused across calls (a fresh 4 MiB np.zeros per commit / prove is an mmap + page faults +
        munmap inside the caller's timed region); contents are overwritten by the library before they are read."""
        b = self._scratch.get(name)
        if b is None or b.shape != tuple(np.atleast_1d(shape)) or b.dtype != np.dtype(dtype):
            b = np.zeros(shape, dtype=dtype)
            self._scratch[name] = b
        return b

    def close(self):
        if self._h:
            lib().lasso_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def init_comm(self, rank=None, world=None):
        """Shard ONE proof over the ranks of a torch.distributed job (one process per GPU, world a power of two
        <= 8, one node).  The 128-byte job id (random bytes naming the job's shared host segments, or the NCCL
        unique id under LASSO_B200_XCHG=nccl) is created on rank 0 and broadcast through torch.distributed
        (any backend).  Collective: every rank must call it."""
        import torch.distributed as dist

        from . import parallel

        rank = dist.get_rank() if rank is None else rank
        world = dist.get_world_size() if world is None else world
        ident = np.zeros(128, dtype=np.uint8)
        if rank == 0:
            _chk(lib().lasso_comm_unique_id(_p(ident)))
        ident = np.frombuffer(parallel.broadcast_bytes(ident.tobytes(), src=0), dtype=np.uint8).copy()
        _chk(lib().lasso_ctx_init_comm(self._h, _p(ident), int(rank), int(world)))
        self.rank, self.world = rank, world

    def bind_host_threads(self):
        """One process per GPU: pin the CALLING thread (the one that proves and spins on the round messages) to a
        dedicated core of the GPU's NUMA node and give the library's helper threads the rest of the node; returns the
        node id or -1 when the topology is not exposed.  Threads created earlier keep their affinity."""
        return int(lib().lasso_ctx_bind_host_threads(self._h))

    @property
    def launches(self):
        return int(lib().lasso_launch_count(self._h))

    def last_timings_ms(self):
        t = (C.c_double * 3)()
        lib().lasso_last_timings(self._h, t)
        return dict(densify=t[0], commit=t[1], prove=t[2])

    def spans(self):
        buf = C.create_string_buffer(8192)
        lib().lasso_spans(self._h, buf, C.c_size_t(8192))
        return dict((kv.split("=")[0], float(kv.split("=")[1])) for kv in buf.value.decode().split(";") if kv)

    def bench_bind(self, length, npolys, iters):
        ms = C.c_double(0)
        _chk(lib().lasso_bench_bind(self._h, C.c_size_t(length), int(npolys), int(iters), C.byref(ms)))
        return ms.value


# ------------------------------------------------------------------ per-loop entry points
def bind_top(ctx, Z, r):
    Z = _fr(Z).copy()
    _chk(lib().lasso_bind_top(ctx._h, _p(Z), C.c_size_t(Z.shape[0]), _p(_fr(r))))
    return Z[: Z.shape[0] // 2]


def bind_bot(ctx, Z, r):
    Z = _fr(Z).copy()
    _chk(lib().lasso_bind_bot(ctx._h, _p(Z), C.c_size_t(Z.shape[0]), _p(_fr(r))))
    return Z[: Z.shape[0] // 2]


def eq_evals(ctx, r):
    r = _fr(r).reshape(-1, 4)
    out = np.zeros((1 << r.shape[0], 4), dtype=np.uint64)
    _chk(lib().lasso_eq_evals(ctx._h, _p(r), int(r.shape[0]), _p(out)))
    return out


def sumcheck_round_arbitrary(ctx, S, polys):
    polys = [_fr(p) for p in polys]
    out = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
    _chk(lib().lasso_sumcheck_round_arbitrary(ctx._h, S.kind, S.C, S.log_m, S.log_r, _ptr_array(polys),
                                              C.c_size_t(polys[0].shape[0]), _p(out)))
    return out


def sumcheck_round_custom(ctx, S, polys):
    """sumcheck_round_arbitrary for a CustomStrategy: g_poly_degree + 2 evaluations."""
    polys = [_fr(p) for p in polys]
    out = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
    _chk(lib().lasso_sumcheck_round_custom(ctx._h, S._h, _ptr_array(polys), C.c_size_t(polys[0].shape[0]), _p(out)))
    return out


def sumcheck_bind_round_arbitrary(ctx, S, polys, r):
    """Bind every polynomial's top variable to r, then evaluate the next round: (bound polys, evals)."""
    polys = [_fr(p).copy() for p in polys]
    out = np.zeros((S.sumcheck_poly_degree + 1, 4), dtype=np.uint64)
    n = polys[0].shape[0]
    _chk(lib().lasso_sumcheck_bind_round_arbitrary(ctx._h, S.kind, S.C, S.log_m, S.log_r, _ptr_array(polys),
                                                   C.c_size_t(n), _p(_fr(r)), _p(out)))
    return [p[: n // 2] for p in polys], out


def sumcheck_round_cubic(ctx, A, B, Ceq):
    A = [_fr(a) for a in A]
    B = [_fr(b) for b in B]
    Ceq = _fr(Ceq)
    out = np.zeros((len(A), 3, 4), dtype=np.uint64)
    _chk(lib().lasso_sumcheck_round_cubic(ctx._h, len(A), _ptr_array(A), _ptr_array(B), _p(Ceq),
                                          C.c_size_t(Ceq.shape[0]), _p(out)))
    return out


def materialize_subtables(ctx, S):
    tabs = [np.zeros((1 << S.log_m, 4), dtype=np.uint64) for _ in range(S.num_subtables)]
    _chk(lib().lasso_materialize_subtables(ctx._h, S.kind, S.C, S.log_m, S.log_r, _ptr_array(tabs)))
    return tabs


def gather_lookup_polys(ctx, S, nz):
    nz = [np.ascontiguousarray(d, dtype=np.uint64) for d in nz]
    s = nz[0].shape[0]
    E = [np.zeros((s, 4), dtype=np.uint64) for _ in range(S.num_memories)]
    _chk(lib().lasso_gather_lookup_polys(ctx._h, S.kind, S.C, S.log_m, S.log_r, _ptr_array(nz), C.c_size_t(s),
                                         _ptr_array(E)))
    return E


def msm(ctx, bases_affine, scalars):
    bases = _fr(bases_affine, 8)
    sc = _fr(scalars)
    if bases.shape[0] != sc.shape[0]:  # VariableBaseMSM::msm -> Err(min_len), msm/mod.rs:36-40
        raise LassoError(1, "msm: bases.len() != scalars.len() (min = %d)" % min(bases.shape[0], sc.shape[0]))
    out = np.zeros(16, dtype=np.uint64)
    _chk(lib().lasso_msm(ctx._h, _p(bases), _p(sc), C.c_size_t(sc.shape[0]), _p(out)))
    return out


class MsmJob:
    """One VariableBaseMSM (msm/mod.rs:36-40) on device-resident inputs: n terms, term i uses base i % len(bases)."""

    def __init__(self, ctx, bases_affine, scalars):
        bases = _fr(bases_affine, 8)
        sc = _fr(scalars)
        h = C.c_void_p()
        _chk(lib().lasso_msm_job_create(ctx._h, _p(bases), C.c_size_t(bases.shape[0]), _p(sc), C.c_size_t(sc.shape[0]),
                                        C.byref(h)))
        self.ctx, self._h, self.n = ctx, h, sc.shape[0]

    def run(self, iters=1):
        """-> (extended point (16 u64), average ms per MSM, info dict)"""
        out = np.zeros(16, dtype=np.uint64)
        ms = C.c_double(0)
        info = (C.c_int * 8)()
        _chk(lib().lasso_msm_job_run(self.ctx._h, self._h, int(iters), C.byref(ms), _p(out), info))
        return out, ms.value, dict(c=info[0], windows=info[1], scalar_bits=info[2], unit=info[3], L=info[4], T2=info[5],
                                   world=info[6])

    def naive(self):
        out = np.zeros(16, dtype=np.uint64)
        _chk(lib().lasso_msm_job_naive(self.ctx._h, self._h, _p(out)))
        return out

    def close(self):
        if self._h:
            lib().lasso_msm_job_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            if self.ctx._h:
                self.close()
        except Exception:
            pass


def commit_rows(ctx, gens_affine, Z, L_size, R_size):
    g = _fr(gens_affine, 8)
    Z = _fr(Z)
    assert g.shape[0] >= R_size and Z.shape[0] == L_size * R_size
    out = np.zeros((L_size, 16), dtype=np.uint64)
    _chk(lib().lasso_commit_rows(ctx._h, _p(g), _p(Z), C.c_size_t(L_size), C.c_size_t(R_size), _p(out)))
    return out


def gens_points_needed(c, s, num_memories, log_m):
    return int(lib().lasso_gens_points_needed(c, s, num_memories, log_m))


def sample_generators(label, count):
    out = np.zeros((count, 8), dtype=np.uint64)
    _chk(lib().lasso_sample_generators(label, C.c_size_t(count), _p(out)))
    return out


# ------------------------------------------------------------------ the reference-shaped surface
class SparsePolyCommitmentGens:
    """src/lasso/surge.rs:25-58"""

    def __init__(self, ctx, handle, stream):
        self.ctx, self._h, self.stream = ctx, handle, stream

    @classmethod
    def new(cls, ctx, label, c, s, num_memories, log_m, stream=None):
        need = gens_points_needed(c, s, num_memories, log_m)
        if stream is None:
            stream = sample_generators(label, need)
        stream = _fr(stream, 8)
        h = C.c_void_p()
        _chk(lib().lasso_gens_create(ctx._h, _p(stream), C.c_size_t(stream.shape[0]), C.c_size_t(c), C.c_size_t(s),
                                     C.c_size_t(num_memories), C.c_size_t(log_m), C.byref(h)))
        return cls(ctx, h, stream)

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                lib().lasso_gens_destroy(self._h)
        except Exception:
            pass


class DensifiedRepresentation:
    """src/lasso/densified.rs:8-96 (device resident)"""

    def __init__(self, ctx, handle, C_, log_m):
        self.ctx, self._h, self.C, self.log_m = ctx, handle, C_, log_m
        self.s = int(lib().lasso_dense_s(handle))
        self.m = 1 << log_m

    @classmethod
    def from_lookup_indices(cls, ctx, indices, log_m):
        """indices: n x C lookup indices.  A numpy array (or anything numpy converts, CPU tensors included) is narrowed
        on the host and uploaded (lasso_densify).  A torch CUDA tensor of dtype int64 or int32 stays where it is
        (lasso_densify_device): any strides, read in the order of torch's current stream of its device; its entries are
        read as unsigned integers, so a negative one is out of range (LassoError code 3)."""
        torch = sys.modules.get("torch")  # a CUDA tensor exists only if torch is loaded already
        if torch is not None and isinstance(indices, torch.Tensor) and indices.is_cuda:
            return cls._from_device_tensor(ctx, indices, log_m, torch)
        idx = np.ascontiguousarray(indices, dtype=np.uint64)
        assert idx.ndim == 2
        h = C.c_void_p()
        _chk(lib().lasso_densify(ctx._h, _p(idx), C.c_size_t(idx.shape[0]), C.c_size_t(idx.shape[1]),
                                 C.c_size_t(log_m), C.byref(h)))
        return cls(ctx, h, idx.shape[1], log_m)

    @classmethod
    def _from_device_tensor(cls, ctx, t, log_m, torch):
        if t.dtype not in (torch.int64, torch.int32):
            raise LassoError(LASSO_ERR_STRATEGY, "CUDA lookup indices must be int64 or int32, not %s" % t.dtype)
        if t.ndim != 2:
            raise LassoError(LASSO_ERR_STRATEGY, "CUDA lookup indices must be an n x C matrix, not %d-dimensional" % t.ndim)
        n, c = t.shape
        row_stride, col_stride = t.stride()
        stream = torch.cuda.current_stream(t.device).cuda_stream
        h = C.c_void_p()
        _chk(lib().lasso_densify_device(ctx._h, C.c_void_p(t.data_ptr()), C.c_size_t(t.element_size()), C.c_size_t(n),
                                        C.c_size_t(c), C.c_size_t(row_stride), C.c_size_t(col_stride), C.c_size_t(log_m),
                                        C.c_void_p(stream), C.byref(h)))
        return cls(ctx, h, c, log_m)

    def _read(self, which, n, width):
        out = np.zeros((n, width) if width > 1 else (n,), dtype=np.uint64)
        got = lib().lasso_dense_read(self.ctx._h, self._h, which, _p(out), C.c_size_t(n))
        assert got == n, (got, n)
        return out

    @property
    def dim_usize(self):
        return self._read(0, self.C * self.s, 1).reshape(self.C, self.s)

    @property
    def dim(self):
        return self._read(1, self.C * self.s, 4).reshape(self.C, self.s, 4)

    @property
    def read(self):
        return self._read(2, self.C * self.s, 4).reshape(self.C, self.s, 4)

    @property
    def final(self):
        return self._read(3, self.C * self.m, 4).reshape(self.C, self.m, 4)

    def commit(self, gens):
        cap = 1 << 22
        out = self.ctx._buf("commitment", cap, np.uint8)
        n = C.c_size_t(0)
        _chk(lib().lasso_commit(self.ctx._h, self._h, gens._h, _p(out), C.c_size_t(cap), C.byref(n)))
        return bytes(out[: n.value])

    def _poly(self, which, j):
        h = C.c_void_p()
        _chk(lib().lasso_dense_poly(self.ctx._h, self._h, which, C.c_size_t(int(j)), C.byref(h)))
        return DensePolynomial._wrap(self.ctx, h)

    def dim_poly(self, j):
        """dim_j (src/lasso/densified.rs:8-18) as a DensePolynomial of its own on ctx's GPU: the same values as
        .dim[j], integer-valued (the u32 mirror).  Single GPU."""
        return self._poly(1, j)

    def read_poly(self, j):
        """read_j, as dim_poly"""
        return self._poly(2, j)

    def final_poly(self, j):
        """final_j (m evaluations), as dim_poly"""
        return self._poly(3, j)

    def outputs(self, strategy):
        """The lookup outputs v[k] = combine_lookups(E_0[k], ..) for k < s (padded lookups included) as a
        DensePolynomial of log2(s) variables on the context's GPU.  Its MLE at r is the claimed evaluation of a proof
        at r: commit to v and open it there to tie the proof to the caller's commitments."""
        h = C.c_void_p()
        if isinstance(strategy, CustomStrategy):
            if strategy._h is None:
                raise LassoError(LASSO_ERR_STRATEGY, "the CustomStrategy was built without a context")
            _chk(lib().lasso_dense_outputs_custom(self.ctx._h, strategy._h, self._h, C.byref(h)))
        else:
            _chk(lib().lasso_dense_outputs(self.ctx._h, strategy.kind, strategy.log_r, self._h, C.byref(h)))
        return DensePolynomial._wrap(self.ctx, h)

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                lib().lasso_dense_destroy(self._h)
        except Exception:
            pass


class SparsePolynomialEvaluationProof:
    """src/lasso/surge.rs:92-211.  `.bytes` is the ark-serialize (compressed) encoding of the proof.  On the label path
    `.challenges` holds every challenge drawn; on a caller's transcript it is None and `.claimed_evaluation` holds the
    primary sumcheck's claim (4 limbs)."""

    def __init__(self, data, challenges, claimed_evaluation=None):
        self.bytes, self.challenges, self.claimed_evaluation = data, challenges, claimed_evaluation

    @classmethod
    def prove(cls, ctx, strategy, dense, r, gens, transcript_label=None, tape_label=None, tape_seed=None,
              transcript=None, random_tape=None):
        """Without transcript / random_tape: on Transcript::new(transcript_label or b"example") and a tape
        RandomTape::new(tape_label or b"proof") seeded with tape_seed (zero by default).  With both: on the caller's
        Transcript and RandomTape, advanced in place; no label or seed may then be given."""
        if transcript is not None or random_tape is not None:
            if transcript is None or random_tape is None:
                raise LassoError(LASSO_ERR_LENGTH, "pass both a transcript and a random_tape, or neither")
            if transcript_label is not None or tape_label is not None or tape_seed is not None:
                raise LassoError(LASSO_ERR_LENGTH, "labels and tape_seed belong to the label path, not to a caller's "
                                                   "transcript and random_tape")
            r = _limbs(r, what="r") if len(r) else np.zeros((0, 4), dtype=np.uint64)
            claim = np.zeros(4, dtype=np.uint64)
            data = cls._call(ctx, strategy, True, dense, r, gens, (transcript._h, random_tape._h), (_p(claim),))
            return cls(data, None, claim)
        transcript_label = b"example" if transcript_label is None else transcript_label
        tape_label = b"proof" if tape_label is None else tape_label
        r = _fr(r).reshape(-1, 4)
        seed = _fr(tape_seed if tape_seed is not None else np.zeros(4, dtype=np.uint64))
        chal = ctx._buf("challenges", (1 << 14, 4), np.uint64)
        nch = C.c_size_t(0)
        data = cls._call(ctx, strategy, False, dense, r, gens, (transcript_label, tape_label, _p(seed)),
                         (_p(chal), C.c_size_t(chal.shape[0]), C.byref(nch)))
        return cls(data, chal[: nch.value].copy())

    @staticmethod
    def _call(ctx, strategy, on_transcript, dense, r, gens, inputs, outputs):
        """lasso_prove[_custom][_transcript] into ctx's proof buffer -> the proof bytes.  inputs: the transcript's
        arguments, between the generators and the proof buffer; outputs: the arguments after proof_len."""
        L = lib()
        if isinstance(strategy, CustomStrategy):
            if strategy._h is None:
                raise LassoError(LASSO_ERR_STRATEGY, "the CustomStrategy was built without a context")
            fn, head = (L.lasso_prove_custom_transcript if on_transcript else L.lasso_prove_custom), (strategy._h,)
        else:
            fn, head = (L.lasso_prove_transcript if on_transcript else L.lasso_prove), (strategy.kind, strategy.log_r)
        cap = 1 << 22
        out = ctx._buf("proof", cap, np.uint8)
        n = C.c_size_t(0)
        _chk(fn(ctx._h, *head, dense._h, _p(r), C.c_size_t(r.shape[0]), gens._h, *inputs, _p(out), C.c_size_t(cap),
                C.byref(n), *outputs))
        return bytes(out[: n.value])


# ------------------------------------------------------------------ dense polynomials on a caller's transcript
def _label(label):
    """a transcript label: bytes (or str) without a NUL byte"""
    if isinstance(label, str):
        label = label.encode()
    if not isinstance(label, (bytes, bytearray)) or b"\0" in label:
        raise LassoError(LASSO_ERR_LENGTH, "a label is bytes without a NUL byte, not %r" % (label,))
    return bytes(label)


def _limbs(a, n=None, what="scalars"):
    """Fr elements as (k, 4) uint64 Montgomery limbs (k = n when given)"""
    a = np.asarray(a)
    if a.dtype != np.uint64 or a.ndim == 0 or a.shape[-1] != 4:
        raise LassoError(LASSO_ERR_LENGTH, "%s are uint64 Montgomery limbs of shape (..., 4)" % what)
    a = np.ascontiguousarray(a).reshape(-1, 4)
    if n is not None and a.shape[0] != n:
        raise LassoError(LASSO_ERR_LENGTH, "%s: %d elements, expected %d" % (what, a.shape[0], n))
    return a


def _compressed(points):
    """32-byte compressed points: one bytes object of 32 k bytes, or a sequence of 32-byte objects"""
    b = bytes(points) if isinstance(points, (bytes, bytearray, memoryview)) else b"".join(bytes(p) for p in points)
    if len(b) % 32:
        raise LassoError(LASSO_ERR_LENGTH, "compressed points are 32 bytes each, got %d bytes" % len(b))
    return b


class Transcript:
    """merlin Transcript with the reference's ProofTranscript methods (src/utils/transcript.rs:6-72).  A host object: no
    context or GPU needed.  Scalars are (4,) uint64 Montgomery limbs, points 32-byte compressed encodings."""

    def __init__(self, label):
        h = C.c_void_p()
        _chk(lib().lasso_transcript_create(_label(label), C.byref(h)))
        self._h = h

    def append_message(self, label, msg):
        msg = bytes(msg)
        _chk(lib().lasso_transcript_append_message(self._h, _label(label), msg, C.c_size_t(len(msg))))

    def append_u64(self, label, x):
        _chk(lib().lasso_transcript_append_u64(self._h, _label(label), int(x)))

    def append_protocol_name(self, name):
        _chk(lib().lasso_transcript_append_protocol_name(self._h, _label(name)))

    def append_scalar(self, label, s):
        _chk(lib().lasso_transcript_append_scalar(self._h, _label(label), _p(_limbs(s, 1, "a scalar"))))

    def append_scalars(self, label, scalars):
        s = _limbs(scalars)
        _chk(lib().lasso_transcript_append_scalars(self._h, _label(label), _p(s), C.c_size_t(s.shape[0])))

    def append_point(self, label, point):
        b = _compressed(point)
        if len(b) != 32:
            raise LassoError(LASSO_ERR_LENGTH, "a point is 32 bytes")
        _chk(lib().lasso_transcript_append_point(self._h, _label(label), b))

    def append_points(self, label, points):
        b = _compressed(points)
        _chk(lib().lasso_transcript_append_points(self._h, _label(label), b, C.c_size_t(len(b) // 32)))

    def append_poly_commitment(self, label, commitment):
        """PolyCommitment::append_to_transcript (src/poly/dense_mlpoly.rs:281-289) of DensePolynomial.commit's bytes"""
        b = bytes(commitment)
        _chk(lib().lasso_transcript_append_poly_commitment(self._h, _label(label), b, C.c_size_t(len(b))))

    def append_sparse_commitment(self, commitment):
        """SparsePolynomialCommitment::append_to_transcript (src/lasso/surge.rs:70-82) of
        DensifiedRepresentation.commit's bytes"""
        b = bytes(commitment)
        _chk(lib().lasso_transcript_append_sparse_commitment(self._h, b, C.c_size_t(len(b))))

    def append_combined_table_commitment(self, commitment, label=b"comm_poly_row_col_ops_val"):
        """CombinedTableCommitment::append_to_transcript (src/subtables/mod.rs:382-393) of PolyCommitment bytes
        (Subtables.commit, DensePolynomial.commit); label is the one surge.rs:139 passes"""
        b = bytes(commitment)
        _chk(lib().lasso_transcript_append_combined_table_commitment(self._h, _label(label), b, C.c_size_t(len(b))))

    def challenge_scalar(self, label):
        out = np.zeros(4, dtype=np.uint64)
        _chk(lib().lasso_transcript_challenge_scalar(self._h, _label(label), _p(out)))
        return out

    def challenge_vector(self, label, n):
        out = np.zeros((int(n), 4), dtype=np.uint64)
        _chk(lib().lasso_transcript_challenge_vector(self._h, _label(label), C.c_size_t(int(n)), _p(out)))
        return out

    def __del__(self):
        try:
            if self._h:
                lib().lasso_transcript_destroy(self._h)
                self._h = None
        except Exception:
            pass


class RandomTape:
    """RandomTape::new(label) (src/utils/random.rs:15-30) seeded with an explicit scalar instead of test_rng()."""

    def __init__(self, label, seed):
        h = C.c_void_p()
        _chk(lib().lasso_random_tape_create(_label(label), _p(_limbs(seed, 1, "the seed")), C.byref(h)))
        self._h = h

    def random_scalar(self, label):
        out = np.zeros(4, dtype=np.uint64)
        _chk(lib().lasso_random_tape_random_scalar(self._h, _label(label), _p(out)))
        return out

    def random_vector(self, label, n):
        out = np.zeros((int(n), 4), dtype=np.uint64)
        _chk(lib().lasso_random_tape_random_vector(self._h, _label(label), C.c_size_t(int(n)), _p(out)))
        return out

    def __del__(self):
        try:
            if self._h:
                lib().lasso_random_tape_destroy(self._h)
                self._h = None
        except Exception:
            pass


def poly_gens_points_needed(num_vars):
    """R + 2 generators, R = 2^(num_vars - num_vars // 2)"""
    return int(lib().lasso_poly_gens_points_needed(C.c_size_t(int(num_vars))))


class PolyCommitmentGens:
    """src/poly/dense_mlpoly.rs:31-45: G_0..G_{R-1}, Q, h from one generator stream (collective on a sharded context,
    where R >= G)"""

    def __init__(self, ctx, handle, stream, num_vars):
        self.ctx, self._h, self.stream, self.num_vars = ctx, handle, stream, num_vars

    @classmethod
    def new(cls, ctx, label, num_vars, stream=None):
        if stream is None:
            stream = sample_generators(_label(label), poly_gens_points_needed(num_vars))
        stream = _fr(stream, 8)
        h = C.c_void_p()
        _chk(lib().lasso_poly_gens_create(ctx._h, _p(stream), C.c_size_t(stream.shape[0]), C.c_size_t(int(num_vars)),
                                          C.byref(h)))
        return cls(ctx, h, stream, int(num_vars))

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                lib().lasso_poly_gens_destroy(self._h)
        except Exception:
            pass


def _poly_source(Z):
    """-> ("host", contiguous (n, 4) uint64 array) or ("device", tensor, row stride); raises on anything else"""
    torch = sys.modules.get("torch")  # a CUDA tensor exists only if torch is loaded already
    if torch is not None and isinstance(Z, torch.Tensor) and Z.is_cuda:
        if Z.dtype not in (torch.int64, getattr(torch, "uint64", torch.int64)):
            raise LassoError(LASSO_ERR_LENGTH, "a CUDA polynomial is int64 or uint64 limbs, not %s" % Z.dtype)
        if Z.ndim != 2 or Z.shape[1] != 4:
            raise LassoError(LASSO_ERR_LENGTH, "a CUDA polynomial is an (n, 4) tensor of limbs, not %s" % (tuple(Z.shape),))
        if Z.stride(1) != 1:
            raise LassoError(LASSO_ERR_LENGTH, "the 4 limbs of an evaluation must be contiguous (stride 1)")
        return "device", Z, (Z.stride(0) if Z.shape[0] > 1 else 4)
    a = np.asarray(Z)
    if a.dtype == np.int64:
        a = a.view(np.uint64)
    if a.dtype != np.uint64 or a.ndim != 2 or a.shape[1] != 4:
        raise LassoError(LASSO_ERR_LENGTH, "a polynomial is an (n, 4) uint64 array of Montgomery limbs")
    return "host", np.ascontiguousarray(a), 4


def _handles(objs):
    """a C array of the handles `_h` of library objects (at least one slot)"""
    objs = list(objs)
    arr = (C.c_void_p * max(len(objs), 1))()
    for i, o in enumerate(objs):
        arr[i] = o._h.value
    return arr


_poly_handles = _handles  # the earlier name, still imported by callers that build their own lasso_poly arrays


def _poly_rows(ctx, Z, padded):
    """a new lasso_poly of Z, in the forms DensePolynomial takes: host rows, or a CUDA tensor read in the order of
    torch's current stream.  padded: new_padded, of any length."""
    kind, src, row_stride = _poly_source(Z)
    h = C.c_void_p()
    L = lib()
    if kind == "device":
        torch = sys.modules["torch"]
        stream = torch.cuda.current_stream(src.device).cuda_stream
        fn = L.lasso_poly_create_padded_device if padded else L.lasso_poly_create_device
        _chk(fn(ctx._h, C.c_void_p(src.data_ptr()), C.c_size_t(src.shape[0]), C.c_size_t(row_stride),
                C.c_void_p(stream), C.byref(h)))
    else:
        fn = L.lasso_poly_create_padded if padded else L.lasso_poly_create
        _chk(fn(ctx._h, _p(src), C.c_size_t(src.shape[0]), C.byref(h)))
    return h


class DensePolynomial:
    """DensePolynomial<Fr> (src/poly/dense_mlpoly.rs:13-235), resident on ctx's GPU.  Z: the 2^num_vars evaluations as
    an (n, 4) uint64 numpy array of Montgomery limbs, or a torch CUDA tensor (int64 or uint64, limbs contiguous, any row
    stride) read in the order of torch's current stream.  The library keeps its own copy.
    On a sharded context (Context.init_comm) creating, committing, evaluating and opening are collective: every rank
    passes the WHOLE polynomial (of the same kind, host or CUDA on its own GPU) and the same arguments, keeps only its
    low-bit shard, and gets the single-GPU bytes and values.  The same holds for prove_cubic_batched and for deriving and
    reading back polynomials (bound_top, bound_bot, split, new_padded, to_numpy, to_tensor, copy_to).  There a
    polynomial needs 2^(num_vars - num_vars // 2) >= G (LASSO_ERR_LENGTH otherwise); prove_arbitrary, grand products and
    DensifiedRepresentation.outputs stay single-GPU."""

    def __init__(self, ctx, Z):
        h = _poly_rows(ctx, Z, False)
        self.ctx, self._h = ctx, h
        self.num_vars = int(lib().lasso_poly_num_vars(h))

    @classmethod
    def _wrap(cls, ctx, h):
        self = cls.__new__(cls)
        self.ctx, self._h = ctx, h
        self.num_vars = int(lib().lasso_poly_num_vars(h))
        return self

    @classmethod
    def eq(cls, ctx, r):
        """EqPolynomial::new(r).evals() (src/poly/eq_poly.rs:21-38) on ctx's GPU, r[0] the most significant variable"""
        r = _limbs(r, what="r") if len(r) else np.zeros((0, 4), dtype=np.uint64)
        h = C.c_void_p()
        _chk(lib().lasso_poly_create_eq(ctx._h, _p(r), C.c_size_t(r.shape[0]), C.byref(h)))
        return cls._wrap(ctx, h)

    @classmethod
    def from_comb(cls, ctx, comb, polys):
        """Q(x) = comb(P_0(x), .., P_{k-1}(x)) at every point of the hypercube, on ctx's GPU (comb.degree is not used),
        e.g. the fingerprints t gamma^2 + v gamma + a - tau of offline memory checking"""
        polys = list(polys)
        h = C.c_void_p()
        _chk(lib().lasso_poly_create_comb(ctx._h, comb._h, _handles(polys), C.c_size_t(len(polys)), C.byref(h)))
        return cls._wrap(ctx, h)

    @classmethod
    def merge(cls, ctx, polys):
        """DensePolynomial::merge (src/poly/dense_mlpoly.rs:251-261): the evaluations of polys one after another,
        zero-padded to a power of two, as a new polynomial with its own copy (the inputs are unchanged and may be
        dropped).  Integer-valued iff every input is."""
        polys = list(polys)
        h = C.c_void_p()
        _chk(lib().lasso_poly_create_merge(ctx._h, _handles(polys), C.c_size_t(len(polys)), C.byref(h)))
        return cls._wrap(ctx, h)

    @staticmethod
    def evaluate_batch(ctx, polys, r):
        """P_j(r) for 1..64 DensePolynomials of one num_vars, over one eq table -> (n, 4) uint64 Montgomery limbs"""
        polys = list(polys)
        r = _limbs(r, what="r") if len(r) else np.zeros((0, 4), dtype=np.uint64)
        out = np.zeros((max(len(polys), 1), 4), dtype=np.uint64)
        _chk(lib().lasso_poly_evaluate_batch(ctx._h, _handles(polys), C.c_size_t(len(polys)), _p(r),
                                             C.c_size_t(r.shape[0]), _p(out)))
        return out[: len(polys)]

    def commit(self, gens):
        """DensePolynomial::commit without blinds -> the ark-serialize bytes of PolyCommitment"""
        cap = 8 + 32 * (1 << (self.num_vars // 2))
        out = np.zeros(cap, dtype=np.uint8)
        n = C.c_size_t(0)
        _chk(lib().lasso_poly_commit(self.ctx._h, self._h, gens._h, _p(out), C.c_size_t(cap), C.byref(n)))
        return bytes(out[: n.value])

    def commit_hiding(self, gens, random_tape):
        """DensePolynomial::commit with Some(random_tape): draws L = 2^(num_vars // 2) blinds as
        random_vector("poly_blinds", L) and commits row i with blind i on h -> (the ark-serialize bytes of
        PolyCommitment, the blinds as an (L, 4) uint64 array of Montgomery limbs).  Advances random_tape in place."""
        L = 1 << (self.num_vars // 2)
        out = np.zeros(8 + 32 * L, dtype=np.uint8)
        blinds = np.zeros((L, 4), dtype=np.uint64)
        n = C.c_size_t(0)
        _chk(lib().lasso_poly_commit_hiding(self.ctx._h, self._h, gens._h, random_tape._h, _p(out), C.c_size_t(out.shape[0]),
                                            C.byref(n), _p(blinds), C.c_size_t(L)))
        return bytes(out[: n.value]), blinds

    def evaluate(self, r):
        r = _limbs(r, what="r")
        out = np.zeros(4, dtype=np.uint64)
        _chk(lib().lasso_poly_evaluate(self.ctx._h, self._h, _p(r), C.c_size_t(r.shape[0]), _p(out)))
        return out

    @classmethod
    def new_padded(cls, ctx, Z):
        """DensePolynomial::new_padded (src/poly/dense_mlpoly.rs:75-87): Z of any length (the forms __init__ takes),
        zero-padded up to the next power of two; an empty Z gives the polynomial of one zero evaluation"""
        return cls._wrap(ctx, _poly_rows(ctx, Z, True))

    def _bound(self, fn, r):
        r = _limbs(np.asarray(r).reshape(-1, 4), what="r")
        h = C.c_void_p()
        _chk(fn(self.ctx._h, self._h, _p(r), C.c_size_t(r.shape[0]), C.byref(h)))
        return DensePolynomial._wrap(self.ctx, h)

    def bound_top(self, r):
        """bound_poly_var_top (dense_mlpoly.rs:209-216) with r[0], r[1], .. in turn, r a (k, 4) or (4,) array: a NEW
        polynomial P(r_0, .., r_{k-1}, x); self is unchanged (the reference binds in place)"""
        return self._bound(lib().lasso_poly_bind_top, r)

    def bound_bot(self, r):
        """bound_poly_var_bot (dense_mlpoly.rs:218-225) with r[0], r[1], .. in turn, r[0] binding the lowest variable:
        a NEW polynomial P(x, r_{k-1}, .., r_0); self is unchanged.  Callers of the reference that bind their challenges
        last first (subtables/mod.rs:256) pass r[::-1]."""
        return self._bound(lib().lasso_poly_bind_bot, r)

    def split(self, idx=None):
        """split(idx) (dense_mlpoly.rs:101-107) -> (Z[:idx], Z[idx:2 idx]) as new polynomials; idx a power of two with
        2 idx <= len, None for len / 2"""
        idx = (1 << self.num_vars) // 2 if idx is None else int(idx)
        lo, hi = C.c_void_p(), C.c_void_p()
        _chk(lib().lasso_poly_split(self.ctx._h, self._h, C.c_size_t(idx), C.byref(lo), C.byref(hi)))
        return DensePolynomial._wrap(self.ctx, lo), DensePolynomial._wrap(self.ctx, hi)

    def to_numpy(self):
        """the 2^num_vars evaluations as an (n, 4) uint64 array of Montgomery limbs (the layout __init__ takes)"""
        out = np.zeros((1 << self.num_vars, 4), dtype=np.uint64)
        _chk(lib().lasso_poly_read(self.ctx._h, self._h, _p(out), C.c_size_t(out.shape[0])))
        return out

    def copy_to(self, tensor):
        """writes the evaluations into an (n, 4) int64 / uint64 CUDA tensor on ctx's GPU (limbs contiguous, any row
        stride), in the order of torch's current stream; returns the tensor"""
        kind, dst, row_stride = _poly_source(tensor)
        if kind != "device":
            raise LassoError(LASSO_ERR_POINTER, "copy_to takes a CUDA tensor")
        if dst.shape[0] != 1 << self.num_vars:
            raise LassoError(LASSO_ERR_LENGTH, "copy_to: the tensor has %d rows, the polynomial %d evaluations"
                             % (dst.shape[0], 1 << self.num_vars))
        torch = sys.modules["torch"]
        stream = torch.cuda.current_stream(dst.device).cuda_stream
        _chk(lib().lasso_poly_read_device(self.ctx._h, self._h, C.c_void_p(dst.data_ptr()), C.c_size_t(row_stride),
                                          C.c_void_p(stream)))
        return tensor

    def to_tensor(self, device=None):
        """the evaluations as a new (n, 4) int64 CUDA tensor (default: torch's current device), written in the order
        of torch's current stream"""
        import torch

        t = torch.empty((1 << self.num_vars, 4), dtype=torch.int64, device=device if device is not None else "cuda")
        return self.copy_to(t)

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                lib().lasso_poly_destroy(self._h)
        except Exception:
            pass


class PolyEvalProof:
    """src/poly/dense_mlpoly.rs:291-359.  `.bytes` is the ark-serialize (compressed) PolyEvalProof, `.C_Zr` the 32-byte
    compressed C_Zr_prime that PolyEvalProof::prove returns alongside it."""

    def __init__(self, data, C_Zr):
        self.bytes, self.C_Zr = data, C_Zr

    @classmethod
    def prove(cls, ctx, poly, r, Zr, gens, transcript, random_tape, *, blinds=None, blind_Zr=None):
        """advances transcript and random_tape in place.  blinds: the (L, 4) row blinds commit_hiding returned (None:
        the commitment was not hiding); blind_Zr: the blind of C_Zr = Zr Q + blind_Zr h (None: zero).  Collective on a
        sharded context: every rank's transcript and tape in the same state, every rank gets the same proof."""
        r = _limbs(r, what="r")
        Zr = _limbs(Zr, 1, "Zr")
        cap = 2 * (8 + 32 * 32) + 4 * 32
        out = np.zeros(cap, dtype=np.uint8)
        czr = np.zeros(32, dtype=np.uint8)
        n = C.c_size_t(0)
        if blinds is None and blind_Zr is None:
            _chk(lib().lasso_poly_eval_prove(ctx._h, poly._h, gens._h, _p(r), C.c_size_t(r.shape[0]), _p(Zr), transcript._h,
                                             random_tape._h, _p(out), C.c_size_t(cap), C.byref(n), _p(czr)))
        else:
            bl = None if blinds is None else _limbs(blinds, what="blinds")
            bz = None if blind_Zr is None else _limbs(blind_Zr, 1, "blind_Zr")
            _chk(lib().lasso_poly_eval_prove_hiding(
                ctx._h, poly._h, gens._h, None if bl is None else _p(bl), C.c_size_t(0 if bl is None else bl.shape[0]),
                _p(r), C.c_size_t(r.shape[0]), _p(Zr), None if bz is None else _p(bz), transcript._h, random_tape._h,
                _p(out), C.c_size_t(cap), C.byref(n), _p(czr)))
        return cls(bytes(out[: n.value]), czr.tobytes())


class CombinedTableEvalProof:
    """src/subtables/mod.rs:225-375 without blinds: n claims P_i(r) about the blocks of one merged polynomial
    (DensePolynomial.merge) opened with one PolyEvalProof.  `.data` is the ark-serialize (compressed) proof."""

    def __init__(self, data):
        self.data = data

    @staticmethod
    def proof_len(num_vars):
        """the serialised size for a merged polynomial of num_vars variables (that of its PolyEvalProof)"""
        lg = num_vars - num_vars // 2
        return 2 * (8 + 32 * lg) + 4 * 32

    @classmethod
    def prove(cls, ctx, combined, evals, r, gens, transcript, random_tape):
        """CombinedTableEvalProof::prove over `combined` for the claims `evals` at r (combined.num_vars == len(r) +
        log2(next_pow2(len(evals)))), on the caller's transcript and tape, advanced in place.  The claims are not checked:
        a wrong one gives a proof the verifier rejects.  Collective on a sharded context, like PolyEvalProof.prove."""
        evals = _limbs(evals, what="evals")
        r = _limbs(r, what="r") if len(r) else np.zeros((0, 4), dtype=np.uint64)
        cap = cls.proof_len(combined.num_vars)
        out = np.zeros(cap, dtype=np.uint8)
        n = C.c_size_t(0)
        _chk(lib().lasso_combined_eval_prove(ctx._h, combined._h, gens._h, _p(evals), C.c_size_t(evals.shape[0]), _p(r),
                                             C.c_size_t(r.shape[0]), transcript._h, random_tape._h, _p(out),
                                             C.c_size_t(cap), C.byref(n)))
        return cls(bytes(out[: n.value]))


# ------------------------------------------------------------------ sumchecks over a caller's polynomials
class Comb:
    """A combining function g(x_0, .., x_{n_inputs-1}) of SumcheckInstanceProof.prove_arbitrary
    (src/subprotocols/sumcheck.rs:149-260): fn(vals), vals a list of n_inputs values, written with + - * and Python
    integers (constants mod l), traced into the program of lasso_comb_create.  degree = combined_degree, the number of
    evaluation points minus one; None means the traced degree.  A host object: no context or GPU needed."""

    def __init__(self, fn, n_inputs, degree=None):
        program, constants, traced = trace_combine_lookups(fn, int(n_inputs))
        self._create(program, constants, int(n_inputs), traced if degree is None else int(degree))
        self.traced_degree = traced

    @classmethod
    def from_program(cls, program, constants, n_inputs, degree):
        """the program format of lasso_comb_create as it is: (n, 3) int32 {op, a, b}, (k, 4) uint64 Montgomery constants"""
        self = cls.__new__(cls)
        program = np.ascontiguousarray(program, dtype=np.int32).reshape(-1, 3)
        constants = np.ascontiguousarray(constants, dtype=np.uint64).reshape(-1, 4)
        self._create(program, constants, int(n_inputs), int(degree))
        self.traced_degree = None
        return self

    def _create(self, program, constants, n_inputs, degree):
        self._h = None
        self.program, self.constants, self.n_inputs, self.degree = program, constants, n_inputs, degree
        h = C.c_void_p()
        _chk(lib().lasso_comb_create(n_inputs, _p(program), int(program.shape[0]), _p(constants) if constants.size else None,
                                     int(constants.shape[0]), degree, C.byref(h)))
        self._h = h

    def __del__(self):
        try:
            if self._h:
                lib().lasso_comb_destroy(self._h)
                self._h = None
        except Exception:
            pass


class SumcheckInstanceProof:
    """src/subprotocols/sumcheck.rs:12-328.  `.bytes` is the ark-serialize (compressed) proof, `.r` the challenges,
    `.final_evals` the value of every polynomial at r after the binds, `.claim` the sum over the hypercube."""

    def __init__(self, data, r, final_evals, claim):
        self.bytes, self.r, self.final_evals, self.claim = data, r, final_evals, claim

    @classmethod
    def prove_arbitrary(cls, ctx, polys, comb, transcript, num_rounds=None):
        """prove_arbitrary over DensePolynomials of ctx (all of one num_vars; the same one may appear several times) on
        the caller's transcript, advanced in place.  The polynomials are not modified.  num_rounds=None: num_vars."""
        polys = list(polys)
        if num_rounds is None:
            num_rounds = polys[0].num_vars if polys else 0
        num_rounds = int(num_rounds)
        cap = 8 + max(num_rounds, 0) * (8 + 32 * comb.degree)
        out = np.zeros(cap, dtype=np.uint8)
        r = np.zeros((max(num_rounds, 1), 4), dtype=np.uint64)
        fin = np.zeros((max(len(polys), 1), 4), dtype=np.uint64)
        claim = np.zeros(4, dtype=np.uint64)
        n = C.c_size_t(0)
        _chk(lib().lasso_sumcheck_prove(ctx._h, comb._h, _handles(polys), C.c_size_t(len(polys)),
                                        C.c_size_t(num_rounds), transcript._h, _p(out), C.c_size_t(cap), C.byref(n), _p(r),
                                        _p(fin), _p(claim)))
        return cls(bytes(out[: n.value]), r[:num_rounds], fin[: len(polys)], claim)

    @classmethod
    def prove_cubic_batched(cls, ctx, A, B, C_poly, coeffs, claim, transcript, num_rounds=None):
        """prove_cubic_batched of claim = sum_x C(x) sum_k coeffs[k] A[k](x) B[k](x) over 1..32 pairs of DensePolynomials
        of ctx and C_poly, all of one num_vars, on the caller's transcript, advanced in place; the claim is not checked.
        The polynomials are not modified, and the same one may appear several times.  num_rounds=None: num_vars.
        `.final_evals` is (2n + 1, 4): A_0.., B_0.., C at (r || 0..0); `.claim` is the caller's claim.  Collective on a
        sharded context."""
        A, B = list(A), list(B)
        if len(A) != len(B):
            raise LassoError(LASSO_ERR_STRATEGY, "prove_cubic_batched: %d A polynomials and %d B" % (len(A), len(B)))
        n = len(A)
        if num_rounds is None:
            num_rounds = C_poly.num_vars
        num_rounds = int(num_rounds)
        coeffs = _limbs(coeffs, n, what="coeffs") if n else np.zeros((1, 4), dtype=np.uint64)
        claim = _limbs(claim, 1, what="claim")
        cap = 8 + max(num_rounds, 0) * 104
        out = np.zeros(cap, dtype=np.uint8)
        r = np.zeros((max(num_rounds, 1), 4), dtype=np.uint64)
        fin = np.zeros((2 * n + 1, 4), dtype=np.uint64)
        ln = C.c_size_t(0)
        _chk(lib().lasso_sumcheck_prove_cubic_batched(
            ctx._h, _handles(A), _handles(B), C.c_size_t(n), C_poly._h, _p(coeffs), _p(claim),
            C.c_size_t(num_rounds), transcript._h, _p(out), C.c_size_t(cap), C.byref(ln), _p(r), _p(fin[:n] if n else fin),
            _p(fin[n:2 * n] if n else fin), _p(fin[2 * n:])))
        return cls(bytes(out[: ln.value]), r[:num_rounds], fin, claim.reshape(4).copy())


# ------------------------------------------------------------------ zero-knowledge sumchecks
class MultiCommitGens:
    """src/poly/commitments.rs:14-70: n points G and h (64-byte affine, (n, 8) and (8,) uint64), 1 <= n <= 1024, on
    ctx's GPU with the digit-multiples table of all n + 1 points.  Usable on a sharded context: no exchange."""

    def __init__(self, ctx, G, h):
        G, h = _fr(G, 8).reshape(-1, 8), _fr(h, 8).reshape(8)
        self._h = None
        hd = C.c_void_p()
        _chk(lib().lasso_mc_gens_create(ctx._h, _p(G), C.c_size_t(G.shape[0]), _p(h), C.byref(hd)))
        self.ctx, self._h, self.G, self.h, self.n = ctx, hd, G, h, G.shape[0]

    @classmethod
    def new(cls, ctx, n, label):
        """MultiCommitGens::new(n, label) (commitments.rs:22-44): G = the first n points of the label's stream, h the
        next"""
        s = sample_generators(_label(label), int(n) + 1)
        return cls(ctx, s[:n], s[n])

    def commit(self, scalars, blind):
        """Commitments::batch_commit (commitments.rs:84-93), commit when n == 1: <scalars, G> + blind h, 32 bytes
        compressed"""
        s = _limbs(scalars, self.n, "scalars")
        b = _limbs(blind, 1, "the blind")
        out = np.zeros(32, dtype=np.uint8)
        _chk(lib().lasso_mc_commit(self.ctx._h, self._h, _p(s), C.c_size_t(self.n), _p(b), _p(out)))
        return out.tobytes()

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                lib().lasso_mc_gens_destroy(self._h)
                self._h = None
        except Exception:
            pass


class DotProductProofGens:
    """src/subprotocols/dot_product.rs:138-150: MultiCommitGens::new(n + 1, label).split_at(n), i.e. gens_n =
    (s[0..n), s[n+1]) and gens_1 = ([s[n]], s[n+1]) of the label's stream s"""

    def __init__(self, n, gens_n, gens_1):
        self.n, self.gens_n, self.gens_1 = n, gens_n, gens_1

    @classmethod
    def new(cls, ctx, n, label):
        n = int(n)
        s = sample_generators(_label(label), n + 2)
        return cls(n, MultiCommitGens(ctx, s[:n], s[n + 1]), MultiCommitGens(ctx, s[n:n + 1], s[n + 1]))


class DotProductProof:
    """src/subprotocols/dot_product.rs:11-136"""

    @staticmethod
    def proof_len(n):
        return 136 + 32 * int(n)

    @staticmethod
    def prove(ctx, gens_1, gens_n, transcript, random_tape, x, blind_x, a, y, blind_y):
        """DotProductProof::prove on the caller's transcript and tape, advanced in place -> (proof bytes, Cx, Cy), the
        commitments 32 bytes compressed.  y is not checked against <x, a>: a wrong one gives a proof the verifier
        rejects."""
        x = _limbs(x, what="x")
        n = x.shape[0]
        a = _limbs(a, n, "a")
        bx, y, by = _limbs(blind_x, 1, "blind_x"), _limbs(y, 1, "y"), _limbs(blind_y, 1, "blind_y")
        cap = DotProductProof.proof_len(n)
        out = np.zeros(cap, dtype=np.uint8)
        cx, cy = np.zeros(32, dtype=np.uint8), np.zeros(32, dtype=np.uint8)
        ln = C.c_size_t(0)
        _chk(lib().lasso_dot_product_prove(ctx._h, gens_1._h, gens_n._h, transcript._h, random_tape._h, _p(x), _p(bx),
                                           _p(a), C.c_size_t(n), _p(y), _p(by), _p(out), C.c_size_t(cap), C.byref(ln),
                                           _p(cx), _p(cy)))
        return bytes(out[: ln.value]), cx.tobytes(), cy.tobytes()


class ZKSumcheckInstanceProof:
    """src/subprotocols/sumcheck.rs:330-447, proven on the GPU.  `.data` is the ark-serialize (compressed) proof, `.r`
    the challenges, `.final_evals` every polynomial at r after the binds, `.claim` the sum over the hypercube,
    `.comm_claim` its commitment claim G_1 + blind_claim h_1 (32 bytes), `.blind_eval` the blind of the last comm_eval."""

    def __init__(self, data, r, final_evals, claim, comm_claim, blind_eval):
        self.data, self.r, self.final_evals = data, r, final_evals
        self.claim, self.comm_claim, self.blind_eval = claim, comm_claim, blind_eval

    @staticmethod
    def proof_len(num_rounds, degree):
        return 24 + int(num_rounds) * (200 + 32 * (int(degree) + 1))

    @classmethod
    def prove(cls, ctx, comb, polys, num_rounds, blind_claim, gens_1, gens_n, transcript, random_tape):
        """the sumcheck of SumcheckInstanceProof.prove_arbitrary, zero-knowledge, on the caller's transcript and tape,
        advanced in place (include/lasso_b200.h lasso_zk_sumcheck_prove).  gens_1.n == 1, gens_n.n == comb.degree + 1.
        num_rounds=None: num_vars.  Single GPU."""
        polys = list(polys)
        if num_rounds is None:
            num_rounds = polys[0].num_vars if polys else 0
        num_rounds = int(num_rounds)
        bc = _limbs(blind_claim, 1, "blind_claim")
        cap = cls.proof_len(max(num_rounds, 0), comb.degree)
        out = np.zeros(cap, dtype=np.uint8)
        r = np.zeros((max(num_rounds, 1), 4), dtype=np.uint64)
        fin = np.zeros((max(len(polys), 1), 4), dtype=np.uint64)
        claim, blind_eval = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
        cc = np.zeros(32, dtype=np.uint8)
        n = C.c_size_t(0)
        _chk(lib().lasso_zk_sumcheck_prove(ctx._h, comb._h, _handles(polys), C.c_size_t(len(polys)),
                                           C.c_size_t(num_rounds), _p(bc), gens_1._h, gens_n._h, transcript._h,
                                           random_tape._h, _p(out), C.c_size_t(cap), C.byref(n), _p(r), _p(fin),
                                           _p(claim), _p(cc), _p(blind_eval)))
        return cls(bytes(out[: n.value]), r[:num_rounds], fin[: len(polys)], claim, cc.tobytes(), blind_eval)


# ------------------------------------------------------------------ Σ-protocols of committed scalars
def _sigma(fn, ctx, gens, transcript, random_tape, names, values, proof_len, n_points):
    """one call of the Σ-provers: values are single Fr elements (uint64 limbs of shape (4,)) named for the errors ->
    (proof bytes, n_points compressed commitments)"""
    vals = [_limbs(v, 1, name) for name, v in zip(names, values)]
    out = np.zeros(proof_len, dtype=np.uint8)
    pts = [np.zeros(32, dtype=np.uint8) for _ in range(n_points)]
    _chk(fn(ctx._h, gens._h, transcript._h, random_tape._h, *[_p(v) for v in vals], _p(out), *[_p(p) for p in pts]))
    return (out.tobytes(),) + tuple(p.tobytes() for p in pts)


class KnowledgeProof:
    """src/subprotocols/zk.rs:11-76: knowledge of x and r behind C = x G + r h"""

    proof_len = 96

    @staticmethod
    def prove(ctx, gens, transcript, random_tape, x, r):
        """KnowledgeProof::prove on the caller's transcript and tape, advanced in place; gens: a MultiCommitGens with
        n == 1 -> (proof bytes {alpha, z1, z2}, C)"""
        return _sigma(lib().lasso_knowledge_prove, ctx, gens, transcript, random_tape, ("x", "r"), (x, r), 96, 1)


class EqualityProof:
    """src/subprotocols/zk.rs:78-154: C1 = v1 G + s1 h and C2 = v2 G + s2 h hide the same value"""

    proof_len = 64

    @staticmethod
    def prove(ctx, gens, transcript, random_tape, v1, s1, v2, s2):
        """EqualityProof::prove on the caller's transcript and tape, advanced in place; gens: a MultiCommitGens with
        n == 1 -> (proof bytes {alpha, z}, C1, C2).  v1 is not checked against v2: a false statement gives a proof the
        verifier rejects."""
        return _sigma(lib().lasso_equality_prove, ctx, gens, transcript, random_tape, ("v1", "s1", "v2", "s2"),
                      (v1, s1, v2, s2), 64, 2)


class ProductProof:
    """src/subprotocols/zk.rs:156-301: Z = z G + rZ h commits to the product of the values behind X and Y"""

    proof_len = 256

    @staticmethod
    def prove(ctx, gens, transcript, random_tape, x, rX, y, rY, z, rZ):
        """ProductProof::prove on the caller's transcript and tape, advanced in place; gens: a MultiCommitGens with
        n == 1 -> (proof bytes {alpha, beta, delta, z[5]}, X, Y, Z).  z is not checked against x y: a false statement
        gives a proof the verifier rejects."""
        return _sigma(lib().lasso_product_prove, ctx, gens, transcript, random_tape, ("x", "rX", "y", "rY", "z", "rZ"),
                      (x, rX, y, rY, z, rZ), 256, 3)


# ------------------------------------------------------------------ grand products over a caller's polynomials
class GrandProductCircuit:
    """src/subprotocols/grand_product.rs:14-66 over a DensePolynomial of ctx with 1 <= num_vars <= 28: the layers above
    the polynomial are built on ctx's GPU; the polynomial itself is layer 0, neither copied nor modified, and the circuit
    keeps a reference to it.  A circuit can be proven once (the proof binds its layers)."""

    def __init__(self, ctx, poly):
        h = C.c_void_p()
        _chk(lib().lasso_gp_circuit_create(ctx._h, poly._h, C.byref(h)))
        self.ctx, self.poly, self._h = ctx, poly, h
        self.num_vars = int(lib().lasso_gp_circuit_num_vars(h))

    def evaluate(self):
        """the product of all evaluations, (4,) uint64 Montgomery limbs"""
        out = np.zeros(4, dtype=np.uint64)
        _chk(lib().lasso_gp_circuit_evaluate(self._h, _p(out)))
        return out

    def __del__(self):
        try:
            if self._h and self.ctx._h:
                lib().lasso_gp_circuit_destroy(self._h)
        except Exception:
            pass


class BatchedGrandProductArgument:
    """src/subprotocols/grand_product.rs:68-262.  `.bytes` is the ark-serialize (compressed) proof, `.r` the point rand
    (num_vars x 4), `.claims` the final claims (n x 4), the circuits' polynomials evaluated at rand."""

    def __init__(self, data, r, claims):
        self.bytes, self.r, self.claims = data, r, claims

    @staticmethod
    def proof_len(n, num_vars):
        return 8 + num_vars * (24 + 64 * n) + 52 * num_vars * (num_vars - 1)

    @classmethod
    def prove(cls, ctx, circuits, transcript):
        """BatchedGrandProductArgument::prove over 1..32 GrandProductCircuits of one num_vars on the caller's transcript,
        advanced in place"""
        circuits = list(circuits)
        v = circuits[0].num_vars if circuits else 0
        cap = cls.proof_len(len(circuits), v)
        out = np.zeros(cap, dtype=np.uint8)
        r = np.zeros((max(v, 1), 4), dtype=np.uint64)
        claims = np.zeros((max(len(circuits), 1), 4), dtype=np.uint64)
        n = C.c_size_t(0)
        _chk(lib().lasso_gp_prove(ctx._h, _handles(circuits), C.c_size_t(len(circuits)), transcript._h, _p(out),
                                  C.c_size_t(cap), C.byref(n), _p(r), _p(claims)))
        return cls(bytes(out[: n.value]), r[:v], claims[: len(circuits)])


# ------------------------------------------------------------------ memory checking inside a caller's protocol
def _strategy_call(strategy, builtin, custom):
    """(function, leading arguments) of a built-in / custom strategy pair of C entry points"""
    if isinstance(strategy, CustomStrategy):
        if strategy._h is None:
            raise LassoError(LASSO_ERR_STRATEGY, "the CustomStrategy was built without a context")
        return custom, (strategy._h,)
    return builtin, (strategy.kind, strategy.log_r)


def _gamma_tau(hash_challenges):
    gamma, tau = hash_challenges
    return _limbs(gamma, 1, "gamma"), _limbs(tau, 1, "tau")


class Subtables:
    """Subtables::new (src/subtables/mod.rs:116-129) of a strategy over a DensifiedRepresentation, on ctx's GPU (single
    GPU).  `.lookup_polys`: the num_memories polynomials E_i[j] = T_sub(i)[dim_i[j]] in memory order, each with its own
    storage and the tables' width; `.combined_poly`: DensePolynomial.merge of them."""

    def __init__(self, ctx, strategy, dense):
        L = lib()
        fn, head = _strategy_call(strategy, L.lasso_lookup_polys, L.lasso_lookup_polys_custom)
        alpha = strategy.num_memories
        hs = (C.c_void_p * max(alpha, 1))()
        _chk(fn(ctx._h, *head, dense._h, hs, C.c_size_t(alpha)))
        self.ctx = ctx
        self.lookup_polys = [DensePolynomial._wrap(ctx, C.c_void_p(hs[i])) for i in range(alpha)]
        self._combined = None

    @property
    def combined_poly(self):
        if self._combined is None:
            self._combined = DensePolynomial.merge(self.ctx, self.lookup_polys)
        return self._combined

    def commit(self, gens):
        """Subtables::commit (src/subtables/mod.rs:177-184) -> the CombinedTableCommitment's bytes (those of its
        PolyCommitment); gens: PolyCommitmentGens of combined_poly.num_vars, e.g. the proof's gens_derefs"""
        return self.combined_poly.commit(gens)


class MemoryCheckingProof:
    """src/subtables/memory_checking.rs:26-147.  `.bytes` is the ark-serialize (compressed) proof: the product layer,
    then the hash layer."""

    def __init__(self, data):
        self.bytes = data

    @classmethod
    def prove(cls, ctx, strategy, dense, hash_challenges, gens, transcript, random_tape):
        """MemoryCheckingProof::prove(dense, (gamma, tau), subtables, gens, transcript, random_tape) on the caller's
        transcript and tape, advanced in place; gens: the SparsePolyCommitmentGens of the lookup proof.  The subtables
        are rebuilt from (strategy, dense).  Single GPU."""
        L = lib()
        fn, head = _strategy_call(strategy, L.lasso_memory_check_prove, L.lasso_memory_check_prove_custom)
        gamma, tau = _gamma_tau(hash_challenges)
        cap = 1 << 22
        out = ctx._buf("proof", cap, np.uint8)
        n = C.c_size_t(0)
        _chk(fn(ctx._h, *head, dense._h, _p(gamma), _p(tau), gens._h, transcript._h, random_tape._h, _p(out),
                C.c_size_t(cap), C.byref(n)))
        return cls(bytes(out[: n.value]))


class GrandProducts:
    """GrandProducts::new(eval_table, dim, dim_usize, read, final, (gamma, tau)) (src/subtables/memory_checking.rs:
    175-310) over a caller's memory: `.polys` are the fingerprint polynomials (init, read, write, final), and `.init`,
    `.read`, `.write`, `.final` GrandProductCircuits over them.  dim doubles as dim_usize and must hold integers below
    M = len(eval_table) (LassoError code 3 otherwise); read and final may be any field elements.  Single GPU."""

    FIELDS = ("init", "read", "write", "final")

    def __init__(self, ctx, polys):
        self.ctx, self.polys = ctx, polys
        for name, p in zip(self.FIELDS, polys):
            setattr(self, name, GrandProductCircuit(ctx, p))

    @classmethod
    def new(cls, ctx, eval_table, dim, read, final, hash_challenges):
        gamma, tau = _gamma_tau(hash_challenges)
        hs = (C.c_void_p * 4)()
        _chk(lib().lasso_memory_fingerprints(ctx._h, eval_table._h, dim._h, read._h, final._h, _p(gamma), _p(tau), hs))
        return cls(ctx, [DensePolynomial._wrap(ctx, C.c_void_p(h)) for h in hs])
