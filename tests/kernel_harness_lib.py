"""ctypes loader for the kernel test harness (tests/kernel_harness/, test infrastructure only): one extern "C" wrapper
per launcher of kernels.cuh / msm.cuh, linked from the library's own kernel objects."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "kernel_harness", "_build", "libkernel_harness.so")

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            raise RuntimeError("libkernel_harness.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(nvcc, sm_90a).")
        L = C.CDLL(SO)
        L.kh_tables_create.argtypes = [C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.POINTER(C.c_void_p)]
        L.kh_tables_destroy.argtypes = [C.c_void_p]
        L.kh_tables_destroy.restype = None
        S, I, V = C.c_size_t, C.c_int, C.c_void_p
        L.kh_cubic.argtypes = [I, I, S, V, V, V, V, V, V, I, V]
        L.kh_product_trees.argtypes = [I, S, I, I, V, V]
        L.kh_bind_heads.argtypes = [I, V, V, V]
        L.kh_bound_u32.argtypes = [V, V, S, S, V]
        L.kh_multi_dot_u32.argtypes = [V, S, I, V, S, V]
        L.kh_fingerprints_mem.argtypes = [V, V, S, I, I, V, V, V, V]
        L.kh_fingerprints_ops.argtypes = [V, V, V, S, V, V, V, V]
        L.kh_fold_ab.argtypes = [V, V, S, V, V]
        L.kh_cross_inner_products.argtypes = [V, V, S, V]
        L.kh_expand_weights.argtypes = [V, S, V, V, V]
        L.kh_bullet_scalars.argtypes = [V, S, V, S, S, S, I, I, I, V, V]
        L.kh_two_row_scalars.argtypes = [V, I, V, V, S, V]
        L.kh_msm_direct.argtypes = [V, V, I, V]
        L.kh_bullet_fused.argtypes = [V, V, V, V, S, S, I, V, V, V, V, V, V, V, V]
        L.kh_msm_rows_direct_u32.argtypes = [V, V, I, I, I, I, I, I, V]
        L.kh_msm_large.argtypes = [V, S, V, S, I, V, V, V]
        L.kh_msm_rows.argtypes = [V, I, V, I, S, I, I, I, I, I, V, V, V]
        L.kh_sum_raw_points.argtypes = [V, I, I, V, V, V]
        L.kh_canonicalize.argtypes = [V, S, C.c_uint, V, V]
        L.kh_msm_rows_direct_raw.argtypes = [V, I, V, I, I, I, I, I, I, V, V]
        L.kh_comb_program.argtypes = [I, V, I, V, I, I, V, V]
        L.kh_comb_eval.argtypes = [I, V, I, V, I, I, V, V, S, I, V]
        L.kh_comb_bind_eval.argtypes = [I, V, I, V, I, I, V, V, S, V, S, I, I, V, V, V]
        L.kh_bind_comb.argtypes = [I, V, V, S, V, I, V]
        L.kh_final_comb.argtypes = [I, V, S, V, I, V]
        L.kh_comb_map.argtypes = [I, V, I, V, I, I, V, V, S, V, S]
        L.kh_product_layer1.argtypes = [V, S, V, S]
        L.kh_bind_ptrs.argtypes = [I, V, V, S, V, V]
        L.kh_poly_ingest.argtypes = [V, S, S, V, V]
        L.kh_poly_mirror_u32.argtypes = [V, S, V]
        L.kh_eq_evals.argtypes = [I, V, V, S, V, V]
        L.kh_densify.argtypes = [V, I, S, S, S, S, I, S, I, I, I, V, S, V, S, V, S, V]
        L.kh_tables_build.argtypes = [V, S, S, S, S, S, C.POINTER(C.c_void_p)]
        L.kh_table_entries.argtypes = [V, I, V, S, V]
        L.kh_arith.argtypes = [I, I, S, V, V, V, V]
        L.kh_arith_op_name.argtypes = [I]
        L.kh_arith_op_name.restype = C.c_char_p
        _lib = L
    return _lib


def call(name, *args):
    """call a wrapper; a non-zero return code is a failure of the launch under test"""
    rc = getattr(lib(), name)(*args)
    assert rc == 0, ("%s returned %d (-1: the launcher threw, -2: CUDA error, -3: publication tag missing, -4: bad "
                     "arguments, -5: a repeated launch published different values)" % (name, rc))


def op_ids(name_fn):
    """{operation name: id} of an arithmetic op table, from its kh_arith_op_name-style name function"""
    ids, i = {}, 0
    while True:
        s = name_fn(i)
        if s is None:
            return ids
        ids[s.decode()] = i
        i += 1


class Tables:
    """window + digit-multiples tables (and optionally 16-bit multiples of ncols16 columns) of a generator set on the
    device, built by the library's launchers"""

    def __init__(self, gens_affine, ncols16=0, col_mul=1, col_add=0):
        import numpy as np

        g = np.ascontiguousarray(gens_affine, dtype=np.uint64)
        h = C.c_void_p()
        call("kh_tables_create", g.ctypes.data, g.shape[0], ncols16, col_mul, col_add, C.byref(h))
        self.h = h
        self.npts = g.shape[0]

    @classmethod
    def as_prover(cls, gens_affine, nd, ncols16=0, col_mul=1, col_add=0):
        """the tables as a proof builds them (kh_tables_build): M over the first nd generators of a T over all of them,
        and with ncols16 the 16-bit multiples of columns jl * col_mul + col_add and their centring constants"""
        import numpy as np

        t = cls.__new__(cls)
        g = np.ascontiguousarray(gens_affine, dtype=np.uint64)
        h = C.c_void_p()
        call("kh_tables_build", g.ctypes.data, g.shape[0], nd, ncols16, col_mul, col_add, C.byref(h))
        t.h = h
        t.npts = g.shape[0]
        return t

    def close(self):
        if self.h:
            lib().kh_tables_destroy(self.h)
            self.h = None
