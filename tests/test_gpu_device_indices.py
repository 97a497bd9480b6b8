"""Lookup indices that are already on the GPU: DensifiedRepresentation.from_lookup_indices with a torch CUDA tensor
(lasso_densify_device).  The densified fields, commitments and proofs must equal those of the host-input path
(lasso_densify) for the same logical matrix, whatever the tensor's dtype (int32 / int64) and strides; an entry >= m,
2^32 + 5 or -1 included, must fail with LASSO_ERR_INDEX_RANGE; a pointer that is not device memory of the context's GPU
must fail with LASSO_ERR_POINTER; the matrix must be read in the order of the caller's stream."""
import ctypes
import hashlib
import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as ol
import workloads as wl

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ERR_INDEX_RANGE, ERR_STRATEGY, ERR_POINTER = 3, 4, 7


@pytest.fixture(scope="module")
def ctx():
    import lasso_b200 as lb

    c = lb.Context(0)
    yield c
    c.close()


def _next_pow2(x):
    return 1 << max(0, (x - 1).bit_length())


def _cuda(a, dtype="int64"):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a).astype(dtype)).cuda()


def _views(dense):
    """sha256 of each of the six lasso_dense_read views: dim_usize, dim, read, final and the two combined polynomials"""
    C, s, m = dense.C, dense.s, dense.m
    shapes = [(0, C * s, 1), (1, C * s, 4), (2, C * s, 4), (3, C * m, 4), (4, _next_pow2(2 * C * s), 4),
              (5, _next_pow2(C) * m, 4)]
    return [hashlib.sha256(dense._read(w, n, width).tobytes()).hexdigest() for w, n, width in shapes]


def _host_mode(monkeypatch, mode):
    """force the host-input path's host scan ("host") or its GPU sort ("gpu"); the device entry ignores both"""
    monkeypatch.setenv("LASSO_B200_HOST_DENSIFY", "1" if mode == "host" else "0")
    monkeypatch.setenv("LASSO_B200_GPU_DENSIFY", "1" if mode == "gpu" else "0")


def _indices(n, C, log_m, seed, skew=False):
    rng = np.random.default_rng(seed)
    idx = rng.integers(0, 1 << log_m, size=(n, C), dtype=np.uint64)
    if skew:  # the skewed columns of test_gpu_densify_matches_host_scan
        idx[:, 1] = rng.integers(0, 3, size=n)
        idx[100:400, 2] = 17
    return idx


# (n, C, log_m, skewed): every n, C and log_m of the issue appears, the smallest and largest of each together
SHAPES = [
    (1, 1, 1, False), (1, 16, 20, False), (3, 3, 7, False), (3, 8, 1, False), (5000, 3, 7, True), (5000, 16, 20, True),
    (2**15 - 1, 4, 16, False), (2**15 - 1, 1, 20, False), (2**15 - 1, 8, 7, False), (2**20, 4, 20, False),
    (2**20, 8, 1, False), (2**20, 1, 16, False),
]


@pytest.mark.parametrize("n,C,log_m,skew", SHAPES)
def test_fields_match_host_input(ctx, monkeypatch, n, C, log_m, skew):
    import lasso_b200 as lb

    idx = _indices(n, C, log_m, n * 31 + C * 7 + log_m, skew)
    dev = _cuda(idx)
    for mode in ("host", "gpu"):
        _host_mode(monkeypatch, mode)
        want = _views(lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m))
        got = _views(lb.DensifiedRepresentation.from_lookup_indices(ctx, dev, log_m))
        assert got == want, (mode, [k for k in range(6) if got[k] != want[k]])


def _layouts(torch, idx, dtype):
    """(name, a non-contiguous CUDA view whose logical value is idx)"""
    n, C = idx.shape
    t = _cuda(idx, dtype)
    transposed = t.T.contiguous().T  # a (C, n) tensor seen as n x C: strides (1, n)
    rows = torch.zeros((2 * n, C), dtype=t.dtype, device=t.device)
    rows[::2] = t
    wide = torch.zeros((n, C + 3), dtype=t.dtype, device=t.device)
    wide[:, 1:C + 1] = t
    return [("contiguous", t), ("transposed", transposed), ("every_other_row", rows[::2]), ("column_slice", wide[:, 1:C + 1])]


@pytest.mark.parametrize("dtype", ["int64", "int32"])
def test_layouts(ctx, dtype):
    import torch

    import lasso_b200 as lb

    n, C, log_m = 3000, 4, 9
    idx = _indices(n, C, log_m, 5)
    want = _views(lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m))
    for name, view in _layouts(torch, idx, dtype):
        assert (view.cpu().numpy().astype(np.uint64) == idx).all()
        if name != "contiguous":
            assert not view.is_contiguous()
        assert _views(lb.DensifiedRepresentation.from_lookup_indices(ctx, view, log_m)) == want, name


RANGE_N, RANGE_C, RANGE_LOG_M = 3000, 3, 8  # XOR needs an even log_m; 2^32 + 5 narrows to 5 < m
BAD = [("m", 1 << RANGE_LOG_M, "int64"), ("m_int32", 1 << RANGE_LOG_M, "int32"), ("2^32+5", 2**32 + 5, "int64"),
       ("minus_one", -1, "int64"), ("minus_one_int32", -1, "int32")]
PLACES = [("first_row", 0, 1), ("last_row", RANGE_N - 1, 1), ("last_column", RANGE_N // 2, RANGE_C - 1)]


def _bad_matrix(value, dtype, row, col):
    idx = _indices(RANGE_N, RANGE_C, RANGE_LOG_M, 9).astype(np.int64)
    idx[row, col] = value
    return _cuda(idx, dtype)


@pytest.mark.parametrize("place,row,col", PLACES)
@pytest.mark.parametrize("label,value,dtype", BAD)
def test_out_of_range_entry(ctx, label, value, dtype, place, row, col):
    """2^32 + 5 narrows to 5 < m and must still fail: the comparison is made in the entry's full width"""
    import lasso_b200 as lb

    with pytest.raises(lb.LassoError) as e:
        lb.DensifiedRepresentation.from_lookup_indices(ctx, _bad_matrix(value, dtype, row, col), RANGE_LOG_M)
    assert e.value.code == ERR_INDEX_RANGE


def _prove(ctx, S, C, log_m, idx, src, seed):
    """commitment, proof bytes and challenges of densify(src) -> commit -> prove, idx the host copy of src"""
    import lasso_b200 as lb

    rng = np.random.default_rng(seed)
    s = _next_pow2(idx.shape[0])
    r = ol.rand_fr(rng, max(1, s.bit_length() - 1))
    tape = ol.rand_fr(rng, 1)[0]
    need = lb.gens_points_needed(C, s, S.num_memories, log_m)
    stream = np.ascontiguousarray(ol.generators(max(need, 300))[:need])
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, s, S.num_memories, log_m, stream=stream)
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, src, log_m)
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=tape)
    return com, proof.bytes, proof.challenges.tobytes()


def test_context_usable_after_range_errors():
    """every rejected matrix of test_out_of_range_entry on one context, then a valid densify and proof on it: the bytes
    equal those of a fresh context"""
    import lasso_b200 as lb

    idx = _indices(RANGE_N, RANGE_C, RANGE_LOG_M, 9)
    S = lb.Strategy(lb.XOR, RANGE_C, RANGE_LOG_M)
    fresh = lb.Context(0)
    want = _prove(fresh, S, RANGE_C, RANGE_LOG_M, idx, idx, 3)
    fresh.close()
    c = lb.Context(0)
    for _, value, dtype in BAD:
        for _, row, col in PLACES:
            with pytest.raises(lb.LassoError) as e:
                lb.DensifiedRepresentation.from_lookup_indices(c, _bad_matrix(value, dtype, row, col), RANGE_LOG_M)
            assert e.value.code == ERR_INDEX_RANGE
    assert _prove(c, S, RANGE_C, RANGE_LOG_M, idx, _cuda(idx), 3) == want
    c.close()


def _raw_densify(ctx, ptr, elem_bytes=8, n=4, C=2, row_stride=2, col_stride=1, log_m=4):
    import lasso_b200 as lb

    h = ctypes.c_void_p()
    rc = lb.lib().lasso_densify_device(ctx._h, ctypes.c_void_p(ptr), ctypes.c_size_t(elem_bytes), ctypes.c_size_t(n),
                                       ctypes.c_size_t(C), ctypes.c_size_t(row_stride), ctypes.c_size_t(col_stride),
                                       ctypes.c_size_t(log_m), ctypes.c_void_p(0), ctypes.byref(h))
    return rc, h.value


def test_pointer_and_parameter_checks(ctx):
    import torch

    import lasso_b200 as lb

    host = np.zeros((4, 2), dtype=np.uint64)
    assert _raw_densify(ctx, host.ctypes.data) == (ERR_POINTER, None)
    pinned = torch.zeros((4, 2), dtype=torch.int64).pin_memory()
    assert _raw_densify(ctx, pinned.data_ptr()) == (ERR_POINTER, None)
    assert _raw_densify(ctx, 0) == (ERR_POINTER, None)
    dev = torch.zeros((4, 2), dtype=torch.int64, device="cuda:0")
    p = dev.data_ptr()
    rc, h = _raw_densify(ctx, p)
    assert rc == 0 and h
    lb.lib().lasso_dense_destroy(ctypes.c_void_p(h))
    for kw in ({"elem_bytes": 2}, {"elem_bytes": 16}, {"n": 0}, {"C": 0}, {"C": 17}, {"log_m": 0}, {"log_m": 29}):
        assert _raw_densify(ctx, p, **kw) == (ERR_STRATEGY, None), kw
    # the binding refuses what it cannot describe to the C ABI
    for bad in (dev.float(), dev[:, 0], dev.reshape(2, 2, 2), dev.to(torch.int16)):
        with pytest.raises(lb.LassoError) as e:
            lb.DensifiedRepresentation.from_lookup_indices(ctx, bad, 4)
        assert e.value.code == ERR_STRATEGY


def test_tensor_on_another_gpu(ctx):
    import torch

    import lasso_b200 as lb

    if torch.cuda.device_count() < 2:
        pytest.skip("needs a second visible GPU")
    with pytest.raises(lb.LassoError) as e:
        lb.DensifiedRepresentation.from_lookup_indices(ctx, torch.zeros((4, 2), dtype=torch.int64, device="cuda:1"), 4)
    assert e.value.code == ERR_POINTER


def test_stream_order(ctx):
    """The indices are written on a side stream after ~0.1 s of device spinning, and densified under that stream with no
    synchronise: the fields must equal the host-input path's, so the matrix was read after the writes.  Then the tensor
    is overwritten on the same stream right after the call returns, and the proof must not change.  That second check
    only catches a missing wait on the caller's stream if the race happens to show: the call has already waited for
    the range verdict, which comes after the last read."""
    import torch

    import lasso_b200 as lb

    n, C, log_m = 1 << 16, 4, 16
    idx = _indices(n, C, log_m, 21)
    S = lb.Strategy(lb.XOR, C, log_m)
    want_views = _views(lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m))
    want = _prove(ctx, S, C, log_m, idx, idx, 4)
    src = _cuda(idx)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.zeros_like(src)
        torch.cuda._sleep(200_000_000)
        x.copy_(src)
        dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, x, log_m)
        x.fill_(1)
    assert _views(dense) == want_views
    del dense
    with torch.cuda.stream(side):
        x = torch.zeros_like(src)
        torch.cuda._sleep(200_000_000)
        x.copy_(src)
        got = _prove(ctx, S, C, log_m, idx, x, 4)
        x.fill_((1 << log_m) - 1)
    assert got == want


def _builtin_cases():
    import lasso_b200 as lb

    return [(lb.AND, 4, 4, 0, 16), (lb.OR, 2, 8, 0, 700), (lb.XOR, 4, 16, 0, 1 << 12), (lb.LT, 8, 8, 0, 512),
            (lb.RANGE_CHECK, 4, 16, 40, 1 << 10)]


@pytest.mark.parametrize("case", range(5))
@pytest.mark.parametrize("dtype", ["int64", "int32"])
def test_builtin_proofs_match_host_input(ctx, case, dtype):
    import lasso_b200 as lb

    kind, C, log_m, log_r, n = _builtin_cases()[case]
    S = lb.Strategy(kind, C, log_m, log_r)
    idx = _indices(n, C, log_m, 40 + case)
    assert _prove(ctx, S, C, log_m, idx, _cuda(idx, dtype), case) == _prove(ctx, S, C, log_m, idx, idx, case)


def test_custom_strategy_proof_matches_host_input(ctx):
    import custom_builtins as cb

    S = cb.NEW_TABLES["product_deg2"](ctx)
    idx = _indices(900, S.C, S.log_m, 50)
    assert _prove(ctx, S, S.C, S.log_m, idx, _cuda(idx), 7) == _prove(ctx, S, S.C, S.log_m, idx, idx, 7)


def test_field_table_strategy_proof_matches_host_input(ctx):
    import field_tables as ft

    S = ft.strategy(ctx, "random_full", 2, 7, 2, nsub=2)
    idx = _indices(600, 2, 7, 51)
    assert _prove(ctx, S, 2, 7, idx, _cuda(idx), 8) == _prove(ctx, S, 2, 7, idx, idx, 8)


@pytest.mark.parametrize("name", ["xor_c4_s20", "lt_c8_s22", "rc40_c4_s24"])
def test_config_from_cuda_tensor_matches_golden(ctx, name):
    """at size: the bytes hash to tests/golden/big_proofs.json, and densify launches as many kernels as the host-input
    path's GPU sort (no extra pass over the matrix)"""
    import lasso_b200 as lb

    g = json.load(open(os.path.join(HERE, "golden", "big_proofs.json")))["cases"][name]
    kind, C, log_m, log_r, log_s, idx, r, tape_seed = wl.config_inputs(name)
    assert hashlib.sha256(idx.tobytes()).hexdigest() == g["indices_sha256"]
    S = lb.Strategy(kind, C, log_m, log_r)
    s = 1 << log_s
    stream = np.ascontiguousarray(ol.generators(g["n_generators"]))
    gens = lb.SparsePolyCommitmentGens.new(ctx, b"gens_sparse_poly", C, s, S.num_memories, log_m, stream=stream)
    before = ctx.launches
    host_dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, idx, log_m)
    host_launches = ctx.launches - before
    del host_dense
    dev = _cuda(idx)
    before = ctx.launches
    dense = lb.DensifiedRepresentation.from_lookup_indices(ctx, dev, log_m)
    assert ctx.launches - before == host_launches
    del dev
    com = dense.commit(gens)
    proof = lb.SparsePolynomialEvaluationProof.prove(ctx, S, dense, r, gens, tape_seed=tape_seed)
    assert hashlib.sha256(com).hexdigest() == g["commitment_sha256"]
    assert proof.challenges[-1].tobytes().hex() == g["last_challenge_hex"]
    assert hashlib.sha256(proof.bytes).hexdigest() == g["proof_sha256"]


def _run_sharded(nproc, same_gpu, timeout=1500):
    """tools/sharded_check.py --device under torchrun (the same launcher as tests/test_gpu_sharded.py)"""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ)
    if same_gpu:
        env["LASSO_SHARD_SAME_GPU"] = "1"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "sharded_check.py"), "--device"]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert "SHARDED_CHECK PASS" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


def test_sharded_two_ranks_one_gpu():
    _run_sharded(2, True)


def test_sharded_four_ranks_one_gpu():
    _run_sharded(4, True)


def test_sharded_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (the one-GPU variants cover the same code)")
    _run_sharded(2, False)
