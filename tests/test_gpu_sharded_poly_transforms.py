"""Deriving polynomials and reading them back on a sharded context: bound_top, bound_bot (fewer, as many and more
variables than lg G, and across the 8-variable passes), split, new_padded (host arrays, CUDA tensors, strided views) and
the read-backs are collective over G ranks, and every rank must return the bytes of a single-GPU context, down to the
smallest results a sharded context holds, and the same error codes.

Rank 0 first runs the same steps on a plain context; every rank then runs them on the sharded one.  Run as a script
under torch.distributed.run it is the worker: 2 and 4 ranks time-slicing GPU 0 (LASSO_SHARD_SAME_GPU=1, gloo for the
plumbing), or one rank per GPU."""
import hashlib
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import dense_poly_cases as dc  # noqa: E402
import lasso_b200 as lb  # noqa: E402
from lasso_b200.api import LASSO_ERR_LENGTH  # noqa: E402

pytestmark = pytest.mark.gpu
MARK = "SHARDED_POLY_TRANSFORMS"


def _run(nproc, same_gpu, timeout=1200):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    env = dict(os.environ)
    if same_gpu:
        env["LASSO_SHARD_SAME_GPU"] = "1"
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc), "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    assert MARK + " PASS" in out.stdout, out.stdout[-4000:] + out.stderr[-4000:]


def test_two_ranks_one_gpu():
    _run(2, True)


def test_four_ranks_one_gpu():
    _run(4, True)


def test_two_ranks_two_gpus():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs (the one-GPU runs cover the same code)")
    _run(2, False)


# ------------------------------------------------------------------------------------------------ the worker
def _h(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _nv_min(G):
    return max(0, 2 * (G.bit_length() - 1) - 1)


def _u16(rng, n):
    return dc.fr_from_u64(rng.integers(0, 1 << 16, size=n, dtype=np.uint64))


def _read(p, dev, out, key):
    """every read-back form of p into out"""
    import torch

    out[key] = _h(p.to_numpy())
    out[key + "/tensor"] = _h(p.to_tensor(dev).cpu().numpy())
    wide = torch.zeros((1 << p.num_vars, 7), dtype=torch.int64, device=dev)
    p.copy_to(wide[:, 2:6])
    torch.cuda.current_stream(dev).synchronize()
    out[key + "/strided"] = _h(wide.cpu().numpy())


def _suite(ctx, G, dev):
    import torch

    out = {}
    lg, m = G.bit_length() - 1, _nv_min(G)
    for nv in (max(m, 4), 10, 14):
        for kind in ("u16", "full"):
            rng = np.random.default_rng(31 * nv + len(kind))
            Z = _u16(rng, 1 << nv) if kind == "u16" else dc.random_full(rng, 1 << nv)
            r = dc.random_full(rng, nv)
            p = lb.DensePolynomial(ctx, Z)
            key = "%d/%s/" % (nv, kind)
            _read(p, dev, out, key + "read")
            # k < lg G, = lg G, > lg G, across a pass boundary, and down to the smallest result
            for k in sorted({1, lg, lg + 1, 3, 9, nv - m} - {0}):
                if k > nv - m:
                    continue
                out[key + "top%d" % k] = _h(p.bound_top(r[:k]).to_numpy())
                out[key + "bot%d" % k] = _h(p.bound_bot(r[:k]).to_numpy())
            q = p.bound_bot(r[: nv - m])
            _read(q, dev, out, key + "bot_min")
            for idx in sorted({1 << (nv - 1), 1 << m}):
                lo, hi = p.split(idx)
                out[key + "split%d" % idx] = _h(lo.to_numpy()) + _h(hi.to_numpy())
            out[key + "unchanged"] = _h(p.to_numpy())
    # new_padded: host, tensor, strided view; lengths whose padding reaches the smallest size a sharded context holds
    for n in sorted({(1 << max(m, 1)) - 1 if m > 1 else 3, 1000, (1 << 12) + 1}):
        rng = np.random.default_rng(n)
        Z = dc.random_full(rng, n)
        t = torch.from_numpy(Z.view(np.int64)).to(dev)
        wide = torch.zeros((n, 9), dtype=torch.int64, device=dev)
        wide[:, 3:7] = t
        for name, src in (("host", Z), ("dev", t), ("strided", wide[:, 3:7])):
            out["padded%d/%s" % (n, name)] = _h(lb.DensePolynomial.new_padded(ctx, src).to_numpy())
    # a bound polynomial of an eq table commits like the single-GPU one (full width on every rank)
    nv = max(m, 6) + 3
    eq = lb.DensePolynomial.eq(ctx, dc.random_full(np.random.default_rng(5), nv))
    b = eq.bound_bot(dc.random_full(np.random.default_rng(6), 3))
    g = lb.PolyCommitmentGens.new(ctx, b"gens_sparse_poly", nv - 3,
                                  stream=np.ascontiguousarray(lb.sample_generators(b"gens_sparse_poly", lb.poly_gens_points_needed(nv - 3))))
    out["eq_bound_commit"] = b.commit(g).hex()
    return out


def _code(fn):
    try:
        fn()
        return 0
    except lb.LassoError as e:
        return e.code


def _errors(ctx, G):
    m = _nv_min(G)
    rng = np.random.default_rng(8)
    nv = max(m, 4)
    p = lb.DensePolynomial(ctx, dc.random_full(rng, 1 << nv))
    r = dc.random_full(rng, nv)
    out = {"top_k0": _code(lambda: p.bound_top(r[:0]))}
    if m >= 1:  # results smaller than the context holds
        out["top_small"] = _code(lambda: p.bound_top(r[: nv - m + 1]))
        out["bot_small"] = _code(lambda: p.bound_bot(r[: nv - m + 1]))
        out["split_small"] = _code(lambda: p.split(1 << (m - 1)))
        out["padded_small"] = _code(lambda: lb.DensePolynomial.new_padded(ctx, dc.random_full(rng, (1 << (m - 1)) - 1 or 1)))
        out["padded_empty"] = _code(lambda: lb.DensePolynomial.new_padded(ctx, np.zeros((0, 4), dtype=np.uint64)))
    out["after"] = _h(p.to_numpy())
    return out


def _expected_errors(G):
    want = {"top_k0": LASSO_ERR_LENGTH}
    if _nv_min(G) >= 1:
        want.update(top_small=LASSO_ERR_LENGTH, bot_small=LASSO_ERR_LENGTH, split_small=LASSO_ERR_LENGTH,
                    padded_small=LASSO_ERR_LENGTH, padded_empty=LASSO_ERR_LENGTH)
    return want


def _worker():
    import torch
    import torch.distributed as dist

    rank, local = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    G = int(os.environ.get("WORLD_SIZE", 1))
    if os.environ.get("LASSO_SHARD_SAME_GPU") == "1":
        local = 0
        torch.cuda.set_device(0)
        dist.init_process_group("gloo")
    else:
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    dev = torch.device("cuda", local)
    single = [None]
    if rank == 0:
        c1 = lb.Context(local)
        single = [(_suite(c1, G, dev), _errors(c1, G)["after"])]
        c1.close()
    dist.broadcast_object_list(single, src=0)
    res1, after1 = single[0]
    c = lb.Context(local)
    c.init_comm()
    res = _suite(c, G, dev)
    errs = _errors(c, G)
    got = [None] * G
    dist.all_gather_object(got, (res, errs))
    if rank == 0:
        fails = []
        want_err = dict(_expected_errors(G), after=after1)
        for g, (rg, eg) in enumerate(got):
            fails += ["rank %d %s" % (g, k) for k in sorted(set(res1) | set(rg)) if res1.get(k) != rg.get(k)]
            fails += ["rank %d error %s: %r != %r" % (g, k, eg.get(k), want_err[k]) for k in want_err if eg.get(k) != want_err[k]]
        print(MARK, "PASS" if not fails else "FAIL %r" % fails[:40], "(%d items)" % len(res1), flush=True)
    dist.barrier()
    c.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker()
