"""gloo world-2 emulation of the sharded Gram + right-hand-side pass of the normal-equation Anderson variants
(csrc/aa.cuh aa_gram_kernel / aa_ne_solve_kernel, Engine::aa_accelerate): every rank keeps [w_x (replicated); w_s on
its rows], sums its 26 scalars per chunk of 8 columns over [lo, dim) (lo = 0 on rank 0, n elsewhere), and one
allreduce of all chunks gives every rank the same M, rhs, eta and candidate as the unsharded restatement."""
import os

import numpy as np
import pytest

import cosmo_b200
from cosmo_b200 import sharding
from tests import anderson_variants as V
from tests.test_sharding_cpu import _free_port

COLS, NR = 8, 26


def _chunk_scalars(Al, Bl, fl, j, l, lo, type1):
    """the partial sums one rank's aa_gram_kernel launches write, all chunks back to back"""
    nch = (l + COLS - 1) // COLS
    out = np.zeros(nch * NR)
    A, B, f = Al[lo:], Bl[lo:], fl[lo:]
    for ch in range(nch):
        o = out[ch * NR:(ch + 1) * NR]
        for c in range(min(COLS, l - ch * COLS)):
            col = ch * COLS + c
            o[c] = A[:, j] @ B[:, col]
            if type1:
                o[COLS + c] = A[:, col] @ B[:, j]
            o[2 * COLS + c] = A[:, col] @ f
        o[3 * COLS] = A[:, j] @ A[:, j]
        if type1:
            o[3 * COLS + 1] = B[:, j] @ B[:, j]
    return out


def _worker(rank, world, port, out):
    import torch
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(60, 150, 0.08, seed=2)
        sh = sharding.make_shard(P, q, A, b, sets, rank, world)
        n, m_full = A.shape[1], A.shape[0]
        dim = n + m_full
        idx = np.concatenate([np.arange(n), n + sh.rows])
        lo = 0 if rank == 0 else n
        ok = True
        for t, mem_kind, reg in (("Type1", "RollingMemory", "NoRegularizer"),
                                 ("Type2{NormalEquations}", "RestartedMemory", "TikonovRegularizer"),
                                 ("Type2{NormalEquations}", "RollingMemory", "FrobeniusNormRegularizer")):
            type1 = t == "Type1"
            mem = 12                                   # two chunks of the Gram pass once l > 8
            full = V.NormalEquationsAccelerator(dim, mem, type1=type1, rolling=mem_kind == "RollingMemory",
                                                regularizer=reg, lam=1e-4)
            loc = V.NormalEquationsAccelerator(len(idx), mem, type1=type1, rolling=mem_kind == "RollingMemory",
                                               regularizer=reg, lam=1e-4)
            rng = np.random.default_rng(0)              # the same operator and start on every rank
            Mop = rng.standard_normal((dim, dim)) * (0.5 / np.sqrt(dim))
            cst = rng.standard_normal(dim)
            xk = rng.standard_normal(dim)
            for k in range(2 * mem + 3):                # crosses a wrap-around / a memory restart
                gk = Mop @ xk + cst
                full.update(gk, xk, k + 2)
                g_acc = gk.copy()
                full.accelerate(g_acc, xk, k + 2)
                # ---- the sharded step: local history, partial scalars, one allreduce, the solve kernel's scatter ----
                loc.update(gk[idx], xk[idx], k + 2)
                cand = gk[idx].copy()
                if loc.fresh:
                    loc.fresh = False
                    l, j = min(loc.iter, loc.mem), loc.j
                    Al = loc.X if type1 else loc.F
                    buf = torch.from_numpy(_chunk_scalars(Al, loc.F, loc.f, j, l, lo, type1))
                    dist.all_reduce(buf, op=dist.ReduceOp.SUM)
                    gsc = buf.numpy()
                    rhs = np.zeros(l)
                    for r in range(l):
                        o = gsc[(r // COLS) * NR:]
                        loc.M[j, r] = o[r % COLS]
                        if r != j:
                            loc.M[r, j] = o[COLS + r % COLS] if type1 else o[r % COLS]
                        rhs[r] = o[2 * COLS + r % COLS]
                    loc.nrmA[j] = gsc[3 * COLS]
                    loc.nrmB[j] = gsc[3 * COLS + 1] if type1 else gsc[3 * COLS]
                    ok = ok and np.allclose(loc.M[:l, :l], full.M[:l, :l], rtol=1e-11, atol=1e-13)
                    if l >= 3:
                        eta = V.lu_solve(loc.system(l), rhs)
                        if eta is not None:
                            cand = gk[idx] - loc.G[:, :l] @ eta
                ok = ok and np.allclose(cand, g_acc[idx], rtol=1e-9, atol=1e-9)
                xk = g_acc
            ok = ok and full.num_accelerated_steps >= mem
        out[rank] = bool(ok)
    finally:
        dist.destroy_process_group()


def test_sharded_gram_pass_matches_full_gloo_world2():
    import torch.multiprocessing as mp
    world = 2
    port = _free_port()
    with mp.Manager() as mgr:
        out = mgr.dict()
        mp.spawn(_worker, args=(world, port, out), nprocs=world, join=True)
        assert dict(out) == {0: True, 1: True}
