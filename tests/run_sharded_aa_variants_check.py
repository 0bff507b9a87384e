"""Launched under torchrun (one rank per GPU) by tests/test_gpu_sharded_aa_variants.py: Type1/RollingMemory and
Type2{NormalEquations}/TikonovRegularizer solves row-sharded over WORLD_SIZE GPUs, checked on rank 0 against the CPU
restatement of tests/anderson_variants.py with the bounds of tests/run_sharded_check.py (5 eps on x, s and mu)."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.distributed as dist

import cosmo_b200
from cosmo_b200 import sharding
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests import anderson_variants as V
from tests.run_sharded_check import gather_rows


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    pr = cosmo_b200.problems
    problems = [("qp", pr.random_sparse_qp(600, 1500, 0.05, seed=4), dict()),
                # accelerated SOCP runs split in the last digits and stop a few tolerances apart (Type1/RollingMemory
                # even unsharded: 523 vs 573 iterations, dx 1.0e-4 at eps = 1e-5); as in run_sharded_check.py, the
                # SOCP is compared at eps = 1e-8 by its end point
                ("socp", pr.portfolio_socp(n=300, k=30, seed=2), dict(max_iter=20000, scaling=0, eps_abs=1e-8, eps_rel=1e-8))]
    variants = [V.variant("Type1", "RollingMemory", "NoRegularizer"),
                V.variant("Type2{NormalEquations}", "RestartedMemory", "TikonovRegularizer")]
    ok = True
    for name, (P, q, A, b, sets), kw in problems:
        for var in variants:
            st = cosmo_b200.Settings(accelerator="AndersonAccelerator", **kw, **var)
            m, n = A.shape
            if st.scaling != 0:
                Ps, qs, As, bs, ss, D, E, c = cosmo_b200.ruiz_equilibrate(P, q, A, b, sets, st)
            else:
                Ps, qs, As, bs, ss, D, E, c = P, q, A, b, sets, None, None, 1.0
            sh = sharding.make_shard(Ps, qs, As, bs, ss, rank, world)
            eng = sharding.create_engine(sh, st, device=local_rank, dist=dist, D=D, E=E, c=c)
            out = eng.solve()
            stats = eng.accelerator_stats()
            x = out.x if D is None else D * out.x
            s = gather_rows(out.s, sh.rows, m, world)
            mu = gather_rows(out.mu, sh.rows, m, world)
            if E is not None:
                s, mu = s / E, E * mu / c
            if rank == 0:
                ref, ws = V.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(kkt_solver="cg", accelerator="anderson", **kw),
                                  **var)
                tight = kw.get("eps_abs", 1e-5) < 1e-6
                tol = 5e-6 if tight else 5e-5      # the bounds of the accelerated cases of run_sharded_check.py
                good = ((tight or out.status == ref.status) and abs(out.obj_val - ref.obj_val) <= tol * max(1, abs(ref.obj_val))
                        and np.max(np.abs(x - ref.x)) <= tol * max(1, np.abs(ref.x).max())
                        and np.max(np.abs(s - ref.s)) <= tol * max(1, np.abs(ref.s).max())
                        and np.max(np.abs(-mu - ref.y)) <= tol * max(1, np.abs(ref.y).max())
                        and stats["accepted"] >= 1)
                print("%-5s %-24s %-16s world=%d status=%s/%s iter=%d/%d dx=%.2e ds=%.2e dmu=%.2e accepted=%d/%d %s" % (
                    name, var["accelerator_type"], var["accelerator_memory"], world, out.status, ref.status, out.iter,
                    ref.iter, np.max(np.abs(x - ref.x)), np.max(np.abs(s - ref.s)), np.max(np.abs(-mu - ref.y)),
                    stats["accepted"], V.stats(ws)["accepted"], "OK" if good else "MISMATCH"), flush=True)
                ok = ok and good
            eng.close()
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.broadcast(flag, src=0)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
