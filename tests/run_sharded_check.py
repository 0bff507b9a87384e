"""Launched under torchrun (one rank per GPU) by tests/test_gpu_sharded.py: solves the same
problems row-sharded over WORLD_SIZE GPUs and checks them against the CPU oracle on rank 0, then runs the
infeasibility certificates of a composite set (every cone family) row-sharded against one unsharded engine."""
import os
import sys

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch
import torch.distributed as dist

import cosmo_b200
from cosmo_b200 import sharding
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones


def gather_rows(local, rows, m, world):
    parts = [None] * world
    dist.all_gather_object(parts, (rows, local))
    full = np.zeros(m)
    for r, v in parts:
        full[r] = v
    return full


def _composite():
    """one set of every family (a large PSD cone among them) and, per case, a point v on the rows (leading
    Nonnegatives row -1, so |v|_inf = 1) where no family, one family or every family fails its certificate"""
    M = cosmo_b200.model
    sets = [M.Nonnegatives(4), M.Box(np.array([-1.0, -2.0, -3.0]), np.array([1.0, np.inf, 3.0])), M.SecondOrderCone(3),
            M.PsdCone(9), M.PsdConeTriangle(6), M.PsdConeTriangle(5050), M.ExponentialCone(), M.DualExponentialCone(),
            M.PowerCone(0.3), M.DualPowerCone(0.6)]
    tri100 = np.concatenate([np.concatenate([np.zeros(j), [-0.5]]) for j in range(100)])
    # the square cone is not symmetric (upper entry 0.2, lower -0.7): certified from its upper triangle
    base = [np.array([-1.0, -0.5, -0.5, -0.5]), np.zeros(3), np.array([-1.0, 0.3, 0.4]),
            np.array([-0.5, -0.7, 0, 0.2, -0.5, 0, 0, 0, -0.5]), np.array([-0.5, 0, -0.5, 0, 0, -0.5]), tri100,
            np.array([0.5, 0.0, -1.0]), np.array([0.0, -0.5, -1.0]), np.array([-0.5, -0.5, 0.0]), np.array([-0.5, -0.5, 0.0])]
    bad = {0: np.array([-1.0, -0.5, 0.5, -0.5]), 2: np.array([1.0, 0.3, 0.4]), 5: -tri100, 6: np.array([-0.5, 0.0, -1.0])}
    cases = [np.concatenate(base)]
    for i, vb in bad.items():
        parts = list(base)
        parts[i] = vb
        cases.append(np.concatenate(parts))
    allbad = list(base)
    for i, vb in bad.items():
        allbad[i] = vb
    cases.append(np.concatenate(allbad))
    return sets, cases


def check_infeasibility_hook(rank, world, local_rank):
    """cosmo_b200_infeasibility_test on row-sharded engines against one unsharded engine on rank 0: the verdict, the
    gate reached, the norms and the failed-family bitmask must be equal, dy'b and the Box support sum (allreduce(sum)
    over the ranks) equal to 1e-14 of their magnitude.  Primal: A = 0, b != 0, delta_y = -v; dual: A = I, P = 0,
    q = -v, delta_x = v (the exact-gate rigs of tests/test_gpu_infeasibility.py)."""
    sets, cases = _composite()
    m = sum(S.dim for S in sets)
    b = np.random.default_rng(3).uniform(-1e-4, 1e-4, m)
    st = cosmo_b200.Settings(scaling=0, eps_prim_inf=2.0 ** -10, eps_dual_inf=2.0 ** -10)
    rigs = {0: (sp.csc_matrix((1, 1)), np.zeros(1), sp.csc_matrix((m, 1)), b),
            1: (sp.csc_matrix((m, m)), np.zeros(m), sp.identity(m, format="csc"), np.zeros(m))}
    ok = True
    for which, (P, q, A, bb) in rigs.items():
        sh = sharding.make_shard(P, q, A, bb, sets, rank, world)
        eng = sharding.create_engine(sh, st, device=local_rank, dist=dist)
        one = sharding.create_engine(sharding.make_shard(P, q, A, bb, sets, 0, 1), st, device=local_rank) if rank == 0 else None
        for k, v in enumerate(cases):
            if which == 0:
                rec = eng.infeasibility_test(0, -v[sh.rows])
            else:
                eng.update_qb(q=-v)
                rec = eng.infeasibility_test(1, v)
            recs = [None] * world
            dist.all_gather_object(recs, rec)
            if rank == 0:
                if which == 1:
                    one.update_qb(q=-v)
                ref = one.infeasibility_test(which, -v if which == 0 else v)
                mag_b = float(np.sum(np.abs(v * b)))
                good = all(r["verdict"] == ref["verdict"] and r["gate"] == ref["gate"] == 4 and r["families"] == ref["families"]
                           and r["norm"] == ref["norm"] and r["psd_unconverged"] == ref["psd_unconverged"] == 0
                           and (which == 1 or (abs(r["gate3"] - ref["gate3"]) <= 1e-14 * mag_b
                                               and abs(r["box_sum"] - ref["box_sum"]) <= 1e-14 * 4.0))
                           for r in recs)
                good = good and ref["families"] == ([0, 1, 2, 4, 8, 15][k])
                print("infeasibility_hook which=%d case=%d world=%d families=%s/%d verdict=%s/%d dyb=%s/%.17g box=%s/%.17g %s" % (
                    which, k, world, [r["families"] for r in recs], ref["families"], [r["verdict"] for r in recs], ref["verdict"],
                    [r["gate3"] for r in recs], ref["gate3"], [r["box_sum"] for r in recs], ref["box_sum"],
                    "OK" if good else "MISMATCH"), flush=True)
                ok = ok and good
        eng.close()
        if one is not None:
            one.close()
    return ok


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local_rank = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local_rank)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    pr = cosmo_b200.problems
    cases = [("qp_default", pr.random_sparse_qp(600, 1500, 0.05, seed=4), dict()),
             ("qp_scaled_off", pr.random_sparse_qp(600, 1500, 0.05, seed=5), dict(scaling=0)),
             ("socp", pr.portfolio_socp(n=300, k=30, seed=2), dict(max_iter=3000, scaling=0)),
             ("sdp", pr.closest_correlation_sdp(N=24, seed=7), dict(scaling=0)),
             # Anderson acceleration over sharded rows: inner products = local part (+ w_x on rank 0) + allreduce
             ("qp_accelerated", pr.random_sparse_qp(600, 1500, 0.05, seed=4), dict(accelerator="AndersonAccelerator")),
             ("socp_accelerated", pr.portfolio_socp(n=300, k=30, seed=2),
              dict(max_iter=3000, scaling=0, accelerator="AndersonAccelerator")),
             # the same two at eps = 1e-8: the distance between two accelerated runs scales with the stopping tolerance
             ("qp_accel_1e-8", pr.random_sparse_qp(600, 1500, 0.05, seed=4),
              dict(accelerator="AndersonAccelerator", eps_abs=1e-8, eps_rel=1e-8, max_iter=20000)),
             ("socp_accel_1e-8", pr.portfolio_socp(n=300, k=30, seed=2),
              dict(max_iter=20000, scaling=0, accelerator="AndersonAccelerator", eps_abs=1e-8, eps_rel=1e-8))]
    ok = True
    for name, (P, q, A, b, sets), kw in cases:
        st = cosmo_b200.Settings(**kw)
        m, n = A.shape
        if st.scaling != 0:
            Ps, qs, As, bs, ss, D, E, c = cosmo_b200.ruiz_equilibrate(P, q, A, b, sets, st)
        else:
            Ps, qs, As, bs, ss, D, E, c = P, q, A, b, sets, None, None, 1.0
        sh = sharding.make_shard(Ps, qs, As, bs, ss, rank, world)
        eng = sharding.create_engine(sh, st, device=local_rank, dist=dist, D=D, E=E, c=c)
        out = eng.solve()
        x = out.x if D is None else D * out.x
        s = gather_rows(out.s, sh.rows, m, world)
        mu = gather_rows(out.mu, sh.rows, m, world)
        if E is not None:
            s, mu = s / E, E * mu / c
        if rank == 0:
            okw = dict(kw)
            if okw.pop("accelerator", None) == "AndersonAccelerator":
                okw["accelerator"] = "anderson"
            ref = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(kkt_solver="cg", **okw))
            # Accelerated runs are chaotic in the rounding of the inner products (the Anderson least-squares problem
            # amplifies the different summation order of the sharded reductions): both runs converge to the same
            # point, their distance is a few stopping tolerances.  Measured on 2 GPUs:
            # socp_accelerated at eps = 1e-5: dx 7.8e-6, ds 2.6e-5, dmu 1.3e-7 with equal status and iteration count;
            # at eps = 1e-8 the distance drops to 3e-7 / 5e-7 / 1e-8 while the iteration counts differ (1962 vs 3438):
            # the bound is 5 eps on x, s and mu separately; the eps = 1e-8 legs compare the end points only.
            accel = "accelerator" in kw
            tight = accel and kw.get("eps_abs", 1e-5) < 1e-6
            tol = (5e-6 if tight else 5e-5) if accel else 1e-5
            tol_sm = tol
            good = ((tight or out.status == ref.status) and abs(out.obj_val - ref.obj_val) <= tol * max(1, abs(ref.obj_val))
                    and np.max(np.abs(x - ref.x)) <= tol * max(1, np.abs(ref.x).max())
                    and np.max(np.abs(s - ref.s)) <= tol_sm * max(1, np.abs(ref.s).max())
                    and np.max(np.abs(-mu - ref.y)) <= tol_sm * max(1, np.abs(ref.y).max()))
            print("%-16s world=%d status=%s/%s iter=%d/%d obj=%.9g/%.9g dx=%.2e ds=%.2e dmu=%.2e (scales %.2g %.2g %.2g) %s" % (
                name, world, out.status, ref.status, out.iter, ref.iter, out.obj_val, ref.obj_val,
                np.max(np.abs(x - ref.x)), np.max(np.abs(s - ref.s)), np.max(np.abs(-mu - ref.y)),
                max(1, np.abs(ref.x).max()), max(1, np.abs(ref.s).max()), max(1, np.abs(ref.y).max()),
                "OK" if good else "MISMATCH"), flush=True)
            ok = ok and good
        eng.close()
    ok = check_infeasibility_hook(rank, world, local_rank) and ok
    flag = torch.tensor([1 if ok else 0], device="cuda")
    dist.broadcast(flag, src=0)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
