"""Timing of the derivatives of a polished solution (cosmo_b200_adjoint) on one GPU, against the solve and the polish it
follows.  Prints the card and its power limit first, then one JSON line per (workload, plugin): random_sparse_qp at
n = 2000, m = 4000 with the simplicial and the supernodal LDL' plugin, and at n = 5000, m = 10000 with the supernodal
one.

After a warm-up (graphs captured, scratch allocated), five rounds each run a solve from a cold start (reset), a polish
and an adjoint with random incoming gradients of x, y and s into host arrays; every call is synchronous.  Reported: the
medians and ranges of the three wall times, the polish factorisation time (ldl_stats after the polish), the
adjoint's statistics and the bytes per adjoint estimated from the shapes (DESIGN.md §3j)."""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from tests.run_polish_timing import card, med


def adjoint_bytes(P, A, nnzL, refine_iter):
    """Bytes one adjoint streams, fp64, counted from the shapes: the right-hand side (one pass over A'), refine_iter + 1
    solves (L twice each), refine_iter + 1 residual passes (A, A' and P: 12 B per nonzero plus the vectors), the vector
    gradients and the P and A gradient passes (index, value map and output per entry of P; index and output per entry
    of A, plus the vectors they gather)."""
    n, m = A.shape[1], A.shape[0]
    spmv = lambda nnz, rows, cols: 12.0 * nnz + 4.0 * rows + 8.0 * (rows + cols)
    res_pass = spmv(A.nnz, m, n) + spmv(A.nnz, n, m) + spmv(P.nnz, n, n)
    rhs = spmv(A.nnz, n, m) + 8.0 * 4 * m
    solves = (refine_iter + 1) * 2 * 12.0 * nnzL
    vec = 8.0 * (4 * n + 9 * m)
    grads = 16.0 * P.nnz + 4.0 * n + 8.0 * 3 * n + 12.0 * A.nnz + 4.0 * n + 8.0 * (3 * n + 4 * m)
    return rhs + solves + (refine_iter + 1) * res_pass + vec + grads


def main():
    print(json.dumps({"card": card()}), flush=True)
    for n, m, plugins in ((2000, 4000, ("DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver")),
                          (5000, 10000, ("DeviceSupernodalKKTSolver",))):
        P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(n, m, 0.01, seed=2)
        rng = np.random.default_rng(0)
        gx, gy, gs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
        outs = [np.empty(k) for k in (n, m, P.nnz, A.nnz, m, m)]
        for plugin in plugins:
            st = cosmo_b200.Settings(kkt_solver=plugin).to_struct()
            eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, equilibrate=True)
            eng.solve()
            eng.polish()
            eng.adjoint(gx, gy, gs)              # warm-up
            t_solve, t_polish, t_factor, t_adj = [], [], [], []
            for k in range(5):
                eng.reset()
                t0 = time.perf_counter()
                out = eng.solve(copy_out=False)
                t_solve.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                _, _, _, pst = eng.polish(x=np.empty(n), y=np.empty(m), s=np.empty(m))
                t_polish.append(time.perf_counter() - t0)
                t_factor.append(eng.ldl_stats()["factor_time"])
                t0 = time.perf_counter()
                _, ast = eng.adjoint(gx, gy, gs, 3, *outs)
                t_adj.append(time.perf_counter() - t0)
            ls = eng.ldl_stats()
            line = {"workload": "random_sparse_qp n=%d m=%d" % (n, m), "plugin": plugin, "nnzA": int(A.nnz),
                    "nnzP": int(P.nnz), "solve_iter": out.iter, "solve_status": out.status, "solve_s": med(t_solve),
                    "polish_s": med(t_polish), "polish_factor_s": med(t_factor), "adjoint_s": med(t_adj),
                    "polish_status": pst["status"], "adjoint": ast, "nnz_L": ls["nnz_L"],
                    "factorizations": ls["factorizations"], "adjoint_bytes_est": adjoint_bytes(P, A, ls["nnz_L"], 3)}
            print(json.dumps(line), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
