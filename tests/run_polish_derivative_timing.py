"""Timing of the forward derivative of a polished solution (cosmo_b200_derivative) against the adjoint
(cosmo_b200_adjoint) on the same polished point, on one GPU.  Prints the card and its power limit first, then one JSON
line per (workload, plugin): random_sparse_qp with scaling = 10 at n = 2000, m = 4000 with the simplicial and the
supernodal LDL' plugin, and at n = 5000, m = 10000 with the supernodal one (DESIGN.md §3j's workloads).

After one solve and one polish, and a warm-up call of each (scratch allocated, the A map derived), the two calls
alternate five times, each synchronous, with host arrays: a random direction of every input for the derivative,
random gradients of x, y and s for the adjoint.  Reported: the medians and ranges of the two wall times, both calls'
statistics and the bytes per derivative counted from the shapes."""
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


def derivative_bytes(P, A, nnzL, refine_iter):
    """Bytes one derivative streams, fp64, counted from the shapes (DESIGN.md §3j): dP x with P's value map (index,
    map, value: 12 B per entry of P plus the vectors), dA' y over CSR(A') (index and value), dA x over CSR(A) with the
    CSR -> CSC map (index, map, value: 16 B per entry), refine_iter + 1 solves (L twice each), refine_iter + 1 residual
    passes (A, A' and P: 12 B per nonzero plus the vectors), one pass over A for ds and the vectors."""
    n, m = A.shape[1], A.shape[0]
    spmv = lambda nnz, rows, cols: 12.0 * nnz + 4.0 * rows + 8.0 * (rows + cols)
    rhs_x = 12.0 * P.nnz + 12.0 * A.nnz + 8.0 * (2 * n + n + m) + 8.0 * 2 * n
    rhs_s = 16.0 * A.nnz + 8.0 * (n + m) + 8.0 * 3 * m + 8.0 * 3 * m
    solves = (refine_iter + 1) * 2 * 12.0 * nnzL
    res_pass = spmv(A.nnz, m, n) + spmv(A.nnz, n, m) + spmv(P.nnz, n, n)
    slack = spmv(A.nnz, m, n) + 8.0 * m
    vec = 8.0 * (4 * n + 9 * m) + 8.0 * (2 * n + 4 * m)
    return rhs_x + rhs_s + solves + (refine_iter + 1) * res_pass + slack + vec


def main():
    print(json.dumps({"card": card()}), flush=True)
    for n, m, plugins in ((2000, 4000, ("DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver")),
                          (5000, 10000, ("DeviceSupernodalKKTSolver",))):
        P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(n, m, 0.01, seed=2)
        rng = np.random.default_rng(0)
        gx, gy, gs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
        d = dict(dPx=rng.standard_normal(P.nnz), dq=rng.standard_normal(n), dAx=rng.standard_normal(A.nnz),
                 db=rng.standard_normal(m), dl=rng.standard_normal(m), du=rng.standard_normal(m))
        adj_outs = [np.empty(k) for k in (n, m, P.nnz, A.nnz, m, m)]
        der_outs = dict(dx=np.empty(n), dy=np.empty(m), ds=np.empty(m))
        for plugin in plugins:
            st = cosmo_b200.Settings(kkt_solver=plugin, scaling=10).to_struct()
            eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, equilibrate=True)
            out = eng.solve(copy_out=False)
            _, _, _, pst = eng.polish(x=np.empty(n), y=np.empty(m), s=np.empty(m))
            eng.adjoint(gx, gy, gs, 3, *adj_outs)              # warm-up
            eng.derivative(**d, refine_iter=3, **der_outs)
            t_adj, t_der = [], []
            for k in range(5):
                t0 = time.perf_counter()
                _, ast = eng.adjoint(gx, gy, gs, 3, *adj_outs)
                t_adj.append(time.perf_counter() - t0)
                t0 = time.perf_counter()
                _, dst = eng.derivative(**d, refine_iter=3, **der_outs)
                t_der.append(time.perf_counter() - t0)
            ls = eng.ldl_stats()
            line = {"workload": "random_sparse_qp n=%d m=%d scaling=10" % (n, m), "plugin": plugin,
                    "nnzA": int(A.nnz), "nnzP": int(P.nnz), "solve_iter": out.iter, "solve_status": out.status,
                    "polish_status": pst["status"], "adjoint_s": med(t_adj), "derivative_s": med(t_der),
                    "adjoint": ast, "derivative": dst, "nnz_L": ls["nnz_L"],
                    "derivative_bytes_est": derivative_bytes(P, A, ls["nnz_L"], 3)}
            print(json.dumps(line), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
