"""Timing of the forward derivative of conic solutions through the fixed point (cosmo_b200_solve_derivative) on one GPU,
beside the solve adjoint and the solve they follow.  Prints the card and its power limit first, then one JSON line per
(workload, plugin), on the workloads of tests/run_solve_adjoint_timing.py.

After a warm-up (scratch allocated, graphs captured), five rounds each run a solve from a cold start (reset), a solve
adjoint with random incoming gradients of x, y and s, and a solve derivative along a random direction of q, b and A,
into host arrays; every call is synchronous.  Reported: the medians and ranges of the three wall times and both calls'
statistics (operator applications, inner iterations, final residual, kink counts)."""
import json
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M
from tests.run_polish_timing import med
from tests.run_solve_adjoint_timing import card, psd_batch


def main():
    print(json.dumps({"card": card()}), flush=True)
    work = [("portfolio_socp n=2000 k=200", cosmo_b200.problems.portfolio_socp(2000, 200), "DeviceSupernodalKKTSolver"),
            ("portfolio_socp n=2000 k=200", cosmo_b200.problems.portfolio_socp(2000, 200), "CGIndirectKKTSolver"),
            ("closest_correlation_sdp N=200", cosmo_b200.problems.closest_correlation_sdp(200), "CGIndirectKKTSolver"),
            ("psd batch 200 x N=6", psd_batch(), "DeviceSupernodalKKTSolver")]
    for name, (P, q, A, b, sets), plugin in work:
        P, A = sp.csc_matrix(P), sp.csc_matrix(A)
        m, n = A.shape
        rng = np.random.default_rng(0)
        gx, gy, gs = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)
        dq, db, dAx = rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(A.nnz)
        st = cosmo_b200.Settings(kkt_solver=plugin).to_struct()
        eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, equilibrate=True)
        outs = [np.empty(k) for k in (n, m, eng.nnzP, eng.nnzA, m, m)]
        douts = [np.empty(k) for k in (n, m, m)]
        eng.solve()
        eng.solve_adjoint(gx, gy, gs)            # warm-up
        eng.solve_derivative(dq=dq, db=db, dAx=dAx)
        t_solve, t_adj, t_der = [], [], []
        for k in range(5):
            eng.reset()
            t0 = time.perf_counter()
            out = eng.solve(copy_out=False)
            t_solve.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            _, ast = eng.solve_adjoint(gx, gy, gs, dq=outs[0], db=outs[1], dPx=outs[2], dAx=outs[3], dl=outs[4],
                                       du=outs[5])
            t_adj.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            _, dst = eng.solve_derivative(dq=dq, db=db, dAx=dAx, dx=douts[0], dy=douts[1], ds=douts[2])
            t_der.append(time.perf_counter() - t0)
        line = {"workload": name, "plugin": plugin, "n": n, "m": m, "nnzA": int(A.nnz), "solve_iter": out.iter,
                "solve_status": out.status, "solve_s": med(t_solve), "solve_adjoint_s": med(t_adj),
                "solve_derivative_s": med(t_der), "adjoint_stats": ast, "derivative_stats": dst}
        print(json.dumps(line), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
