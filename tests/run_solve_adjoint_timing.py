"""Timing of the derivatives of conic solutions through the fixed point (cosmo_b200_solve_adjoint) on one GPU, against
the solve they follow.  Prints the card and its power limit first, then one JSON line per (workload, plugin):
portfolio_socp at n = 2000, k = 200 with the supernodal plugin and with CG, closest_correlation_sdp at N = 200, and a
seeded batch of small PSD cones.

After a warm-up (scratch allocated, graphs captured), five rounds each run a solve from a cold start (reset) and a
solve adjoint with random incoming gradients of x, y and s into host arrays; every call is synchronous.  Reported: the
medians and ranges of both wall times and the adjoint's statistics (operator applications, inner iterations, final
residual, kink counts)."""
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
from tests.run_polish_timing import card, med


def psd_batch(n_cones=200, N=6, seed=3):
    """min 1/2 |x|^2 + q'x over a batch of PsdConeTriangle constraints mat(b_k - A_k x) >= 0 with strictly feasible x = 0."""
    rng = np.random.default_rng(seed)
    d = N * (N + 1) // 2
    n = 4 * n_cones
    iu = np.triu_indices(N)
    order = np.lexsort((iu[0], iu[1]))
    eye = np.where(iu[0][order] == iu[1][order], 1.0, 0.0)
    blocks = [sp.random(d, n, density=8.0 / n, random_state=seed + k) for k in range(n_cones)]
    A = sp.csc_matrix(sp.vstack(blocks))
    b = np.tile(eye, n_cones)
    q = rng.standard_normal(n)
    sets = [cosmo_b200.PsdConeTriangle(d) for _ in range(n_cones)]
    return sp.identity(n, format="csc"), q, A, b, sets


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
        st = cosmo_b200.Settings(kkt_solver=plugin).to_struct()
        eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, equilibrate=True)
        outs = [np.empty(k) for k in (n, m, eng.nnzP, eng.nnzA, m, m)]
        eng.solve()
        eng.solve_adjoint(gx, gy, gs)            # warm-up
        t_solve, t_adj = [], []
        for k in range(5):
            eng.reset()
            t0 = time.perf_counter()
            out = eng.solve(copy_out=False)
            t_solve.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            _, ast = eng.solve_adjoint(gx, gy, gs, dq=outs[0], db=outs[1], dPx=outs[2], dAx=outs[3], dl=outs[4],
                                       du=outs[5])
            t_adj.append(time.perf_counter() - t0)
        line = {"workload": name, "plugin": plugin, "n": n, "m": m, "nnzA": int(A.nnz), "solve_iter": out.iter,
                "solve_status": out.status, "solve_s": med(t_solve), "solve_adjoint_s": med(t_adj), "stats": ast}
        print(json.dumps(line), flush=True)
        eng.close()


if __name__ == "__main__":
    main()
