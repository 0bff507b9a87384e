"""Timing of solution polishing (cosmo_b200_polish) on one GPU, against the solve it follows.  Prints the card and its
power limit first, then one JSON line per (workload, plugin): random_sparse_qp at n = 2000, m = 4000 and at
n = 5000, m = 10000, with the direct LDL' plugin and the supernodal one.

Five rounds alternate a solve followed by a polish with a solve alone, each from a cold start (reset).  Reported: the
medians and ranges of the solve and of the polish wall time (both calls are synchronous), the polish factorisation
time (ldl_stats after the polish), the polish outcome and the residuals before and after.  The bytes per polish are
estimated from the shapes (DESIGN.md §3i)."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cosmo_b200
from cosmo_b200 import engine as E
from cosmo_b200 import model as M


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:                      # the measurement still runs; the line says why the card is unknown
        return "nvidia-smi failed: %r" % (e,)


def polish_bytes(P, A, nnzL, refine_iter):
    """Bytes one polish streams, fp64, counted from the shapes: one factorisation (read K, write and read L), the
    refine_iter + 1 solves (L twice), the refine_iter + 1 residual passes (A, A' and P: 12 B per nonzero plus the
    vectors) and the finishing pass (A once more, the projection and the two compute_residuals of 3 passes each)."""
    n, m = A.shape[1], A.shape[0]
    spmv = lambda nnz, rows, cols: 12.0 * nnz + 4.0 * rows + 8.0 * (rows + cols)
    res_pass = spmv(A.nnz, m, n) + spmv(A.nnz, n, m) + spmv(P.nnz, n, n)
    factor = 12.0 * (P.nnz + A.nnz) + 3 * 12.0 * nnzL
    solves = (refine_iter + 1) * 2 * 12.0 * nnzL
    finish = spmv(A.nnz, m, n) + 2 * res_pass + 8.0 * 6 * m
    return factor + solves + (refine_iter + 1) * res_pass + finish


def med(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}


def main():
    print(json.dumps({"card": card()}), flush=True)
    for n, m in ((2000, 4000), (5000, 10000)):
        P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(n, m, 0.01, seed=2)
        for plugin in ("DeviceLdlKKTSolver", "DeviceSupernodalKKTSolver"):
            if plugin == "DeviceLdlKKTSolver" and n > 2000:
                # the simplicial factor is already 2.2 s at n = 2000 (H100, 700 W); 11 solves of several
                # factorisations each do not fit one measurement call at n = 5000
                print(json.dumps({"workload": "random_sparse_qp n=%d m=%d" % (n, m), "plugin": plugin,
                                  "skipped": "simplicial factor too slow at this size"}), flush=True)
                continue
            st = cosmo_b200.Settings(kkt_solver=plugin).to_struct()
            eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, equilibrate=True)
            eng.solve()
            eng.polish()                         # warm-up: graphs captured, scratch allocated
            t_solve, t_solve_alone, t_polish, t_factor, outs = [], [], [], [], []
            for k in range(5):
                for with_polish in (True, False):
                    eng.reset()
                    t0 = time.perf_counter()
                    out = eng.solve(copy_out=False)
                    ts = time.perf_counter() - t0
                    if not with_polish:
                        t_solve_alone.append(ts)
                        continue
                    t_solve.append(ts)
                    t0 = time.perf_counter()
                    _, _, _, pst = eng.polish(x=np.empty(n), y=np.empty(m), s=np.empty(m))
                    t_polish.append(time.perf_counter() - t0)
                    t_factor.append(eng.ldl_stats()["factor_time"])
                    outs.append((out, pst))
            out, pst = outs[-1]
            ls = eng.ldl_stats()
            line = {"workload": "random_sparse_qp n=%d m=%d" % (n, m), "plugin": plugin, "nnzA": int(A.nnz),
                    "nnzP": int(P.nnz), "solve_iter": out.iter, "solve_status": out.status,
                    "solve_s": med(t_solve), "solve_alone_s": med(t_solve_alone), "polish_s": med(t_polish),
                    "polish_factor_s": med(t_factor), "polish_status": pst["status"],
                    "active": [pst["n_lower"], pst["n_upper"], pst["n_equality"]],
                    "r_prim": [out.r_prim, pst["r_prim"]], "r_dual": [out.r_dual, pst["r_dual"]],
                    "refine_residual": pst["refine_residual"], "nnz_L": ls["nnz_L"],
                    "polish_bytes_est": polish_bytes(P, A, ls["nnz_L"], 3)}
            print(json.dumps(line), flush=True)
            eng.close()


if __name__ == "__main__":
    main()
