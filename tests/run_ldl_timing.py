"""Timing of the direct LDL' KKT plugin on one GPU: symbolic analysis, factorisation, KKT phase per ADMM iteration,
levels, kernel launches per solve, nnz(L), and time to Solved against the CG plugin.  Prints the card and its power
limit first, then one JSON line per workload: C5 MAXCUT |V| = 10 000 (chordal, parent_child), the portfolio SOCP
n = 2000, k = 200, and the closest correlation matrix N = 200."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cosmo_b200
from cosmo_b200 import chordal


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:                      # the measurement still runs; the line says why the card is unknown
        return "nvidia-smi failed: %r" % (e,)


def workloads():
    rows, cols, w = cosmo_b200.problems.banded_random_graph(10_000, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(10_000, rows, cols, w)
    P2, q2, A2, b2, sets2, _ = chordal.decompose(P, q, A, b, sets, merge="parent_child")
    yield "C5 MAXCUT |V|=10000 chordal parent_child", (P2, q2, A2, b2, sets2)
    yield "portfolio SOCP n=2000 k=200", cosmo_b200.problems.portfolio_socp(2000, 200, seed=1)
    yield "closest correlation N=200", cosmo_b200.problems.closest_correlation_sdp(N=200)


def main():
    print(json.dumps({"card": card()}), flush=True)
    for name, (P, q, A, b, sets) in workloads():
        line = {"workload": name, "n": int(A.shape[1]), "m": int(A.shape[0])}
        # fixed iteration count with the phase timers on: KKT phase time per iteration (the solve graph + fused tail)
        iters = 200
        for plugin in ("DeviceLdlKKTSolver", "CGIndirectKKTSolver"):
            model = cosmo_b200.Model()
            model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=plugin, max_iter=iters, eps_abs=0.0, eps_rel=0.0,
                                                            adaptive_rho=False, verbose_timing=True))
            res = model.optimize()
            key = "ldl" if plugin.startswith("Device") else "cg"
            line[key + "_kkt_ms_per_iter"] = 1e3 * res.times["kkt_time"] / max(res.iter, 1)
            line[key + "_iter_ms_device"] = 1e3 * res.times["iter_time_device"] / max(res.iter, 1)
            if key == "ldl":
                st = model.engine.ldl_stats()
                line.update({"N": st["N"], "nnz_triu_K": st["nnz_triu_K"], "nnz_L": st["nnz_L"], "levels": st["levels"],
                             "solve_graph_nodes": st["solve_nodes"], "symbolic_s": st["symbolic_time"],
                             "factor_ms": 1e3 * st["factor_time"]})
                # refactorisations on a warm handle: the factor graph replayed after update_rho
                eng = model.engine
                rv = eng.rho_vec()
                times = []
                for k in range(5):
                    eng.update_rho(rv * (1.0 + 0.1 * (k + 1)), 0.1)
                    eng.kkt_solve(np.ones(eng.n + eng.m))
                    times.append(eng.ldl_stats()["factor_time"])
                line["refactor_ms_median"] = 1e3 * float(np.median(times))
        # time to Solved with default settings
        for plugin in ("DeviceLdlKKTSolver", "CGIndirectKKTSolver"):
            model = cosmo_b200.Model()
            model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=plugin, max_iter=5000))
            t0 = time.perf_counter()
            res = model.optimize()
            key = "ldl" if plugin.startswith("Device") else "cg"
            line[key + "_to_solved"] = {"status": res.status, "iter": int(res.iter), "wall_s": time.perf_counter() - t0,
                                        "solver_s": res.times["solver_time"], "obj": res.obj_val}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
