"""Timing of the supernodal LDL' KKT plugin (code 4) against the simplicial one (code 3) and CG on one GPU.  Prints
the card and its power limit first, then one JSON line per workload: C5 MAXCUT |V| = 10 000 (chordal, parent_child),
the portfolio SOCP n = 2000, k = 200, the closest correlation matrix N = 200 and the random QP n = 2000, m = 4000.
Per plugin, alternating and `--runs` times each (median reported): symbolic time, factor time on a warm handle after
update_rho, KKT phase per iteration from the phase timers, iterations and time to Solved; the supernode stats; and the
largest differences in x, s and mu between codes 4 and 3 at Solved."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cosmo_b200
from cosmo_b200 import chordal

PLUGINS = {"sn": "DeviceSupernodalKKTSolver", "ldl": "DeviceLdlKKTSolver", "cg": "CGIndirectKKTSolver"}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:
        return "nvidia-smi failed: %r" % (e,)


def workloads(only):
    if "c5" in only:
        rows, cols, w = cosmo_b200.problems.banded_random_graph(10_000, 3.0, 20, seed=1)
        P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(10_000, rows, cols, w)
        P2, q2, A2, b2, sets2, _ = chordal.decompose(P, q, A, b, sets, merge="parent_child")
        yield "C5 MAXCUT |V|=10000 chordal parent_child", (P2, q2, A2, b2, sets2)
    if "portfolio" in only:
        yield "portfolio SOCP n=2000 k=200", cosmo_b200.problems.portfolio_socp(2000, 200, seed=1)
    if "corr" in only:
        yield "closest correlation N=200", cosmo_b200.problems.closest_correlation_sdp(N=200)
    if "qp" in only:
        yield "random QP n=2000 m=4000", cosmo_b200.problems.random_sparse_qp(2000, 4000, 0.002, seed=0)


def one_run(key, P, q, A, b, sets, iters):
    out = {}
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=PLUGINS[key], max_iter=iters, eps_abs=0.0, eps_rel=0.0,
                                                    adaptive_rho=False, verbose_timing=True))
    res = model.optimize()
    out["kkt_ms_per_iter"] = 1e3 * res.times["kkt_time"] / max(res.iter, 1)
    if key != "cg":
        eng = model.engine
        st = eng.ldl_stats()
        out["symbolic_s"] = st["symbolic_time"]
        rv = eng.rho_vec()
        times = []
        for k in range(3):
            eng.update_rho(rv * (1.0 + 0.1 * (k + 1)), 0.1)
            eng.kkt_solve(np.ones(eng.n + eng.m))
            times.append(eng.ldl_stats()["factor_time"])
        out["refactor_ms"] = 1e3 * float(np.median(times))
        out["ldl_stats"] = {k: st[k] for k in ("N", "nnz_L", "levels", "solve_nodes")}
        if key == "sn":
            out["sn_stats"] = eng.ldl_sn_stats()
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(kkt_solver=PLUGINS[key], max_iter=5000))
    t0 = time.perf_counter()
    res = model.optimize()
    out["to_solved"] = {"status": res.status, "iter": int(res.iter), "wall_s": time.perf_counter() - t0}
    return out, (res.x, res.s, res.y)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--only", default="c5,portfolio,corr,qp")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for name, (P, q, A, b, sets) in workloads(args.only.split(",")):
        runs = {k: [] for k in PLUGINS}
        sol = {}
        for _ in range(args.runs):
            for key in PLUGINS:                    # alternating: sn, ldl, cg, sn, ...
                r, s = one_run(key, P, q, A, b, sets, args.iters)
                runs[key].append(r)
                sol[key] = s
        line = {"workload": name, "n": int(A.shape[1]), "m": int(A.shape[0])}
        for key, rs in runs.items():
            med = lambda f: float(np.median([f(r) for r in rs]))
            d = {"kkt_ms_per_iter": med(lambda r: r["kkt_ms_per_iter"]),
                 "to_solved_s": med(lambda r: r["to_solved"]["wall_s"]),
                 "status": rs[-1]["to_solved"]["status"], "iter": rs[-1]["to_solved"]["iter"]}
            if key != "cg":
                d.update(symbolic_s=med(lambda r: r["symbolic_s"]), refactor_ms=med(lambda r: r["refactor_ms"]),
                         **rs[-1]["ldl_stats"])
            if key == "sn":
                d["sn_stats"] = rs[-1]["sn_stats"]
            line[key] = d
        line["max_diff_sn_ldl"] = {v: float(np.max(np.abs(a - c))) if a.size else 0.0
                                   for v, a, c in zip(("x", "s", "mu"), sol["sn"], sol["ldl"])}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
