"""Timing of the derivatives through custom cones with the Jacobian hook (COSMO_B200_CUSTOM_HAS_JACOBIAN) on one GPU:
portfolio_socp(n=2000, k=200) with its second-order cone built in (SecondOrderCone) and as the hooked custom type
soc2_jac of tests/custom_cone_jacobians.py, with the supernodal LDL' and the CG plugin.  Prints the card and its power
limit first, then one JSON line per (plugin, variant), then one line of the Dpi kernel times per (plugin, variant).

Both calls run a fixed number of operator applications (tol below any reachable residual, max_iter = APPS), so the two
variants do the same work apart from Dpi.  After a warm-up, five rounds alternate the variants; each round runs one
solve_adjoint and one solve_derivative into host arrays, synchronously.  Reported: the median and range of the wall
time per operator application.  The Dpi kernel times come from a separate torch.profiler run of one call of each kind:
the SOC kernels of sa_dpi (sa_soc_dot_chunk_kernel, sa_soc_dot_final_kernel) and sa_dpi_rows_kernel for the built-in
cone, sa_dpi_rows_kernel and cosmo_custom_jacobian for the custom one, per operator application."""
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
from tests import custom_cone_jacobians as CJ
from tests.run_solve_adjoint_timing import card

APPS = 200
KW = dict(tol=1e-30, max_iter=APPS)
DPI_KERNELS = ("sa_soc_dot_chunk_kernel", "sa_soc_dot_final_kernel", "sa_dpi_rows_kernel", "cosmo_custom_jacobian")


def _variants():
    P, q, A, b, sets = cosmo_b200.problems.portfolio_socp(2000, 200)
    custom = sets[:-1] + [M.CustomCone(CJ.soc2_type(), sets[-1].dim)]
    return sp.csc_matrix(P), q, sp.csc_matrix(A), b, {"builtin": sets, "custom": custom}


def _engine(P, q, A, b, sets, plugin):
    st = cosmo_b200.Settings(kkt_solver=plugin).to_struct()
    eng = E.Engine(P, q, A, b, [M.set_tuple(S) for S in sets], st, equilibrate=True)
    eng.solve()
    return eng


def _rng_inputs(n, m, nnzA):
    rng = np.random.default_rng(0)
    return (rng.standard_normal(n), rng.standard_normal(m), rng.standard_normal(m)), \
        dict(dq=rng.standard_normal(n), db=rng.standard_normal(m), dAx=rng.standard_normal(nnzA))


def wall(P, q, A, b, variants, plugin):
    m, n = A.shape
    g, d = _rng_inputs(n, m, A.nnz)
    engs = {k: _engine(P, q, A, b, s, plugin) for k, s in variants.items()}
    for e in engs.values():                                 # warm-up: scratch, graphs
        e.solve_adjoint(*g, **KW)
        e.solve_derivative(**d, **KW)
    times = {k: {"adjoint": [], "derivative": []} for k in engs}
    stats = {}
    for _ in range(5):
        for k, e in engs.items():
            t0 = time.perf_counter()
            _, ast = e.solve_adjoint(*g, **KW)
            times[k]["adjoint"].append((time.perf_counter() - t0) / ast["operator_applications"])
            t0 = time.perf_counter()
            _, dst = e.solve_derivative(**d, **KW)
            times[k]["derivative"].append((time.perf_counter() - t0) / dst["operator_applications"])
            stats[k] = (ast, dst)
    for k, e in engs.items():
        line = {"workload": "portfolio_socp n=2000 k=200", "plugin": plugin, "variant": k, "n": n, "m": m}
        for call, ts in times[k].items():
            line[call + "_ms_per_application"] = {"median": 1e3 * float(np.median(ts)), "min": 1e3 * min(ts),
                                                  "max": 1e3 * max(ts)}
        line["adjoint_stats"], line["derivative_stats"] = stats[k]
        print(json.dumps(line), flush=True)
        e.close()


def kernels(P, q, A, b, variants, plugin):
    import torch
    from torch.profiler import ProfilerActivity, profile
    m, n = A.shape
    g, d = _rng_inputs(n, m, A.nnz)
    for k, sets in variants.items():
        eng = _engine(P, q, A, b, sets, plugin)
        eng.solve_adjoint(*g, **KW)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _, ast = eng.solve_adjoint(*g, **KW)
            _, dst = eng.solve_derivative(**d, **KW)
            torch.cuda.synchronize()
        apps = ast["operator_applications"] + dst["operator_applications"]
        us = {}
        for ev in prof.key_averages():
            name = next((kk for kk in DPI_KERNELS if kk in ev.key), None)
            if name:
                us[name] = us.get(name, 0.0) + ev.device_time_total / apps
        print(json.dumps({"plugin": plugin, "variant": k, "dpi_us_per_application": us,
                          "dpi_total_us_per_application": sum(us.values())}), flush=True)
        eng.close()


def main():
    print(json.dumps({"card": card()}), flush=True)
    P, q, A, b, variants = _variants()
    for plugin in ("DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"):
        wall(P, q, A, b, variants, plugin)
    for plugin in ("DeviceSupernodalKKTSolver", "CGIndirectKKTSolver"):
        kernels(P, q, A, b, variants, plugin)


if __name__ == "__main__":
    main()
