"""Cost of custom cones on one GPU: NVRTC compile time per type (cold and cached), and the projection time per
iteration (ResultTimes.proj_time, CUDA events) and iterations per second of the `soc2` warp cone against the built-in
SecondOrderCone, on one large cone and on 10^5 small ones.  Prints one JSON line and writes it to --out.

    python tests/run_custom_cone_timing.py --out custom_cone_timing.json
"""
import argparse
import json
import os
import subprocess
import sys
import time
import uuid

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import cosmo_b200  # noqa: E402
from cosmo_b200 import model as M  # noqa: E402
from tests import custom_cones as CC  # noqa: E402


def gpu_name():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def compile_times():
    out = {}
    for make in (CC.nonpos_type, CC.soc2_type, CC.linf_type):
        k = make()
        fresh = M.CustomConeType(k.name, k.source + "// %s\n" % uuid.uuid4().hex, k.granularity, k.n_params, k.in_dual,
                                 k.in_pol_recc)
        t0 = time.perf_counter()
        assert fresh.compile()
        t1 = time.perf_counter()
        assert not fresh.compile()
        t2 = time.perf_counter()
        out[k.name] = {"cold_s": t1 - t0, "cached_s": t2 - t1}
    return out


def socp(dims, kind, seed=0):
    """min 1/2 |x|^2 + q'x s.t. A x + s = b, s in the cones of `dims`: A = [I; random], m = sum(dims) rows"""
    rng = np.random.default_rng(seed)
    m = int(sum(dims))
    n = 1000
    A = (sp.random(m, n, density=min(1.0, 4.0 / n), random_state=seed, format="csc") + sp.eye(m, n, format="csc")).tocsc()
    sets = [M.SecondOrderCone(d) if kind is None else M.CustomCone(kind, d) for d in dims]
    s0 = np.concatenate([np.concatenate([[np.linalg.norm(v) + 1.0], v]) for v in (rng.standard_normal(d - 1) for d in dims)])
    return sp.eye(n, format="csc"), rng.standard_normal(n), A, A @ rng.standard_normal(n) + s0, sets


def proj_timing(dims, iters):
    out = {}
    for name, kind in (("soc", None), ("soc2", CC.soc2_type())):
        P, q, A, b, sets = socp(dims, kind)
        model = cosmo_b200.Model()
        st = cosmo_b200.Settings(max_iter=iters, eps_abs=1e-14, eps_rel=1e-14, check_termination=iters,
                                 check_infeasibility=iters, adaptive_rho=False, verbose_timing=True, scaling=0)
        model.set(P, q, A, b, sets, st)
        model.optimize()                                   # warm-up: module loads, CG graphs
        res = model.optimize()
        out[name] = {"iter": res.iter, "proj_ms_per_iter": 1e3 * res.times["proj_time"] / res.iter,
                     "iter_per_s": res.iter / res.times["iter_time"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rec = {"gpu": gpu_name(), "compile": compile_times(),
           "one_cone_1e6": proj_timing([1_000_000], a.iters),
           "small_cones_1e5x10": proj_timing([10] * 100_000, a.iters)}
    line = json.dumps(rec)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
