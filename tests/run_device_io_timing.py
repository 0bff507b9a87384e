"""Host arrays against device arrays (torch CUDA tensors) for the calls that move a re-solve's data, alternating the
two paths; median of --reps with the range (min-max), wall time of each call (every call returns synchronised):

- C2 (bench.py's problem) update_matrices with all four arrays;
- C2 update_qb, then a --steps iteration solve, then the solution: host (update_qb + solve with copy-out + the host
  reverse_scaling!) against device (update_qb_original + solve without copy-out + cosmo_b200_solution into tensors);
- C5 (MAXCUT dual SDP, decomposed, --nv vertices): Model.update(q, b) with NumPy arrays against CUDA tensors, and the
  host copy-out + reverse against cosmo_b200_solution into tensors, without and with complete_dual.

Prints one JSON line per measurement with the card's name and power limit.
Usage: python tests/run_device_io_timing.py [--nv 10000] [--reps 5] [--skip-c5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cosmo_b200
from cosmo_b200 import engine as E


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, check=True).stdout.splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return "unknown", "unknown"


def stats(ts):
    return {"median_s": statistics.median(ts), "min_s": min(ts), "max_s": max(ts), "runs": len(ts)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def alternate(reps, host, device):
    th, td = [], []
    for _ in range(reps):
        th.append(timed(host))
        td.append(timed(device))
    return stats(th), stats(td)


def emit(base, what, h, d):
    print(json.dumps(dict(base, what=what, host=h, device=d)), flush=True)


def c2(a, base):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(50_000, 100_000, 0.01, 2)
    P.sort_indices()
    A.sort_indices()
    st = cosmo_b200.Settings(scaling=0, adaptive_rho=False, max_iter=a.steps, eps_abs=0.0, eps_rel=0.0).to_struct()
    eng = E.Engine(P, q, A, b, [cosmo_b200.model.set_tuple(S) for S in sets], st)
    base = dict(base, workload="C2 n=50000 m=100000 density=0.01 nnz(A)=%d" % A.nnz)
    host = [P.data, A.data, q, b]
    dev = [torch.as_tensor(v, device="cuda") for v in host]
    eng.update_matrices(*host)                       # the value maps are made by the first update
    emit(base, "update_matrices (Px, Ax, q, b)", *alternate(a.reps, lambda: eng.update_matrices(*host),
                                                             lambda: eng.update_matrices(*dev)))
    xo, yo, so = (torch.empty(k, dtype=torch.float64, device="cuda") for k in (eng.n, eng.m, eng.m))

    def host_path():
        eng.update_qb(q, b)
        o = eng.solve()
        return o.x.astype(np.float64), -o.mu.astype(np.float64), o.s.astype(np.float64)   # D = E = 1, c = 1

    def device_path():
        eng.update_qb_original(dev[2], dev[3])
        eng.solve(copy_out=False)
        eng.solution(False, xo, yo, so)
    emit(base, "update_qb + %d iterations + solution" % a.steps, *alternate(a.reps, host_path, device_path))
    eng.close()


def c5(a, base):
    rows, cols, w = cosmo_b200.problems.banded_random_graph(a.nv, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(a.nv, rows, cols, w)
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(decompose=True, reverse_on_device=True, max_iter=50))
    model.optimize()
    base = dict(base, workload="C5 MAXCUT dual SDP |V|=%d, decomposed: n=%d m=%d, n'=%d m'=%d"
                % (a.nv, model.n, model.m, model.engine.n, model.engine.m))
    qh, bh = model.q0.copy(), model.b0.copy()
    qd, bd = torch.as_tensor(qh, device="cuda"), torch.as_tensor(bh, device="cuda")
    emit(base, "Model.update(q, b)", *alternate(a.reps, lambda: model.update(q=qh, b=bh), lambda: model.update(q=qd, b=bd)))
    eng = model.engine
    eng.solve(copy_out=False)
    xo, yo, so = (torch.empty(k, dtype=torch.float64, device="cuda") for k in (model.n, model.m, model.m))
    for cd in (False, True):
        def host_path():
            xs, ss, mus, _ = eng.reverse_decomposition(complete_dual=cd)
            return xs, -mus, ss
        emit(base, "solution (complete_dual=%s): reverse_decomposition to host vs solution into tensors" % cd,
             *alternate(a.reps, host_path, lambda: eng.solution(cd, xo, yo, so)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nv", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--skip-c5", action="store_true")
    a = ap.parse_args()
    name, power = card()
    base = {"gpu": name, "power_limit": power}
    c2(a, base)
    if not a.skip_c5:
        c5(a, base)


if __name__ == "__main__":
    main()
