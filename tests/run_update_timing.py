"""Engine creation against cosmo_b200_update_matrices on config C2 at full size with the bench.py settings (CG, scaling 0,
fixed rho, cold start), and the ADMM rate of an updated engine against a fresh one.

create, first update (uploads the value maps) and later updates: median of 5 with the spread (min-max); the rate is
iterations / device iteration time of a --steps solve, fresh and updated engines alternating.  Prints one JSON line per
measurement with the card name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import cosmo_b200
from cosmo_b200 import engine as E


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, check=True).stdout.splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return "unknown", "unknown"


def stats(ts):
    return {"median_s": statistics.median(ts), "min_s": min(ts), "max_s": max(ts), "runs": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50_000)
    ap.add_argument("--m", type=int, default=100_000)
    ap.add_argument("--density", type=float, default=0.01)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    a = ap.parse_args()
    name, power = card()
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(a.n, a.m, a.density, a.seed)
    P.sort_indices()
    A.sort_indices()
    rng = np.random.default_rng(a.seed + 1)
    A2 = A.data * (1.0 + 0.01 * rng.standard_normal(A.nnz))          # same pattern, new values (still 9 B)
    P2 = P.data * 1.01
    tuples = [cosmo_b200.model.set_tuple(S) for S in sets]
    st = cosmo_b200.Settings(scaling=0, adaptive_rho=False, max_iter=a.steps, eps_abs=0.0, eps_rel=0.0).to_struct()
    base = {"workload": "C2 n=%d m=%d density=%g nnz(A)=%d" % (a.n, a.m, a.density, A.nnz), "gpu": name,
            "power_limit": power}

    def timed(fn):
        t0 = time.perf_counter()
        r = fn()
        return time.perf_counter() - t0, r

    creates, firsts = [], []
    eng = None
    for i in range(a.reps):
        if eng is not None:
            eng.close()
        t, eng = timed(lambda: E.Engine(P, q, A, b, tuples, st))
        creates.append(t)
        firsts.append(timed(lambda: eng.update_matrices(P2, A2))[0])
    later = []
    for i in range(a.reps):
        vals = (P.data, A.data) if i % 2 == 0 else (P2, A2)
        later.append(timed(lambda: eng.update_matrices(*vals))[0])
    print(json.dumps(dict(base, what="create", **stats(creates))), flush=True)
    print(json.dumps(dict(base, what="first update", **stats(firsts))), flush=True)
    print(json.dumps(dict(base, what="later update", **stats(later))), flush=True)

    # the engine now holds (P2, A2) if reps is even, else the original values: compare with a fresh engine of the same data
    cur = (P.data, A.data) if a.reps % 2 == 1 else (P2, A2)
    Pf, Af = P.copy(), A.copy()
    Pf.data, Af.data = cur[0].copy(), cur[1].copy()
    fresh = E.Engine(Pf, q, Af, b, tuples, st)
    rates = {"updated": [], "fresh": []}
    for _ in range(3):
        for label, e in (("updated", eng), ("fresh", fresh)):
            e.reset()
            o = e.solve()
            rates[label].append(o.iter / o.times["iter_time_device"])
    for label, r in rates.items():
        print(json.dumps(dict(base, what="iterations/s after %s" % ("an update" if label == "updated" else "create"),
                              median=statistics.median(r), min=min(r), max=max(r), steps=a.steps)), flush=True)
    eng.close()
    fresh.close()


if __name__ == "__main__":
    main()
