"""C5 (MAXCUT dual SDP on the banded graph, default |V| = 2000): the compact and the traditional transformation side by
side.  For each: the size of the decomposed problem (n', m', nnz(A')), the host time of chordal.decompose (median of
`repeats`), then one solve to Solved with the settings of the benchmark: iterations, iteration time and iter/s from the
engine's timers.

Usage: python tests/run_traditional_timing.py [|V|] [repeats] [merge] [solver]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

import cosmo_b200  # noqa: E402
from cosmo_b200 import chordal, model as M  # noqa: E402

MERGE = {"CliqueGraphMerge": "clique_graph", "ParentChildMerge": "parent_child_reference", "NoMerge": "none"}


def main():
    nv = int(sys.argv[1]) if len(sys.argv) > 1 else 2000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    merge = sys.argv[3] if len(sys.argv) > 3 else "CliqueGraphMerge"
    solver = sys.argv[4] if len(sys.argv) > 4 else "CGIndirectKKTSolver"
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement needs the GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
    rows, cols, w = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    P, A = M._sorted_csc(P), M._sorted_csc(A)
    for compact in (True, False):
        out = {"card": card, "nv": nv, "merge": merge, "kkt_solver": solver, "compact_transformation": compact,
               "n": A.shape[1], "m": A.shape[0]}
        t = []
        for _ in range(reps):
            t0 = time.perf_counter()
            P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge=MERGE[merge], compact=compact)
            t.append(time.perf_counter() - t0)
        out.update({"n_decomposed": A2.shape[1], "m_decomposed": A2.shape[0], "nnzA_decomposed": int(A2.nnz),
                    "cliques": len(info.clique_sizes), "largest_clique": max(info.clique_sizes),
                    "decompose_s_median": float(np.median(t)), "decompose_s_min": float(np.min(t))})
        model = cosmo_b200.Model()
        model.set(P, q, A, b, sets, cosmo_b200.Settings(decompose=True, merge_strategy=merge, kkt_solver=solver,
                                                        compact_transformation=compact))
        res = model.optimize()
        model.empty_model()
        it_time = res.times.get("iter_time_device") or res.times.get("iter_time")
        out.update({"status": res.status, "iterations": int(res.iter), "obj_val": float(res.obj_val),
                    "setup_time_s": float(res.times["setup_time"]), "iter_time_s": float(it_time),
                    "iter_per_s": float(res.iter / it_time) if it_time else None})
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
