"""C5 (MAXCUT dual SDP on the banded graph, default |V| = 10 000): what new weights cost a chordally decomposed model.

Route (a) is the rebuild a decomposed model paid for every update before the forward map: chordal analysis (elimination,
cliques, merge), augmentation (the rest of chordal.decompose), engine create (with the LDL' symbolic analysis inside,
reported apart from the engine's own timer), set_decomposition, and the forward map itself (forward_arrays +
set_forward_map, the one-off price of route (b)).  Route (b) is cosmo_b200_update_matrices_original on the live engine:
the first call (it derives the value maps) and later calls.  The two routes alternate; every figure is the median of
`repeats` with the range.  Wall clock around calls that end in a device synchronise.  Then the iterations to Solved after
a small change of the weights, from the kept clique iterates and from a cold fresh model.

Usage: python tests/run_decomposed_update_timing.py [|V|] [repeats] [merge,...] [solver,...]"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402

import cosmo_b200  # noqa: E402
from cosmo_b200 import chordal, engine as E, model as M  # noqa: E402

MERGE = {"CliqueGraphMerge": "clique_graph", "ParentChildMerge": "parent_child_reference"}


def _problem(nv, seed):
    rows, cols, _ = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=1)
    w = np.random.default_rng(seed).integers(1, 11, size=len(rows)).astype(np.float64)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    return M._sorted_csc(P), q, M._sorted_csc(A), b, sets


def _stat(t):
    return {"median_s": float(np.median(t)), "min_s": float(np.min(t)), "max_s": float(np.max(t))}


def _analysis(A, b, sets, merge):
    """the pattern analysis of chordal.decompose for the one PSD cone of C5, alone"""
    S = sets[0]
    Ar = sp.csr_matrix(A)
    nz = np.unique(np.concatenate([np.nonzero(np.diff(Ar.indptr))[0], np.nonzero(b)[0]]))
    ii, jj = chordal.svec_to_ij(nz)
    tree = chordal.chordal_cliques(S.sqrt_dim, ii, jj)
    return chordal.clique_graph_merge(tree) if merge == "clique_graph" else chordal.parent_child_merge_reference(tree)


def _rebuild(data, merge, st):
    """route (a), timed step by step; returns (times, engine, forward map)"""
    P, q, A, b, sets = data
    t = {}
    t0 = time.perf_counter()
    _analysis(A, b, sets, merge)
    t["chordal_analysis"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    P2, q2, A2, b2, sets2, info = chordal.decompose(P, q, A, b, sets, merge=merge)
    t["augmentation"] = time.perf_counter() - t0 - t["chordal_analysis"]      # decompose runs the analysis again
    t0 = time.perf_counter()
    eng = E.Engine(P2, q2, A2, b2, [M.set_tuple(S) for S in sets2], st.to_struct(), equilibrate=st.scaling != 0)
    eng.scaling()
    t["engine_create"] = time.perf_counter() - t0
    t["symbolic_analysis"] = eng.ldl_stats()["symbolic_time"]
    t0 = time.perf_counter()
    eng.set_decomposition(chordal.decomposition_arrays(info, eng.n, eng.m))
    t["set_decomposition"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    f = chordal.forward_arrays(info, A, eng.n, eng.m)
    eng.set_forward_map(f)
    t["forward_map"] = time.perf_counter() - t0
    t["rebuild_total"] = sum(v for k, v in t.items() if k not in ("symbolic_analysis", "forward_map"))
    return t, eng, f


def main():
    nv = int(sys.argv[1]) if len(sys.argv) > 1 else 10000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    merges = sys.argv[3].split(",") if len(sys.argv) > 3 else list(MERGE)
    solvers = sys.argv[4].split(",") if len(sys.argv) > 4 else ["CGIndirectKKTSolver", "DeviceLdlKKTSolver"]
    import torch
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this measurement needs the GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
    data = [_problem(nv, seed) for seed in (3, 4)]                        # two sets of weights on one graph
    for merge_name in merges:
        for solver in solvers:
            st = cosmo_b200.Settings(decompose=True, merge_strategy=merge_name, kkt_solver=solver)
            out = {"card": card, "nv": nv, "merge": merge_name, "kkt_solver": solver, "repeats": reps}
            steps, first, later = {}, [], []
            eng = None
            for r in range(reps):                                         # (a) and (b) alternate
                if eng is not None:
                    eng.close()
                t, eng, f = _rebuild(data[r % 2], MERGE[merge_name], st)
                for k, v in t.items():
                    steps.setdefault(k, []).append(v)
                for k in range(3):
                    P, q, A, b, _ = data[(r + k + 1) % 2]
                    t0 = time.perf_counter()
                    eng.update_matrices_original(P.data, A.data, q, b)
                    (first if k == 0 else later).append(time.perf_counter() - t0)
            out.update({"n_decomposed": eng.n, "m_decomposed": eng.m, "m_orig": f.m_orig, "nnzA_decomposed": len(f.a_src)})
            eng.close()
            out["rebuild"] = {k: _stat(v) for k, v in steps.items()}
            out["update_matrices_original_first"] = _stat(first)
            out["update_matrices_original_later"] = _stat(later)
            # iterations to Solved after a small change of the weights
            P, q, A, b, sets = data[0]
            b2 = b * (1.0 + 1e-3 * np.random.default_rng(9).standard_normal(len(b)))
            model = cosmo_b200.Model()
            model.set(P, q, A, b, sets, st)
            r0 = model.optimize()
            model.update(b=b2, A=A)
            kept = model.engine is not None
            rw = model.optimize()
            model.empty_model()
            cold = cosmo_b200.Model()
            cold.set(P, q, A, b2, sets, st)
            rc = cold.optimize()
            cold.empty_model()
            out["iterations"] = {"first_solve": [r0.iter, r0.status], "engine_kept": kept,
                                 "after_update_warm": [rw.iter, rw.status], "cold_fresh_model": [rc.iter, rc.status]}
            print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
