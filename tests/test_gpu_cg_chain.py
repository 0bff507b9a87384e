"""The chained CG loop on problems whose A and A' run through the column-windowed kernel.

Every kernel of a CG iteration is a programmatic dependent of the one before it, the P rows of the reduced KKT operator
are summed inside the windowed A' pass, and the warm-start product rho .* (A x) of each CG solve is taken from the
previous ADMM iteration's fused tail."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests.gpu_helpers import _engine

pytestmark = pytest.mark.gpu

W_MAX = 25600          # doubles of one column window (200 KB of shared memory)


def _windows(M):
    """(nwin, windowed) by the engine's rule (build_windows): W_MAX-column windows, at most 16 of them, and on average
    at least 24 entries per row segment"""
    rows, cols = M.shape
    nwin = -(-cols // W_MAX)
    return nwin, bool(nwin <= 16 and M.nnz / (rows * nwin) >= 24.0)


def _kernel_counts(fn, tmp_path):
    """kernel names `fn` launches, with their counts (torch.profiler trace)"""
    import json
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    trace = str(tmp_path / "trace.json")
    prof.export_chrome_trace(trace)
    with open(trace) as f:
        events = json.load(f).get("traceEvents", [])
    counts = {}
    for e in events:
        if e.get("cat") == "kernel":
            counts[e["name"]] = counts.get(e["name"], 0) + 1
    assert counts, "no kernels in the trace"
    return counts


def _count(counts, *parts):
    return sum(c for name, c in counts.items() if all(p in name for p in parts))


@pytest.mark.parametrize("nwin,m,p_half,lanes", [(1, 20000, 20, 32), (2, 40000, 20, 32), (4, 90000, 20, 32), (2, 40000, 5, 8),
                                               (4, 90000, 0.5, 2)])
def test_windowed_kkt_operator_with_fused_p_rows(nwin, m, p_half, lanes, tmp_path):
    """y = A' x2 + P x1 + sigma x1 with A' windowed (nwin = 1, 2, 4) and P's rows (32, 8 and 2 lanes, the 32-lane rows
    longer than the A' row segments) summed by the window CTAs of each chunk, against SciPy"""
    n = 30000
    rng = np.random.default_rng(int(nwin * 100 + p_half * 10))
    per_row = 30 * nwin                                   # entries per row of A' (per column of A): ~30 per window
    rows = rng.integers(0, m, size=n * per_row)
    cols = np.repeat(np.arange(n), per_row)
    A = sp.csc_matrix((rng.standard_normal(n * per_row), (rows, cols)), shape=(m, n))
    B = sp.random(n, n, density=p_half / n, random_state=rng, format="csr")
    P = sp.csc_matrix(B + B.T + sp.identity(n))
    assert _windows(A.T.tocsr()) == (nwin, True)
    assert not _windows(P)[1]                             # P stays plain CSR: its rows are folded into the A' pass
    mean_p = P.nnz / n                                    # the engine's lane choice for P (pick_lanes)
    assert lanes == (32 if mean_p > 24 else 8 if mean_p > 3 else 2)
    eng = _engine(P, np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], scaling=0)
    x1, x2 = rng.standard_normal(n), rng.standard_normal(m)
    sigma = cosmo_b200.Settings().sigma
    counts = _kernel_counts(lambda: eng.spmv(3, np.concatenate([x1, x2])), tmp_path)
    got = eng.spmv(3, np.concatenate([x1, x2]))
    assert _count(counts, "spmv_win_kernel", "EpiKktOp", ", %d>" % lanes) == 1 and _count(counts, "spmv_kernel") == 0, counts
    ref = A.T @ x2 + P @ x1 + sigma * x1
    scale = abs(A.T) @ np.abs(x2) + abs(P) @ np.abs(x1) + sigma * np.abs(x1) + 1e-300
    assert np.max(np.abs(got - ref) / scale) < 1e-14
    # the fused P rows against the separate P launch: equal up to the rounding of the final three-term sum
    pu = eng.spmv(2, x1)
    at = eng.spmv(1, x2)
    assert np.max(np.abs(got - (at + pu + sigma * x1)) / scale) < 1e-15
    eng.close()


def test_windowed_admm_solve_with_rho_adaptation_and_warm_start_matches_oracle(tmp_path):
    # n = 30k, m = 60k, 120 entries per column: A (2 windows, ~60 per row) and A' (3 windows, ~120 per row)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30000, 60000, 0.002, seed=3)
    assert _windows(sp.csr_matrix(A)) == (2, True) and _windows(sp.csr_matrix(A.T)) == (3, True)
    assert not _windows(sp.csr_matrix(P))[1]
    cones = to_oracle_cones(sets)
    iters = 30
    kw = dict(scaling=0, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14, rho=1e-5, adaptive_rho=True, adaptive_rho_interval=10)
    eng = _engine(P, q, A, b, sets, **kw)
    ref = O.solve(P, q, A, b, cones, O.Settings(kkt_solver="cg", **kw))
    assert len(ref.info.rho_updates) >= 2          # the adaptation happens inside the compared iterations

    # CG iterations of every KKT solve: the solve of the first k iterations (initialisation step included), from the
    # same cold start, runs the oracle's first k + 1 CG solves
    totals = []
    for k in range(1, iters + 1):
        st = cosmo_b200.Settings(**dict(kw, max_iter=k)).to_struct()
        eng.update_settings(st)
        eng.reset()
        totals.append(int(eng.solve().kkt_inner_iterations))
    assert totals == [int(v) for v in np.cumsum(ref.kkt.inner_iterations)[1:]]

    # the full solve: four kernels per CG iteration, the warm-start pass only in the first ADMM iteration and after each
    # rho change
    outs = []

    def full_solve():
        eng.reset()
        outs.append(eng.solve())

    counts = _kernel_counts(full_solve, tmp_path)
    out = outs[0]
    assert out.iter == ref.iter
    assert len(out.rho_updates) == len(ref.info.rho_updates)
    assert np.allclose(out.rho_updates, ref.info.rho_updates, rtol=1e-6)
    w = eng.w()
    assert np.linalg.norm(w - ref.w) <= 1e-8 * np.linalg.norm(ref.w)
    n_u = _count(counts, "cg_update_u")
    assert _count(counts, "cg_update_xr") == n_u
    kkt_solves = _count(counts, "spmv_win_kernel", "EpiAddVec")                     # one rhs pass per KKT solve
    assert _count(counts, "spmv_win_kernel", "EpiKktOp") == n_u + kkt_solves        # CG loop + one warm start each
    assert _count(counts, "spmv_kernel", "EpiStore") == 0, counts                   # no separate P launch
    warm = _count(counts, "spmv_win_kernel", "EpiScale") - n_u
    assert warm == len(out.rho_updates), (warm, out.rho_updates)   # the first solve + one after each rho change

    # reset + warm start from the first solve's answer (cosmo's y = -mu)
    x0, s0, mu0 = out.x.copy(), out.s.copy(), out.mu.copy()
    eng.reset()
    eng.warm_start(x0, s0, mu0)
    out2 = eng.solve()
    ref2 = O.solve(P, q, A, b, cones, O.Settings(kkt_solver="cg", **kw), x0=x0, s0=s0, y0=-mu0)
    assert out2.iter == ref2.iter and out2.kkt_inner_iterations == sum(ref2.kkt.inner_iterations)
    assert np.allclose(out2.rho_updates, ref2.info.rho_updates, rtol=1e-6)
    assert np.linalg.norm(eng.w() - ref2.w) <= 1e-8 * np.linalg.norm(ref2.w)
    eng.close()
