"""The packed (9 B per entry) fp64 column-windowed slabs: which matrices get them, and that they compute what the 10 B
slabs compute.

An fp64 windowed matrix is packed (csrc/win_pack.h) unless more than 1/256 of its stored entries fall outside its best
14 binades; an engine that equilibrates on the device applies that rule to the scaled values.  The layout is read from
the kernel names of a profiler trace (`spmv_win_kernel<double, true, ...>` is the packed kernel) and from the
COSMO_B200_SETUP_DEBUG report."""
import json
import re

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones
from tests.gpu_helpers import _engine, _tuples

pytestmark = pytest.mark.gpu

PACKED, PLAIN = "spmv_win_kernel<double, true", "spmv_win_kernel<double, false"


def _kernel_counts(fn, tmp_path, reps=20):
    """kernel names `reps` calls of `fn` launch, with their counts (torch.profiler trace; a capture of a single short
    call can come back empty)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
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


def _count(counts, part):
    return sum(c for name, c in counts.items() if part in name)


def _layouts(capfd):
    """(layout, ebase, escapes, windows, window width) of every windowed matrix the last engine creation reported, A
    first, then A'"""
    err = capfd.readouterr().err
    return [(m.group(3), int(m.group(4)), int(m.group(5)), int(m.group(1)), int(m.group(2)))
            for m in re.finditer(r"\[setup\] windows (\d+) x (\d+), \d+ rows: (\d+ B) layout, ebase (\d+), (\d+) escapes", err)]


def _assert_layout_rule(A, lay):
    """The layouts reported for A and A', recomputed with NumPy: the exponent window is the first of the 14-binade
    windows that hold the most finite normal values, the escapes are the stored nonzero values outside it, and a slab
    is packed iff escapes * 256 <= its slots (every (row, window) segment padded to a multiple of 8 entries)."""
    data = np.ascontiguousarray(A.data, dtype=np.float64)
    e = ((data.view(np.uint64) >> np.uint64(52)) & np.uint64(0x7FF)).astype(np.int64)
    hist = np.bincount(e[(e != 0) & (e != 0x7FF)], minlength=2048)
    ebase = 1 + int(np.argmax(np.convolve(hist[1:2047], np.ones(14, dtype=np.int64), "valid")))
    nesc = int(np.count_nonzero((data != 0) & ((e < ebase) | (e > ebase + 13))))
    assert len(lay) == 2, lay
    for M, (layout, eb, esc, nwin, W) in zip((sp.coo_matrix(A), sp.coo_matrix(A.T)), lay):
        seg = np.bincount(M.row.astype(np.int64) * nwin + M.col // W, minlength=M.shape[0] * nwin)
        slots = int(((seg + 7) // 8 * 8).sum())
        assert (layout == "9 B") == (nesc * 256 <= slots), (layout, nesc, slots)
        if layout == "9 B":
            assert (eb, esc) == (ebase, nesc), (eb, esc, ebase, nesc)


def _windowed_matrix(rng, values, m=20000, n=40000, per_col=30):
    """m x n with `per_col` entries per column at random rows: A (2 windows, ~60 per row) and A' (1 window) windowed"""
    rows = rng.integers(0, m, size=n * per_col)
    cols = np.repeat(np.arange(n), per_col)
    return sp.csc_matrix((values(n * per_col), (rows, cols)), shape=(m, n))


def _check_products(eng, A, rng, tol=1e-14):
    """spmv 0 (A x), 1 (A' y) and 3 (A' y + P x + sigma x, P = I) against SciPy, relative to |A||x|"""
    m, n = A.shape
    x, y = rng.standard_normal(n), rng.standard_normal(m)
    sigma = cosmo_b200.Settings().sigma
    for which, arg, ref, scale in ((0, x, A @ x, abs(A) @ np.abs(x)), (1, y, A.T @ y, abs(A.T) @ np.abs(y)),
                                   (3, np.concatenate([x, y]), A.T @ y + x + sigma * x,
                                    abs(A.T) @ np.abs(y) + (1 + sigma) * np.abs(x))):
        got = eng.spmv(which, arg)
        assert np.max(np.abs(got - ref) / (scale + 1e-300)) < tol, which


def _eye_engine(A, **kw):
    m, n = A.shape
    return _engine(sp.identity(n, format="csc"), np.zeros(n), A, np.zeros(m), [cosmo_b200.Nonnegatives(m)], scaling=0, **kw)


def test_gaussian_values_are_packed_with_escapes(tmp_path, capfd, monkeypatch):
    rng = np.random.default_rng(11)
    A = _windowed_matrix(rng, rng.standard_normal)
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    capfd.readouterr()
    eng = _eye_engine(A)
    lay = _layouts(capfd)
    assert [l[0] for l in lay] == ["9 B", "9 B"], lay
    assert all(0 < esc <= A.nnz / 256 for _, _, esc, _, _ in lay), lay      # the smallest |values| escape
    _assert_layout_rule(A, lay)
    counts = _kernel_counts(lambda: eng.spmv(0, np.ones(A.shape[1])), tmp_path)
    assert _count(counts, PACKED) > 0 and _count(counts, PLAIN) == 0, counts
    _check_products(eng, A, rng)
    eng.close()


def test_special_values_stay_packed_and_exact(tmp_path, capfd, monkeypatch):
    rng = np.random.default_rng(12)
    A = _windowed_matrix(rng, rng.standard_normal).tolil()
    j = 777                                                     # one column holds every special value
    specials = [0.0, -0.0, 1e-300, -1e-300, 5e-324, -5e-324, 1e300, -1e300, 2.5e-310]
    for i, v in enumerate(specials):
        A[100 * i + 3, j] = v if v != 0.0 else 1.0              # placeholder: lil drops explicit zeros
    A = A.tocsc()
    A.sort_indices()
    for i, v in enumerate(specials):
        k = A.indptr[j] + np.searchsorted(A.indices[A.indptr[j]:A.indptr[j + 1]], 100 * i + 3)
        A.data[k] = v                                           # explicit +-0 entries stay stored
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    capfd.readouterr()
    eng = _eye_engine(A)
    lay = _layouts(capfd)
    assert [l[0] for l in lay] == ["9 B", "9 B"], lay
    _assert_layout_rule(A, lay)
    # A e_j is column j exactly: every special value comes back as stored (zeros compare equal up to their sign)
    e = np.zeros(A.shape[1])
    e[j] = 1.0
    got = eng.spmv(0, e)
    assert np.array_equal(got, A[:, j].toarray().ravel())
    for i, v in enumerate(specials):
        assert got[100 * i + 3] == v
    # A' e_r picks row r of A: the rows holding the subnormals and the large values
    for i in (4, 6, 8):
        r = 100 * i + 3
        er = np.zeros(A.shape[0])
        er[r] = 1.0
        assert np.array_equal(eng.spmv(1, er), A[r, :].toarray().ravel())
    eng.close()

    # Inf entries: the same non-finite rows as SciPy, the finite ones within the usual bound
    B = A.copy()
    B.data[B.indptr[5]] = np.inf
    B.data[B.indptr[9] + 1] = -np.inf
    eng = _eye_engine(B)
    x = rng.standard_normal(B.shape[1])
    with np.errstate(invalid="ignore"):
        ref = B @ x
        scale = abs(B) @ np.abs(x)
    got = eng.spmv(0, x)
    fin = np.isfinite(ref)
    assert (~fin).sum() >= 2 and np.array_equal(np.isfinite(got), fin)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(got[np.isinf(ref)], ref[np.isinf(ref)])
    assert np.max(np.abs(got[fin] - ref[fin]) / (scale[fin] + 1e-300)) < 1e-14
    eng.close()


def test_wide_value_range_keeps_the_10_byte_layout(tmp_path, capfd, monkeypatch):
    rng = np.random.default_rng(13)
    A = _windowed_matrix(rng, lambda k: rng.choice([-1.0, 1.0], k) * 10.0 ** rng.uniform(-40, 40, k))
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    capfd.readouterr()
    eng = _eye_engine(A)
    lay = _layouts(capfd)
    assert [l[0] for l in lay] == ["10 B", "10 B"], lay
    _assert_layout_rule(A, lay)
    counts = _kernel_counts(lambda: eng.spmv(1, np.ones(A.shape[0])), tmp_path)
    assert _count(counts, PLAIN) > 0 and _count(counts, PACKED) == 0, counts
    _check_products(eng, A, rng)
    eng.close()


def _ruiz_scaled(A, D, E):
    """E A D of a CSC matrix as the engine forms it: every entry times the product D_j E_i"""
    S = A.copy()
    S.data = A.data * (D[np.repeat(np.arange(A.shape[1]), np.diff(A.indptr))] * E[A.indices])
    return S


def test_device_equilibration_fills_the_slabs_with_the_scaled_values(tmp_path, capfd, monkeypatch):
    """scale_ruiz! scales the CSR copies and the slabs are filled from the scaled A' afterwards: they take the layout
    the rule picks for the scaled values and hold exactly the numbers of the CSR copies"""
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30000, 40000, 0.002, seed=5)   # A and A' windowed
    A.sort_indices()
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    capfd.readouterr()
    eng = E.Engine(P, q, A, b, _tuples(sets), cosmo_b200.Settings().to_struct(), equilibrate=True)
    lay = _layouts(capfd)
    D, Ev, c = eng.scaling()
    Ps, qs, As, bs, cones, sm = O.scale_ruiz(P, q, A, b, to_oracle_cones(sets), O.Settings())
    assert np.max(np.abs(D - sm.D) / sm.D) <= 1e-13
    assert np.max(np.abs(Ev - sm.E) / sm.E) <= 1e-13
    S = _ruiz_scaled(A, D, Ev)
    _assert_layout_rule(S, lay)
    rng = np.random.default_rng(1)
    x, y = rng.standard_normal(A.shape[1]), rng.standard_normal(A.shape[0])
    for which, arg, (layout, *_) in ((0, x, lay[0]), (1, y, lay[1])):
        want, other = (PACKED, PLAIN) if layout == "9 B" else (PLAIN, PACKED)
        counts = _kernel_counts(lambda: eng.spmv(which, arg), tmp_path)
        assert _count(counts, want) > 0 and _count(counts, other) == 0, (which, counts)
    # A e_j and A' e_i are a column and a row of the slabs, on both sides of a window edge: bit for bit those of E A D
    Sr = S.tocsr()
    (*_, WA), (*_, WAt) = lay
    for j in (0, WA - 1, WA, A.shape[1] - 1):
        e = np.zeros(A.shape[1])
        e[j] = 1.0
        assert np.array_equal(eng.spmv(0, e), S[:, j].toarray().ravel()), j
    for i in (0, WAt - 1, WAt, A.shape[0] - 1):
        e = np.zeros(A.shape[0])
        e[i] = 1.0
        assert np.array_equal(eng.spmv(1, e), Sr[i, :].toarray().ravel()), i
    for which, got_in, ref in ((0, x, As @ x), (1, y, As.T @ y), (2, x, Ps @ x)):
        got = eng.spmv(which, got_in)
        assert np.max(np.abs(got - ref)) <= 1e-12 * max(1.0, np.max(np.abs(ref))), which
    eng.close()


def test_admm_solve_on_packed_slabs_matches_oracle(tmp_path, capfd, monkeypatch):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30000, 40000, 0.002, seed=4)
    iters = 15
    kw = dict(scaling=0, max_iter=iters, eps_abs=1e-14, eps_rel=1e-14, rho=1e-4, adaptive_rho=False)
    monkeypatch.setenv("COSMO_B200_SETUP_DEBUG", "1")
    capfd.readouterr()
    eng = _engine(P, q, A, b, sets, **kw)
    lay = _layouts(capfd)
    assert [l[0] for l in lay] == ["9 B", "9 B"], lay
    _assert_layout_rule(A, lay)
    ref = O.solve(P, q, A, b, to_oracle_cones(sets), O.Settings(kkt_solver="cg", **kw))
    outs = []
    counts = _kernel_counts(lambda: outs.append(eng.solve()), tmp_path, reps=1)
    out = outs[0]
    assert _count(counts, PACKED) > 0 and _count(counts, PLAIN) == 0, counts
    assert out.iter == ref.iter == iters
    assert int(out.kkt_inner_iterations) == int(sum(ref.kkt.inner_iterations))
    assert np.linalg.norm(eng.w() - ref.w) <= 1e-8 * np.linalg.norm(ref.w)
    eng.close()
