"""Helpers shared by the GPU test modules: engine construction and the test matrices of the PSD projections."""
import numpy as np
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E
from oracle import cosmo_oracle as O
from oracle.bridge import to_oracle_cones

U32 = 2.0 ** -24        # unit roundoff of IEEE single precision
U64 = 2.0 ** -53


def _tuples(sets):
    return [cosmo_b200.model.set_tuple(S) for S in sets]


def _engine(P, q, A, b, sets, dtype=np.float64, **kw):
    st = cosmo_b200.Settings(**kw).to_struct()
    return E.Engine(P, q, A, b, _tuples(sets), st, dtype=dtype)


def _project_engine(sets, dtype=np.float64, **kw):
    """an engine whose only job is to project: n = 1, A = 0"""
    m = sum(S.dim for S in sets)
    return _engine(sp.identity(1, format="csc"), np.zeros(1), sp.csc_matrix((m, 1)), np.zeros(m), sets, dtype=dtype, **kw)


def _oracle_project(ws, sets):
    """the fp64 oracle projection of ws (whatever its type) as float64"""
    ref = np.asarray(ws, dtype=np.float64).copy()
    O.project(ref, to_oracle_cones(sets))
    return ref


def _round32(a):
    """fp64 data rounded to fp32 and back: the exact input an fp32 kernel sees, in the oracle's type"""
    return np.asarray(a, dtype=np.float64).astype(np.float32).astype(np.float64)


def _psd_test_matrix(kind, N, rng):
    B = rng.standard_normal((N, N))
    if kind == "wigner":
        return (B + B.T) / 2
    if kind == "rank_deficient":
        k = max(N // 10, 2)
        return B[:, :k] @ B[:, :k].T - B[:, k:2 * k] @ B[:, k:2 * k].T
    if kind == "shifted":
        return (B + B.T) / 2 + 3.0 * np.sqrt(N) * np.eye(N)
    if kind == "zero":
        return np.zeros((N, N))
    if kind == "admm_like":      # w_s = s - mu / rho near a solution: PSD part, scaled negative part, a cluster near zero
        Q, _ = np.linalg.qr(B)
        lam = np.concatenate([np.abs(rng.standard_normal(N // 3)), -10.0 * np.abs(rng.standard_normal(N // 3)),
                              1e-7 * rng.standard_normal(N - 2 * (N // 3))])
        return (Q * lam) @ Q.T
    if kind == "graded":         # eigenvalues spread over 12 orders of magnitude, both signs
        Q, _ = np.linalg.qr(B)
        lam = np.logspace(0, -12, N) * np.where(np.arange(N) % 2 == 0, 1.0, -1.0)
        return (Q * lam) @ Q.T
    raise ValueError(kind)


def _hermitian_ws(N, rng, kind):
    Z = rng.standard_normal((N, N)) + 1j * rng.standard_normal((N, N))
    H = (Z + Z.conj().T) / 2
    if kind == "shifted":
        H = H - 0.3 * np.sqrt(N) * np.eye(N)
    elif kind == "low_rank_plus_noise":          # an ADMM-like iterate: a PSD part plus a small indefinite perturbation
        Y = rng.standard_normal((N, N // 4)) + 1j * rng.standard_normal((N, N // 4))
        H = Y @ Y.conj().T / N + 1e-3 * H
    return O.extract_upper_triangle_complex(H, np.sqrt(2.0)), H
