"""CPU test of the host glue of Model.update(q, b, P=, A=): pattern checks, which values reach the engine (unscaled
with device equilibration, as given without), the decomposed fallback, and that update(q, b) alone keeps its own
path.  The CUDA engine is replaced by a stand-in that records the calls (the engine is covered by the GPU tests)."""
import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import model as M


class _RecordingEngine:
    """stand-in with the call surface Model uses; scaling() hands back a fixed D, E, c for equilibrating engines"""
    instances = []

    def __init__(self, P, q, A, b, sets, settings, D=None, E=None, c=1.0, dtype=np.float64, device=0, equilibrate=False):
        self.m, self.n = A.shape
        self.equilibrate = equilibrate
        self.calls = []
        self.scale = 1.0
        _RecordingEngine.instances.append(self)

    def scaling(self):
        if not self.equilibrate:
            return np.ones(self.n), np.ones(self.m), 1.0
        return np.full(self.n, 2.0 * self.scale), np.full(self.m, 0.5 * self.scale), 0.25 * self.scale

    def update_settings(self, st):
        pass

    def set_accelerator(self, acc):
        pass

    def warm_start(self, x, s, mu):
        self.calls.append(("warm_start", x, s, mu))

    def update_qb(self, q, b):
        self.calls.append(("update_qb", q, b))

    def update_matrices(self, Px=None, Ax=None, q=None, b=None):
        self.calls.append(("update_matrices", Px, Ax, q, b))
        self.scale = 3.0

    def solve(self):
        raise AssertionError("not solved in this test")

    def close(self):
        pass


@pytest.fixture
def engine(monkeypatch):
    _RecordingEngine.instances.clear()
    monkeypatch.setattr(M._eng, "Engine", _RecordingEngine)
    return _RecordingEngine


def _model(scaling):
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(40, 60, 0.2, seed=1)
    model = cosmo_b200.Model()
    model.set(P, q, A, b, sets, cosmo_b200.Settings(scaling=scaling))
    model._setup()
    return model


def _shuffled_copy(M0, values):
    """the same matrix pattern with new values, its row indices stored unsorted within every column"""
    M1 = sp.csc_matrix((values, M0.indices.copy(), M0.indptr.copy()), shape=M0.shape)
    idx, dat = M1.indices.copy(), M1.data.copy()
    for j in range(M1.shape[1]):
        a, e = M1.indptr[j], M1.indptr[j + 1]
        idx[a:e], dat[a:e] = idx[a:e][::-1], dat[a:e][::-1]
    return sp.csc_matrix((dat, idx, M1.indptr), shape=M1.shape)


def test_set_keeps_sorted_indices(engine):
    model = _model(0)
    A = _shuffled_copy(model.A0, model.A0.data)
    assert not A.has_sorted_indices
    model.set(model.P0, model.q0, A, model.b0, model.sets0)
    assert model.A0.has_sorted_indices and model.P0.has_sorted_indices
    assert not A.has_sorted_indices                      # the caller's matrix is not reordered in place


def test_pattern_and_shape_errors(engine):
    model = _model(0)
    A = model.A0.tolil()
    A[0, 0] = 0.0 if model.A0[0, 0] != 0 else 1.0
    A = A.tocsc()
    with pytest.raises(ValueError, match="set!"):
        model.update(A=A)
    with pytest.raises(ValueError, match="set!"):
        model.update(P=sp.identity(model.n + 1, format="csc"))
    with pytest.raises(ValueError):
        model.update(P=model.P0, q=np.zeros(model.n + 1))
    assert not [c for c in engine.instances[-1].calls if c[0] == "update_matrices"]


def test_unsorted_input_reaches_the_engine_in_csc_order(engine):
    model = _model(0)
    vals = np.arange(1.0, model.A0.nnz + 1.0)
    model.update(A=_shuffled_copy(model.A0, vals))
    name, Px, Ax, q, b = engine.instances[-1].calls[-1]
    assert name == "update_matrices" and Px is None and q is None and b is None
    assert np.array_equal(Ax, vals) and np.array_equal(model.A0.data, vals)


def test_without_scaling_the_given_values_go_as_they_are(engine):
    model = _model(0)
    P2 = model.P0.copy()
    P2.data *= 2.0
    q2 = np.arange(model.n, dtype=np.float64)
    model.update(q=q2, P=P2)
    name, Px, Ax, q, b = engine.instances[-1].calls[-1]
    assert name == "update_matrices" and Ax is None and b is None
    assert np.array_equal(Px, P2.data) and np.array_equal(q, q2)
    assert np.array_equal(model.q0, q2) and np.array_equal(model.P0.data, P2.data)


def test_equilibrating_engine_gets_every_unscaled_array_and_new_scaling(engine):
    model = _model(10)
    assert (model.D[0], model.E[0], model.c) == (2.0, 0.5, 0.25)
    A2 = model.A0.copy()
    A2.data = -A2.data
    model.update(A=A2)
    eng = engine.instances[-1]
    name, Px, Ax, q, b = eng.calls[-1]
    assert name == "update_matrices"
    assert np.array_equal(Px, model.P0.data) and np.array_equal(Ax, A2.data)
    assert np.array_equal(q, model.q0) and np.array_equal(b, model.b0)          # unscaled, not D q c / E b
    assert (model.D[0], model.E[0], model.c) == (6.0, 1.5, 0.75)                 # read back after the update
    assert len(engine.instances) == 1


def test_engine_creation_not_current_settings_decides_the_path(engine):
    model = _model(10)                  # the engine equilibrates on the device
    model.settings.scaling = 0          # a later solve's settings do not change how the engine was built
    model.update(P=model.P0.copy())
    name, Px, Ax, q, b = engine.instances[-1].calls[-1]
    assert name == "update_matrices" and Ax is not None and q is not None and b is not None
    plain = _model(0)
    plain.settings.scaling = 10
    plain.update(P=plain.P0.copy())
    name, Px, Ax, q, b = engine.instances[-1].calls[-1]
    assert name == "update_matrices" and Px is not None and Ax is None and q is None and b is None


def test_decomposed_model_drops_the_engine(engine):
    model = _model(0)
    model._dec = object()          # as after a chordal decomposition
    model.update(P=model.P0.copy())
    assert model.engine is None and model._x2 is None
    assert not [c for c in engine.instances[-1].calls if c[0] == "update_matrices"]


def test_q_b_update_keeps_its_path(engine):
    model = _model(10)
    q2, b2 = np.ones(model.n), np.ones(model.m)
    model.update(q=q2, b=b2)
    calls = [c for c in engine.instances[-1].calls if c[0] != "warm_start"]
    assert [c[0] for c in calls] == ["update_qb"]
    _, q, b = calls[0]
    assert np.array_equal(q, model.D * q2 * model.c) and np.array_equal(b, model.E * b2)
