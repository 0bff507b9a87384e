"""CPU side of re-solving from device memory: the __cuda_array_interface__ checks (fake objects), the Model routing of
CUDA q and b and of optimize(solution="device") (a recording stand-in for the engine), and the new entry points in the
header, the signature table and the library."""
import ctypes as C

import numpy as np
import pytest

import cosmo_b200
from cosmo_b200 import engine as E, model as M

NEW = ("cosmo_b200_set_caller_stream", "cosmo_b200_update_qb_original", "cosmo_b200_original_qb", "cosmo_b200_solution",
       "cosmo_b200_rescale_iterates")


class FakeCuda:
    """an object that only carries a __cuda_array_interface__ (no memory behind it)"""

    def __init__(self, n, typestr="<f8", strides=None, readonly=False, stream=None, shape=None, ptr=0x7000_0000):
        self.__cuda_array_interface__ = {"shape": shape or (n,), "typestr": typestr, "data": (ptr, readonly),
                                         "strides": strides, "version": 3}
        if stream is not None:
            self.__cuda_array_interface__["stream"] = stream


def test_new_entry_points_are_declared_and_exported():
    header = open(E._build.LIB.replace("cosmo.jl_b200/libcosmo_b200.so", "include/cosmo_b200.h")).read()
    lib = E.load_library()
    for name in NEW:
        assert name + "(" in header
        assert name in E.SIGNATURES
        assert isinstance(getattr(lib, name), C._CFuncPtr)


def test_cuda_array_checks():
    assert E.cuda_array(FakeCuda(5), np.float64, 5) == (0x7000_0000, None)
    assert E.cuda_array(FakeCuda(5, typestr="<f4"), np.float32, 5)[0] == 0x7000_0000
    assert E.cuda_array(FakeCuda(5, strides=(8,)), np.float64)[0] == 0x7000_0000
    assert E.cuda_array(FakeCuda(5, stream=7), np.float64, 5)[1] == 7
    bad = [(FakeCuda(5, typestr="<f4"), np.float64, 5, False), (FakeCuda(5), np.float64, 6, False),
           (FakeCuda(5, shape=(5, 1)), np.float64, None, False), (FakeCuda(5, strides=(16,)), np.float64, 5, False),
           (FakeCuda(5, readonly=True), np.float64, 5, True), (FakeCuda(5, stream=0), np.float64, 5, False)]
    for a, dt, n, out in bad:
        with pytest.raises(E.EngineError) as e:
            E.cuda_array(a, dt, n, out)
        assert e.value.code == E.ERR_INVALID
    assert E.cuda_array(FakeCuda(5, readonly=True), np.float64, 5, False)[0]   # a read-only input is fine
    assert E.caller_stream_handle(1) is None and E.caller_stream_handle(2) == 2 and E.caller_stream_handle(99) == 99


class _Rec:
    """stand-in engine recording the calls Model makes"""

    def __init__(self, P, q, A, b, sets, settings, D=None, E=None, c=1.0, dtype=np.float64, device=0, equilibrate=False):
        self.m, self.n = A.shape
        self.calls = []
        self.n_orig = self.m_orig = 0
        self.q0, self.b0 = np.asarray(q, dtype=np.float64), np.asarray(b, dtype=np.float64)

    def scaling(self):
        return np.full(self.n, 2.0), np.full(self.m, 0.5), 0.25

    def update_settings(self, st):
        pass

    def set_accelerator(self, acc):
        pass

    def warm_start(self, x, s, mu):
        self.calls.append("warm_start")

    def rescale_iterates(self):
        self.calls.append("rescale_iterates")

    def update_qb(self, q, b):
        self.calls.append("update_qb")

    def update_qb_original(self, q, b):
        self.calls.append(("update_qb_original", q, b))

    def original_qb(self, q=None, b=None):
        self.calls.append(("original_qb", q is not None, b is not None))
        if q is not None:
            q[:] = 7.0
        if b is not None:
            b[:] = 8.0
        return q, b

    def update_matrices(self, Px=None, Ax=None, q=None, b=None):
        self.calls.append(("update_matrices", q, b))

    def solution(self, complete_dual, x=None, y=None, s=None):
        self.calls.append("solution")
        for a, v in ((x, 1.0), (y, -3.0), (s, 2.0)):
            if a is not None:
                a[:] = v
        return x, y, s

    def solve(self, copy_out=True):
        self.calls.append(("solve", copy_out))
        o = E.SolveOutput()
        o.x = np.zeros(self.n) if copy_out else None
        o.s = np.zeros(self.m) if copy_out else None
        o.mu = np.zeros(self.m) if copy_out else None
        o.obj_val, o.iter, o.status, o.safeguarding_iter = 0.0, 1, "Solved", 0
        o.r_prim = o.r_dual = o.max_norm_prim = o.max_norm_dual = 0.0
        o.rho, o.rho_updates, o.times = 0.1, [0.1], {}
        o.kkt_inner_iterations = o.kkt_multiplications = o.kernel_launches = 0
        return o

    def close(self):
        pass


@pytest.fixture
def model(monkeypatch):
    monkeypatch.setattr(M._eng, "Engine", _Rec)
    P, q, A, b, sets = cosmo_b200.problems.random_sparse_qp(30, 40, 0.2, seed=1)
    m = cosmo_b200.Model()
    m.set(P, q, A, b, sets, cosmo_b200.Settings())
    return m


def test_cuda_q_b_go_to_update_qb_original_and_q0_b0_are_read_back_lazily(model, monkeypatch):
    model.optimize()
    eng = model.engine
    q, b = FakeCuda(model.n), FakeCuda(model.m)
    model.update(q=q, b=b)
    assert eng.calls[-1] == ("update_qb_original", q, b)
    assert model._qb_on_device == [True, True]
    assert not any(c[0] == "original_qb" for c in eng.calls if isinstance(c, tuple))
    assert np.all(model.b0 == 8.0)                          # read on first use, both in one call
    assert eng.calls[-1] == ("original_qb", True, True)
    assert np.all(model.q0 == 7.0) and model._qb_on_device == [False, False]
    assert eng.calls[-1] == ("original_qb", True, True)
    with pytest.raises(ValueError):
        model.update(q=FakeCuda(model.n + 1))


def test_without_an_engine_cuda_arrays_are_copied_to_the_host(model, monkeypatch):
    monkeypatch.setattr(M._eng, "to_host", lambda a, dtype=np.float64: np.full(a.__cuda_array_interface__["shape"][0], 5.0))
    model.update(q=FakeCuda(model.n))
    assert model.engine is None and np.all(model.q0 == 5.0)


def test_device_solution_loop(model):
    r = model.optimize(solution="device")
    eng = model.engine
    assert r.x is None and r.y is None and r.s is None and eng.calls[-1] == ("solve", False)
    x, y, s = np.empty(model.n), np.empty(model.m), np.empty(model.m)
    model.solution_into(x, y, s)
    assert eng.calls[-1] == "solution" and np.all(y == -3.0)
    eng.calls.clear()
    model.optimize(solution="device")
    assert eng.calls[0] == "rescale_iterates" and "warm_start" not in eng.calls
    # a host warm start cancels the device round trip, after fetching the solution it completes
    model.warm_start_slack(np.zeros(model.m))
    assert np.all(model.x == 1.0) and np.all(model.mu == 3.0)
    eng.calls.clear()
    model.optimize()
    assert "warm_start" in eng.calls and "rescale_iterates" not in eng.calls
    x2 = np.empty(model.n)
    model.solution_into(x=x2)                               # after a host solve: the host copies
    assert np.all(x2 == model.x)
    with pytest.raises(ValueError):
        model.optimize(solution="gpu")


def test_new_matrices_fetch_the_device_solution_first(model):
    model.optimize(solution="device")
    model.update(P=model.P0.copy())
    assert model.engine.calls[-2] == "solution" and model.engine.calls[-1][0] == "update_matrices"
    assert not model._solution_on_device and np.all(model.x == 1.0)


def test_dropping_the_engine_keeps_a_q_that_lived_only_in_it(model):
    # a decomposed model with a forward map (faked): q as a CUDA array, then a host b that is nonzero on an uncovered row
    from types import SimpleNamespace
    model.optimize()
    eng = model.engine
    model._dec = object()
    unc = np.zeros(model.m, dtype=np.uint8)
    unc[3] = 1
    model._fwd = SimpleNamespace(b_uncovered=unc)
    model.update(q=FakeCuda(model.n))
    assert model._qb_on_device == [True, False]
    b = np.array(model.b0)
    b[3] = 1.0
    model.update(b=b)                                       # the host route drops the engine
    assert model.engine is None and ("original_qb", True, False) in eng.calls
    assert np.all(model.q0 == 7.0) and np.array_equal(model.b0, b) and model._qb_on_device == [False, False]
    model._dec = None
    model.optimize()                                        # the rebuild reads q0 and b0 from the host
    assert model.engine is not eng and "warm_start" in model.engine.calls
