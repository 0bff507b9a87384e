"""Re-solves from device memory: q and b given as CUDA tensors (cosmo_b200_update_qb_original), the solution written
into CUDA tensors (cosmo_b200_solution), the round trip between solves on the device (cosmo_b200_rescale_iterates) and
device pointers in the existing data entry points.  Each is compared bit for bit with the host route it replaces."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import cosmo_b200
from cosmo_b200 import engine as E

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


def _maxcut(nv, seed, graph_seed=1):
    rows, cols, _ = cosmo_b200.problems.banded_random_graph(nv, 3.0, 20, seed=graph_seed)
    rng = np.random.default_rng(seed)
    w = rng.integers(1, 11, size=len(rows)).astype(np.float64)
    P, q, A, b, sets = cosmo_b200.problems.maxcut_dual_sdp(nv, rows, cols, w)
    A = sp.csc_matrix(A)
    A.sort_indices()
    P = sp.diags(rng.uniform(0.001, 0.01, nv), format="csc")
    return P, q * rng.uniform(0.9, 1.1, nv), A, b * rng.uniform(0.9, 1.1, b.size), sets


def _qp(seed):
    return cosmo_b200.problems.random_sparse_qp(300, 500, 0.05, seed=seed)


def _bits(a):
    a = a.cpu().numpy() if torch.is_tensor(a) else a
    return np.ascontiguousarray(a, dtype=np.float64).view(np.int64)


def _same(a, b):
    assert np.array_equal(_bits(a), _bits(b))


def _cuda(a, dtype=torch.float64):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


KINDS = ["plain", "compact", "traditional"]


def _model(kind, seed, **st):
    dtype = st.pop("dtype", np.float64)
    if kind == "plain":
        data = _qp(seed)
    else:
        data = _maxcut(200, seed)
        st.update(decompose=True, compact_transformation=kind == "compact")
    m = cosmo_b200.Model(dtype=dtype)
    m.set(*data, cosmo_b200.Settings(**st))
    return m


def _new_qb(m, seed):
    rng = np.random.default_rng(seed)
    q = m.q0 * rng.uniform(0.8, 1.2, m.n)
    b = m.b0 * rng.uniform(0.8, 1.2, m.m)
    return q, b


def _engine_state(m, r):
    eng = m.engine
    return (eng.w(), eng.rho_vec(), r.status, r.iter, r.x, r.s, r.y)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("solver", ["CGIndirectKKTSolver", "DeviceLdlKKTSolver"])
@pytest.mark.parametrize("scaling", [0, 10])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_update_qb_original_leaves_the_host_route_state(kind, solver, scaling, dtype):
    st = dict(kkt_solver=solver, scaling=scaling, dtype=dtype, max_iter=120)
    models = [_model(kind, 1, **st) for _ in range(3)]
    for m in models:
        m.optimize()
    q, b = _new_qb(models[0], 5)
    models[0].update(q=q, b=b)                                       # host route: scaled on the host, update_qb
    models[1].engine.update_qb_original(q, b)                       # host arrays through the device scaling
    models[1]._qb_on_device = [True, True]
    models[2].update(q=_cuda(q), b=_cuda(b))                         # CUDA tensors
    assert models[2]._qb_on_device == [True, True]
    states = [_engine_state(m, m.optimize()) for m in models]
    for other in states[1:]:
        for a, c in zip(states[0], other):
            if isinstance(a, np.ndarray):
                _same(a, c)
            else:
                assert a == c
    _same(models[2].q0, q)
    _same(models[2].b0, b)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("complete_dual", [False, True])
def test_solution_into_cuda_tensors_is_the_host_result(kind, complete_dual):
    m = _model(kind, 2, complete_dual=complete_dual, reverse_on_device=True, max_iter=150)
    r = m.optimize()
    n, mm = m.n, m.m
    x, y, s = (torch.empty(k, dtype=torch.float64, device="cuda") for k in (n, mm, mm))
    m.engine.solution(complete_dual, x, y, s)
    _same(x, r.x), _same(y, r.y), _same(s, r.s)
    x2, y2, s2 = (torch.empty(k, dtype=torch.float64, device="cuda") for k in (n, mm, mm))
    m.solution_into(x2, y2, s2)                                      # host copies into CUDA tensors
    _same(x2, r.x), _same(y2, r.y), _same(s2, r.s)


def _loop(kind, device, steps, **st):
    m = _model(kind, 3, **st)
    out = []
    for k in range(steps):
        q, b = _new_qb(m, 10 + k) if k else (None, None)
        if device:
            if k:
                m.update(q=_cuda(q), b=_cuda(b))
            r = m.optimize(solution="device")
            assert r.x is None
            x, y, s = (torch.empty(k_, dtype=torch.float64, device="cuda") for k_ in (m.n, m.m, m.m))
            m.solution_into(x, y, s)
            out.append((r.status, r.iter, r.info.rho_updates, x.cpu().numpy(), y.cpu().numpy(), s.cpu().numpy()))
        else:
            if k:
                m.update(q=q, b=b)
            r = m.optimize()
            out.append((r.status, r.iter, r.info.rho_updates, r.x, r.y, r.s))
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_device_loop_is_the_host_loop(kind):
    # a rho check every 25 iterations with a tolerance of 1.5: the loop crosses rho adaptations
    st = dict(max_iter=200, adaptive_rho_interval=25, adaptive_rho_tolerance=1.5, reverse_on_device=True,
              complete_dual=kind != "plain")
    host, dev = _loop(kind, False, 4, **st), _loop(kind, True, 4, **st)
    assert any(len(h[2]) > 1 for h in host)
    for h, d in zip(host, dev):
        assert h[:3] == d[:3]
        for a, c in zip(h[3:], d[3:]):
            _same(a, c)


def test_device_loop_with_a_matrix_update_reads_q0_b0_from_the_engine():
    def run(device):
        m = _model("plain", 4, max_iter=150)           # scaling 10: an equilibrating engine
        m.optimize(solution="device" if device else "host")
        q, b = _new_qb(m, 21)
        m.update(q=_cuda(q) if device else q, b=_cuda(b) if device else b)
        m.optimize(solution="device" if device else "host")
        P2 = m.P0.copy()
        P2.data = P2.data * 1.5
        m.update(P=P2)                                 # an equilibrating engine re-runs Ruiz from q0, b0
        if device:
            assert m._qb_on_device == [False, False]
        r = m.optimize()
        return r, m.q0, m.b0
    (rh, qh, bh), (rd, qd, bd) = run(False), run(True)
    _same(qh, qd), _same(bh, bd)
    assert (rh.status, rh.iter) == (rd.status, rd.iter)
    _same(rh.x, rd.x), _same(rh.y, rd.y), _same(rh.s, rd.s)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_existing_entry_points_take_device_pointers(dtype):
    P, q, A, b, sets = _qp(6)
    st = cosmo_b200.Settings(max_iter=100).to_struct()
    from cosmo_b200 import model as M
    tsets = [M.set_tuple(S) for S in sets]
    engs = [E.Engine(P, q, A, b, tsets, st, dtype=dtype) for _ in range(2)]
    tdt = torch.float64 if dtype == np.float64 else torch.float32
    rng = np.random.default_rng(0)
    Ac = sp.csc_matrix(A); Ac.sort_indices()
    Pc = sp.csc_matrix(P); Pc.sort_indices()
    Px, Ax = Pc.data * 1.1, Ac.data * rng.uniform(0.9, 1.1, Ac.nnz)
    q2, b2 = q * 1.2, b * 0.9
    x0, s0, mu0 = rng.standard_normal(A.shape[1]), rng.standard_normal(A.shape[0]), rng.standard_normal(A.shape[0])
    outs = []
    for k, eng in enumerate(engs):
        f = (lambda a: _cuda(np.asarray(a, dtype=dtype), tdt)) if k else (lambda a: np.asarray(a, dtype=dtype))
        eng.update_matrices(f(Px), f(Ax), f(q2), f(b2))
        eng.update_qb(f(q2 * 1.01), f(b2))
        eng.warm_start(f(x0), f(s0), f(mu0))
        if k:
            xs = [torch.empty(v, dtype=tdt, device="cuda") for v in (eng.n, eng.m, eng.m)]
            o = eng.solve(*xs)
            outs.append((o.iter, o.status, *[t.cpu().numpy() for t in xs], eng.w()))
        else:
            o = eng.solve()
            outs.append((o.iter, o.status, o.x, o.s, o.mu, eng.w()))
    assert outs[0][:2] == outs[1][:2]
    for a, c in zip(outs[0][2:], outs[1][2:]):
        _same(a, c)


def test_stream_ordering_on_a_side_stream():
    m = _model("plain", 7, max_iter=100)
    m.optimize()
    ref = _model("plain", 7, max_iter=100)
    ref.optimize()
    q, b = _new_qb(m, 30)
    ref.update(q=q, b=b)
    r_ref = ref.optimize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        m.engine.set_caller_stream(side.cuda_stream)
        big = torch.randn(4096, 4096, device="cuda", dtype=torch.float64)
        qd = _cuda(np.zeros(m.n))
        bd = _cuda(np.zeros(m.m))
        _ = big @ big                                  # keep the side stream busy before the inputs are written
        qd.copy_(_cuda(q) * 1.0)
        bd.copy_(_cuda(b) * 1.0)
        m.update(q=qd, b=bd)
        m.optimize(solution="device")
        x = torch.full((m.n,), float("nan"), dtype=torch.float64, device="cuda")
        _ = big @ big
        m.solution_into(x=x)
        x2 = x * 2.0                                   # consumed on the side stream
    side.synchronize()
    _same(x2.cpu().numpy() / 2.0, r_ref.x)


def test_refusals():
    m = _model("compact", 8, max_iter=100)
    m.optimize()
    twin = _model("compact", 8, max_iter=100)
    twin.optimize()
    unc = np.nonzero(np.asarray(m._fwd.b_uncovered))[0]
    assert unc.size
    b = m.b0.copy()
    b[unc[0]] = 1.0
    eng = m.engine
    with pytest.raises(E.EngineError) as e:
        eng.update_qb_original(None, _cuda(b))
    assert e.value.code == E.ERR_INVALID
    r1, r2 = m.optimize(), twin.optimize()
    _same(r1.x, r2.x), _same(r1.s, r2.s), _same(r1.y, r2.y)
    # the Model drops the engine, as the host route does, and keeps the new b
    m.update(b=_cuda(b))
    assert m.engine is None
    _same(m.b0, b)
    with pytest.raises(E.EngineError) as e:                       # no q was ever given to update_qb_original
        twin.engine.original_qb(np.empty(twin.n), None)
    assert e.value.code == E.ERR_INVALID


def test_fallback_copies_are_ordered_on_a_side_stream():
    # the host copies of the Model: a host solution into a CUDA tensor, and a CUDA q copied to the host without an engine
    m = _model("plain", 9, max_iter=100)
    r = m.optimize()
    side = torch.cuda.Stream()
    big = torch.randn(4096, 4096, device="cuda", dtype=torch.float64)
    with torch.cuda.stream(side):
        x = torch.zeros(m.n, dtype=torch.float64, device="cuda")
        _ = big @ big                                  # the zero fill lands late unless the copy waits for it
        x.zero_()
        m.solution_into(x=x)
        x2 = x * 2.0
        fresh = _model("plain", 9, max_iter=100)
        qd = torch.zeros(fresh.n, dtype=torch.float64, device="cuda")
        _ = big @ big
        qd.copy_(_cuda(fresh.q0) * 3.0)                # written on the side stream just before the host copy
        fresh.update(q=qd)
    side.synchronize()
    _same(x2.cpu().numpy() / 2.0, r.x)
    assert fresh.engine is None
    _same(fresh.q0, _qp(9)[1] * 3.0)


@pytest.mark.parametrize("kind", ["compact", "traditional"])
def test_decomposed_entry_points_take_device_pointers(kind):
    # update_matrices_original with device arrays, reverse_decomposition into device outputs
    models = [_model(kind, 11, max_iter=100, reverse_on_device=True) for _ in range(2)]
    for m in models:
        m.optimize()
    m0 = models[0]
    vals = [m0.P0.data * 1.2, m0.A0.data * 0.9, m0.q0 * 1.1, m0.b0 * 0.95]   # all four: the engines equilibrate
    models[0].engine.update_matrices_original(*vals)
    models[1].engine.update_matrices_original(*[_cuda(v) for v in vals])
    outs = []
    for k, m in enumerate(models):
        o = m.engine.solve()
        n0, m_0 = m.n, m.m
        if k:
            outs_d = [torch.empty(v, dtype=torch.float64, device="cuda") for v in (n0, m_0, m_0)]
            m.engine.reverse_decomposition(True, *outs_d)
            rev = [t.cpu().numpy() for t in outs_d]
        else:
            rev = list(m.engine.reverse_decomposition(True)[:3])
        outs.append((o.iter, o.status, o.x, o.s, o.mu, m.engine.w(), *rev))
    assert outs[0][:2] == outs[1][:2]
    for a, c in zip(outs[0][2:], outs[1][2:]):
        _same(a, c)


def test_managed_memory_is_taken_like_device_memory():
    m1, m2 = _model("plain", 12, max_iter=100), _model("plain", 12, max_iter=100)
    for m in (m1, m2):
        m.optimize()
    q, b = _new_qb(m1, 40)
    m1.engine.update_qb_original(q, b)
    rt = E._cudart()
    rt.cudaMallocManaged.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_uint]
    rt.cudaFree.argtypes = [C.c_void_p]
    ptrs = []
    try:
        for v in (q, b):
            p = C.c_void_p()
            assert rt.cudaMallocManaged(C.byref(p), v.nbytes, 1) == 0
            ptrs.append(p.value)
            C.memmove(p.value, v.ctypes.data, v.nbytes)
        qm, bm = (_Managed(p, v.size) for p, v in zip(ptrs, (q, b)))
        m2.engine.update_qb_original(qm, bm)
        r1, r2 = m1.engine.solve(), m2.engine.solve()
        assert (r1.iter, r1.status) == (r2.iter, r2.status)
        _same(r1.x, r2.x), _same(r1.s, r2.s), _same(r1.mu, r2.mu)
        out = _Managed(ptrs[0], m2.n)                  # an output in managed memory
        m2.engine.solution(False, x=out)
        got = np.empty(m2.n)
        C.memmove(got.ctypes.data, ptrs[0], got.nbytes)
        x1 = np.empty(m1.n)
        m1.engine.solution(False, x=x1)
        _same(got, x1)
    finally:
        for p in ptrs:
            rt.cudaFree(p)


class _Managed:
    """a managed allocation seen through __cuda_array_interface__"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "strides": None,
                                         "version": 3}
