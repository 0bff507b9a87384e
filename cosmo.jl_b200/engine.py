"""ctypes binding of libcosmo_b200.so (include/cosmo_b200.h).

This is the stub a maintainer would write for any host language: plain
pointers and sizes, no torch types.  The Julia equivalent (``ccall``) is shown
in INTEGRATION.md.  There is no CPU fallback here: if the shared library is
missing or no CUDA device is present every call raises ``EngineError``.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Sequence

import numpy as np

from . import build as _build

OK = 0
ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA, ERR_ALLOC, ERR_NCCL, ERR_NUMERICAL = -1, -2, -3, -4, -5, -6
F64, F32 = 0, 1
ZERO, NONNEG, BOX, SOC, PSD_SQUARE, PSD_TRIANGLE, EXP, DUAL_EXP, POW, DUAL_POW, PSD_TRIANGLE_COMPLEX, CUSTOM = range(12)
CUSTOM_THREAD, CUSTOM_WARP, CUSTOM_BLOCK = 0, 1, 2
CUSTOM_HAS_IN_DUAL, CUSTOM_HAS_IN_POL_RECC = 1, 2
STATUS = {0: "Undetermined", 1: "Solved", 2: "Max_iter_reached", 3: "Time_limit_reached",
          4: "Primal_infeasible", 5: "Dual_infeasible", 6: "Unsolved"}
KKT_CG, KKT_MINRES_REDUCED, KKT_MINRES, KKT_LDL, KKT_LDL_SUPERNODAL = 0, 1, 2, 3, 4
ACC_EMPTY, ACC_ANDERSON = 0, 1
AA_TYPE2_QR, AA_TYPE2_NORMAL, AA_TYPE1 = 0, 1, 2
AA_RESTARTED_MEMORY, AA_ROLLING_MEMORY = 0, 1
AA_NO_REGULARIZER, AA_TIKONOV, AA_FROBENIUS = 0, 1, 2
AA_IMMEDIATE, AA_ITER, AA_ACCURACY = 0, 1, 2


class EngineError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("cosmo_b200 error %d: %s" % (code, msg))
        self.code = code


class CscStruct(C.Structure):
    _fields_ = [("nrows", C.c_int64), ("ncols", C.c_int64), ("colptr", C.c_void_p), ("rowval", C.c_void_p),
                ("nzval", C.c_void_p)]


class SetStruct(C.Structure):
    _fields_ = [("type", C.c_int32), ("max_iter", C.c_int32), ("dim", C.c_int64), ("l", C.c_void_p), ("u", C.c_void_p),
                ("alpha", C.c_double), ("tol", C.c_double)]


class CustomConeStruct(C.Structure):
    """cosmo_b200_custom_cone: a cone type whose device functions the engine compiles (include/cosmo_b200.h)."""
    _fields_ = [("name", C.c_char_p), ("source", C.c_char_p), ("granularity", C.c_int32), ("n_params", C.c_int32),
                ("flags", C.c_int32), ("reserved", C.c_int32)]


class ProblemStruct(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("index_base", C.c_int32), ("device", C.c_int32), ("flags", C.c_int32),
                ("m", C.c_int64), ("n", C.c_int64), ("P", CscStruct), ("A", CscStruct),
                ("q", C.c_void_p), ("b", C.c_void_p), ("n_sets", C.c_int64), ("sets", C.c_void_p),
                ("D", C.c_void_p), ("Dinv", C.c_void_p), ("E", C.c_void_p), ("Einv", C.c_void_p), ("c", C.c_double)]


class SettingsStruct(C.Structure):
    _fields_ = [("rho", C.c_double), ("sigma", C.c_double), ("alpha", C.c_double),
                ("eps_abs", C.c_double), ("eps_rel", C.c_double), ("eps_prim_inf", C.c_double),
                ("eps_dual_inf", C.c_double),
                ("max_iter", C.c_int64), ("check_termination", C.c_int32), ("check_infeasibility", C.c_int32),
                ("scaling", C.c_int32), ("adaptive_rho", C.c_int32), ("adaptive_rho_interval", C.c_int32),
                ("kkt_solver", C.c_int32),
                ("adaptive_rho_tolerance", C.c_double), ("adaptive_rho_max_adaptions", C.c_int64),
                ("RHO_MIN", C.c_double), ("RHO_MAX", C.c_double), ("RHO_TOL", C.c_double),
                ("RHO_EQ_OVER_RHO_INEQ", C.c_double), ("COSMO_INFTY", C.c_double), ("MIN_SCALING", C.c_double),
                ("time_limit", C.c_double), ("tol_constant", C.c_double), ("tol_exponent", C.c_double),
                ("verbose", C.c_int32), ("psd_max_sweeps", C.c_int32),
                ("accelerator", C.c_int32), ("accelerator_mem", C.c_int32), ("accelerator_min_mem", C.c_int32),
                ("safeguard", C.c_int32), ("safeguard_tol", C.c_double),
                ("adaptive_rho_fraction", C.c_double), ("setup_time", C.c_double), ("MAX_SCALING", C.c_double),
                ("obj_true", C.c_double), ("obj_true_tol", C.c_double)]


class ResultStruct(C.Structure):
    _fields_ = [("x", C.c_void_p), ("s", C.c_void_p), ("mu", C.c_void_p),
                ("obj_val", C.c_double), ("iter", C.c_int64), ("safeguarding_iter", C.c_int64),
                ("status", C.c_int32), ("_pad", C.c_int32),
                ("r_prim", C.c_double), ("r_dual", C.c_double), ("max_norm_prim", C.c_double),
                ("max_norm_dual", C.c_double), ("rho", C.c_double),
                ("rho_updates", C.c_void_p), ("rho_updates_cap", C.c_int64), ("n_rho_updates", C.c_int64),
                ("solver_time", C.c_double), ("setup_time", C.c_double), ("iter_time", C.c_double),
                ("proj_time", C.c_double), ("kkt_time", C.c_double), ("res_time", C.c_double),
                ("iter_time_device", C.c_double),
                ("kkt_inner_iterations", C.c_int64), ("kkt_multiplications", C.c_int64),
                ("kernel_launches", C.c_int64)]


class AcceleratorStruct(C.Structure):
    _fields_ = [("type", C.c_int32), ("memory", C.c_int32), ("regularizer", C.c_int32), ("activation", C.c_int32),
                ("lambda_", C.c_double), ("start_iter", C.c_int64), ("start_accuracy", C.c_double)]


class CompletionStruct(C.Structure):
    _fields_ = [("N", C.c_int64), ("row_offset", C.c_int64), ("dim", C.c_int64), ("new_of", C.c_void_p),
                ("n_steps", C.c_int64), ("steps", C.c_void_p), ("n_idx", C.c_int64), ("idx", C.c_void_p)]


class DecompositionStruct(C.Structure):
    _fields_ = [("n_orig", C.c_int64), ("m_orig", C.c_int64), ("n", C.c_int64), ("m", C.c_int64),
                ("n_plain", C.c_int64), ("plain", C.c_void_p), ("n_rows", C.c_int64), ("row", C.c_void_p),
                ("s_ptr", C.c_void_p), ("s_src", C.c_void_p), ("mu_src", C.c_void_p),
                ("n_cones", C.c_int64), ("cones", C.c_void_p)]


class ForwardMapStruct(C.Structure):
    _fields_ = [("n_orig", C.c_int64), ("m_orig", C.c_int64), ("n", C.c_int64), ("m", C.c_int64),
                ("nnzA_orig", C.c_int64), ("nnzA", C.c_int64), ("a_src", C.c_void_p), ("b_src", C.c_void_p),
                ("b_uncovered", C.c_void_p)]


def _signatures():
    """(restype, argtypes) of every entry point of include/cosmo_b200.h, in the header's order."""
    vp, i32, i64, f64, P = C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.POINTER
    rc = C.c_int
    return {
        "cosmo_b200_abi_version": (rc, []),
        "cosmo_b200_default_settings": (rc, [P(SettingsStruct)]),
        "cosmo_b200_create": (rc, [P(vp), P(ProblemStruct), P(SettingsStruct)]),
        "cosmo_b200_destroy": (None, [vp]),
        "cosmo_b200_last_error": (C.c_char_p, [vp]),
        "cosmo_b200_update_settings": (rc, [vp, P(SettingsStruct)]),
        "cosmo_b200_warm_start": (rc, [vp, vp, vp, vp]),
        "cosmo_b200_update_qb": (rc, [vp, vp, vp]),
        "cosmo_b200_update_matrices": (rc, [vp, vp, i64, vp, i64, vp, vp]),
        "cosmo_b200_update_rho": (rc, [vp, vp, f64]),
        "cosmo_b200_reset": (rc, [vp]),
        "cosmo_b200_set_accelerator": (rc, [vp, P(AcceleratorStruct)]),
        "cosmo_b200_accelerator_stats": (rc, [vp, P(i64)]),
        "cosmo_b200_solve": (rc, [vp, P(ResultStruct)]),
        "cosmo_b200_project": (rc, [vp, vp, vp]),
        "cosmo_b200_kkt_solve": (rc, [vp, vp, vp, P(i64)]),
        "cosmo_b200_residuals": (rc, [vp, vp, vp, vp, i32, P(f64)]),
        "cosmo_b200_spmv": (rc, [vp, i32, vp, vp]),
        "cosmo_b200_spmv_bench": (rc, [vp, i32, i32, P(f64), P(f64)]),
        "cosmo_b200_get_rho_vec": (rc, [vp, vp]),
        "cosmo_b200_get_scaling": (rc, [vp, vp, vp, P(f64)]),
        "cosmo_b200_get_w": (rc, [vp, vp]),
        "cosmo_b200_infeasibility_test": (rc, [vp, i32, vp, P(f64)]),
        "cosmo_b200_psd_lambda_max": (rc, [vp, vp, P(f64)]),
        "cosmo_b200_ldl_stats": (rc, [vp, P(f64)]),
        "cosmo_b200_ldl_symbolic": (rc, [P(ProblemStruct), P(i64), P(i64), P(i64), P(i64)]),
        "cosmo_b200_ldl_sn_stats": (rc, [vp, P(i64)]),
        "cosmo_b200_ldl_sn_symbolic": (rc, [P(ProblemStruct), P(i64), P(i64), P(i64), P(i64)]),
        "cosmo_b200_set_decomposition": (rc, [vp, P(DecompositionStruct)]),
        "cosmo_b200_set_decomposition_noncompact": (rc, [vp, P(DecompositionStruct)]),
        "cosmo_b200_reverse_decomposition": (rc, [vp, i32, vp, vp, vp, P(i64)]),
        "cosmo_b200_psd_complete": (rc, [i64, P(CompletionStruct), vp, P(i64)]),
        "cosmo_b200_set_forward_map": (rc, [vp, P(ForwardMapStruct)]),
        "cosmo_b200_update_matrices_original": (rc, [vp, vp, i64, vp, i64, vp, vp]),
        "cosmo_b200_set_caller_stream": (rc, [vp, vp]),
        "cosmo_b200_update_qb_original": (rc, [vp, vp, vp]),
        "cosmo_b200_original_qb": (rc, [vp, vp, vp]),
        "cosmo_b200_solution": (rc, [vp, i32, vp, vp, vp]),
        "cosmo_b200_rescale_iterates": (rc, [vp]),
        "cosmo_b200_comm_unique_id": (rc, [vp]),
        "cosmo_b200_comm_init": (rc, [vp, i32, i32, vp]),
        "cosmo_b200_comm_p2p_export": (rc, [vp, vp]),
        "cosmo_b200_comm_p2p_attach": (rc, [vp, vp, i32]),
        "cosmo_b200_custom_cone_compile": (rc, [P(CustomConeStruct), i32, C.c_char_p, i64]),
        "cosmo_b200_custom_cone_stats": (rc, [vp, P(i64)]),
        "cosmo_b200_psd_stats": (rc, [vp, P(i64)]),
        "cosmo_b200_tc_gemm_test": (rc, [i32, i32, i32, i32, vp, vp, vp, i32, P(f64), P(f64)]),
    }


SIGNATURES = _signatures()
EXPORTS = list(SIGNATURES)


def _check_rc(lib, rc, h=None):
    """EngineError unless rc is OK, with the last error of handle `h` (None: of the calls without a handle)."""
    if rc != OK:
        raise EngineError(rc, (lib.cosmo_b200_last_error(h) or b"").decode())


def _keyed(lib, h, fn, *args, ctype, keys, ints=()):
    """fn(*args, out) for an out array of len(keys) `ctype`s, checked as _check_rc does.  Returns the array as a dict in
    the order of `keys`, without the slots whose key is None and with the values of the keys in `ints` cast to int."""
    out = (ctype * len(keys))()
    _check_rc(lib, fn(*args, out), h)
    return {k: int(v) if k in ints else v for k, v in zip(keys, out) if k is not None}


def _i64(a, keep):
    a = np.ascontiguousarray(a, dtype=np.int64)
    keep.append(a)
    return _ptr(a)


def completion_struct(c, keep) -> CompletionStruct:
    """cosmo_b200_completion of a chordal.CompletionSchedule; the arrays it points to are appended to `keep`."""
    st = np.asarray(c.steps, dtype=np.int64).reshape(-1, 6)
    return CompletionStruct(int(c.N), int(c.row_offset), int(c.dim), _i64(c.new_of, keep), st.shape[0], _i64(st, keep),
                            len(c.idx), _i64(c.idx, keep))


def problem_struct(P, A, dtype, index_base, keep) -> ProblemStruct:
    """cosmo_b200_problem with dtype, index_base, m, n, P and A set from CSC matrices P and A with sorted indices
    (values as `dtype`, indices shifted by `index_base`); the arrays it points to are appended to `keep`."""
    prob = ProblemStruct()
    prob.dtype = F64 if np.dtype(dtype) == np.float64 else F32
    prob.index_base = index_base
    prob.m, prob.n = A.shape
    for name, M in (("P", P), ("A", A)):
        arrs = [np.ascontiguousarray(M.indptr, dtype=np.int64) + index_base,
                np.ascontiguousarray(M.indices, dtype=np.int64) + index_base, np.ascontiguousarray(M.data, dtype=dtype)]
        keep.extend(arrs)
        setattr(prob, name, CscStruct(M.shape[0], M.shape[1], *[_ptr(a) for a in arrs]))
    return prob


# cosmo_b200_reverse_decomposition / cosmo_b200_psd_complete stats[4]
REVERSE_STATS = ("cones_completed", "pinv_fallbacks", "workspace_bytes", "device_us")

_lib = None


def lib_path():
    return _build.LIB


def load_library(rebuild_if_stale=True):
    """dlopen the in-tree shared library (building it with nvcc when stale)."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if rebuild_if_stale and (not os.path.exists(path)):
        _build.build()
    if not os.path.exists(path):
        raise EngineError(ERR_CUDA, "libcosmo_b200.so is missing (run `python -c 'import __graft_entry__ as g; g.build()'`)")
    lib = C.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = argtypes, restype
    _lib = lib
    return lib


_nvrtc_ready = False


def preload_nvrtc():
    """Make libnvrtc.so.12 loadable for the engine's dlopen: the system's copy when the loader finds one, else the copy
    of the `nvidia-cuda-nvrtc` wheel that PyTorch installs, loaded with RTLD_GLOBAL so that the engine's
    dlopen("libnvrtc.so.12") finds it by its soname.  Without either, custom cones fail with ERR_UNSUPPORTED."""
    global _nvrtc_ready
    if _nvrtc_ready:
        return
    try:
        C.CDLL("libnvrtc.so.12", mode=C.RTLD_GLOBAL)
    except OSError:
        try:
            import nvidia.cuda_nvrtc as _w
        except ImportError:
            return
        for d in _w.__path__:
            path = os.path.join(d, "lib", "libnvrtc.so.12")
            if os.path.exists(path):
                C.CDLL(path, mode=C.RTLD_GLOBAL)
                break
        else:
            return
    _nvrtc_ready = True


def custom_cone_compile(cone_struct: CustomConeStruct, dtype=np.float64) -> bool:
    """cosmo_b200_custom_cone_compile: check and compile a cone type for `dtype` (no device needed).  True when this
    call compiled it, False when it was in the process-wide cache; EngineError with the compiler log otherwise."""
    lib = load_library()
    preload_nvrtc()
    log = C.create_string_buffer(1 << 16)
    rc = lib.cosmo_b200_custom_cone_compile(C.byref(cone_struct), F64 if np.dtype(dtype) == np.float64 else F32, log,
                                            len(log))
    if rc < 0:
        raise EngineError(rc, log.value.decode(errors="replace"))
    return rc == 1


def default_settings() -> SettingsStruct:
    s = SettingsStruct()
    rc = load_library().cosmo_b200_default_settings(C.byref(s))
    if rc != OK:
        raise EngineError(rc, "default_settings failed")
    return s


def _ptr(a):
    """The pointer argument of a NumPy array (None stays None; a device pointer from cuda_array passes as it is)."""
    if a is None or isinstance(a, C.c_void_p):
        return a
    return a.ctypes.data_as(C.c_void_p)


def is_cuda_array(a) -> bool:
    return hasattr(a, "__cuda_array_interface__")


def cuda_array(a, dtype, size=None, output=False):
    """(device pointer, stream) of an object with ``__cuda_array_interface__`` (torch, CuPy), after the checks the C
    calls rely on: the typestr of `dtype`, one dimension of length `size` (any length when None), C-contiguous and, for
    an output, not read-only.  `stream` is the interface's stream field (None: no ordering is needed)."""
    cai = a.__cuda_array_interface__
    want = np.dtype(dtype).newbyteorder("<").str
    if cai.get("typestr") != want:
        raise EngineError(ERR_INVALID, "CUDA array of typestr %r where %r is needed" % (cai.get("typestr"), want))
    shape = tuple(cai.get("shape", ()))
    if len(shape) != 1 or (size is not None and shape[0] != size):
        raise EngineError(ERR_INVALID, "CUDA array of shape %s where (%s,) is needed" % (shape, "n" if size is None else size))
    strides = cai.get("strides")
    if strides is not None and shape[0] > 1 and tuple(strides) != (np.dtype(dtype).itemsize,):
        raise EngineError(ERR_INVALID, "CUDA array is not C-contiguous (strides %s)" % (tuple(strides),))
    ptr, readonly = cai["data"]
    if output and readonly:
        raise EngineError(ERR_INVALID, "CUDA array given as an output is read-only")
    stream = cai.get("stream")
    if stream == 0:
        raise EngineError(ERR_INVALID, "__cuda_array_interface__ stream 0 is not allowed (1: legacy, 2: per-thread)")
    return ptr, stream


def caller_stream_handle(stream):
    """The cudaStream_t of cosmo_b200_set_caller_stream for an interface stream field: 1 is the legacy default stream
    (NULL), 2 the per-thread default stream (cudaStreamPerThread, the same value), any other integer the stream."""
    return None if stream == 1 else int(stream)


_cudart_lib = None


def _cudart():
    """libcudart.so.12: the system's copy, else the one of the `nvidia-cuda-runtime` wheel that PyTorch installs."""
    global _cudart_lib
    if _cudart_lib is None:
        try:
            lib = C.CDLL("libcudart.so.12")
        except OSError:
            import nvidia.cuda_runtime as _w
            lib = C.CDLL(os.path.join(list(_w.__path__)[0], "lib", "libcudart.so.12"))
        lib.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
        lib.cudaStreamSynchronize.argtypes = [C.c_void_p]
        _cudart_lib = lib
    return _cudart_lib


def _ordered_copy(dst, src, nbytes, stream):
    """cudaMemcpy(cudaMemcpyDefault) between a CUDA array and host memory, ordered on both sides.  Before: the array's
    stream (the interface's stream field) is synchronised, or, when it names none (torch), the whole device, so a write
    on any stream of this process, the caller stream of an engine included, has landed.  After: the legacy stream the
    copy ran on is synchronised, so the data is in place for every stream when this returns."""
    rt = _cudart()
    rc = rt.cudaStreamSynchronize(caller_stream_handle(stream)) if stream is not None else rt.cudaDeviceSynchronize()
    if rc == 0 and nbytes:
        rc = rt.cudaMemcpy(dst, src, nbytes, 4) or rt.cudaStreamSynchronize(None)   # 4: cudaMemcpyDefault
    if rc != 0:
        raise EngineError(ERR_CUDA, "copy between a CUDA array and host memory failed (cudaError %d)" % rc)


def copy_into(dst, src: np.ndarray):
    """Write the host array `src` into `dst`: a CUDA array (checked by cuda_array) or a NumPy array of src's dtype."""
    if not is_cuda_array(dst):
        dst[...] = src
        return
    src = np.ascontiguousarray(src)
    ptr, stream = cuda_array(dst, src.dtype, src.size, output=True)
    _ordered_copy(ptr, src.ctypes.data, src.nbytes, stream)


def to_host(a, dtype=np.float64) -> np.ndarray:
    """A NumPy copy of a 1-D CUDA array of `dtype`, or np.asarray of anything else."""
    if not is_cuda_array(a):
        return np.asarray(a, dtype=dtype)
    ptr, stream = cuda_array(a, dtype)
    out = np.empty(a.__cuda_array_interface__["shape"][0], dtype=dtype)
    _ordered_copy(out.ctypes.data, ptr, out.nbytes, stream)
    return out


def nccl_unique_id() -> bytes:
    buf = (C.c_char * 128)()
    lib = load_library()
    _check_rc(lib, lib.cosmo_b200_comm_unique_id(C.cast(buf, C.c_void_p)))
    return bytes(buf)


class SolveOutput:
    __slots__ = ("x", "s", "mu", "obj_val", "iter", "safeguarding_iter", "status", "r_prim", "r_dual", "max_norm_prim", "max_norm_dual",
                 "rho", "rho_updates", "times", "kkt_inner_iterations", "kkt_multiplications", "kernel_launches")


class Engine:
    """Owns one ``cosmo_b200_handle`` (one problem resident in HBM on one GPU).

    ``P`` and ``A`` are SciPy CSC matrices (the same three arrays Julia's
    SparseMatrixCSC holds); ``sets`` is a list of ``(type, dim, l, u)`` or, for the
    exponential / power cones, ``(type, 3, None, None, {"alpha": a, "max_iter": k, "tol": t})``.
    """

    def __init__(self, P, q, A, b, sets: Sequence[tuple], settings: Optional[SettingsStruct] = None,
                 D=None, E=None, c: float = 1.0, dtype=np.float64, device: int = 0, julia_indexing: bool = True,
                 equilibrate: bool = False):
        """equilibrate=True: the data are unscaled and settings.scaling != 0 -- the engine runs scale_ruiz! on the
        device (COSMO_B200_PROBLEM_EQUILIBRATE); read D, E, c back with scaling()."""
        import scipy.sparse as sp
        self._lib = load_library()
        self.dtype = np.dtype(dtype)
        if self.dtype not in (np.dtype(np.float64), np.dtype(np.float32)):
            raise EngineError(ERR_UNSUPPORTED, "dtype must be float64 or float32")
        T = self.dtype
        P = sp.csc_matrix(P)
        A = sp.csc_matrix(A)
        P.sort_indices()
        A.sort_indices()
        self.m, self.n = A.shape
        self.n_psd = sum(1 for t in sets if t[0] in (PSD_SQUARE, PSD_TRIANGLE, PSD_TRIANGLE_COMPLEX) and int(t[1]) > 0)
        keep = []  # keep host arrays alive during create
        set_arr = (SetStruct * max(len(sets), 1))()
        for i, (typ, dim, l, u, *extra) in enumerate(sets):
            set_arr[i].type = int(typ)
            set_arr[i].dim = int(dim)
            if typ == CUSTOM:
                # u: the cone type (anything with a `struct()` -> CustomConeStruct, model.CustomConeType), l: parameters
                preload_nvrtc()
                cs = u.struct()
                keep.append(cs)
                set_arr[i].u = C.cast(C.pointer(cs), C.c_void_p)
                if l is not None and len(l):
                    pa = np.ascontiguousarray(l, dtype=T)
                    keep.append(pa)
                    set_arr[i].l = _ptr(pa)
                continue
            if extra and extra[0]:
                set_arr[i].alpha = float(extra[0].get("alpha", 0.0))
                set_arr[i].max_iter = int(extra[0].get("max_iter", 0))
                set_arr[i].tol = float(extra[0].get("tol", 0.0))
            if l is not None:
                la = np.ascontiguousarray(l, dtype=T)
                ua = np.ascontiguousarray(u, dtype=T)
                keep.extend([la, ua])
                set_arr[i].l = _ptr(la)
                set_arr[i].u = _ptr(ua)
        prob = problem_struct(P, A, T, 1 if julia_indexing else 0, keep)
        prob.device = device
        prob.flags = 1 if equilibrate else 0
        qa = np.ascontiguousarray(q, dtype=T)
        ba = np.ascontiguousarray(b, dtype=T)
        keep.extend([qa, ba])
        prob.q, prob.b = _ptr(qa), _ptr(ba)
        prob.n_sets = len(sets)
        prob.sets = C.cast(set_arr, C.c_void_p)
        if D is not None and E is not None:
            Da = np.ascontiguousarray(D, dtype=T)
            Ea = np.ascontiguousarray(E, dtype=T)
            Di = np.ascontiguousarray(1.0 / np.asarray(D, dtype=np.float64), dtype=T)
            Ei = np.ascontiguousarray(1.0 / np.asarray(E, dtype=np.float64), dtype=T)
            keep.extend([Da, Ea, Di, Ei])
            prob.D, prob.Dinv, prob.E, prob.Einv = _ptr(Da), _ptr(Di), _ptr(Ea), _ptr(Ei)
        prob.c = float(c)
        self.settings = settings if settings is not None else default_settings()
        h = C.c_void_p()
        _check_rc(self._lib, self._lib.cosmo_b200_create(C.byref(h), C.byref(prob), C.byref(self.settings)))
        self._h = h
        self.n_orig, self.m_orig = 0, 0     # the original problem of a decomposition map (set_decomposition)
        self._fwd_sizes = None              # (n_orig, m_orig) of the forward map (set_forward_map)
        del keep

    # ---- lifecycle --------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None):
            self._lib.cosmo_b200_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        _check_rc(self._lib, rc, self._h)

    def _arr(self, a, size=None, dtype=None, output=False):
        """An array argument of the calls that take host or device memory.  A CUDA array passes as its device pointer
        (checked by cuda_array; its stream, when it names one, becomes the caller stream).  A host input goes as _vec
        makes it; a host output must be a writable C-contiguous NumPy array of the dtype and size."""
        dtype = np.dtype(dtype or self.dtype)
        if a is None:
            return None
        if is_cuda_array(a):
            ptr, stream = cuda_array(a, dtype, size, output)
            if stream is not None:
                self.set_caller_stream(caller_stream_handle(stream))
            return C.c_void_p(ptr)
        if not output:
            return self._vec(a, size) if dtype == self.dtype else self._vec_of(a, size, dtype)
        if not (isinstance(a, np.ndarray) and a.dtype == dtype and a.flags.c_contiguous and a.flags.writeable
                and a.ndim == 1 and (size is None or a.shape[0] == size)):
            raise EngineError(ERR_INVALID, "an output must be a writable C-contiguous 1-D %s array of length %s" % (dtype, size))
        return a

    @staticmethod
    def _vec_of(a, size, dtype):
        a = np.ascontiguousarray(a, dtype=dtype)
        if size is not None and a.shape != (size,):
            raise EngineError(ERR_INVALID, "vector has wrong length")
        return a

    def _vec(self, a, size=None):
        """`a` as a flat contiguous array of the engine's dtype (None stays None), of length `size` if one is given."""
        if a is None:
            return None
        a = np.ascontiguousarray(a, dtype=self.dtype)
        if size is not None and a.shape != (size,):
            raise EngineError(ERR_INVALID, "vector has wrong length")
        return a.ravel()

    # ---- updates ------------------------------------------------------------
    def update_settings(self, settings: SettingsStruct):
        self.settings = settings
        self._check(self._lib.cosmo_b200_update_settings(self._h, C.byref(settings)))

    def warm_start(self, x=None, s=None, mu=None):
        x, s, mu = self._arr(x, self.n), self._arr(s, self.m), self._arr(mu, self.m)
        self._check(self._lib.cosmo_b200_warm_start(self._h, _ptr(x), _ptr(s), _ptr(mu)))

    def update_qb(self, q=None, b=None):
        q, b = self._arr(q, self.n), self._arr(b, self.m)
        self._check(self._lib.cosmo_b200_update_qb(self._h, _ptr(q), _ptr(b)))

    # ---- caller arrays in device memory ------------------------------------------
    def set_caller_stream(self, stream=None):
        """cosmo_b200_set_caller_stream: the cudaStream_t (an integer; None: the legacy default stream) that caller device
        memory is ordered on, e.g. ``torch.cuda.current_stream().cuda_stream``."""
        self._check(self._lib.cosmo_b200_set_caller_stream(self._h, None if stream is None else C.c_void_p(stream)))

    def _orig_sizes(self):
        return self._fwd_sizes or (self.n, self.m)

    def update_qb_original(self, q=None, b=None):
        """cosmo_b200_update_qb_original: update!(q=, b=) with the model's unscaled fp64 values (host or CUDA arrays;
        None: unchanged), mapped through the forward map when one is set and scaled on the device."""
        n0, m0 = self._orig_sizes()
        q, b = self._arr(q, n0, np.float64), self._arr(b, m0, np.float64)
        self._check(self._lib.cosmo_b200_update_qb_original(self._h, _ptr(q), _ptr(b)))

    def original_qb(self, q=None, b=None):
        """cosmo_b200_original_qb into the given fp64 outputs (host or CUDA arrays; None: skipped); returns (q, b)."""
        n0, m0 = self._orig_sizes()
        pq, pb = self._arr(q, n0, np.float64, output=True), self._arr(b, m0, np.float64, output=True)
        self._check(self._lib.cosmo_b200_original_qb(self._h, _ptr(pq), _ptr(pb)))
        return q, b

    def solution(self, complete_dual=False, x=None, y=None, s=None):
        """cosmo_b200_solution: the last solve's unscaled solution (x, y = -mu, s) in fp64 in the original coordinates,
        into the given outputs (host or CUDA arrays; None: skipped).  Returns (x, y, s)."""
        n0, m0 = (self.n_orig, self.m_orig) if self.n_orig or self.m_orig else (self.n, self.m)
        px, py, ps = (self._arr(a, k, np.float64, output=True) for a, k in ((x, n0), (y, m0), (s, m0)))
        self._check(self._lib.cosmo_b200_solution(self._h, int(bool(complete_dual)), _ptr(px), _ptr(py), _ptr(ps)))
        return x, y, s

    def rescale_iterates(self):
        """cosmo_b200_rescale_iterates: the host's unscale / rescale round trip between two solves, on the device."""
        self._check(self._lib.cosmo_b200_rescale_iterates(self._h))

    def update_matrices(self, Px=None, Ax=None, q=None, b=None):
        """cosmo_b200_update_matrices: new values of P and A on the pattern of create -- ``Px`` / ``Ax`` are the ``data``
        arrays of the CSC matrices with sorted indices -- and optionally q and b (None: unchanged).  The engine is left
        as a new Engine with these data would be; an equilibrating engine needs all four, unscaled."""
        self._update_values(self._lib.cosmo_b200_update_matrices, (self.n, self.m), Px, Ax, q, b)

    def update_rho(self, rho_vec, rho):
        rv = self._vec(rho_vec, self.m)
        self._check(self._lib.cosmo_b200_update_rho(self._h, _ptr(rv), float(rho)))

    def reset(self):
        self._check(self._lib.cosmo_b200_reset(self._h))

    def set_accelerator(self, acc: Optional[AcceleratorStruct]):
        """cosmo_b200_set_accelerator: the Anderson variant and activation reason (None: the default)."""
        self._check(self._lib.cosmo_b200_set_accelerator(self._h, None if acc is None else C.byref(acc)))

    def comm_init(self, nranks, rank, unique_id: Optional[bytes]):
        buf = C.create_string_buffer(unique_id, 128) if unique_id is not None else None
        self._check(self._lib.cosmo_b200_comm_init(self._h, nranks, rank, C.cast(buf, C.c_void_p) if buf else None))

    def p2p_export(self) -> bytes:
        buf = (C.c_char * 128)()
        self._check(self._lib.cosmo_b200_comm_p2p_export(self._h, C.cast(buf, C.c_void_p)))
        return bytes(buf)

    def p2p_attach(self, blobs: bytes, nranks: int):
        buf = C.create_string_buffer(blobs, len(blobs))
        self._check(self._lib.cosmo_b200_comm_p2p_attach(self._h, C.cast(buf, C.c_void_p), nranks))

    # ---- the hot loop ----------------------------------------------------------
    def solve(self, out_x=None, out_s=None, out_mu=None, copy_out=True) -> SolveOutput:
        """cosmo_b200_solve.  Output buffers may be caller-provided (e.g. pinned, or CUDA arrays); copy_out=False leaves
        the iterates on the device only (x, s, mu None)."""
        T = self.dtype
        x, s, mu = ((o if o is not None or not copy_out else np.empty(k, dtype=T))
                    for o, k in ((out_x, self.n), (out_s, self.m), (out_mu, self.m)))
        rho_updates = np.zeros(256, dtype=np.float64)
        r = ResultStruct()
        r.x, r.s, r.mu = (_ptr(self._arr(a, k, output=True)) for a, k in ((x, self.n), (s, self.m), (mu, self.m)))
        r.rho_updates = _ptr(rho_updates)
        r.rho_updates_cap = rho_updates.shape[0]
        self._check(self._lib.cosmo_b200_solve(self._h, C.byref(r)))
        o = SolveOutput()
        o.x, o.s, o.mu = x, s, mu
        o.obj_val, o.iter, o.status = r.obj_val, r.iter, STATUS[r.status]
        o.safeguarding_iter = r.safeguarding_iter
        o.r_prim, o.r_dual, o.max_norm_prim, o.max_norm_dual = r.r_prim, r.r_dual, r.max_norm_prim, r.max_norm_dual
        o.rho = r.rho
        o.rho_updates = rho_updates[:min(r.n_rho_updates, rho_updates.shape[0])].copy()
        o.times = {"solver_time": r.solver_time, "setup_time": r.setup_time, "iter_time": r.iter_time,
                   "proj_time": r.proj_time, "kkt_time": r.kkt_time, "res_time": r.res_time,
                   "iter_time_device": r.iter_time_device}
        o.kkt_inner_iterations, o.kkt_multiplications = r.kkt_inner_iterations, r.kkt_multiplications
        o.kernel_launches = r.kernel_launches
        return o

    # ---- plugin-granularity entry points ------------------------------------
    def project(self, w_s):
        w_s = self._vec(w_s, self.m)
        out = np.empty(self.m, dtype=self.dtype)
        self._check(self._lib.cosmo_b200_project(self._h, _ptr(w_s), _ptr(out)))
        return out

    def kkt_solve(self, rhs):
        rhs = self._vec(rhs, self.n + self.m)
        sol = np.empty(self.n + self.m, dtype=self.dtype)
        inner = C.c_int64(0)
        self._check(self._lib.cosmo_b200_kkt_solve(self._h, _ptr(rhs), _ptr(sol), C.byref(inner)))
        return sol, inner.value

    def residuals(self, x, s, mu, ignore_scaling=False):
        x, s, mu = self._vec(x, self.n), self._vec(s, self.m), self._vec(mu, self.m)
        out = (C.c_double * 5)()
        self._check(self._lib.cosmo_b200_residuals(self._h, _ptr(x), _ptr(s), _ptr(mu), int(ignore_scaling), out))
        return tuple(out)

    def spmv(self, which, x):
        size_in = self.m if which == 1 else self.n + self.m if which == 3 else self.n
        size_out = self.m if which == 0 else self.n
        x = self._vec(x, size_in)
        y = np.empty(size_out, dtype=self.dtype)
        self._check(self._lib.cosmo_b200_spmv(self._h, which, _ptr(x), _ptr(y)))
        return y

    def spmv_bench(self, which, reps=20):
        ms, nbytes = C.c_double(0), C.c_double(0)
        self._check(self._lib.cosmo_b200_spmv_bench(self._h, which, reps, C.byref(ms), C.byref(nbytes)))
        return ms.value, nbytes.value

    def rho_vec(self):
        out = np.empty(self.m, dtype=self.dtype)
        self._check(self._lib.cosmo_b200_get_rho_vec(self._h, _ptr(out)))
        return out

    def w(self):
        out = np.empty(self.n + self.m, dtype=self.dtype)
        self._check(self._lib.cosmo_b200_get_w(self._h, _ptr(out)))
        return out

    def scaling(self):
        """(D, E, c) as used by the engine (cosmo_b200_get_scaling)."""
        D = np.empty(self.n, dtype=self.dtype)
        E = np.empty(self.m, dtype=self.dtype)
        c = C.c_double(1.0)
        self._check(self._lib.cosmo_b200_get_scaling(self._h, _ptr(D), _ptr(E), C.byref(c)))
        return D.astype(np.float64), E.astype(np.float64), float(c.value)

    def _read_out(self, fn, *args, ctype, keys, ints=()):
        return _keyed(self._lib, self._h, fn, self._h, *args, ctype=ctype, keys=keys, ints=ints)

    def psd_stats(self):
        """Which path projected the large PSD cones so far (cosmo_b200_psd_stats)."""
        keys = ("tc_projections", "tc_fallbacks", "tc_last_steps", "tc_last_checks", None, None, "jacobi_last_sweeps", "tc_slices")
        return self._read_out(self._lib.cosmo_b200_psd_stats, ctype=C.c_int64, keys=keys)

    def custom_cone_stats(self):
        """cosmo_b200_custom_cone_stats, keyed by CUSTOM_CONE_STATS."""
        return self._read_out(self._lib.cosmo_b200_custom_cone_stats, ctype=C.c_int64, keys=CUSTOM_CONE_STATS)

    def accelerator_stats(self):
        """Accelerator events of the last solve (cosmo_b200_accelerator_stats), keyed by ACCELERATOR_STATS."""
        return self._read_out(self._lib.cosmo_b200_accelerator_stats, ctype=C.c_int64, keys=ACCELERATOR_STATS)

    def infeasibility_test(self, which, delta):
        """cosmo_b200_infeasibility_test: is_primal_infeasible! (which = 0, delta = delta_y, m) or is_dual_infeasible!
        (which = 1, delta = delta_x, n) on the engine's data; returns a dict keyed by INFEASIBILITY_RECORD."""
        delta = self._vec(delta, self.m if which == 0 else self.n)
        return self._read_out(self._lib.cosmo_b200_infeasibility_test, int(which), _ptr(delta), ctype=C.c_double,
                              keys=INFEASIBILITY_RECORD, ints=("verdict", "gate", "families", "psd_unconverged"))

    def psd_lambda_max(self, v):
        """cosmo_b200_psd_lambda_max: lambda_max of every PSD cone of mat(v) (set order) as the certificate computes it."""
        v = self._vec(v, self.m)
        lam = np.zeros(max(self.n_psd, 1), dtype=np.float64)
        self._check(self._lib.cosmo_b200_psd_lambda_max(self._h, _ptr(v), lam.ctypes.data_as(C.POINTER(C.c_double))))
        return lam[:self.n_psd]

    def ldl_stats(self):
        """State of the direct LDL' plugin (cosmo_b200_ldl_stats), keyed by LDL_STATS."""
        return self._read_out(self._lib.cosmo_b200_ldl_stats, ctype=C.c_double, keys=LDL_STATS, ints=LDL_STATS[:6])

    def ldl_sn_stats(self):
        """State of the supernodal LDL' plugin (cosmo_b200_ldl_sn_stats), keyed by LDL_SN_STATS."""
        return self._read_out(self._lib.cosmo_b200_ldl_sn_stats, ctype=C.c_int64, keys=LDL_SN_STATS)

    # ---- reverse of a chordal decomposition ---------------------------------
    def set_decomposition(self, d):
        """cosmo_b200_set_decomposition, or cosmo_b200_set_decomposition_noncompact for the map of the traditional
        transformation (d.traditional): hand over the map of a chordal.DecompositionArrays (None clears it)."""
        if d is None:
            self._check(self._lib.cosmo_b200_set_decomposition(self._h, None))
            self.n_orig, self.m_orig = 0, 0
            return
        keep = []
        cones = (CompletionStruct * max(len(d.cones), 1))()
        for k, c in enumerate(d.cones):
            cones[k] = completion_struct(c, keep)
        sptr = np.asarray(d.s_ptr, dtype=np.int64)
        ds = DecompositionStruct(int(d.n_orig), int(d.m_orig), int(d.n), int(d.m),
                                 np.asarray(d.plain).reshape(-1, 3).shape[0], _i64(d.plain, keep),
                                 len(d.row), _i64(d.row, keep), _i64(sptr, keep), _i64(d.s_src, keep),
                                 None if d.traditional else _i64(d.mu_src, keep), len(d.cones), C.cast(cones, C.c_void_p))
        setter = self._lib.cosmo_b200_set_decomposition_noncompact if d.traditional else self._lib.cosmo_b200_set_decomposition
        self._check(setter(self._h, C.byref(ds)))
        self.n_orig, self.m_orig = int(d.n_orig), int(d.m_orig)

    def reverse_decomposition(self, complete_dual=False, x=True, s=True, mu=True):
        """cosmo_b200_reverse_decomposition: the unscaled (x, s, mu) of the original problem in fp64 from the iterates of
        the last solve (a False argument skips that output: None in its place; an fp64 array, host or CUDA, is written
        into), and the stats keyed by REVERSE_STATS."""
        out = [(np.empty(n, dtype=np.float64) if want else None) if isinstance(want, bool) else want
               for want, n in ((x, self.n_orig), (s, self.m_orig), (mu, self.m_orig))]
        ptrs = [_ptr(self._arr(a, n, np.float64, output=True)) for a, n in zip(out, (self.n_orig, self.m_orig, self.m_orig))]
        stats = self._read_out(self._lib.cosmo_b200_reverse_decomposition, int(bool(complete_dual)), *ptrs,
                               ctype=C.c_int64, keys=REVERSE_STATS)
        return out[0], out[1], out[2], stats

    # ---- values of the original problem onto the decomposed one ---------------
    def set_forward_map(self, f):
        """cosmo_b200_set_forward_map: hand over a chordal.ForwardArrays (None clears it)."""
        if f is None:
            self._check(self._lib.cosmo_b200_set_forward_map(self._h, None))
            self._fwd_sizes = None
            return
        keep = []
        unc = np.ascontiguousarray(f.b_uncovered, dtype=np.uint8)
        fs = ForwardMapStruct(int(f.n_orig), int(f.m_orig), int(f.n), int(f.m), int(f.nnzA_orig), len(f.a_src),
                              _i64(f.a_src, keep), _i64(f.b_src, keep), _ptr(unc))
        self._check(self._lib.cosmo_b200_set_forward_map(self._h, C.byref(fs)))
        self._fwd_sizes = (int(f.n_orig), int(f.m_orig))

    def update_matrices_original(self, Px=None, Ax=None, q=None, b=None):
        """cosmo_b200_update_matrices_original: update_matrices with the ``data`` arrays of P and A (sorted CSC), q and b
        of the problem the chordal decomposition started from; the forward map (set_forward_map) carries them onto the
        decomposed problem on the device."""
        # without a map the engine reads none of q, b and answers ERR_INVALID: their lengths go unchecked here
        sizes = self._fwd_sizes or (None, None)
        self._update_values(self._lib.cosmo_b200_update_matrices_original, sizes, Px, Ax, q, b)

    def _update_values(self, fn, qb_sizes, Px, Ax, q, b):
        nnz = [0 if a is None else a.__cuda_array_interface__["shape"][0] if is_cuda_array(a) else None for a in (Px, Ax)]
        Px, Ax = self._arr(Px), self._arr(Ax)
        q, b = self._arr(q, qb_sizes[0]), self._arr(b, qb_sizes[1])
        nnz = [a.size if k is None else k for a, k in zip((Px, Ax), nnz)]
        self._check(fn(self._h, _ptr(Px), nnz[0], _ptr(Ax), nnz[1], _ptr(q), _ptr(b)))


def psd_complete(Y, schedule):
    """cosmo_b200_psd_complete: the device completion of the symmetric matrix Y (upper triangle read) along a
    chordal.CompletionSchedule.  Returns (completed matrix, stats keyed by REVERSE_STATS)."""
    lib = load_library()
    W = np.array(Y, dtype=np.float64, order="F", copy=True)
    keep = []
    cs = completion_struct(schedule, keep)
    stats = _keyed(lib, None, lib.cosmo_b200_psd_complete, int(cs.N), C.byref(cs), W.ctypes.data_as(C.c_void_p),
                   ctype=C.c_int64, keys=REVERSE_STATS)
    return W, stats


# cosmo_b200_infeasibility_test's out[8]: "gate2" is |Dinv A'dy|_inf (primal) or q'dx (dual), "gate3" dy'b of the
# normalized -dy (primal) or |Dinv P dx|_inf (dual); "families" has bit 0 rows, 1 SOC, 2 PSD, 3 Exp/Pow, 4 custom cones
INFEASIBILITY_RECORD = ("verdict", "gate", "norm", "gate2", "gate3", "box_sum", "families", "psd_unconverged")
FAMILY_ROWS, FAMILY_SOC, FAMILY_PSD, FAMILY_C3, FAMILY_CUSTOM = 1, 2, 4, 8, 16

CUSTOM_CONE_STATS = ("types", "cones", "compilations", "cache_hits")

LDL_STATS = ("N", "nnz_triu_K", "nnz_L", "levels", "solve_nodes", "factorizations", "factor_time", "symbolic_time")

LDL_SN_STATS = ("supernodes", "max_width", "explicit_zeros", "levels", "small_path", "tiled_path", "solve_nodes",
                "update_flops")
LDL_SN_SYMBOLIC_STATS = ("supernodes", "max_width", "stored", "explicit_zeros", "levels", "simplicial_levels", "nnz_L",
                         "update_flops")

ACCELERATOR_STATS = ("accepted", "declined", "rejected", "rho_restarts", "memory_restarts", "activated_at")


def ldl_symbolic(P, A):
    """cosmo_b200_ldl_symbolic: the host symbolic analysis of K = [P + sigma I, A'; A, -diag(1/rho)] (no GPU needed).
    Returns (perm, parent, colcount, level), each of length n + m and in pivot order."""
    import scipy.sparse as sp
    lib = load_library()
    P = sp.csc_matrix(P, dtype=np.float64)
    A = sp.csc_matrix(A, dtype=np.float64)
    P.sort_indices()
    A.sort_indices()
    keep = []
    prob = problem_struct(P, A, np.float64, 0, keep)
    out = [np.zeros(prob.n + prob.m, dtype=np.int64) for _ in range(4)]
    _check_rc(lib, lib.cosmo_b200_ldl_symbolic(C.byref(prob), *[o.ctypes.data_as(C.POINTER(C.c_int64)) for o in out]))
    return tuple(out)


def ldl_sn_symbolic(P, A):
    """cosmo_b200_ldl_sn_symbolic: the supernodal symbolic analysis (no GPU needed).  Returns (perm, snode_ptr,
    snode_parent, stats): the postordered pivots, the supernodes' column pointers and parents, and a dict keyed by
    LDL_SN_SYMBOLIC_STATS."""
    import scipy.sparse as sp
    lib = load_library()
    P = sp.csc_matrix(P, dtype=np.float64)
    A = sp.csc_matrix(A, dtype=np.float64)
    P.sort_indices()
    A.sort_indices()
    keep = []
    prob = problem_struct(P, A, np.float64, 0, keep)
    N = prob.n + prob.m
    perm, sptr, spar = np.zeros(N, dtype=np.int64), np.zeros(N + 1, dtype=np.int64), np.zeros(max(N, 1), dtype=np.int64)
    stats = _keyed(lib, None, lib.cosmo_b200_ldl_sn_symbolic, C.byref(prob),
                   *[o.ctypes.data_as(C.POINTER(C.c_int64)) for o in (perm, sptr, spar)], ctype=C.c_int64,
                   keys=LDL_SN_SYMBOLIC_STATS)
    ns = stats["supernodes"]
    return perm, sptr[:ns + 1].copy(), spar[:ns].copy(), stats


def tc_gemm(A, B, slices=8, groups=0, reps=0):
    """C = A @ B for symmetric commuting fp64 matrices through the int8-sliced wgmma product kernel
    (diagnostic entry `cosmo_b200_tc_gemm_test`).  Returns (C, ms_per_product, (|C|_F^2, |I - C|_F^2))."""
    lib = load_library()
    A = np.asfortranarray(A, dtype=np.float64)
    B = np.asfortranarray(B, dtype=np.float64)
    N = A.shape[0]
    assert A.shape == (N, N) and B.shape == (N, N)
    Cm = np.zeros((N, N), dtype=np.float64, order="F")
    ms = C.c_double(0.0)
    fr = (C.c_double * 2)()
    _check_rc(lib, lib.cosmo_b200_tc_gemm_test(N, slices, groups, 0, A.ctypes.data, B.ctypes.data, Cm.ctypes.data, reps,
                                               C.byref(ms), fr))
    return Cm, ms.value, (fr[0], fr[1])
