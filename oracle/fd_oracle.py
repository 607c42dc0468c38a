"""ctypes binding of the CPU oracle (oracle/libfd_oracle.so).

TEST INFRASTRUCTURE ONLY — see oracle/fd_oracle.h.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs import this module; the product
package (finitediff.jl_b200/) never does.

Index conventions follow the reference (Julia): all index arrays are Int64 and 1-based.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libfd_oracle.so"

FORWARD, CENTRAL = 0, 1
SP_NONE, SP_CSC_SAME, SP_CSC, SP_COO, SP_BANDED = 0, 1, 2, 3, 4
J_NZVAL, J_DENSE, J_BAND, J_SLOTS = 0, 1, 2, 3

_i64p = C.POINTER(C.c_int64)
_f64p = C.POINTER(C.c_double)

FDO_FN = C.CFUNCTYPE(None, C.c_void_p, _f64p, _f64p)


class _Problem(C.Structure):
    _fields_ = [
        ("sp_kind", C.c_int), ("j_kind", C.c_int),
        ("m", C.c_int64), ("n", C.c_int64),
        ("colptr", _i64p), ("rowval", _i64p),
        ("rows_index", _i64p), ("cols_index", _i64p), ("nnz", C.c_int64),
        ("slots", _i64p),
        ("l", C.c_int64), ("u", C.c_int64),
        ("ldJ", C.c_int64), ("j_len", C.c_int64),
    ]


class _Cache(C.Structure):
    _fields_ = [("x1", _f64p), ("x2", _f64p), ("fx", _f64p), ("fx1", _f64p)]


class _Opts(C.Structure):
    _fields_ = [
        ("fdtype", C.c_int), ("relstep", C.c_double), ("absstep", C.c_double), ("dir", C.c_double),
        ("colorvec", _i64p), ("f_in", _f64p), ("eps_override", _f64p), ("eps_out", _f64p),
        ("no_drift", C.c_int), ("nthreads", C.c_int), ("fcalls", C.c_int64),
    ]


class SynthTridiagCtx(C.Structure):
    _fields_ = [("n", C.c_int64), ("nthreads", C.c_int)]


class SynthLap5Ctx(C.Structure):
    _fields_ = [("g", C.c_int64), ("nthreads", C.c_int)]


class SynthEllCtx(C.Structure):
    _fields_ = [("m", C.c_int64), ("K", C.c_int64), ("cols", C.POINTER(C.c_int32)), ("coef", _f64p),
                ("nthreads", C.c_int)]


class SynthRank1Ctx(C.Structure):
    _fields_ = [("n", C.c_int64), ("w", _f64p), ("nthreads", C.c_int)]


def build(force: bool = False) -> Path:
    """Compile the oracle with the committed Makefile (gcc, no GPU needed)."""
    srcs = [_HERE / "fd_oracle.c", _HERE / "synth_fns.c", _HERE / "fd_oracle.h", _HERE / "Makefile"]
    if force or not _LIB_PATH.exists() or any(s.stat().st_mtime > _LIB_PATH.stat().st_mtime for s in srcs):
        env = dict(os.environ)
        env.pop("CC", None)
        subprocess.run(["make", "-C", str(_HERE)], check=True, env=env, capture_output=True)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            build()
        L = C.CDLL(str(_LIB_PATH))
        L.fdo_norm2.restype = C.c_double
        L.fdo_norm2.argtypes = [C.c_void_p, C.c_int64]
        L.fdo_default_relstep.restype = C.c_double
        L.fdo_default_relstep.argtypes = [C.c_int]
        L.fdo_compute_epsilon.restype = C.c_double
        L.fdo_compute_epsilon.argtypes = [C.c_int, C.c_double, C.c_double, C.c_double, C.c_double]
        L.fdo_max_color.restype = C.c_int64
        L.fdo_max_color.argtypes = [_i64p, C.c_int64]
        L.fdo_findstructralnz_dense.restype = C.c_int64
        L.fdo_findstructralnz_dense.argtypes = [_f64p, C.c_int64, C.c_int64, _i64p, _i64p]
        for name in ("fdo_finite_difference_jacobian",):
            fn = getattr(L, name)
            fn.restype = C.c_int
            fn.argtypes = [C.POINTER(_Problem), _f64p, C.c_void_p, C.c_void_p, _f64p, C.POINTER(_Cache),
                           C.POINTER(_Opts)]
        L.fdo_finite_difference_jacobian_cacheless.restype = C.c_int
        L.fdo_finite_difference_jacobian_cacheless.argtypes = [C.POINTER(_Problem), _f64p, C.c_void_p, C.c_void_p,
                                                               _f64p, C.POINTER(_Opts)]
        L.synth_fill_x.restype = None
        L.synth_fill_x.argtypes = [_f64p, C.c_int64, C.c_uint64, C.c_int]
        L.synth_ellrows.restype = None
        L.synth_ellrows.argtypes = [C.c_void_p, _f64p, _f64p]
        L.synth_ellrows_c.restype = None
        L.synth_ellrows_c.argtypes = [C.c_void_p, _f64p, _f64p]     # complex128 arrays as interleaved doubles
        L.synth_blocked_sum.restype = C.c_double
        L.synth_blocked_sum.argtypes = [_f64p, C.c_int64]
        _lib = L
    return _lib


def _p64(a):
    return a.ctypes.data_as(_f64p) if a is not None else None


def _pi64(a):
    return a.ctypes.data_as(_i64p) if a is not None else None


def _as_i64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int64)


def norm2(v) -> float:
    """LinearAlgebra.norm of a Float64 vector as the reference evaluates it (generic_norm2 below 32 elements, OpenBLAS
    dnrm2 from 32 on) — fd_oracle.c:fdo_norm2."""
    a = np.ascontiguousarray(v, dtype=np.float64)
    return lib().fdo_norm2(a.ctypes.data, a.size)


def color_eps(x, colorvec, k: int, fdtype: int, relstep=None, absstep=None, dir: float = 1.0) -> float:
    """Step size of colour k (1-based) exactly as jacobians.jl:559-561 / :600-602 form it from a pristine x:
    x2 = x .* (colorvec .== k); eps = compute_epsilon(fd, sqrt(norm(x2)), relstep, absstep, dir)."""
    x = np.asarray(x, dtype=np.float64)
    mask = np.asarray(colorvec) == k
    x2 = np.where(mask, x, np.copysign(0.0, x))
    rs = default_relstep(fdtype) if relstep is None else relstep
    ab = rs if absstep is None else absstep
    return compute_epsilon(fdtype, float(np.sqrt(norm2(x2))), rs, ab, dir)


def default_relstep(fdtype: int) -> float:
    return lib().fdo_default_relstep(fdtype)


def compute_epsilon(fdtype: int, x: float, relstep: float, absstep: float, dir: float = 1.0) -> float:
    return lib().fdo_compute_epsilon(fdtype, x, relstep, absstep, dir)


def findstructralnz_dense(A: np.ndarray):
    """jacobians.jl:473-488 on a dense prototype (any dtype; nonzero test)."""
    A = np.asarray(A)
    if A.ndim == 1:
        A = A.reshape(1, -1)
    m, n = A.shape
    Af = np.asfortranarray(A.astype(np.float64))
    nnz = lib().fdo_findstructralnz_dense(_p64(Af.reshape(-1, order="F")), m, n, None, None)
    rows = np.zeros(nnz, np.int64)
    cols = np.zeros(nnz, np.int64)
    flat = np.ascontiguousarray(Af.reshape(-1, order="F"))
    lib().fdo_findstructralnz_dense(_p64(flat), m, n, _pi64(rows), _pi64(cols))
    return rows, cols


class Problem:
    """Describes (sparsity, J storage) the way the reference's dispatch sees them."""

    def __init__(self, sp_kind, j_kind, m, n, *, colptr=None, rowval=None, rows=None, cols=None, slots=None,
                 l=0, u=0, ldJ=0, j_len=0):
        self.sp_kind, self.j_kind, self.m, self.n = sp_kind, j_kind, int(m), int(n)
        self.colptr, self.rowval = _as_i64(colptr), _as_i64(rowval)
        self.rows, self.cols, self.slots = _as_i64(rows), _as_i64(cols), _as_i64(slots)
        self.l, self.u, self.ldJ, self.j_len = int(l), int(u), int(ldJ), int(j_len)
        nnz = len(self.rows) if self.rows is not None else 0
        self._c = _Problem(sp_kind, j_kind, self.m, self.n, _pi64(self.colptr), _pi64(self.rowval),
                           _pi64(self.rows), _pi64(self.cols), nnz, _pi64(self.slots), self.l, self.u,
                           self.ldJ, self.j_len)

    # -- constructors mirroring the reference's J / sparsity combinations --
    @staticmethod
    def dense(m, n):
        return Problem(SP_NONE, J_DENSE, m, n, ldJ=m, j_len=m * n)

    @staticmethod
    def csc_same(m, n, colptr, rowval):
        return Problem(SP_CSC_SAME, J_NZVAL, m, n, colptr=colptr, rowval=rowval, j_len=len(rowval))

    @staticmethod
    def csc_to_dense(m, n, colptr, rowval):
        return Problem(SP_CSC, J_DENSE, m, n, colptr=colptr, rowval=rowval, ldJ=m, j_len=m * n)

    @staticmethod
    def coo_to_dense(m, n, rows, cols):
        return Problem(SP_COO, J_DENSE, m, n, rows=rows, cols=cols, ldJ=m, j_len=m * n)

    @staticmethod
    def coo_to_slots(m, n, rows, cols, slots, j_len):
        return Problem(SP_COO, J_SLOTS, m, n, rows=rows, cols=cols, slots=slots, j_len=j_len)

    @staticmethod
    def banded(m, n, l, u):
        return Problem(SP_BANDED, J_BAND, m, n, l=l, u=u, j_len=(l + u + 1) * n)

    @staticmethod
    def banded_to_dense(m, n, l, u):
        return Problem(SP_BANDED, J_DENSE, m, n, l=l, u=u, ldJ=m, j_len=m * n)


def as_fn(f):
    """Wrap a Python callable f(fx: ndarray, x: ndarray) as an fdo_fn; returns (cfunc, keepalive)."""
    state = {}

    def tramp(_ctx, pfx, px):
        m, n = state["m"], state["n"]
        fx = np.ctypeslib.as_array(pfx, shape=(m,))
        x = np.ctypeslib.as_array(px, shape=(n,))
        f(fx, x)

    return FDO_FN(tramp), state


def jacobian(P: Problem, J: np.ndarray, f, x: np.ndarray, *, fdtype=FORWARD, relstep=None, absstep=None, dir=1.0,
             colorvec=None, f_in=None, eps_override=None, no_drift=False, nthreads=1, cache=None, cacheless=False,
             ctx=None):
    """Run the oracle's cached (default) or cache-less finite_difference_jacobian!.

    J: flat float64 storage (nzval / column-major dense / band data), modified in place.
    f: Python callable f(fx, x) or a (cfunc_pointer, ctx_struct) native pair via `ctx`.
    Returns dict(fcalls=..., eps=ndarray[maxcolor]).
    """
    L = lib()
    assert J.dtype == np.float64 and J.flags.c_contiguous or J.flags.f_contiguous
    assert x.dtype == np.float64 and x.flags.c_contiguous
    cv = _as_i64(colorvec)
    maxcolor = int(cv.max()) if cv is not None and len(cv) else (P.n if cv is None else 0)
    eps_out = np.zeros(max(maxcolor, 1), np.float64)
    eo = None if eps_override is None else np.ascontiguousarray(eps_override, dtype=np.float64)
    fin = None if f_in is None else np.ascontiguousarray(f_in, dtype=np.float64)
    relstep = float("nan") if relstep is None else float(relstep)     # NaN = keyword not given
    absstep = float("nan") if absstep is None else float(absstep)
    opts = _Opts(fdtype, relstep, absstep, float(dir), _pi64(cv), _p64(fin), _p64(eo), _p64(eps_out),
                 int(bool(no_drift)), int(nthreads), 0)
    if ctx is None:
        cf, st = as_fn(f)
        st["m"], st["n"] = P.m, P.n
        fptr, cptr = C.cast(cf, C.c_void_p), None
    else:
        fptr, cptr = C.cast(f, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p)
    Jp = J.ctypes.data_as(_f64p)
    if cacheless:
        rc = L.fdo_finite_difference_jacobian_cacheless(C.byref(P._c), Jp, fptr, cptr, _p64(x), C.byref(opts))
    else:
        if cache is None:
            cache = dict(x1=np.zeros(max(P.n, 1)), x2=np.zeros(max(P.n, 1)), fx=np.zeros(max(P.m, 1)),
                         fx1=np.zeros(max(P.m, 1)))
        cc = _Cache(_p64(cache["x1"]), _p64(cache["x2"]), _p64(cache["fx"]), _p64(cache["fx1"]))
        rc = L.fdo_finite_difference_jacobian(C.byref(P._c), Jp, fptr, cptr, _p64(x), C.byref(cc), C.byref(opts))
    if rc != 0:
        raise RuntimeError(f"oracle returned {rc}")
    return {"fcalls": int(opts.fcalls), "eps": eps_out[:maxcolor].copy(), "cache": cache}


FDO_FN_C = C.CFUNCTYPE(None, C.c_void_p, _f64p, _f64p)   # complex128 arrays as interleaved doubles


def jacobian_complex(P: Problem, J: np.ndarray, f, x: np.ndarray, *, colorvec=None, nthreads=1, ctx=None):
    """Complex-step Jacobian (jacobians.jl:623-648).  f: Python callable f(fx, x) on complex128 numpy views, or a
    native fdo_fn_c with `ctx`.  Returns dict(fcalls=...)."""
    L = lib()
    if not hasattr(L.fdo_finite_difference_jacobian_complex, "_bound"):
        L.fdo_finite_difference_jacobian_complex.restype = C.c_int
        L.fdo_finite_difference_jacobian_complex.argtypes = [C.POINTER(_Problem), _f64p, C.c_void_p, C.c_void_p, _f64p,
                                                             _i64p, C.c_int, C.POINTER(C.c_int64)]
        L.fdo_finite_difference_jacobian_complex._bound = True
    cv = _as_i64(colorvec)
    if ctx is None:
        m, n = P.m, P.n

        def tramp(_ctx, pfx, px):
            fx = np.ctypeslib.as_array(pfx, shape=(2 * m,)).view(np.complex128)
            xx = np.ctypeslib.as_array(px, shape=(2 * n,)).view(np.complex128)
            f(fx, xx)

        cf = FDO_FN_C(tramp)
        fptr, cptr = C.cast(cf, C.c_void_p), None
    else:
        fptr, cptr = C.cast(f, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p)
    calls = C.c_int64(0)
    rc = L.fdo_finite_difference_jacobian_complex(C.byref(P._c), J.ctypes.data_as(_f64p), fptr, cptr, _p64(x), _pi64(cv),
                                                  int(nthreads), C.byref(calls))
    if rc != 0:
        raise RuntimeError(f"oracle returned {rc}")
    return {"fcalls": int(calls.value)}


def jvp(f, x: np.ndarray, v: np.ndarray, m: int, *, fdtype=FORWARD, relstep=None, absstep=None, dir=1.0, f_in=None,
        eps_override=None, ctx=None, alias_x1=False):
    """finite_difference_jvp!(jvp, f, x, v, cache, f_in) (src/jvp.jl:238-274).  Returns dict(jvp, eps, fcalls, x1, fx1).

    alias_x1=True passes x's own buffer (a copy of the x given here) as cache.x1, as JVPCache(x, fx1) does
    (jvp.jl:73-80): central mode then evaluates f at (x - eps*v) + eps*v, and the returned x1 is x's end state."""
    L = lib()
    fn = L.fdo_finite_difference_jvp
    if not hasattr(fn, "_bound"):
        fn.restype = C.c_int
        fn.argtypes = [_f64p, C.c_void_p, C.c_void_p, _f64p, _f64p, C.c_int64, C.c_int64, _f64p, _f64p, _f64p, C.c_int,
                       C.c_double, C.c_double, C.c_double, _f64p, _f64p, C.POINTER(C.c_int64)]
        fn._bound = True
    n = len(x)
    out = np.zeros(max(m, 1))
    x1, fx1 = np.zeros(max(n, 1)), np.zeros(max(m, 1))
    if ctx is None:
        cf, st = as_fn(f)
        st["m"], st["n"] = m, n
        fptr, cptr = C.cast(cf, C.c_void_p), None
    else:
        fptr, cptr = C.cast(f, C.c_void_p), C.cast(C.pointer(ctx), C.c_void_p)
    fin = None if f_in is None else np.ascontiguousarray(f_in, dtype=np.float64)
    eo = None if eps_override is None else np.array([eps_override], dtype=np.float64)
    eps_out = np.zeros(1)
    calls = C.c_int64(0)
    relstep = float("nan") if relstep is None else float(relstep)
    absstep = float("nan") if absstep is None else float(absstep)
    xa = np.ascontiguousarray(x, dtype=np.float64)
    if alias_x1:
        xa = x1 = np.array(xa if n else np.zeros(1), dtype=np.float64, copy=True)    # fd_oracle.c has no restrict
    rc = fn(_p64(out), fptr, cptr, _p64(xa), _p64(np.ascontiguousarray(v)), m, n, _p64(x1), _p64(fx1),
            _p64(fin), fdtype, relstep, absstep, float(dir), _p64(eo), _p64(eps_out), C.byref(calls))
    if rc != 0:
        raise RuntimeError(f"oracle returned {rc}")
    return {"jvp": out[:m], "eps": float(eps_out[0]), "fcalls": int(calls.value), "x1": x1, "fx1": fx1}


def fill_x(n: int, seed: int, nthreads: int = 1) -> np.ndarray:
    x = np.empty(n, np.float64)
    lib().synth_fill_x(_p64(x), n, seed, nthreads)
    return x


def native_fn(name: str):
    """Address of a native synthetic f! (synth_tridiag / synth_lap5 / synth_ellrows / synth_rank1)."""
    return getattr(lib(), name)
