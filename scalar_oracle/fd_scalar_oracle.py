"""ctypes binding of the CPU restatement of the reference's Hessian and gradient (scalar_oracle/libfd_scalar_oracle.so).

TEST INFRASTRUCTURE ONLY — see fd_scalar_oracle.h.  Only tests/, __graft_entry__.smoke() and scripts/ import it; the
product package (finitediff.jl_b200/) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libfd_scalar_oracle.so"

FORWARD, CENTRAL, COMPLEX, HCENTRAL = 0, 1, 2, 3

_f64p = C.POINTER(C.c_double)
FDSO_FN = C.CFUNCTYPE(C.c_double, C.c_void_p, _f64p)
FDSO_FN_C = C.CFUNCTYPE(None, C.c_void_p, _f64p, _f64p)
FDSO_LOG = C.CFUNCTYPE(None, C.c_void_p, _f64p, C.c_int64)
FDSO_EFN = C.CFUNCTYPE(C.c_double, C.c_void_p, C.c_int64, C.c_double)
FDSO_EFN_C = C.CFUNCTYPE(None, C.c_void_p, C.c_int64, _f64p, _f64p)
FDSO_VFN = C.CFUNCTYPE(None, C.c_void_p, _f64p, C.c_double)
FDSO_VFN_C = C.CFUNCTYPE(None, C.c_void_p, _f64p, _f64p)


class SynthScalarCtx(C.Structure):
    _fields_ = [("n", C.c_int64), ("a", _f64p), ("w", _f64p)]


def build(force: bool = False) -> Path:
    """Compile with the committed Makefile (gcc, no GPU needed)."""
    srcs = [_HERE / "fd_scalar_oracle.c", _HERE / "synth_scalar.c", _HERE / "fd_scalar_oracle.h", _HERE / "Makefile"]
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
        L.fdso_hessian.restype = C.c_int
        L.fdso_hessian.argtypes = [_f64p, C.c_int64, C.c_void_p, C.c_void_p, _f64p, C.c_int64, C.c_double, C.c_double,
                                   _f64p, _f64p, _f64p, _f64p, _f64p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
        L.fdso_gradient.restype = C.c_int
        L.fdso_gradient.argtypes = [_f64p, C.c_void_p, C.c_void_p, _f64p, C.c_int64, C.c_int, _f64p, C.c_double,
                                    C.c_double, C.c_double, _f64p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
        L.fdso_gradient_complex.restype = C.c_int
        L.fdso_gradient_complex.argtypes = [_f64p, C.c_void_p, C.c_void_p, _f64p, C.c_int64, _f64p, C.c_void_p,
                                            C.c_void_p, C.POINTER(C.c_int64)]
        L.fdso_default_relstep.restype = C.c_double
        L.fdso_default_relstep.argtypes = [C.c_int]
        L.synth_quartic.restype = C.c_double
        L.synth_quartic.argtypes = [C.c_void_p, _f64p]
        L.synth_sumsq.restype = C.c_double
        L.synth_sumsq.argtypes = [C.c_void_p, _f64p]
        L.synth_guarded.restype = C.c_double
        L.synth_guarded.argtypes = [C.c_void_p, _f64p]
        L.synth_quartic_c.restype = None
        L.synth_quartic_c.argtypes = [C.c_void_p, _f64p, _f64p]
        L.fdso_derivative.restype = C.c_int
        L.fdso_derivative.argtypes = [_f64p, C.c_void_p, C.c_void_p, _f64p, C.c_int64, C.c_int, _f64p, C.c_double,
                                      C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
        L.fdso_derivative_complex.restype = C.c_int
        L.fdso_derivative_complex.argtypes = [_f64p, C.c_void_p, C.c_void_p, _f64p, C.c_int64, C.c_void_p, C.c_void_p,
                                              C.POINTER(C.c_int64)]
        L.fdso_scalar_gradient.restype = C.c_int
        L.fdso_scalar_gradient.argtypes = [_f64p, C.c_void_p, C.c_void_p, C.c_double, C.c_int64, C.c_int, _f64p,
                                           C.c_double, C.c_double, C.c_double, _f64p, _f64p, C.c_void_p, C.c_void_p,
                                           C.POINTER(C.c_int64)]
        L.fdso_scalar_gradient_complex.restype = C.c_int
        L.fdso_scalar_gradient_complex.argtypes = [_f64p, C.c_void_p, C.c_void_p, C.c_double, C.c_int64, _f64p,
                                                   C.c_void_p, C.c_void_p, C.POINTER(C.c_int64)]
        for nm in ("synth_poly", "synth_poly_guarded"):
            getattr(L, nm).restype = C.c_double
            getattr(L, nm).argtypes = [C.c_void_p, C.c_int64, C.c_double]
        for nm in ("synth_poly_c", "synth_poly_guarded_c"):
            getattr(L, nm).restype = None
            getattr(L, nm).argtypes = [C.c_void_p, C.c_int64, _f64p, _f64p]
        for nm in ("synth_tpoly", "synth_tpoly_guarded"):
            getattr(L, nm).restype = None
            getattr(L, nm).argtypes = [C.c_void_p, _f64p, C.c_double]
        for nm in ("synth_tpoly_c", "synth_tpoly_guarded_c"):
            getattr(L, nm).restype = None
            getattr(L, nm).argtypes = [C.c_void_p, _f64p, _f64p]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(_f64p)


def _step(v):
    return float("nan") if v is None else float(v)        # NaN = keyword not given


def default_relstep(fdtype: int) -> float:
    return lib().fdso_default_relstep(fdtype)


class SynthScalar:
    """CPU twin of fdbs_quartic / fdbs_sumsq / fdbs_guarded / fdbs_quartic_c: keeps a and w alive with the ctx struct.
    Calling it evaluates `name` (default: synth_quartic when a is given, else synth_sumsq)."""

    def __init__(self, n, a=None, w=None, name=None):
        self.n = int(n)
        self.a = None if a is None else np.ascontiguousarray(a, dtype=np.float64)
        self.w = None if w is None else np.ascontiguousarray(w, dtype=np.float64)
        self.ctx = SynthScalarCtx(self.n, _p(self.a), _p(self.w))
        self.name = name or ("synth_quartic" if self.a is not None else "synth_sumsq")

    def native(self, name: str):
        """(function address, ctx) for the oracle entry points: name = synth_quartic / synth_sumsq / synth_guarded /
        synth_quartic_c, or synth_poly[_guarded][_c] / synth_tpoly[_guarded][_c] for derivative / scalar_gradient."""
        return C.cast(getattr(lib(), name), C.c_void_p), C.cast(C.pointer(self.ctx), C.c_void_p)

    def __call__(self, x) -> float:
        x = np.ascontiguousarray(x, dtype=np.float64)
        return getattr(lib(), self.name)(C.byref(self.ctx), _p(x))


def _fn(f, n, complex_=False):
    """(address, ctx, keepalive) of a Python f(x) -> float (or complex), or a native (address, ctx) pair."""
    if isinstance(f, tuple):
        return f[0], f[1], None
    if complex_:
        def tramp_c(_ctx, px, pout):
            z = complex(f(np.ctypeslib.as_array(px, shape=(2 * n,)).copy().view(np.complex128)))
            pout[0], pout[1] = z.real, z.imag
        cf = FDSO_FN_C(tramp_c)
    else:
        cf = FDSO_FN(lambda _ctx, px: float(f(np.ctypeslib.as_array(px, shape=(n,)).copy())))
    return C.cast(cf, C.c_void_p), None, cf


def _log(points):
    if points is None:
        return None, None
    cb = FDSO_LOG(lambda _c, px, cnt: points.append(np.ctypeslib.as_array(px, shape=(cnt,)).copy()))
    return C.cast(cb, C.c_void_p), cb


def hessian(f, x, *, relstep=None, absstep=None, ldH=None, H=None, cache=None, log=False):
    """finite_difference_hessian!(H, f, x, cache) (hessians.jl:202-292).  f: Python f(x) -> float or a native pair from
    SynthScalar.native.  Returns dict(H (ldH x n, Fortran order), fx, fcalls, points (list of arrays when log))."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    n = x.size
    ld = max(n, 1) if ldH is None else int(ldH)
    if H is None:
        H = np.zeros((ld, n), dtype=np.float64, order="F")
    cache = [np.zeros(max(n, 1)) for _ in range(4)] if cache is None else [np.ascontiguousarray(c, dtype=np.float64) for c in cache]
    fptr, ctx, keep = _fn(f, n)
    points = [] if log else None
    lptr, lkeep = _log(points)
    fx = np.zeros(1)
    calls = C.c_int64(0)
    rc = lib().fdso_hessian(H.ctypes.data_as(_f64p), ld, fptr, ctx, _p(x), n, _step(relstep), _step(absstep),
                            *[_p(c) for c in cache], _p(fx), lptr, None, C.byref(calls))
    if rc != 0:
        raise ValueError(f"oracle returned {rc}")
    return {"H": H, "fx": float(fx[0]), "fcalls": calls.value, "points": points}


def gradient(f, x, fdtype=FORWARD, *, fx=None, relstep=None, absstep=None, dir=1.0, log=False):
    """finite_difference_gradient!(df, f, x, cache) (gradients.jl:390-473) for real x and df: forward (fx = the cache's
    fx or None), central, complex.  Returns dict(df, fcalls, points)."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    n = x.size
    df = np.zeros(max(n, 1))
    points = [] if log else None
    lptr, lkeep = _log(points)
    calls = C.c_int64(0)
    if fdtype == COMPLEX:
        fptr, ctx, keep = _fn(f, n, complex_=True)
        c1 = np.zeros(max(2 * n, 2))
        rc = lib().fdso_gradient_complex(_p(df), fptr, ctx, _p(x), n, _p(c1), lptr, None, C.byref(calls))
    else:
        fptr, ctx, keep = _fn(f, n)
        c3 = np.zeros(max(n, 1))
        fxa = None if fx is None else np.array([float(fx)])
        rc = lib().fdso_gradient(_p(df), fptr, ctx, _p(x), n, int(fdtype), _p(fxa), _step(relstep), _step(absstep),
                                 float(dir), _p(c3), lptr, None, C.byref(calls))
    if rc != 0:
        raise ValueError(f"oracle returned {rc}")
    return {"df": df[:n], "fcalls": calls.value, "points": points}


def _efn(f, complex_=False):
    """(address, ctx, keepalive) of a Python scalar f(v) (index-free, as the reference's f) or a native pair."""
    if isinstance(f, tuple):
        return f[0], f[1], None
    if complex_:
        def tramp_c(_ctx, _i, px, pout):
            z = complex(f(complex(px[0], px[1])))
            pout[0], pout[1] = z.real, z.imag
        cf = FDSO_EFN_C(tramp_c)
    else:
        cf = FDSO_EFN(lambda _ctx, _i, v: float(f(v)))
    return C.cast(cf, C.c_void_p), None, cf


def _vfn(f, m, complex_=False):
    """(address, ctx, keepalive) of a Python in-place f(fx, t) on numpy arrays (fx float64 or complex128 of length m, t a
    float or complex) or a native pair."""
    if isinstance(f, tuple):
        return f[0], f[1], None
    if complex_:
        def tramp_c(_ctx, pfx, pt):
            fx = np.zeros(m, dtype=np.complex128)
            f(fx, complex(pt[0], pt[1]))
            np.ctypeslib.as_array(pfx, shape=(2 * m,))[:] = fx.view(np.float64)
        cf = FDSO_VFN_C(tramp_c)
    else:
        def tramp(_ctx, pfx, t):
            fx = np.zeros(m)
            f(fx, t)
            np.ctypeslib.as_array(pfx, shape=(m,))[:] = fx
        cf = FDSO_VFN(tramp)
    return C.cast(cf, C.c_void_p), None, cf


def derivative(f, x, fdtype=CENTRAL, *, fx=None, relstep=None, absstep=None, dir=1.0, log=False):
    """finite_difference_derivative!(df, f, x::StridedArray, cache) (derivatives.jl:197-233).  f: Python f(v) -> float
    (complex for COMPLEX) or a native pair from SynthScalar.native.  Returns dict(df, fcalls, points (each argument: a
    float, or a (re, im) array for complex))."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    n = x.size
    df = np.zeros(max(n, 1))
    points = [] if log else None
    lptr, lkeep = _log(points)
    calls = C.c_int64(0)
    fptr, ctx, keep = _efn(f, fdtype == COMPLEX)
    if fdtype == COMPLEX:
        rc = lib().fdso_derivative_complex(_p(df), fptr, ctx, _p(x), n, lptr, None, C.byref(calls))
    else:
        fxa = None if fx is None else np.ascontiguousarray(fx, dtype=np.float64)
        rc = lib().fdso_derivative(_p(df), fptr, ctx, _p(x), n, int(fdtype), _p(fxa), _step(relstep), _step(absstep),
                                   float(dir), lptr, None, C.byref(calls))
    if rc != 0:
        raise ValueError(f"oracle returned {rc}")
    if points is not None and fdtype != COMPLEX:
        points = [float(p[0]) for p in points]
    return {"df": df[:n], "fcalls": calls.value, "points": points}


def scalar_gradient(f, x, m, fdtype=CENTRAL, *, fx=None, relstep=None, absstep=None, dir=1.0, log=False):
    """finite_difference_gradient!(df, f, x::Number, cache) (gradients.jl:477-533).  f: Python in-place f(fx, t) or a
    native pair.  Returns dict(df, fcalls, points)."""
    df = np.zeros(max(m, 1))
    points = [] if log else None
    lptr, lkeep = _log(points)
    calls = C.c_int64(0)
    fptr, ctx, keep = _vfn(f, m, fdtype == COMPLEX)
    if fdtype == COMPLEX:
        c1 = np.zeros(max(2 * m, 2))
        rc = lib().fdso_scalar_gradient_complex(_p(df), fptr, ctx, float(x), m, _p(c1), lptr, None, C.byref(calls))
    else:
        c1, c2 = np.zeros(max(m, 1)), np.zeros(max(m, 1))
        fxa = None if fx is None else np.ascontiguousarray(fx, dtype=np.float64)
        rc = lib().fdso_scalar_gradient(_p(df), fptr, ctx, float(x), m, int(fdtype), _p(fxa), _step(relstep),
                                        _step(absstep), float(dir), _p(c1), _p(c2), lptr, None, C.byref(calls))
    if rc != 0:
        raise ValueError(f"oracle returned {rc}")
    if points is not None and fdtype != COMPLEX:
        points = [float(p[0]) for p in points]
    return {"df": df[:m], "fcalls": calls.value, "points": points}
