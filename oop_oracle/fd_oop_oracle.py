"""ctypes binding of the C restatement of the out-of-place forms (oop_oracle/fd_oop_oracle.c; test infrastructure).

jacobian_oop / jvp_oop take the same arguments and return the same values as tests/_literal_oop.py, so that the two
restatements can be compared with each other and the device with either.  f is a Python callable on numpy arrays (called
through a ctypes callback, so it can record the points) or a native callback given as (address, ctx) — e.g. a synthetic
f of the oracle library in oracle/ with its context struct."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "libfd_oop_oracle.so"
_f64p = C.POINTER(C.c_double)
_i64p = C.POINTER(C.c_int64)
FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_void_p)
FD = {"forward": 0, "central": 1, "complex": 2}
RAW, DENSE, SPARSE = 0, 1, 2


class Args(C.Structure):
    _fields_ = [("m", C.c_int64), ("n", C.c_int64), ("fdtype", C.c_int32), ("kind", C.c_int32), ("ncols", C.c_int64),
                ("colorvec", _i64p), ("colptr", _i64p), ("rowval", _i64p), ("f_in", _f64p),
                ("relstep", C.c_double), ("absstep", C.c_double), ("dir", C.c_double), ("eps_override", _f64p),
                ("J", _f64p), ("out_colptr", _i64p), ("out_rowval", _i64p), ("out_nzval", _f64p),
                ("nnz", C.c_int64), ("fcalls", C.c_int64), ("eps_out", _f64p)]


class OracleThrows(Exception):
    """The reference throws here (_make_Ji on an invalid colouring, sparse() with a colour past the prototype)."""


def build(force: bool = False) -> Path:
    """Compile with the committed Makefile (gcc, no GPU needed)."""
    srcs = [_HERE / "fd_oop_oracle.c", _HERE / "Makefile"]
    if force or not _LIB_PATH.exists() or any(s.stat().st_mtime > _LIB_PATH.stat().st_mtime for s in srcs):
        env = dict(os.environ)
        env.pop("CC", None)
        subprocess.run(["make", "-C", str(_HERE)], check=True, env=env, capture_output=True)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(str(_LIB_PATH))
        L.fdoo_jacobian_oop.restype = C.c_int
        L.fdoo_jacobian_oop.argtypes = [C.POINTER(Args), _f64p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.fdoo_jvp_oop.restype = C.c_int
        L.fdoo_jvp_oop.argtypes = [C.c_int64, C.c_int64, C.c_int, _f64p, _f64p, _f64p, C.c_double, C.c_double, C.c_double,
                                   _f64p, C.c_void_p, C.c_void_p, _f64p, _f64p, _i64p]
        _lib = L
    return _lib


def _p(a, t=_f64p):
    return None if a is None else a.ctypes.data_as(t)


def _callback(f, m, n, complex_):
    """(function pointer, ctx, keepalive) for a Python f on numpy arrays or a native (address, ctx)"""
    if isinstance(f, tuple):
        addr, ctx = f
        return C.c_void_p(addr), (C.cast(C.pointer(ctx), C.c_void_p) if ctx is not None else None), None

    def tramp(_ctx, p_fx, p_x):
        if complex_:
            x = np.ctypeslib.as_array(C.cast(p_x, _f64p), (2 * n,)).view(np.complex128) if n else np.zeros(0, complex)
            out = np.ctypeslib.as_array(C.cast(p_fx, _f64p), (2 * m,)).view(np.complex128) if m else None
        else:
            x = np.ctypeslib.as_array(C.cast(p_x, _f64p), (n,)) if n else np.zeros(0)
            out = np.ctypeslib.as_array(C.cast(p_fx, _f64p), (m,)) if m else None
        y = np.asarray(f(np.array(x, copy=True)))
        if m:
            out[:] = y.reshape(-1)
    cb = FN(tramp)
    return C.cast(cb, C.c_void_p), None, cb


def jacobian_oop(f, x, fdtype="forward", f_in=None, *, relstep=None, absstep=None, colorvec=None, sparsity=None,
                 jac_prototype=None, dir=1.0, eps_override=None, cacheless=False, m=None):
    """finite_difference_jacobian(f, x, cache, f_in; …) (jacobians.jl:277-429); cacheless=True: :240-259."""
    x = np.ascontiguousarray(x, np.float64)
    n = x.size
    if cacheless:
        fx = np.asarray(f(x.copy())) if f_in is None else np.asarray(f_in)                # :250-254
        return jacobian_oop(f, x, fdtype, np.real(fx) if np.iscomplexobj(fx) else fx, relstep=relstep, absstep=absstep,
                            colorvec=colorvec, sparsity=sparsity, jac_prototype=jac_prototype, dir=dir,
                            eps_override=eps_override, m=m)
    if m is None:
        m = (sparsity[0] if sparsity is not None else jac_prototype[1] if jac_prototype is not None
             else np.asarray(f_in).size if f_in is not None else n)
    cv = np.ascontiguousarray(np.arange(1, n + 1) if colorvec is None else colorvec, np.int64)
    a = Args()
    a.m, a.n, a.fdtype, a.dir = m, n, FD[fdtype], float(dir)
    a.relstep = float("nan") if relstep is None else float(relstep)
    a.absstep = float("nan") if absstep is None else float(absstep)
    keep = [cv, x]
    a.colorvec = _p(cv, _i64p)
    if sparsity is not None:
        cp = np.ascontiguousarray(sparsity[2], np.int64)
        rv = np.ascontiguousarray(sparsity[3], np.int64)
        keep += [cp, rv]
        a.colptr, a.rowval = _p(cp, _i64p), _p(rv, _i64p)
    if f_in is not None and fdtype == "forward":
        fin = np.ascontiguousarray(f_in, np.float64).reshape(-1)
        keep.append(fin)
        a.f_in = _p(fin)
    if eps_override is not None:
        eo = np.ascontiguousarray(eps_override, np.float64)
        keep.append(eo)
        a.eps_override = _p(eo)
    C_ = int(cv.max()) if n else 0
    if jac_prototype is None:
        a.kind, a.ncols = (RAW, C_) if sparsity is None else (DENSE, sparsity[1])
    else:
        a.kind = SPARSE if jac_prototype[0] == "sparse" else DENSE
        a.ncols = jac_prototype[2]
    ncols = a.ncols
    J = np.zeros(max(m * ncols, 1) if a.kind != SPARSE else 1)
    a.J = _p(J)
    cap = max(m * ncols if sparsity is None else len(sparsity[3]), 1)
    ocp, orv, onz = np.zeros(ncols + 1, np.int64), np.zeros(cap, np.int64), np.zeros(cap)
    a.out_colptr, a.out_rowval, a.out_nzval = _p(ocp, _i64p), _p(orv, _i64p), _p(onz)
    eps = np.zeros(max(n, C_, 1))
    a.eps_out = _p(eps)
    fn, ctx, cb = _callback(f, m, n, fdtype == "complex")
    real_fn, cplx_fn = (None, fn) if fdtype == "complex" else (fn, None)
    rc = lib().fdoo_jacobian_oop(C.byref(a), _p(x), real_fn, cplx_fn, ctx)
    if rc == 1:
        raise OracleThrows("the reference throws (_make_Ji / sparse())")
    if rc != 0:
        raise ValueError("rejected by the restatement (empty colorvec, colour past length(x), ...)")
    if a.kind == SPARSE:
        return ("sparse", m, ncols, ocp, orv[: a.nnz].copy(), onz[: a.nnz].copy())
    return ("dense", J[: m * ncols].reshape((ncols, m)).T.copy())


def jvp_oop(f, x, v, fdtype="forward", f_in=None, *, relstep=None, absstep=None, dir=1.0, eps_override=None,
            cacheless=False, m=None):
    """finite_difference_jvp(f, x, v, cache, f_in; …) (jvp.jl:159-189); cacheless=True: :133-146.  Returns (jvp, eps)."""
    x = np.ascontiguousarray(x, np.float64)
    v = np.ascontiguousarray(v, np.float64)
    if cacheless:
        fx = np.asarray(f(x.copy())) if f_in is None else np.asarray(f_in)                # :139-143
        return jvp_oop(f, x, v, fdtype, fx, relstep=relstep, absstep=absstep, dir=dir, eps_override=eps_override)
    n = x.size
    if m is None:
        m = np.asarray(f_in).size if f_in is not None else n
    fin = np.ascontiguousarray(f_in, np.float64).reshape(-1) if f_in is not None else None
    eo = None if eps_override is None else np.array([float(eps_override)])
    out, e, calls = np.zeros(max(m, 1)), np.zeros(1), C.c_int64()
    fn, ctx, cb = _callback(f, m, n, False)
    rc = lib().fdoo_jvp_oop(m, n, FD[fdtype], _p(x), _p(v), _p(fin), float("nan") if relstep is None else float(relstep),
                            float("nan") if absstep is None else float(absstep), float(dir), _p(eo), fn, ctx, _p(out),
                            _p(e), C.byref(calls))
    if rc != 0:
        raise ValueError("rejected by the restatement")
    return out[:m].copy(), float(e[0])
