"""Line-by-line transcription of the reference's OUT-OF-PLACE forms, in numpy:

    finite_difference_jacobian(f, x, cache, f_in; relstep, absstep, colorvec, sparsity, jac_prototype, dir)
                                                          src/jacobians.jl:277-429 (cache-less form :240-259)
    _make_Ji (dense result, both methods)                 src/jacobians.jl:151-187
    _make_Ji (SparseMatrixCSC result, both methods)       ext/FiniteDiffSparseArraysExt.jl:7-17
    J + Ji on SparseMatrixCSC                             SparseArrays' zero-preserving map: a result is stored only when
                                                          it is not iszero (restated from the stdlib; parity unpinned at
                                                          source level)
    finite_difference_jvp(f, x, v, cache, f_in; …)        src/jvp.jl:159-189 (cache-less form :133-146)

It is the CPU side of the out-of-place tests: it evaluates f on the host and records every point f is called with.
`norm` (LinearAlgebra's, jacobians.jl:338,378) and `dot` (jvp.jl:172) only decide the step size; their summation order is
not pinned, so callers may pass the step sizes (eps_override) the device computed.

A result is ("dense", J) with J an m x ncols float64 array, or ("sparse", m, ncols, colptr, rowval, nzval) with 1-based
Int64 colptr / rowval in storage order.
"""
from __future__ import annotations

import numpy as np

EPS = np.finfo(np.float64).eps


def jl_max(a, b):
    """Julia's max on Float64: NaN if either is NaN, +0.0 above -0.0."""
    a, b = float(a), float(b)
    if a != a or b != b:
        return a - b
    return b if np.signbit(a - b) else a


def default_relstep(fdtype):
    return {"forward": float(np.sqrt(EPS)), "central": float(np.cbrt(EPS)), "complex": 1.0}[fdtype]


def eps_forward(x, relstep, absstep, dir):
    """compute_epsilon(Val(:forward), x, relstep, absstep, dir) = max(relstep*abs(x), absstep)*dir  (epsilons.jl:26-29)"""
    return float(np.float64(jl_max(np.float64(relstep) * abs(np.float64(x)), absstep)) * np.float64(dir))


def eps_central(x, relstep, absstep):
    """compute_epsilon(Val(:central), x, relstep, absstep) = max(relstep*abs(x), absstep)  (epsilons.jl:50-53)"""
    return jl_max(np.float64(relstep) * abs(np.float64(x)), absstep)


def bool_mul(e, mask):
    """e .* (colorvec .== k): Julia's Bool product is a strong zero, e*false = copysign(0, e)."""
    return np.where(mask, np.float64(e), np.copysign(0.0, np.float64(e)))


class Recorder:
    """Wraps an out-of-place f (numpy in, numpy out) and records a copy of every point it is called with."""

    def __init__(self, f):
        self.f, self.points = f, []

    def __call__(self, x):
        self.points.append(np.array(x, copy=True))
        return np.asarray(self.f(np.array(x, copy=True)))


class MakeJiError(Exception):
    """What _make_Ji throws on a colouring with two columns of one colour in a row (ArgumentError / BoundsError)."""


def _make_Ji_dense_sparsity(rows_index, cols_index, dx, colorvec, color_i, nrows, ncols):
    """_make_Ji(::AbstractArray, rows_index, cols_index, dx, colorvec, color_i, nrows, ncols)  jacobians.jl:151-162"""
    pick = [i for i in range(len(rows_index)) if colorvec[cols_index[i] - 1] == color_i]        # :153
    rows_c = [rows_index[i] for i in pick]                                                        # :154
    cols_c = [cols_index[i] for i in pick]                                                        # :155
    len_rows = len(pick)                                                                          # :156
    seen = set(rows_c)
    unused = [r for r in range(1, nrows + 1) if r not in seen]                                    # :157 setdiff
    if nrows - len_rows < 0:
        raise MakeJiError("zeros(Int, negative): ArgumentError")                                  # :159
    key = rows_c + unused
    perm = sorted(range(len(key)), key=lambda i: key[i])                                          # :158 sortperm (stable)
    padded = cols_c + [0] * (nrows - len_rows)
    if any(p >= len(padded) for p in perm):
        raise MakeJiError("BoundsError")                                                          # :159 [perm_rows]
    cols_c = [padded[p] for p in perm]
    Ji = np.zeros((nrows, ncols))                                                                 # `false` -> 0.0
    for i in range(nrows):                                                                        # :160: row i holds dx[i]
        if 1 <= cols_c[i] <= ncols:                                                               # in column cols_c[i] only
            Ji[i, cols_c[i] - 1] = dx[i]
    return Ji


def _make_Ji_dense(dx, color_i, nrows, ncols):
    """_make_Ji(::AbstractArray, xtype, dx, color_i, nrows, ncols)  jacobians.jl:184-187"""
    # mapreduce(i -> i == color_i ? dx : zero(dx), hcat, 1:ncols): zero(dx) is +0.0
    Ji = np.zeros((len(dx), ncols))
    if 1 <= color_i <= ncols:
        Ji[:, color_i - 1] = dx
    if Ji.shape != (nrows, ncols):
        if Ji.size != nrows * ncols:
            raise MakeJiError("DimensionMismatch in reshape")
        Ji = Ji.reshape((nrows, ncols), order="F")
    return Ji


def _make_Ji_sparse_sparsity(rows_index, cols_index, dx, colorvec, color_i, nrows, ncols):
    """ext/FiniteDiffSparseArraysExt.jl:7-13: sparse(rows_c, cols_c, dx[rows_c], nrows, ncols) — explicit values kept"""
    return {(rows_index[i], cols_index[i]): dx[rows_index[i] - 1]
            for i in range(len(rows_index)) if colorvec[cols_index[i] - 1] == color_i}


def _make_Ji_sparse(dx, color_i, nrows, ncols):
    """ext/FiniteDiffSparseArraysExt.jl:15-17: sparse(1:nrows, fill(color_i, nrows), dx, nrows, ncols)"""
    if color_i > ncols:
        raise MakeJiError("sparse(): column index out of bounds (ArgumentError)")
    return {(r, color_i): dx[r - 1] for r in range(1, nrows + 1)}


def _sparse_plus(A, B):
    """A + B of two SparseMatrixCSC: the union of the patterns, implicit entries +0.0, and only results that are not
    iszero stored (NaN is stored; +-0.0 are not).  Every entry A stores is nonzero (A is itself such a sum), and
    v + 0.0 is v for those, so only B's keys need the addition; A is updated in place."""
    for k, b in B.items():
        v = np.float64(A.get(k, 0.0)) + np.float64(b)
        if v != 0.0 or v != v:
            A[k] = v
        else:
            A.pop(k, None)
    return A


def _csc(m, ncols, entries):
    keys = sorted(entries, key=lambda rc: (rc[1], rc[0]))
    colptr = np.ones(ncols + 1, np.int64)
    for (r, c) in keys:
        colptr[c:] += 1
    rowval = np.array([r for (r, c) in keys], np.int64)
    nzval = np.array([entries[k] for k in keys], np.float64)
    return ("sparse", m, ncols, colptr, rowval, nzval)


def findstructralnz(colptr, rowval):
    """rows_index, cols_index of a CSC pattern in storage order (jacobians.jl:313)"""
    rows, cols = [], []
    for c in range(len(colptr) - 1):
        for p in range(colptr[c] - 1, colptr[c + 1] - 1):
            rows.append(int(rowval[p]))
            cols.append(c + 1)
    return rows, cols


def jacobian_oop(f, x, fdtype="forward", f_in=None, *, relstep=None, absstep=None, colorvec=None, sparsity=None,
                 jac_prototype=None, dir=1.0, eps_override=None, cacheless=False):
    """finite_difference_jacobian(f, x, cache, f_in; …)  jacobians.jl:277-429.

    f: a Recorder (or any numpy f); x: float64 array; sparsity: None or (m, n, colptr, rowval) 1-based;
    jac_prototype: None, ("dense", m, n) or ("sparse", m, n); colorvec: None (1:n) or 1-based ints;
    eps_override: step sizes per colour of a coloured call (index k-1).  cacheless=True: the form :240-259, which
    evaluates f(x) first and passes it on as f_in."""
    x = np.asarray(x, np.float64)
    n = x.size
    if cacheless:
        fx = f(x) if f_in is None else f_in                                                      # :250-254
        if fdtype == "complex":
            fx = np.real(fx)
        return jacobian_oop(f, x, fdtype, fx, relstep=relstep, absstep=absstep, colorvec=colorvec, sparsity=sparsity,
                            jac_prototype=jac_prototype, dir=dir, eps_override=eps_override)
    relstep = default_relstep(fdtype) if relstep is None else relstep                            # :282
    absstep = relstep if absstep is None else absstep                                            # :283
    colorvec = np.arange(1, n + 1) if colorvec is None else np.asarray(colorvec, np.int64)
    if colorvec.size == 0:
        raise MakeJiError("maximum of an empty collection")
    C = int(colorvec.max())
    if f_in is not None:                                                                         # :297-305
        vecfx = np.asarray(f_in, np.float64)
    elif fdtype == "forward":
        vecfx = np.asarray(f(x), np.float64)
    else:
        vecfx = None                                                                             # cache.fx: not read below
    # J = zero(jac_prototype) / zeros(size(sparsity)) / an m x 0 matrix   :307-310
    if jac_prototype is not None:
        pkind, nrows, ncols = jac_prototype
    elif sparsity is not None:
        pkind, nrows, ncols = "dense", sparsity[0], sparsity[1]
    else:
        pkind, nrows, ncols = None, None, None
    J = {} if pkind == "sparse" else (np.zeros((nrows, ncols)) if pkind == "dense" else None)
    if sparsity is not None:
        rows_index, cols_index = findstructralnz(sparsity[2], sparsity[3])                      # :312-316

    def step(e_k, xs):
        return eps_override[e_k] if eps_override is not None else xs

    def column(i):
        """calculate_Ji_forward / _central / _complex (i)   :319-327, :356-367, :397-404"""
        xs = x[i - 1]
        if fdtype == "forward":
            e = eps_forward(xs, relstep, absstep, dir)                                           # :321
            x1 = x.copy(); x1[i - 1] = xs + e                                                     # :322 setindex
            return (np.asarray(f(x1), np.float64) - vecfx) / e                                   # :324-325
        if fdtype == "central":
            e = eps_forward(xs, relstep, absstep, dir)                                           # :358 Val(:forward)
            x1 = x.copy(); x1[i - 1] = xs + e                                                     # :359
            x2 = x.copy(); x2[i - 1] = xs - e                                                     # :360
            fx1 = np.asarray(f(x1), np.float64)                                                  # :363
            fx = np.asarray(f(x2), np.float64)                                                   # :364
            return (fx1 - fx) / (2 * e)                                                          # :365
        e = EPS                                                                                  # :395
        xc = x.astype(np.complex128)                                                             # complex.(vecx)
        xc[i - 1] = complex(xs + 0.0, e)                                                         # x_save + im*epsilon :399
        return np.imag(np.asarray(f(xc))) / e                                                    # :401-402

    def colour(k):
        """the coloured branch per colour_i   :338-344, :378-387, :415-418"""
        mask = colorvec == k
        if fdtype == "complex":
            e = EPS
            # vecx + im*eps*(c==k)  :415 — every real part is x + 0.0, the imaginary part eps or +0.0
            xc = np.array([complex(a, b) for a, b in zip(x + 0.0, np.where(mask, e, 0.0))], np.complex128)
            return np.imag(np.asarray(f(xc))) / e                                                # :417-418
        tmp = np.linalg.norm(np.where(mask, x, 0.0))                                             # :338 / :378
        e = eps_override[k - 1] if eps_override is not None else eps_forward(np.sqrt(tmp), relstep, absstep, dir)
        if fdtype == "forward":
            x1 = x + bool_mul(e, mask)                                                           # :341
            return (np.asarray(f(x1), np.float64) - vecfx) / e                                   # :343-344
        x1 = x + bool_mul(e, mask)                                                               # :381
        x2 = x - bool_mul(e, mask)                                                               # :382
        fx1 = np.asarray(f(x1), np.float64)                                                      # :385
        fx = np.asarray(f(x2), np.float64)                                                       # :386
        return (fx1 - fx) / (2 * e)                                                              # :387

    if jac_prototype is None and sparsity is None:                                               # :329-331 mapreduce hcat
        if C < 1:
            raise MakeJiError("mapreduce over an empty collection")
        if C > n:
            raise MakeJiError("BoundsError in setindex")
        return ("dense", np.stack([column(i) for i in range(1, C + 1)], axis=1))
    for k in range(1, C + 1):                                                                    # :333
        if sparsity is None:
            if k > n:
                raise MakeJiError("BoundsError in setindex")
            dx = column(k)
            if pkind == "sparse":
                J = _sparse_plus(J, _make_Ji_sparse(dx, k, nrows, ncols))                        # :336
            else:
                J = J + _make_Ji_dense(dx, k, nrows, ncols)
        else:
            dx = colour(k)
            if pkind == "sparse":
                J = _sparse_plus(J, _make_Ji_sparse_sparsity(rows_index, cols_index, dx, colorvec, k, nrows, ncols))
            else:
                J = J + _make_Ji_dense_sparsity(rows_index, cols_index, dx, colorvec, k, nrows, ncols)   # :345-347
    if pkind == "sparse":
        return _csc(nrows, ncols, J)
    return ("dense", J)


def jvp_oop(f, x, v, fdtype="forward", f_in=None, *, relstep=None, absstep=None, dir=1.0, eps_override=None,
            cacheless=False):
    """finite_difference_jvp(f, x, v, cache, f_in; relstep, absstep, dir)  jvp.jl:159-189 (cache-less :133-146)"""
    x, v = np.asarray(x, np.float64), np.asarray(v, np.float64)
    if cacheless:
        fx = f(x) if f_in is None else f_in                                                      # :139-143
        return jvp_oop(f, x, v, fdtype, fx, relstep=relstep, absstep=absstep, dir=dir, eps_override=eps_override)
    relstep = default_relstep(fdtype) if relstep is None else relstep
    absstep = relstep if absstep is None else absstep
    if eps_override is not None:
        e = eps_override
    else:
        tmp = np.sqrt(abs(float(np.dot(x, v))))                                                  # :172
        e = eps_forward(tmp, relstep, absstep, dir) if fdtype == "forward" else eps_central(tmp, relstep, absstep)   # :173
    if fdtype == "forward":
        fx = np.asarray(f(x) if f_in is None else f_in, np.float64)                              # :175
        x1 = x + e * v                                                                           # :176
        fx1 = np.asarray(f(x1), np.float64)                                                      # :177
        return (fx1 - fx) / e, e                                                                 # :178
    x1 = x + e * v                                                                               # :180
    fx1 = np.asarray(f(x1), np.float64)                                                          # :181
    x1 = x - e * v                                                                               # :182
    fx = np.asarray(f(x1), np.float64)                                                           # :183
    return (fx1 - fx) / (2 * e), e                                                               # :184


def jacobian_oop_csc_fast(f, x, fdtype, eps, m, colptr, rowval, colorvec, *, f_in=None, sparse=True):
    """The coloured branch with a CSC sparsity, vectorised over the entries, for sizes the literal loop cannot take:
    the same points, calls and quotients as jacobian_oop (checked against it in test_oop_cpu.py), with the step sizes
    given.  Returns the CSC result (sparse=True) or (rows0, cols0, values) of the dense result's structural slots."""
    x = np.asarray(x, np.float64)
    colorvec = np.asarray(colorvec, np.int64)
    C = int(colorvec.max())
    colptr = np.asarray(colptr, np.int64)
    rowval = np.asarray(rowval, np.int64)
    n = colptr.size - 1
    cols0 = np.repeat(np.arange(n), np.diff(colptr))
    rows0 = rowval - 1
    ecol = colorvec[cols0]
    vals = np.zeros(rows0.size)
    vecfx = None
    if fdtype == "forward":
        vecfx = np.asarray(f(x) if f_in is None else f_in, np.float64)
    for k in range(1, C + 1):
        mask = colorvec == k
        e = eps[k - 1]
        if fdtype == "forward":
            dx = (np.asarray(f(x + bool_mul(e, mask)), np.float64) - vecfx) / e
        else:
            fx1 = np.asarray(f(x + bool_mul(e, mask)), np.float64)
            fx = np.asarray(f(x - bool_mul(e, mask)), np.float64)
            dx = (fx1 - fx) / (2 * e)
        sel = ecol == k
        vals[sel] = dx[rows0[sel]]
    if not sparse:
        return rows0, cols0, vals + 0.0
    keep = (vals != 0.0) | np.isnan(vals)
    kept_cols = cols0[keep]
    cp = np.concatenate([[1], 1 + np.cumsum(np.bincount(kept_cols, minlength=n))]).astype(np.int64)
    return ("sparse", m, n, cp, rowval[keep], vals[keep])
