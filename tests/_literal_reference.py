"""A second, independent reading of the reference: finite_difference_jacobian!(J, f, x, cache, f_in; ...) transcribed
line by line into Python/numpy with Julia's 1-based loops kept (src/jacobians.jl:504-622; hooks: ext/FiniteDiffSparseArraysExt.jl
:20-28,:38-47,:51-52, ext/FiniteDiffBandedMatricesExt.jl:13-27, src/iteration_utils.jl:25-32, src/jacobians.jl:473-488,
src/epsilons.jl:26-29,50-53).  It exists to cross-check oracle/fd_oracle.c on random inputs (tests/test_oracle_literal.py):
two restatements written separately agreeing bit for bit is stronger evidence than either alone.  Test infrastructure only.

Matrix stand-ins: CSC(m, n, colptr, rowval, nzval) (1-based Int64 arrays), Banded(m, n, l, u, data[(l+u+1), n]),
dense = 2-D float64 array (column-major or not: indexed as J[row, col]).
"""
import math

import numpy as np


class CSC:
    def __init__(self, m, n, colptr, rowval, nzval=None):
        self.m, self.n = m, n
        self.colptr, self.rowval = np.asarray(colptr, np.int64), np.asarray(rowval, np.int64)
        self.nzval = np.zeros(len(self.rowval)) if nzval is None else nzval

    def setindex(self, v, row, col):          # J[row, col] = v on a stored entry (rows sorted inside a column)
        lo, hi = self.colptr[col - 1] - 1, self.colptr[col] - 1
        p = lo + int(np.searchsorted(self.rowval[lo:hi], row))
        assert p < hi and self.rowval[p] == row, "entry not stored (the reference would insert it)"
        self.nzval[p] = v


class Banded:
    def __init__(self, m, n, l, u, data=None):
        self.m, self.n, self.l, self.u = m, n, l, u
        self.data = np.zeros((l + u + 1, n)) if data is None else data

    def setindex(self, v, row, col):          # BandedMatrices storage: data[u + row - col + 1, col]
        self.data[self.u + row - col, col - 1] = v


def _size(J):
    return (J.m, J.n) if isinstance(J, (CSC, Banded)) else J.shape


def _setindex(J, v, row, col):
    if isinstance(J, (CSC, Banded)):
        J.setindex(v, row, col)
    else:
        J[row - 1, col - 1] = v


def _bool_mul(v, mask):
    """Julia's Float64 * Bool, elementwise: v * true = v, v * false = copysign(0.0, v) (a "strong zero", never NaN:
    NaN * false and Inf * false are zeros too, unlike numpy's v * False)."""
    v = np.broadcast_to(np.asarray(v, dtype=np.float64), np.shape(mask))
    return np.where(mask, v, np.copysign(0.0, v))


def _max(a, b):
    """Julia's max(::Float64, ::Float64): NaN if either is NaN, and -0.0 < 0.0 (Python's max keeps its first argument on
    a tie, so max(-0.0, 0.0) would be -0.0, and max(1.0, nan) would be 1.0)."""
    if math.isnan(a) or math.isnan(b):
        return a - b
    if a == b:
        return b if math.copysign(1.0, a) < 0 else a
    return a if a > b else b


def compute_epsilon(fdtype, x, relstep, absstep, dir):
    if fdtype == "forward":
        return _max(relstep * abs(x), absstep) * dir           # epsilons.jl:26-29
    return _max(relstep * abs(x), absstep)                     # epsilons.jl:50-53


def norm(x2):
    """LinearAlgebra.norm(::Vector{Float64}) (stdlib: norm2 -> generic_norm2 below 32 elements, BLAS.nrm2 from 32 on),
    written independently of oracle/fd_oracle.c: plain Python floats in order for the short branch, numpy's x87
    `longdouble` with four interleaved accumulators for OpenBLAS's nrm2.S."""
    n = len(x2)
    if n == 0:
        return 0.0
    if n < 32:
        maxabs = abs(float(x2[0]))                             # normInf: max propagates NaN (Python's max does not)
        for v in x2[1:]:
            a = abs(float(v))
            maxabs = maxabs if (math.isnan(maxabs) or maxabs > a) else a
        if maxabs == 0.0 or math.isinf(maxabs):
            return maxabs
        if math.isfinite(n * maxabs * maxabs) and maxabs * maxabs != 0.0:
            s = 0.0
            for v in x2:
                s += float(v) * float(v)
            return math.sqrt(s)
        s = 0.0
        for v in x2:
            t = abs(float(v)) / maxabs
            s += t * t
        return maxabs * math.sqrt(s)
    L = np.longdouble
    acc = [L(0), L(0), L(0), L(0)]
    body = n - n % 8
    for i in range(body):
        t = L(x2[i])
        acc[i % 4] = acc[i % 4] + t * t
    for i in range(body, n):
        t = L(x2[i])
        acc[0] = acc[0] + t * t
    return float(np.sqrt((acc[0] + acc[1]) + (acc[2] + acc[3])))


def default_relstep(fdtype):
    eps = np.finfo(np.float64).eps
    return math.sqrt(eps) if fdtype == "forward" else float(np.cbrt(eps))   # epsilons.jl:134-144: sqrt(eps(T)) / cbrt(eps(T))


def _findstructralnz(A):                                       # jacobians.jl:473-488
    I, Jc = [], []
    for j in range(1, A.shape[1] + 1):
        for i in range(1, A.shape[0] + 1):
            if A[i - 1, j - 1] != 0:
                I.append(i)
                Jc.append(j)
    return I, Jc


def _fill_matrix(J, v):                                        # jacobians.jl:663 / ext Sparse :30
    if isinstance(J, CSC):
        J.nzval[:] = v
    elif isinstance(J, Banded):
        J.data[:] = v
    else:
        J[:] = v


def _colorediteration(J, sparsity, rows_index, cols_index, vfx, colorvec, color_i, ncols, common):
    if common:                                                 # ext Sparse :38-47
        for col_index in range(1, ncols + 1):
            if colorvec[col_index - 1] == color_i:
                for spidx in range(J.colptr[col_index - 1], J.colptr[col_index]):      # nzrange
                    row_index = J.rowval[spidx - 1]
                    J.nzval[spidx - 1] = vfx[row_index - 1]
    elif isinstance(sparsity, CSC):                            # ext Sparse :20-28
        for col_index in range(1, ncols + 1):
            if colorvec[col_index - 1] == color_i:
                for row_index in sparsity.rowval[sparsity.colptr[col_index - 1] - 1:sparsity.colptr[col_index] - 1]:
                    _setindex(J, vfx[row_index - 1], int(row_index), col_index)
    elif isinstance(sparsity, Banded):                         # ext Banded :13-27
        nrows = _size(J)[0]
        l, u = sparsity.l, sparsity.u
        for col_index in range(max(1, 1 - l), min(ncols, ncols + u) + 1):
            if colorvec[col_index - 1] == color_i:
                for row_index in range(max(1, col_index - u), min(nrows, col_index + l) + 1):
                    _setindex(J, vfx[row_index - 1], row_index, col_index)
    else:                                                      # iteration_utils.jl:25-32
        for i in range(1, len(cols_index) + 1):
            if colorvec[cols_index[i - 1] - 1] == color_i:
                _setindex(J, vfx[rows_index[i - 1] - 1], rows_index[i - 1], cols_index[i - 1])


def finite_difference_jacobian(J, f, x, cache, f_in=None, *, fdtype="forward", relstep=None, absstep=None, colorvec,
                               sparsity, dir=1.0):
    """Returns dict(eps=[per colour], fcalls=int).  cache = dict(x1, x2, fx, fx1) of numpy arrays (mutated like the
    reference mutates them); x is mutated and restored in central mode exactly as jacobians.jl:604,620 do."""
    if relstep is None:
        relstep = default_relstep(fdtype)                      # :508
    if absstep is None:
        absstep = relstep                                      # :509
    m, n = _size(J)                                            # :515
    _color = np.asarray(colorvec)
    x1, x2, fx, fx1 = cache["x1"], cache["x2"], cache["fx"], cache["fx1"]
    x1[:] = x                                                  # :519
    vfx = fx
    calls = 0
    rows_index = cols_index = None
    if sparsity is not None and not isinstance(sparsity, (CSC, Banded)):   # :524-528  (DenseMatrix prototype)
        rows_index, cols_index = _findstructralnz(sparsity)
    if sparsity is not None:
        _fill_matrix(J, 0.0)                                   # :530-532
    common = isinstance(J, CSC) and isinstance(sparsity, CSC) and np.array_equal(J.colptr, sparsity.colptr) and \
        np.array_equal(J.rowval, sparsity.rowval)              # ext Sparse :51-52
    maxcolor = int(_color.max()) if len(_color) else 0
    eps_list = []
    if fdtype == "forward":
        vfx1 = fx1
        if f_in is None:
            f(fx, x); calls += 1                               # :540-542
            vfx = fx
        else:
            vfx = f_in
        for color_i in range(1, maxcolor + 1):                 # :547
            if sparsity is None:                               # :548-557
                x1_save = x1[color_i - 1]
                epsilon = compute_epsilon("forward", x1_save, relstep, absstep, dir)
                x1[color_i - 1] = x1_save + epsilon
                f(fx1, x1); calls += 1
                J[:, color_i - 1] = (vfx1 - vfx) / epsilon
                x1[color_i - 1] = x1_save
            else:
                mask = (_color == color_i)
                x2[:] = _bool_mul(x1, mask)                    # :559
                tmp = norm(x2)                                 # norm(x2) :560
                epsilon = compute_epsilon("forward", math.sqrt(tmp), relstep, absstep, dir)   # :561
                x1[:] = x1 + _bool_mul(epsilon, mask)          # :562
                f(fx1, x1); calls += 1                         # :563
                vfx1[:] = (vfx1 - vfx) / epsilon               # :565
                _colorediteration(J, sparsity, rows_index, cols_index, vfx1, _color, color_i, n, common)
                x1[:] = x1 - _bool_mul(epsilon, mask)          # :584
            eps_list.append(epsilon)
    elif fdtype == "central":
        vfx1 = fx1
        for color_i in range(1, maxcolor + 1):                 # :589
            if sparsity is None:                               # :590-598
                x_save = x[color_i - 1]
                epsilon = compute_epsilon("central", x_save, relstep, absstep, dir)
                x1[color_i - 1] = x_save + epsilon
                f(fx1, x1); calls += 1
                x1[color_i - 1] = x_save - epsilon
                f(fx, x1); calls += 1
                J[:, color_i - 1] = (vfx1 - vfx) / (2 * epsilon)
                x1[color_i - 1] = x_save
            else:
                mask = (_color == color_i)
                x2[:] = _bool_mul(x1, mask)                    # :600
                tmp = norm(x2)                                 # :601
                epsilon = compute_epsilon("central", math.sqrt(tmp), relstep, absstep, dir)
                x1[:] = x1 + _bool_mul(epsilon, mask)          # :603
                x[:] = x - _bool_mul(epsilon, mask)            # :604
                f(fx1, x1); calls += 1
                f(fx, x); calls += 1
                vfx1[:] = (vfx1 - vfx) / (2 * epsilon)         # :607
                _colorediteration(J, sparsity, rows_index, cols_index, vfx1, _color, color_i, n, common)
                x1[:] = x1 - _bool_mul(epsilon, mask)          # :619
                x[:] = x + _bool_mul(epsilon, mask)            # :620
            eps_list.append(epsilon)
    else:
        raise ValueError("fdtype")
    return {"eps": np.array(eps_list), "fcalls": calls}


def finite_difference_jacobian_complex(J, f, x, cache, *, colorvec, sparsity):
    """fdtype = Val(:complex), returntype <: Real (jacobians.jl:623-648).  cache = dict(x1, fx) of complex128 arrays."""
    m, n = _size(J)
    _color = np.asarray(colorvec)
    x1, fx = cache["x1"], cache["fx"]
    x1[:] = x                                                  # :519 (complex copy of the real x)
    vfx = fx
    rows_index = cols_index = None
    if sparsity is not None and not isinstance(sparsity, (CSC, Banded)):
        rows_index, cols_index = _findstructralnz(sparsity)
    if sparsity is not None:
        _fill_matrix(J, 0.0)
    common = isinstance(J, CSC) and isinstance(sparsity, CSC) and np.array_equal(J.colptr, sparsity.colptr) and \
        np.array_equal(J.rowval, sparsity.rowval)
    epsilon = float(np.finfo(np.float64).eps)                  # :624
    calls = 0
    for color_i in range(1, (int(_color.max()) if len(_color) else 0) + 1):
        if sparsity is None:                                   # :626-631
            x1_save = x1[color_i - 1]
            x1[color_i - 1] = x1_save + 1j * epsilon
            f(fx, x1); calls += 1
            J[:, color_i - 1] = vfx.imag / epsilon
            x1[color_i - 1] = x1_save
        else:
            mask = (_color == color_i)
            # im*epsilon = Complex(epsilon*false, epsilon*true); times a Bool each part is a strong zero where false
            x1[:] = x1 + (_bool_mul(0.0, mask) + 1j * _bool_mul(epsilon, mask))   # :634
            f(fx, x1); calls += 1
            q = vfx.imag / epsilon                             # :636  @. vfx = imag(vfx) / epsilon
            vfx[:] = q
            _colorediteration(J, sparsity, rows_index, cols_index, q, _color, color_i, n, common)
            x1[:] = x1 - (_bool_mul(0.0, mask) + 1j * _bool_mul(epsilon, mask))   # :644
    return {"fcalls": calls}


def finite_difference_jvp(jvp, f, x, v, cache, f_in=None, *, fdtype="forward", relstep=None, absstep=None, dir=1.0):
    """finite_difference_jvp!(jvp, f, x, v, cache::JVPCache, f_in; relstep, absstep, dir)  (src/jvp.jl:238-274).
    cache = dict(x1, fx1).  Returns dict(eps, fcalls)."""
    if relstep is None:
        relstep = default_relstep(fdtype)
    if absstep is None:
        absstep = relstep
    x1, fx1 = cache["x1"], cache["fx1"]
    tmp = math.sqrt(abs(float(np.dot(x, v))))                 # :253
    epsilon = compute_epsilon(fdtype, tmp, relstep, absstep, dir)
    calls = 0
    if fdtype == "forward":
        if f_in is None:
            f(fx1, x); calls += 1                              # :256
        else:
            fx1 = f_in                                         # :258 (rebinds the local only)
        x1[:] = x + epsilon * v                                # :260
        f(jvp, x1); calls += 1
        jvp[:] = (jvp - fx1) / epsilon                         # :262
    elif fdtype == "central":
        x1[:] = x - epsilon * v                                # :264
        f(fx1, x1); calls += 1
        x1[:] = x + epsilon * v                                # :266
        f(jvp, x1); calls += 1
        jvp[:] = (jvp - fx1) / (2 * epsilon)                   # :268
    else:
        raise ValueError("fdtype")
    return {"eps": epsilon, "fcalls": calls}


_DEFAULT = object()


def finite_difference_jacobian_cacheless(J, f, x, fdtype="forward", f_in=None, *, relstep=None, absstep=None,
                                         colorvec=None, sparsity=_DEFAULT):
    """The cache-less method (jacobians.jl:446-471): builds the cache, evaluates f(fx, x) itself in forward mode and
    forwards cache.fx as f_in.  Returns dict(eps, fcalls)."""
    m, n = _size(J)
    if colorvec is None:
        colorvec = np.arange(1, len(x) + 1)                    # :454
    if sparsity is _DEFAULT:
        sparsity = J if isinstance(J, (CSC, Banded)) else None # :455  ArrayInterface.has_sparsestruct(J) ? J : nothing
    extra = 0
    if f_in is None and fdtype == "forward":
        fx = np.zeros_like(x) if m == len(x) else np.zeros(m)  # :457-461
        f(fx, x); extra = 1                                    # :462
        cache = dict(x1=x.copy(), x2=np.zeros_like(x), fx=fx, fx1=fx.copy())          # JacobianCache(x, fx, ...) :50-57
    elif f_in is None:
        cache = dict(x1=x.copy(), x2=np.zeros_like(x), fx=np.zeros(m), fx1=np.zeros(m))
    else:
        cache = dict(x1=x.copy(), x2=np.zeros_like(x), fx=f_in, fx1=f_in.copy())
    r = finite_difference_jacobian(J, f, x, cache, cache["fx"], fdtype=fdtype, relstep=relstep, absstep=absstep,
                                   colorvec=colorvec, sparsity=sparsity)               # :469-470
    r["fcalls"] += extra
    return r
