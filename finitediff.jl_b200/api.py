"""Host-side mirror of the reference interface for the coloured-Jacobian path, over the C ABI.

The reference is Julia and this image has no `julia`, so the executable host side is this Python mirror (the Julia
`ccall` wrapper with the same surface is shipped, unexecuted, in julia/FiniteDiffB200.jl).  Names, argument meaning
and error behaviour follow src/jacobians.jl:

    JacobianCache(x[, fx[, fx1]], fdtype="forward", returntype=float64; colorvec=1:length(x), sparsity=nothing)
                                                                       (jacobians.jl:11-17, :50-57, :94-102)
    finite_difference_jacobian_(J, f, x, cache, f_in=None; relstep, absstep, colorvec, sparsity, dir)   (:504-514)
    finite_difference_jacobian_(J, f, x, fdtype="forward", returntype, f_in; relstep, absstep, colorvec, sparsity)
                                                                       (cache-less, :446-455)
    resize_(cache, i)                                                  (:655-661)
    default_relstep / compute_epsilon                                  (epsilons.jl:26-29,50-53,134-144)

(`!` is not a Python identifier character: `finite_difference_jacobian!` is spelled with a trailing underscore.)
Index arrays keep Julia's convention: Int64, 1-based.  PyTorch is used only for device memory and streams.
All compute happens in libfdjac_b200.so; there is no eager/CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import numbers
import warnings
import weakref
import zlib
from typing import Callable, Optional

import numpy as np
import torch

from . import _lib as L

__all__ = [
    "SparseMatrixCSC", "BandedMatrix", "Tridiagonal", "Diagonal", "Bidiagonal", "SymTridiagonal", "BandedBlockBandedMatrix",
    "BlockSkylineMatrix", "DenseColumnBlock", "SparseMatrixCSR", "NativeFn", "JacobianCache", "Plan",
    "finite_difference_jacobian_", "finite_difference_jacobian_b", "resize_", "default_relstep", "compute_epsilon",
    "zeros_colmajor", "pinned_empty", "HessianCache", "finite_difference_hessian_", "finite_difference_hessian",
    "GradientCache", "finite_difference_gradient_", "finite_difference_gradient", "DerivativeCache",
    "finite_difference_derivative_", "finite_difference_derivative",
]

_DEFAULT = object()

_FDTYPES = {"forward": L.FDB_FORWARD, "central": L.FDB_CENTRAL, "complex": L.FDB_COMPLEX, L.FDB_FORWARD: L.FDB_FORWARD,
            L.FDB_CENTRAL: L.FDB_CENTRAL, L.FDB_COMPLEX: L.FDB_COMPLEX}


def _fdtype_code(fdtype) -> int:
    if isinstance(fdtype, str):
        fdtype = fdtype.lstrip(":")
    if fdtype not in _FDTYPES:
        # epsilons.jl:159-167 fdtype_error
        raise ValueError("Unrecognized fdtype: valid values are 'forward', 'central' and 'complex'.")
    return _FDTYPES[fdtype]


def default_relstep(fdtype, T=torch.float64) -> float:
    """src/epsilons.jl:134-144"""
    return L.lib().fdb_default_relstep(_fdtype_code(fdtype))


def compute_epsilon(fdtype, x: float, relstep: float, absstep: float, dir: float = 1.0) -> float:
    """src/epsilons.jl:26-29 (forward) / :50-53 (central)"""
    return L.lib().fdb_compute_epsilon(_fdtype_code(fdtype), float(x), float(relstep), float(absstep), float(dir))


# ------------------------------------------------------------------------------------------------ array helpers
class PeerValues:
    """J value storage that lives in ANOTHER process / on another GPU and is only mapped here (CUDA IPC, peer access): a
    raw device pointer + length, deliberately NOT a torch tensor — torch would attribute the mapping to the exporting
    device and copy it on any device mismatch, and stores into a copy never reach the owner."""
    is_cuda = True
    dtype = torch.float64

    def __init__(self, ptr: int, numel: int):
        self._ptr, self._numel = int(ptr), int(numel)

    def data_ptr(self) -> int:
        return self._ptr

    def numel(self) -> int:
        return self._numel


def _is_cuda(t) -> bool:
    return (isinstance(t, torch.Tensor) and t.is_cuda) or isinstance(t, PeerValues)


def _index_ptr(a):
    """(pointer, keepalive) of an Int64 index array living on the host (numpy / CPU tensor) or the device."""
    if a is None:
        return None, None
    if isinstance(a, torch.Tensor):
        if a.dtype != torch.int64:
            raise TypeError("index arrays must be Int64 (as SparseMatrixCSC{Float64,Int64} stores them)")
        a = a.contiguous()
        return a.data_ptr(), a
    if isinstance(a, range):
        a = np.arange(a.start, a.stop, a.step, dtype=np.int64)
    arr = np.ascontiguousarray(a, dtype=np.int64)
    return arr.ctypes.data, arr


def _is_identity_colorvec(colorvec, n: int) -> bool:
    """colorvec == 1:n (the JacobianCache default, jacobians.jl:16), whatever container holds it."""
    if colorvec is None:
        return True
    if isinstance(colorvec, range):
        return colorvec == range(1, n + 1)
    if isinstance(colorvec, torch.Tensor):
        return colorvec.numel() == n and bool(torch.equal(colorvec.reshape(-1).cpu().to(torch.int64),
                                                          torch.arange(1, n + 1, dtype=torch.int64)))
    arr = np.asarray(colorvec).reshape(-1)
    return arr.size == n and bool(np.array_equal(arr, np.arange(1, n + 1)))


def _index_key(a):
    if a is None:
        return None
    if isinstance(a, torch.Tensor):
        return ("t", a.data_ptr(), a.numel(), a._version, str(a.device))
    if isinstance(a, range):
        return ("r", a.start, a.stop, a.step)
    arr = np.asarray(a)
    if arr.size <= 4096:
        return ("v", arr.shape, arr.astype(np.int64).tobytes())
    # large host arrays: identity + a strided content sample (4096 elements, first and last included), so that an
    # in-place edit of colorvec / colptr / rowval is noticed in all but contrived cases without an O(n) pass on every
    # call.  The plan holds a private compressed copy: after an in-place edit that the sample cannot see, call
    # cache.invalidate() (documented in JacobianCache).
    flat = arr.reshape(-1)
    step = max(1, flat.size // 4096)
    sample = np.ascontiguousarray(flat[::step]).tobytes() + np.ascontiguousarray(flat[-1:]).tobytes()
    return ("n", arr.__array_interface__["data"][0], arr.size, zlib.crc32(sample))


def zeros_colmajor(m: int, n: int, device="cuda") -> torch.Tensor:
    """A Julia-style dense Matrix{Float64}: logical (m, n), column-major storage (stride (1, m))."""
    return torch.zeros((n, m), dtype=torch.float64, device=device).t()


def pinned_empty(count: int) -> np.ndarray:
    """float64 host array in pinned memory (fdb_host_alloc) — what fdb_jacobian_host needs to reach PCIe speed."""
    p = C.c_void_p()
    L.check(L.lib().fdb_host_alloc(C.byref(p), max(int(count), 1) * 8))
    buf = (C.c_double * max(int(count), 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=np.float64, count=int(count))
    weakref.finalize(buf, L.lib().fdb_host_free, p)
    return arr


class _DevArray:
    """Zero-copy view of raw device memory for torch.as_tensor (CUDA array interface v3)."""

    def __init__(self, ptr: int, shape, strides=None, typestr: str = "<f8"):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 3, "strides": strides}


# ------------------------------------------------------------------------------------------------ matrix types
class SparseMatrixCSC:
    """Mirror of SparseArrays.SparseMatrixCSC{Float64,Int64}: m, n, colptr[n+1], rowval[nnz] (Int64, 1-based),
    nzval[nnz] (float64; CUDA tensor for the device path, numpy array for the host path)."""

    def __init__(self, m, n, colptr, rowval, nzval):
        self.m, self.n = int(m), int(n)
        self.colptr, self.rowval, self.nzval = colptr, rowval, nzval

    @property
    def shape(self):
        return (self.m, self.n)

    @property
    def nnz(self):
        return int(self.rowval.shape[0]) if hasattr(self.rowval, "shape") else len(self.rowval)

    @staticmethod
    def from_scipy(A, device="cuda", index_device=None):
        import scipy.sparse as sp
        A = sp.csc_matrix(A)
        A.sort_indices()
        colptr = torch.from_numpy(A.indptr.astype(np.int64) + 1)
        rowval = torch.from_numpy(A.indices.astype(np.int64) + 1)
        if index_device is not None:
            colptr, rowval = colptr.to(index_device), rowval.to(index_device)
        nz = torch.zeros(A.nnz, dtype=torch.float64, device=device) if device != "host" else np.zeros(A.nnz)
        return SparseMatrixCSC(A.shape[0], A.shape[1], colptr, rowval, nz)

    def similar(self):
        nz = torch.empty_like(self.nzval) if isinstance(self.nzval, torch.Tensor) else np.empty_like(self.nzval)
        return SparseMatrixCSC(self.m, self.n, self.colptr, self.rowval, nz)

    def to_dense(self) -> np.ndarray:
        cp = np.asarray(self.colptr.cpu() if isinstance(self.colptr, torch.Tensor) else self.colptr) - 1
        rv = np.asarray(self.rowval.cpu() if isinstance(self.rowval, torch.Tensor) else self.rowval) - 1
        nz = self.nzval.cpu().numpy() if isinstance(self.nzval, torch.Tensor) else np.asarray(self.nzval)
        import scipy.sparse as sp
        return sp.csc_matrix((nz, rv, cp), shape=(self.m, self.n)).toarray()


class SparseMatrixCSR:
    """Mirror of a row-compressed sparse matrix (CUDA.jl's CuSparseMatrixCSR{Float64} with Int64 indices, the input format
    of cuSPARSE, cuDSS and AMGX): m, n, rowptr[m+1], colval[nnz] (Int64, 1-based), nzval[nnz] (float64).  Columns within a
    row may come in any order and an (r, c) may repeat: each stored entry is its own slot of nzval."""

    def __init__(self, m, n, rowptr, colval, nzval):
        self.m, self.n = int(m), int(n)
        self.rowptr, self.colval, self.nzval = rowptr, colval, nzval

    @property
    def shape(self):
        return (self.m, self.n)

    @property
    def nnz(self):
        return int(self.colval.shape[0]) if hasattr(self.colval, "shape") else len(self.colval)

    @staticmethod
    def from_scipy(A, device="cuda", index_device=None):
        """The CSR of A as scipy stores it: its column order within a row (and its duplicates) are kept."""
        import scipy.sparse as sp
        A = A if sp.isspmatrix_csr(A) or isinstance(A, sp.csr_array) else sp.csr_matrix(A)
        rowptr = torch.from_numpy(A.indptr.astype(np.int64) + 1)
        colval = torch.from_numpy(A.indices.astype(np.int64) + 1)
        if index_device is not None:
            rowptr, colval = rowptr.to(index_device), colval.to(index_device)
        nz = torch.zeros(A.nnz, dtype=torch.float64, device=device) if device != "host" else np.zeros(A.nnz)
        return SparseMatrixCSR(A.shape[0], A.shape[1], rowptr, colval, nz)

    def similar(self):
        nz = torch.empty_like(self.nzval) if isinstance(self.nzval, torch.Tensor) else np.empty_like(self.nzval)
        return SparseMatrixCSR(self.m, self.n, self.rowptr, self.colval, nz)

    def findstructralnz(self):
        """(rows, cols), 1-based, one per stored entry in storage order: the entry list of the slot route, whose slots
        are 1:nnz."""
        rp = np.asarray(self.rowptr.cpu() if isinstance(self.rowptr, torch.Tensor) else self.rowptr, dtype=np.int64)
        cv = np.asarray(self.colval.cpu() if isinstance(self.colval, torch.Tensor) else self.colval, dtype=np.int64)
        rows = np.repeat(np.arange(1, self.m + 1, dtype=np.int64), np.diff(rp))
        return rows, cv.copy()

    def to_dense(self) -> np.ndarray:
        """Dense copy; a repeated (r, c) shows the value of its last slot."""
        rows, cols = self.findstructralnz()
        nz = self.nzval.cpu().numpy() if isinstance(self.nzval, torch.Tensor) else np.asarray(self.nzval)
        out = np.zeros((self.m, self.n))
        out[rows - 1, cols - 1] = nz[: len(rows)]
        return out


class BandedMatrix:
    """Mirror of BandedMatrices.BandedMatrix: data is the (l+u+1) x n column-major band storage (flat float64),
    entry (r,c) at data[u+r-c+1, c] (1-based; ext/FiniteDiffBandedMatricesExt.jl:22)."""

    def __init__(self, m, n, l, u, data=None, device="cuda"):
        self.m, self.n, self.l, self.u = int(m), int(n), int(l), int(u)
        if data is None:
            data = torch.zeros((self.l + self.u + 1) * self.n, dtype=torch.float64, device=device)
        self.data = data

    @property
    def shape(self):
        return (self.m, self.n)

    def to_dense(self) -> np.ndarray:
        d = self.data.cpu().numpy() if isinstance(self.data, torch.Tensor) else np.asarray(self.data)
        w = self.l + self.u + 1
        J = np.zeros((self.m, self.n))
        for c in range(1, self.n + 1):
            for r in range(max(1, c - self.u), min(self.m, c + self.l) + 1):
                J[r - 1, c - 1] = d[(c - 1) * w + (self.u + r - c)]
        return J


class Tridiagonal:
    """Mirror of LinearAlgebra.Tridiagonal(dl, d, du): one buffer [dl; d; du]; its structural nonzeros are
    enumerated band by band like ArrayInterface.findstructralnz does (order is irrelevant to the result)."""

    def __init__(self, n, buf=None, device="cuda"):
        self.n = int(n)
        if buf is None:
            buf = torch.zeros(max(3 * self.n - 2, 0), dtype=torch.float64, device=device)
        self.buf = buf

    @property
    def shape(self):
        return (self.n, self.n)

    @property
    def dl(self):
        return self.buf[: self.n - 1]

    @property
    def d(self):
        return self.buf[self.n - 1: 2 * self.n - 1]

    @property
    def du(self):
        return self.buf[2 * self.n - 1:]

    def findstructralnz(self):
        n = self.n
        rows = np.concatenate([np.arange(2, n + 1), np.arange(1, n + 1), np.arange(1, n)]).astype(np.int64)
        cols = np.concatenate([np.arange(1, n), np.arange(1, n + 1), np.arange(2, n + 1)]).astype(np.int64)
        slots = np.arange(1, 3 * n - 1, dtype=np.int64)
        return rows, cols, slots

    def to_dense(self) -> np.ndarray:
        b = self.buf.cpu().numpy()
        n = self.n
        return np.diag(b[n - 1: 2 * n - 1]) + np.diag(b[: n - 1], -1) + np.diag(b[2 * n - 1:], 1)


def _band_entries(n, l, u):
    """1-based (rows, cols, slots) of the in-matrix band (l, u), l, u in {0, 1}, in the packed diagonal storage:
    sub-diagonal, main diagonal, super-diagonal, each from the top left (the layout of FDB_J_DIAGONALS)."""
    rows, cols = [], []
    if l and n > 1:
        rows.append(np.arange(2, n + 1))
        cols.append(np.arange(1, n))
    rows.append(np.arange(1, n + 1))
    cols.append(np.arange(1, n + 1))
    if u and n > 1:
        rows.append(np.arange(1, n))
        cols.append(np.arange(2, n + 1))
    rows = np.concatenate(rows).astype(np.int64)
    cols = np.concatenate(cols).astype(np.int64)
    return rows, cols, np.arange(1, len(rows) + 1, dtype=np.int64)


class Diagonal:
    """Mirror of LinearAlgebra.Diagonal(d): one buffer [d] of n values; its structural nonzeros are the main diagonal,
    the band (0, 0)."""

    l, u = 0, 0

    def __init__(self, n, buf=None, device="cuda"):
        self.n = int(n)
        if buf is None:
            buf = torch.zeros(self.n, dtype=torch.float64, device=device)
        self.buf = buf

    @property
    def shape(self):
        return (self.n, self.n)

    def findstructralnz(self):
        return _band_entries(self.n, 0, 0)

    def to_dense(self) -> np.ndarray:
        return np.diag(self.buf.cpu().numpy())


class Bidiagonal:
    """Mirror of LinearAlgebra.Bidiagonal(dv, ev, uplo): one buffer in ascending row-minus-column order, [dv; ev] for
    uplo = :U (band (0, 1)) and [ev; dv] for :L (band (1, 0)); dv holds n values, ev n-1."""

    def __init__(self, n, uplo, buf=None, device="cuda"):
        self.n = int(n)
        self.uplo = str(uplo).lstrip(":").upper()
        if self.uplo not in ("U", "L"):
            raise ValueError(f"uplo must be :U or :L, got {uplo!r}")
        if buf is None:
            buf = torch.zeros(max(2 * self.n - 1, 0), dtype=torch.float64, device=device)
        self.buf = buf

    @property
    def l(self):
        return 1 if self.uplo == "L" else 0

    @property
    def u(self):
        return 1 if self.uplo == "U" else 0

    @property
    def shape(self):
        return (self.n, self.n)

    @property
    def dv(self):
        return self.buf[: self.n] if self.uplo == "U" else self.buf[self.n - 1: 2 * self.n - 1]

    @property
    def ev(self):
        return self.buf[self.n: 2 * self.n - 1] if self.uplo == "U" else self.buf[: max(self.n - 1, 0)]

    def findstructralnz(self):
        return _band_entries(self.n, self.l, self.u)

    def to_dense(self) -> np.ndarray:
        dv, ev = self.dv.cpu().numpy(), self.ev.cpu().numpy()
        return np.diag(dv) + (np.diag(ev, 1) if self.uplo == "U" else np.diag(ev, -1))


class SymTridiagonal:
    """Mirror of LinearAlgebra.SymTridiagonal as a sparsity: the band (1, 1), the same entry lists as Tridiagonal.  It
    holds no values by default; `buf` = [dv; ev] may be given for n <= 1, where it is a valid Jacobian target.  As a
    target with n >= 2 it is refused before any f call: LinearAlgebra's setindex! refuses its off-diagonal entries."""

    l, u = 1, 1

    def __init__(self, n, buf=None):
        self.n = int(n)
        self.buf = buf

    @property
    def shape(self):
        return (self.n, self.n)

    def findstructralnz(self):
        return _band_entries(self.n, 1, 1)


class BandedBlockBandedMatrix:
    """Mirror of BlockBandedMatrices.BandedBlockBandedMatrix: square blocks structure given by `rowblocks` / `colblocks`
    (block lengths), block bandwidths (l, u) and sub-block bandwidths (lam, mu).  The decompression hook
    ext/FiniteDiffBlockBandedMatricesExt.jl:16-42 writes, for every column j of block-column J and every block-row
    K in blockcolrange(J) = max(1,J-u):min(N,J+l), the in-sub-band rows k in max(1,j-mu):min(m_K, j+lam).
    Storage here: one band-data column of (l+u+1)*(lam+mu+1) slots per matrix column — slot
    (K-J+u)*(lam+mu+1) + (mu+k-j) for entry (k, j) of block (K, J) (the BlockBandedMatrices layout as documented; the
    package source is not vendored in the reference tree, so the LAYOUT is this mirror's own — the ENTRY SET and the
    values are what parity is about, coloring_tests.jl:99-119)."""

    def __init__(self, rowblocks, colblocks, blockbandwidths, subblockbandwidths, data=None, device="cuda"):
        self.rb, self.cb = [int(b) for b in rowblocks], [int(b) for b in colblocks]
        (self.l, self.u), (self.lam, self.mu) = blockbandwidths, subblockbandwidths
        self.m, self.n = sum(self.rb), sum(self.cb)
        self.w = (self.l + self.u + 1) * (self.lam + self.mu + 1)
        if data is None:
            data = torch.zeros(self.w * self.n, dtype=torch.float64, device=device)
        self.data = data
        self._nz = None

    @property
    def shape(self):
        return (self.m, self.n)

    def findstructralnz(self):
        """(rows, cols, slots), 1-based, in the order the reference's hook visits them."""
        if self._nz is None:
            ro = np.concatenate([[0], np.cumsum(self.rb)])
            co = np.concatenate([[0], np.cumsum(self.cb)])
            sw = self.lam + self.mu + 1
            rows, cols, slots = [], [], []
            N_r, N_c = len(self.rb), len(self.cb)
            for J in range(1, N_c + 1):
                for K in range(max(1, J - self.u), min(N_r, J + self.l) + 1):
                    mK = self.rb[K - 1]
                    for j in range(1, self.cb[J - 1] + 1):
                        k = np.arange(max(1, j - self.mu), min(mK, j + self.lam) + 1)
                        if len(k) == 0:
                            continue
                        gc = co[J - 1] + j
                        rows.append(ro[K - 1] + k)
                        cols.append(np.full(len(k), gc))
                        slots.append((gc - 1) * self.w + (K - J + self.u) * sw + (self.mu + k - j) + 1)
            cat = lambda a: np.concatenate(a).astype(np.int64) if a else np.zeros(0, np.int64)
            self._nz = (cat(rows), cat(cols), cat(slots))
        return self._nz

    def to_dense(self) -> np.ndarray:
        rows, cols, slots = self.findstructralnz()
        d = self.data.cpu().numpy() if isinstance(self.data, torch.Tensor) else np.asarray(self.data)
        J = np.zeros((self.m, self.n))
        J[rows - 1, cols - 1] = d[slots - 1]
        return J

    def matrix_colors(self) -> np.ndarray:
        """A valid colouring for the full structure: block colour (cycle l+u+1) x sub-band colour (cycle lam+mu+1)
        — the scheme of ArrayInterface.matrix_colors(::BandedBlockBandedMatrix) for uniform blocks."""
        sw, bw = self.lam + self.mu + 1, self.l + self.u + 1
        out = []
        for J, nb in enumerate(self.cb):
            out.append((J % bw) * sw + (np.arange(nb) % sw) + 1)
        return np.concatenate(out).astype(np.int64)


class BlockBandedMatrix(BandedBlockBandedMatrix):
    """Mirror of BlockBandedMatrices.BlockBandedMatrix: dense blocks inside the block band.  Hook
    ext/FiniteDiffBlockBandedMatricesExt.jl:44-68: for every column j of block-column J, ALL rows of every block-row K
    in blockcolrange(J).  Expressed as a BandedBlockBandedMatrix whose sub-block bandwidths cover the whole block."""

    def __init__(self, rowblocks, colblocks, blockbandwidths, data=None, device="cuda"):
        full = max(max(rowblocks), max(colblocks)) - 1 if len(rowblocks) and len(colblocks) else 0
        super().__init__(rowblocks, colblocks, blockbandwidths, (full, full), data=data, device=device)


class BlockSkylineMatrix:
    """Mirror of BlockBandedMatrices.BlockBandedMatrix as that package stores it (a BlockSkylineMatrix with constant
    block bandwidths (l, u)): dense blocks inside the block band, hook ext/FiniteDiffBlockBandedMatricesExt.jl:44-68.
    Block column J (0-based here) covers block rows max(0, J-u) .. min(N-1, J+l); its data is one column-major slab of
    height h_J (the rows of those blocks) and cb[J] columns, starting at slot start_J = sum_{J'<J} h_J' cb[J'].  Entry
    (r, c) of block (K, J) sits at start_J + c h_J + rowoff_J(K) + r.  Every slot is a structural entry, so `data` holds
    j_len = start_N values and nothing else.  (BlockBandedMatrix above is this structure in the padded band layout.)"""

    def __init__(self, rowblocks, colblocks, blockbandwidths, data=None, device="cuda"):
        self.rb, self.cb = [int(b) for b in rowblocks], [int(b) for b in colblocks]
        self.l, self.u = (int(b) for b in blockbandwidths)
        self.m, self.n = sum(self.rb), sum(self.cb)
        ro = np.concatenate([[0], np.cumsum(self.rb, dtype=np.int64)]).astype(np.int64)
        Nr = len(self.rb)
        J = np.arange(len(self.cb), dtype=np.int64)
        k0 = np.clip(J - self.u, 0, Nr)                                 # block rows [k0, k1) of block column J
        k1 = np.clip(J + self.l + 1, k0, Nr)
        self.row0 = ro[k0]                                              # first row of each slab, 0-based
        self.heights = ro[k1] - ro[k0]
        self.col0 = np.concatenate([[0], np.cumsum(self.cb, dtype=np.int64)])[:-1].astype(np.int64)
        self.starts = np.concatenate([[0], np.cumsum(self.heights * np.asarray(self.cb, np.int64))]).astype(np.int64)
        self.j_len = int(self.starts[-1])
        if data is None:
            data = torch.zeros(self.j_len, dtype=torch.float64, device=device)
        self.data = data
        self._nz = None

    @property
    def shape(self):
        return (self.m, self.n)

    def findstructralnz(self):
        """(rows, cols, slots), 1-based, in the order the reference's hook visits them: block column J, its column j,
        then every row of every block row in blockcolrange(J) — which is storage order, so slots = 1:j_len."""
        if self._nz is None:
            s = np.arange(self.j_len, dtype=np.int64)
            J = np.searchsorted(self.starts, s, side="right") - 1     # an empty slab shares its start with the next
            rel = s - self.starts[J]
            h = self.heights[J]
            self._nz = (self.row0[J] + rel % h + 1, self.col0[J] + rel // h + 1, s + 1)
        return self._nz

    def to_dense(self) -> np.ndarray:
        rows, cols, slots = self.findstructralnz()
        d = self.data.cpu().numpy() if isinstance(self.data, torch.Tensor) else np.asarray(self.data)
        J = np.zeros((self.m, self.n))
        J[rows - 1, cols - 1] = d[slots - 1]
        return J

    def matrix_colors(self) -> np.ndarray:
        """A valid colouring for the full structure: block colour (cycle l+u+1) x column within the block, b colours
        per block colour — ArrayInterface.matrix_colors(::BlockBandedMatrix) for uniform blocks of size b, so
        (l+u+1)*b colours.  Non-uniform blocks take b = the largest block."""
        bw, b = max(self.l + self.u + 1, 1), max(self.cb, default=0)
        out = [(J % bw) * b + np.arange(nb) + 1 for J, nb in enumerate(self.cb)]
        return np.concatenate(out).astype(np.int64) if out else np.zeros(0, np.int64)


class DenseColumnBlock:
    """Columns [col0, col0+ncols) of a dense m x n Jacobian held by ONE rank (north_star config 5: the dense Jacobian is
    column-partitioned over the GPUs and may stay that way): `slab` is the rank's own column-major (m, ncols) storage.
    Use it as J with a JacobianCache built with rank=, world= and sparsity=None; the plan's column range must be the
    block (checked on first use)."""

    def __init__(self, m, n, col0, ncols, device="cuda", slab=None):
        self.m, self.n, self.col0, self.ncols = int(m), int(n), int(col0), int(ncols)
        self.slab = zeros_colmajor(self.m, max(self.ncols, 1), device) if slab is None else slab

    @property
    def shape(self):
        return (self.m, self.n)


def _findstructralnz_dense(A):
    """src/jacobians.jl:473-488: column-major scan of a dense 0/1 prototype."""
    A = np.asarray(A.cpu() if isinstance(A, torch.Tensor) else A)
    if A.ndim == 1:
        A = A.reshape(1, -1)
    c, r = np.nonzero(A.T)
    return (r + 1).astype(np.int64), (c + 1).astype(np.int64)


# ------------------------------------------------------------------------------------------------ user functions
class NativeFn:
    """A native fdb_fn (function address + context struct), e.g. the synthetic f! of libfdjac_synth.so."""

    def __init__(self, address: int, ctx=None, max_batch: int = 1, keepalive=None):
        self.address = int(address)
        self.ctx = ctx
        self.max_batch = int(max_batch)
        self._keepalive = keepalive

    @property
    def ctx_ptr(self):
        return C.cast(C.pointer(self.ctx), C.c_void_p) if self.ctx is not None else None


class _PyFn:
    """Wraps a Python f!(fx, x) working on CUDA tensors as an fdb_fn.  `batched=True` callables receive 2-D
    (batch, m) / (batch, n) tensors; otherwise they are called once per point with 1-D tensors."""

    def __init__(self, f: Callable, m: int, n: int, device: torch.device, batched: bool, complex_: bool = False,
                 scalar: bool = False, elementwise: bool = False, tvec: bool = False, oop: bool = False):
        self.f, self.m, self.n, self.device, self.batched = f, m, n, device, batched
        # scalar (m = 1) functions are called as f(x) and RETURN their value (a 0-d CUDA tensor needs no host sync)
        self.scalar = scalar
        # elementwise functions (derivatives) are called as f(x) and return a tensor of x's shape; scalar -> vector
        # functions (tvec, n = 1) are called in place as f(fx, t) with t a 0-d tensor
        self.elementwise, self.tvec = elementwise, tvec
        # out-of-place functions (finite_difference_jacobian / _jvp) are called as f(x) and return a new array of m values
        # (batched: (batch, m)), which is copied into the slot f! would have written
        self.oop = oop
        self.exc: Optional[BaseException] = None
        self.calls = 0
        # complex-step callbacks (fdb_fn_c) see complex128 tensors; ld* then count complex elements
        self.typestr, self.esize = ("<c16", 16) if complex_ else ("<f8", 8)
        self.cfunc = L.FDB_FN(self._tramp)

    def _view(self, ptr, batch, k, ld):
        if k == 0:                  # an empty array has no storage: its pointer may be NULL (None through ctypes)
            dt = torch.complex128 if self.esize == 16 else torch.float64
            return torch.empty((batch, 0), dtype=dt, device=self.device)
        es = self.esize
        return torch.as_tensor(_DevArray(ptr, (batch, k), (ld * es, es), self.typestr), device=self.device)

    def _tramp(self, _ctx, p_fx, p_x, batch, ldfx, ldx, stream):
        try:
            cur = torch.cuda.current_stream(self.device)
            ctx = None
            if (stream or 0) != cur.cuda_stream:
                ctx = torch.cuda.stream(torch.cuda.ExternalStream(stream or 0, device=self.device))
                ctx.__enter__()
            try:
                fx2 = self._view(p_fx, batch, self.m, ldfx)
                x2 = self._view(p_x, batch, self.n, ldx)
                if self.oop:
                    self.calls += int(batch)
                    if self.batched:
                        fx2.copy_(_oop_result(self.f(x2), fx2.shape, complex_ok=self.esize == 16))
                    else:
                        for b in range(int(batch)):
                            fx2[b].copy_(_oop_result(self.f(x2[b]), fx2[b].shape, complex_ok=self.esize == 16))
                elif self.elementwise and self.batched:
                    self.calls += int(batch)
                    fx2.copy_(torch.as_tensor(self.f(x2), dtype=fx2.dtype, device=self.device))
                elif self.elementwise:
                    for b in range(int(batch)):
                        self.calls += 1
                        fx2[b].copy_(torch.as_tensor(self.f(x2[b]), dtype=fx2.dtype, device=self.device))
                elif self.tvec:
                    for b in range(int(batch)):
                        self.calls += 1
                        self.f(fx2[b], x2[b, 0])
                elif self.scalar and self.batched:
                    self.calls += int(batch)
                    # dtype of the slot (float64 / complex128): a Python float or complex must not pass through
                    # torch's default float32 / complex64
                    fx2[:, 0].copy_(torch.as_tensor(self.f(x2), dtype=fx2.dtype, device=self.device).reshape(-1))
                elif self.scalar:
                    for b in range(int(batch)):
                        self.calls += 1
                        fx2[b, 0].copy_(torch.as_tensor(self.f(x2[b]), dtype=fx2.dtype, device=self.device).reshape(()))
                elif self.batched:
                    self.calls += int(batch)
                    self.f(fx2, x2)
                else:
                    for b in range(int(batch)):
                        self.calls += 1
                        self.f(fx2[b], x2[b])
            finally:
                if ctx is not None:
                    ctx.__exit__(None, None, None)
            return 0
        except BaseException as e:  # never let an exception cross the C ABI
            self.exc = e
            return 1


def _oop_result(r, shape, complex_ok=False):
    """The array an out-of-place f returned, checked against the slot it is copied into."""
    if not isinstance(r, torch.Tensor) or not r.is_cuda:
        raise TypeError("an out-of-place f must return a CUDA tensor")
    if r.is_complex() and not complex_ok:
        raise TypeError("not built: f returns a complex array (complex-valued results of the out-of-place path)")
    if shape == (-1,):
        return r.reshape(-1)
    if r.numel() != int(np.prod(shape)):
        raise ValueError(f"f returned {r.numel()} values where {int(np.prod(shape))} were expected")
    return r.reshape(shape)


# ------------------------------------------------------------------------------------------------ plans
class Plan:
    """Owner of an fdb_plan* (the per-(pattern, colorvec, fdtype) state)."""

    def __init__(self, handle: int, keep=(), owned: bool = True):
        self._h = C.c_void_p(handle)
        self._keep = keep
        # members of an fdb_group are owned (and destroyed) by the group: owned=False gives a plain view
        self._fin = weakref.finalize(self, L.lib().fdb_plan_destroy, C.c_void_p(handle)) if owned else (lambda: None)

    @property
    def handle(self):
        return self._h

    def info(self) -> dict:
        i = L.PlanInfo()
        L.check(L.lib().fdb_plan_info(self._h, C.byref(i)))
        return i.as_dict()

    def counters(self) -> dict:
        c = L.Counters()
        L.check(L.lib().fdb_plan_counters(self._h, C.byref(c)))
        return c.as_dict()

    def eps(self, stream=None) -> np.ndarray:
        i = self.info()
        count = i["n_local_colors"] if i["sp_kind"] == 0 else i["n_colors"]
        out = np.zeros(max(count, 1))
        L.check(L.lib().fdb_plan_get_eps(self._h, out.ctypes.data_as(C.POINTER(C.c_double)), len(out),
                                         C.c_void_p(stream or 0)))
        return out[:count]

    def color_owner(self) -> np.ndarray:
        i = self.info()
        out = np.zeros(max(i["n_colors"], 1), np.int32)
        L.check(L.lib().fdb_plan_color_owner(self._h, out.ctypes.data_as(C.POINTER(C.c_int32)), len(out)))
        return out[: i["n_colors"]]

    def dense_range(self):
        b, e = C.c_int64(), C.c_int64()
        L.check(L.lib().fdb_plan_dense_range(self._h, C.byref(b), C.byref(e)))
        return b.value, e.value

    def set_peers(self, ptrs):
        arr = (C.c_void_p * max(len(ptrs), 1))(*ptrs)
        L.check(L.lib().fdb_plan_set_peers(self._h, len(ptrs), arr))

    def enable_timing(self, on=True):
        L.check(L.lib().fdb_plan_enable_timing(self._h, int(bool(on))))

    def read_timing(self):
        """(summed scatter milliseconds, scatter launches) since the last read; synchronises the recorded events."""
        ms, cnt = C.c_double(), C.c_int64()
        L.check(L.lib().fdb_plan_read_timing(self._h, C.byref(ms), C.byref(cnt)))
        return ms.value, cnt.value

    def destroy(self):
        self._fin()


def _opts(fdtype, device_index, *, no_drift=False, max_batch=1, scratch_bytes=0, rank=0, world=1, partition=0,
          strategy=0, use_graph=False, shared_j=False):
    return L.PlanOpts(fdtype=fdtype, device=device_index, use_current_device=0, no_drift=int(bool(no_drift)),
                      max_batch=int(max_batch), scratch_bytes=int(scratch_bytes), rank=int(rank), world=int(world),
                      partition=int(partition), strategy=int(strategy), use_graph=int(bool(use_graph)), shared_j=int(bool(shared_j)))


def _device_index(device) -> int:
    d = torch.device(device)
    return d.index if d.index is not None else torch.cuda.current_device()


def _dense_ld(J: torch.Tensor):
    """(m, n, ldJ) of a column-major dense J (Julia Matrix).  Row-major tensors are rejected loudly."""
    if isinstance(J, DenseColumnBlock):
        return J.m, J.n, max(int(J.slab.stride(1)) if J.slab.dim() == 2 and J.slab.shape[1] > 1 else J.m, J.m, 1)
    if J.dim() == 1:
        return J.shape[0], 1, max(J.shape[0], 1)
    m, n = J.shape
    if J.dtype != torch.float64:
        raise TypeError("J must be float64")
    if m > 1 and J.stride(0) != 1:
        raise ValueError("dense J must be column-major (Julia Matrix layout): use zeros_colmajor(m, n) or X.t()")
    ld = J.stride(1) if n > 1 else max(m, 1)
    if m == 1 and n > 1:
        ld = J.stride(1)
    return m, n, max(int(ld), m, 1)


def _new_handle(creator: str, *args):
    """The handle fdb_<creator>(&h, *args) creates."""
    h = C.c_void_p()
    L.check(getattr(L.lib(), creator)(C.byref(h), *args))
    return h


def _cached_plan(cache, key, create) -> Plan:
    """cache._plans[key], created by create() on first use."""
    p = cache._plans.get(key)
    if p is None:
        p = cache._plans[key] = create()
    return p


def _stream(stream, device) -> int:
    """The call's stream: the one given, else the current stream of `device`."""
    return torch.cuda.current_stream(device).cuda_stream if stream is None else stream


def _steps(relstep, absstep):
    return (L.STEP_DEFAULT if relstep is None else float(relstep), L.STEP_DEFAULT if absstep is None else float(absstep))


def _call(device, pyfns, fn, *args):
    """fn(*args) on `device`.  When a Python f failed (FDB_ERR_CALLBACK), the first exception pending on the call's
    wrappers `pyfns` propagates as itself, as Julia propagates it; any other failure raises FdbError."""
    with torch.cuda.device(device):
        st = fn(*args)
    if st == L.FDB_ERR_CALLBACK:
        for w in pyfns:
            if w is not None and w.exc is not None:
                exc, w.exc = w.exc, None
                raise exc
    L.check(st)


def _device_slot(owner, attr: str, device, stream, value=None) -> torch.Tensor:
    """owner.<attr>: a one-element float64 tensor on `device` that keeps its pointer from call to call (the arguments of
    a call, and a captured graph's key under use_graph, stay the same), with `value` written on `stream` when given."""
    slot = getattr(owner, attr, None)
    if slot is None or slot.device != device:
        slot = torch.empty(1, dtype=torch.float64, device=device)
        setattr(owner, attr, slot)
    if value is not None:
        with torch.cuda.stream(torch.cuda.ExternalStream(stream, device=device)):
            slot.fill_(float(value))
    return slot


def _plan_route(J, sparsity, colorvec):
    """(kind, args, keep) for (typeof(J), sparsity, colorvec) — the dispatch the reference performs with
    _use_findstructralnz / _use_sparseCSC_common_sparsity / typeof(J) (jacobians.jl:522-535): the plan is made by
    fdb_plan_create_<kind>(&h, *args, &opts) (or fdb_group_create_<kind>(&h, n_devices, devices, *args, &opts)), and
    `keep` holds the host arrays the pointers in args point into."""
    diag_route = _diagonals_route(J, sparsity)     # first: a refused target raises before anything is built
    cv_ptr, cv_keep = _index_ptr(colorvec)
    keep = [cv_keep]
    if diag_route is not None:
        # Diagonal / Bidiagonal / SymTridiagonal sparsity: the banded plan with the band (l, u) of the type, into the packed
        # diagonal storage of the same type or into a dense J
        return "banded", (*diag_route, cv_ptr), keep
    if isinstance(J, SparseMatrixCSR) and not isinstance(sparsity, SparseMatrixCSR):
        raise TypeError(f"not built: a SparseMatrixCSR J with a {type(sparsity).__name__} sparsity")
    if sparsity is None:
        # dense column branch (jacobians.jl:548-557): column i of J from perturbing component i, colorvec = 1:n.
        # With sparsity === nothing and any OTHER colorvec the reference loops color_i in 1:maximum(colorvec) and
        # perturbs COMPONENT color_i (the colour id used as an index), writing only those leading columns of J (J is
        # not zero-filled on this branch) — reproduced as written by fdb_plan_create_dense_colorvec.
        m, n, ld = _dense_ld(J)
        if colorvec is not None and not _is_identity_colorvec(colorvec, n):
            return "dense_colorvec", (m, n, ld, cv_ptr), keep
        return "dense", (m, n, ld), keep
    if isinstance(sparsity, SparseMatrixCSC):
        cp, k1 = _index_ptr(sparsity.colptr)
        rv, k2 = _index_ptr(sparsity.rowval)
        keep += [k1, k2]
        if isinstance(J, SparseMatrixCSC):
            if J is sparsity or (J.colptr is sparsity.colptr and J.rowval is sparsity.rowval):
                jcp = jrv = None
            else:
                jcp, k3 = _index_ptr(J.colptr)
                jrv, k4 = _index_ptr(J.rowval)
                keep += [k3, k4]
            return "csc", (sparsity.m, sparsity.n, cp, rv, L.FDB_J_CSC_NZVAL, jcp, jrv, 0, cv_ptr), keep
        if isinstance(J, torch.Tensor):
            m, n, ld = _dense_ld(J)
            if (m, n) != (sparsity.m, sparsity.n):
                raise ValueError("size(J) != size(sparsity)")
            return "csc", (m, n, cp, rv, L.FDB_J_DENSE, None, None, ld, cv_ptr), keep
        raise TypeError(f"unsupported J type {type(J)} for a SparseMatrixCSC sparsity")
    if isinstance(sparsity, SparseMatrixCSR):
        if isinstance(J, SparseMatrixCSR):
            # J's own pattern: the nzval scatter (rowptr / colval / nzval as the solver holds them)
            if not (J is sparsity or (J.rowptr is sparsity.rowptr and J.colval is sparsity.colval) or _same_csr(J, sparsity)):
                raise TypeError("not built: a SparseMatrixCSR J with a different pattern than its sparsity")
            rp, k1 = _index_ptr(J.rowptr)
            cv, k2 = _index_ptr(J.colval)
            return "csr", (J.m, J.n, rp, cv, cv_ptr), keep + [k1, k2]
        if isinstance(J, torch.Tensor):
            rows, cols = sparsity.findstructralnz()
            m, nn, ld = _dense_ld(J)
            if (m, nn) != (sparsity.m, sparsity.n):
                raise ValueError("size(J) != size(sparsity)")
            return "coo", (m, nn, len(rows), rows.ctypes.data, cols.ctypes.data, L.FDB_J_DENSE, None, ld, cv_ptr), \
                keep + [rows, cols]
        raise TypeError(f"not built: J of type {type(J).__name__} with a SparseMatrixCSR sparsity")
    if isinstance(sparsity, BandedMatrix):
        if isinstance(J, BandedMatrix):
            if (J.l, J.u) != (sparsity.l, sparsity.u):
                raise ValueError("J and sparsity must have the same bandwidths")
            return "banded", (sparsity.m, sparsity.n, sparsity.l, sparsity.u, L.FDB_J_BAND, 0, cv_ptr), keep
        if isinstance(J, torch.Tensor):
            m, n, ld = _dense_ld(J)
            return "banded", (m, n, sparsity.l, sparsity.u, L.FDB_J_DENSE, ld, cv_ptr), keep
        raise TypeError(f"unsupported J type {type(J)} for a BandedMatrix sparsity")
    if isinstance(sparsity, BandedBlockBandedMatrix) and (bb := _block_banded_plan_args(J, sparsity)) is not None:
        # J and sparsity are one square block-banded structure: the closed-form plan, no entry lists on the host
        blocks, l, u, lam, mu, ldata = bb
        return "block_banded", (len(blocks), blocks.ctypes.data if len(blocks) else None, l, u, lam, mu, ldata,
                                cv_ptr), keep + [blocks]
    if isinstance(sparsity, BlockSkylineMatrix):
        # ext/FiniteDiffBlockBandedMatricesExt.jl:44-68 takes the row and the colour blocks from axes(Jac, 1)
        if sparsity.rb != sparsity.cb:
            raise L.FdbError(L.FDB_ERR_INVALID, "a BlockBandedMatrix Jacobian needs square blocks (rowblocks == colblocks)")
        if isinstance(J, BlockSkylineMatrix):
            if (J.rb, J.cb, J.l, J.u) != (sparsity.rb, sparsity.cb, sparsity.l, sparsity.u):
                raise ValueError("J and sparsity must have the same block structure")
            blocks = np.asarray(J.rb, dtype=np.int64)
            ldata = J.data.numel() if isinstance(J.data, torch.Tensor) else J.j_len
            return "block_dense", (len(blocks), blocks.ctypes.data if len(blocks) else None, J.l, J.u, ldata, cv_ptr), \
                keep + [blocks]
    if isinstance(sparsity, (Tridiagonal, SymTridiagonal)):
        rows, cols, slots = sparsity.findstructralnz()
        n = sparsity.n
        if isinstance(J, Tridiagonal):
            jargs = (n, n, L.FDB_J_SLOTS, slots.ctypes.data, 3 * n - 2)
        elif isinstance(J, torch.Tensor):
            m, nn, ld = _dense_ld(J)
            jargs = (m, nn, L.FDB_J_DENSE, None, ld)
        else:
            raise TypeError(f"unsupported J type {type(J)} for a Tridiagonal sparsity")
    elif isinstance(sparsity, BandedBlockBandedMatrix):
        # ext/FiniteDiffBlockBandedMatricesExt.jl:16-42: the hook's (block-row, sub-band) entry set, written by slot
        rows, cols, slots = sparsity.findstructralnz()
        if isinstance(J, BandedBlockBandedMatrix):
            if (J.rb, J.cb, J.l, J.u, J.lam, J.mu) != (sparsity.rb, sparsity.cb, sparsity.l, sparsity.u, sparsity.lam, sparsity.mu):
                raise ValueError("J and sparsity must have the same block structure")
            jargs = (sparsity.m, sparsity.n, L.FDB_J_SLOTS, slots.ctypes.data, sparsity.w * sparsity.n)
        elif isinstance(J, torch.Tensor):
            m, nn, ld = _dense_ld(J)
            jargs = (m, nn, L.FDB_J_DENSE, None, ld)
        else:
            raise TypeError(f"unsupported J type {type(J)} for a BandedBlockBandedMatrix sparsity")
    elif isinstance(sparsity, BlockSkylineMatrix):
        # a dense J: the hook's entry set, written by (row, column)
        rows, cols, slots = sparsity.findstructralnz()
        slots = None
        if not isinstance(J, torch.Tensor):
            raise TypeError(f"unsupported J type {type(J)} for a BlockSkylineMatrix sparsity")
        m, nn, ld = _dense_ld(J)
        jargs = (m, nn, L.FDB_J_DENSE, None, ld)
    elif isinstance(sparsity, (torch.Tensor, np.ndarray, list)):
        # dense 0/1 prototype: rows/cols from _findstructralnz (jacobians.jl:526-527), J must be dense
        rows, cols = _findstructralnz_dense(sparsity)
        slots = None
        if not isinstance(J, torch.Tensor):
            raise TypeError("a dense prototype sparsity needs a dense J")
        m, n, ld = _dense_ld(J)
        jargs = (m, n, L.FDB_J_DENSE, None, ld)
    else:
        raise TypeError(f"unsupported sparsity type {type(sparsity)}")
    m, n, jkind, slot_ptr, ld = jargs          # the entry lists (rows, cols) go into J's slots or into a dense J
    return "coo", (m, n, len(rows), rows.ctypes.data, cols.ctypes.data, jkind, slot_ptr, ld, cv_ptr), \
        keep + [rows, cols, slots]


def _same_csr(A, B) -> bool:
    """A and B are CSRs with the same size, row pointer and columns (the same pattern in the same storage order)."""
    def host(a):
        return np.asarray(a.cpu() if isinstance(a, torch.Tensor) else a, dtype=np.int64)
    return A.shape == B.shape and np.array_equal(host(A.rowptr), host(B.rowptr)) and np.array_equal(host(A.colval), host(B.colval))


def make_plan(J, sparsity, colorvec, fdtype, x_len: int, device, **plan_kw) -> Plan:
    """Create the fdb_plan for (typeof(J), sparsity, colorvec, fdtype) by the creator _plan_route chooses."""
    kind, args, keep = _plan_route(J, sparsity, colorvec)
    o = _opts(_fdtype_code(fdtype), _device_index(device), **plan_kw)
    return Plan(_new_handle(f"fdb_plan_create_{kind}", *args, C.byref(o)).value, tuple(keep))


def _block_banded_plan_args(J, sparsity):
    """(blocks, l, u, lam, mu, ldata) for fdb_plan_create_block_banded when J and `sparsity` are the same block-banded
    structure with square blocks and non-negative bandwidths (BlockBandedMatrix included, in this mirror's layout);
    None otherwise: a dense J, rectangular block lists or two different structures keep the slot-addressed route."""
    if not isinstance(J, BandedBlockBandedMatrix) or not isinstance(sparsity, BandedBlockBandedMatrix):
        return None
    key = (J.rb, J.cb, J.l, J.u, J.lam, J.mu)
    if key != (sparsity.rb, sparsity.cb, sparsity.l, sparsity.u, sparsity.lam, sparsity.mu) or J.rb != J.cb:
        return None
    if min(J.l, J.u, J.lam, J.mu) < 0:
        return None
    ldata = J.data.numel() if isinstance(J.data, torch.Tensor) else J.w * J.n
    return np.asarray(J.rb, dtype=np.int64), J.l, J.u, J.lam, J.mu, ldata


_LA_BANDED = (Diagonal, Bidiagonal, SymTridiagonal)


def _diagonals_route(J, sparsity):
    """(m, n, l, u, jkind, ldJ) for fdb_plan_create_banded when `sparsity` is a Diagonal, Bidiagonal or SymTridiagonal:
    its band (l, u) written into the packed diagonal storage of a J of the same type and size (FDB_J_DIAGONALS), or into
    a dense J (FDB_J_DENSE).  None for every other sparsity, which keeps its route (a Tridiagonal sparsity stays on the
    slot-addressed COO route, and so does a Tridiagonal J with a SymTridiagonal sparsity).

    A SymTridiagonal J with n >= 2 raises ValueError (Julia: ArgumentError) here, before any f call; the reference
    throws the same from LinearAlgebra's setindex! at the first off-diagonal store, after colour 1's f calls.  A J of
    another structured type than the sparsity raises TypeError."""
    if isinstance(J, SymTridiagonal) and J.n >= 2:
        raise ValueError("ArgumentError: a SymTridiagonal cannot be a Jacobian target: its off-diagonal entries cannot be "
                         "set one at a time (use Tridiagonal)")
    if not isinstance(sparsity, _LA_BANDED):
        return None
    n, l, u = sparsity.n, sparsity.l, sparsity.u
    if isinstance(J, torch.Tensor):
        m, nn, ld = _dense_ld(J)
        if (m, nn) != (n, n):
            raise ValueError("size(J) != size(sparsity)")
        return n, n, l, u, L.FDB_J_DENSE, ld
    if isinstance(J, Tridiagonal) and isinstance(sparsity, SymTridiagonal):
        return None
    if type(J) is not type(sparsity) or (isinstance(J, SymTridiagonal) and J.buf is None):
        raise TypeError(f"unsupported J type {type(J)} for a {type(sparsity).__name__} sparsity")
    if J.n != n or (J.l, J.u) != (l, u):
        raise ValueError("J and sparsity must have the same size and bands")
    if isinstance(J, SymTridiagonal):
        l = u = 0                                       # n <= 1: the main diagonal is the whole structure
    return n, n, l, u, L.FDB_J_DIAGONALS, J.buf.numel()


def _has_sparsestruct(J) -> bool:
    """ArrayInterface.has_sparsestruct(J) as used at jacobians.jl:455."""
    return isinstance(J, (SparseMatrixCSC, SparseMatrixCSR, BandedMatrix, Tridiagonal, BandedBlockBandedMatrix,
                          BlockSkylineMatrix) + _LA_BANDED)


def _j_values(J):
    if isinstance(J, (SparseMatrixCSC, SparseMatrixCSR)):
        return J.nzval
    if isinstance(J, BandedMatrix):
        return J.data
    if isinstance(J, (Tridiagonal,) + _LA_BANDED):
        return J.buf
    if isinstance(J, (BandedBlockBandedMatrix, BlockSkylineMatrix)):
        return J.data
    if isinstance(J, DenseColumnBlock):
        return J.slab
    return J


def _j_key(J):
    if isinstance(J, SparseMatrixCSC):
        return ("csc", J.m, J.n, _index_key(J.colptr), _index_key(J.rowval))
    if isinstance(J, SparseMatrixCSR):
        return ("csr", J.m, J.n, _index_key(J.rowptr), _index_key(J.colval))
    if isinstance(J, BandedMatrix):
        return ("band", J.m, J.n, J.l, J.u)
    if isinstance(J, Tridiagonal):
        return ("tri", J.n)
    if isinstance(J, Diagonal):
        return ("diag", J.n)
    if isinstance(J, Bidiagonal):
        return ("bidiag", J.n, J.uplo)
    if isinstance(J, SymTridiagonal):
        return ("symtri", J.n)
    if isinstance(J, BandedBlockBandedMatrix):
        return ("bbb", tuple(J.rb), tuple(J.cb), J.l, J.u, J.lam, J.mu)
    if isinstance(J, BlockSkylineMatrix):
        return ("bsky", tuple(J.rb), tuple(J.cb), J.l, J.u)
    if isinstance(J, torch.Tensor):
        return ("dense", tuple(J.shape), tuple(J.stride()))
    if isinstance(J, DenseColumnBlock):
        return ("denseblock", J.m, J.n, J.col0, J.ncols, tuple(J.slab.stride()))
    if isinstance(J, np.ndarray):
        return ("hdense", J.shape, J.strides)
    return ("obj", id(J))


def _sp_key(sp):
    if sp is None:
        return None
    if isinstance(sp, (SparseMatrixCSC, SparseMatrixCSR, BandedMatrix, Tridiagonal, BandedBlockBandedMatrix,
                       BlockSkylineMatrix) + _LA_BANDED):
        return _j_key(sp)
    if isinstance(sp, torch.Tensor):
        return ("proto", sp.data_ptr(), tuple(sp.shape), sp._version)
    a = np.asarray(sp)
    return ("protov", a.shape, a.tobytes())


# ------------------------------------------------------------------------------------------------ JacobianCache
class JacobianCache:
    """Mirror of FiniteDiff.JacobianCache (jacobians.jl:1-9) with its three constructors:

        JacobianCache(x, fdtype=..)                 allocating, square (x1=copy(x), fx=copy(x), fx1=copy(x))   :11-36
        JacobianCache(x, fx, fdtype=..)             allocating (fx1 = copy(fx))                               :50-80
        JacobianCache(x1, fx, fx1, fdtype=..)       non-allocating: ALIASES the arrays passed in              :94-128

    Fields x1, x2, fx, fx1, colorvec, sparsity keep their names.  The GPU path keeps the perturbed points and the
    stacked f! outputs in plan-owned scratch; of the cache arrays only `fx` is written (forward mode: fx = f(x),
    jacobians.jl:540-542).  x1/x2/fx1 are not touched (documented drop: in the reference they end as x (with drift),
    the last colour's mask*x, and the last colour's divided difference).
    Extra keywords (GPU path only): max_batch, scratch_bytes, no_drift, rank, world, partition.
    Plans are cached per (typeof(J), sparsity, colorvec, fdtype) and hold private compressed copies of the index arrays:
    index arrays are treated as immutable while cached (torch tensors are tracked by their version counter, large numpy
    arrays by identity + a content sample); after editing one in place call `cache.invalidate()`.
    """

    def __init__(self, x1, fx=None, fx1=None, fdtype="forward", returntype=torch.float64, *, colorvec=None,
                 sparsity=None, inplace=True, **plan_kw):
        if isinstance(fx, str):          # JacobianCache(x, "central")
            fdtype, fx = fx, None
        if isinstance(fx1, str):         # JacobianCache(x, fx, "central")
            fdtype, fx1 = fx1, None
        self.fdtype = fdtype.lstrip(":") if isinstance(fdtype, str) else fdtype
        _fdtype_code(self.fdtype)
        if returntype not in (torch.float64, float, np.float64):
            raise TypeError("only Float64 is supported by the GPU path")
        if not _is_cuda(x1):
            raise TypeError("JacobianCache needs CUDA float64 tensors (this path has no CPU implementation)")
        if _fdtype_code(self.fdtype) == L.FDB_COMPLEX:
            # complex step: x1 and fx are complex (`false .* im .* x`), fx1 === nothing  (:20-32, :60-76, :105-117)
            fx_like = x1 if fx is None else fx
            self.x1 = torch.zeros(x1.shape, dtype=torch.complex128, device=x1.device)
            self.fx = torch.zeros(fx_like.shape, dtype=torch.complex128, device=x1.device)
            self.fx1 = None
        elif fx is None and fx1 is None:
            self.x1, self.fx, self.fx1 = x1.clone(), x1.clone(), x1.clone()           # :25-33
        elif fx1 is None:
            self.x1, self.fx, self.fx1 = x1.clone(), fx.clone(), fx.clone()           # :62-76
        else:
            if fx.dtype != torch.float64 or fx1.dtype != torch.float64:              # @assert eltype :120-121
                raise AssertionError("eltype(fx) == eltype(fx1) == returntype")
            self.x1, self.fx, self.fx1 = x1, fx, fx1                                  # aliases :118-122
        self.x2 = torch.zeros_like(self.x1)                                           # :124
        n = self.x1.numel()
        self.colorvec = range(1, n + 1) if colorvec is None else colorvec             # :16
        self.sparsity = sparsity
        self._plan_kw = plan_kw
        self._plans = {}

    def plan_for(self, J, sparsity, colorvec, x_len) -> Plan:
        default_cv = isinstance(colorvec, range) and colorvec == range(1, x_len + 1)
        key = (_j_key(J), _sp_key(sparsity), None if default_cv else _index_key(colorvec), self.fdtype)
        return _cached_plan(self, key, lambda: make_plan(J, sparsity, None if default_cv else colorvec, self.fdtype, x_len,
                                                         self.x1.device, **self._plan_kw))

    def _oop_plan_for(self, kind, sparsity, colorvec, pn, m, n, device, csr=False) -> Plan:
        """The out-of-place plan (finite_difference_jacobian) for a result of `kind` with m rows and n = length(x) (csr:
        a CSR result, which a CSC sparsity gives with a CSR prototype); of the plan keywords it takes max_batch and
        scratch_bytes."""
        def create():
            suffix, args, keep = _oop_plan_route(kind, sparsity, colorvec, pn, m, n, csr)
            o = _opts(_fdtype_code(self.fdtype), _device_index(device),
                      **{k: v for k, v in self._plan_kw.items() if k in ("max_batch", "scratch_bytes")})
            with torch.cuda.device(device):
                return Plan(_new_handle(f"fdb_oop_plan_create_{suffix}", *args, C.byref(o)).value)
        key = ("oop", kind, _sp_key(sparsity) if sparsity is not None else None, _index_key(colorvec), pn, m, n)
        if csr:
            key += ("csr",)
        return _cached_plan(self, key, create)

    def invalidate(self):
        for p in self._plans.values():
            p.destroy()
        self._plans.clear()


def resize_(cache: JacobianCache, i: int):
    """resize!(cache, i)  jacobians.jl:655-661: resizes x1, fx, fx1 and resets colorvec to 1:i."""
    i = int(i)

    def rs(t):
        out = torch.zeros(i, dtype=t.dtype, device=t.device)
        k = min(i, t.numel())
        out[:k] = t.reshape(-1)[:k]
        return out

    cache.x1 = rs(cache.x1)
    cache.x2 = torch.zeros_like(cache.x1)
    cache.fx = rs(cache.fx)
    if cache.fx1 is not None:
        cache.fx1 = rs(cache.fx1)
    cache.colorvec = range(1, i + 1)
    cache.invalidate()
    return None


# ------------------------------------------------------------------------------------------------ colouring
def matrix_colors(A, device=None) -> torch.Tensor:
    """ArrayInterface.matrix_colors(A) on the device: an Int64 CUDA tensor of 1-based colours, ready to be passed as
    `colorvec`.  Tridiagonal and SymTridiagonal -> 1,2,3,...; Diagonal -> all 1; Bidiagonal -> 1,2,1,2,...;
    BandedMatrix(l,u) -> cycle 1:(l+u+1) (ArrayInterface's closed forms);
    SparseMatrixCSC -> a valid distance-2 column colouring (deterministic Jones-Plassmann, fdb_matrix_colors_csc);
    SparseMatrixCSR -> the same colouring of the same matrix (fdb_matrix_colors_csr);
    dense tensors -> 1:n (ArrayInterface: eachindex of the columns)."""
    lib = L.lib()
    if isinstance(A, Tridiagonal):
        n, l, u = A.n, 1, 1
        dev = A.buf.device if device is None else torch.device(device)
    elif isinstance(A, _LA_BANDED):
        n, l, u = A.n, A.l, A.u
        buf_dev = A.buf.device if isinstance(A.buf, torch.Tensor) and A.buf.is_cuda else torch.device("cuda")
        dev = buf_dev if device is None else torch.device(device)
    elif isinstance(A, BandedMatrix):
        n, l, u = A.n, A.l, A.u
        dev = (A.data.device if isinstance(A.data, torch.Tensor) and A.data.is_cuda else torch.device("cuda")) if device is None else torch.device(device)
    elif isinstance(A, (SparseMatrixCSC, SparseMatrixCSR)):
        dev = torch.device("cuda") if device is None else torch.device(device)
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        out = torch.zeros(max(A.n, 1), dtype=torch.int64, device=dev)
        csr = isinstance(A, SparseMatrixCSR)
        cp, k1 = _index_ptr(A.rowptr if csr else A.colptr)
        rv, k2 = _index_ptr(A.colval if csr else A.rowval)
        nc, nr = C.c_int64(), C.c_int64()
        _call(dev, (), lib.fdb_matrix_colors_csr if csr else lib.fdb_matrix_colors_csc, A.m, A.n, cp, rv, out.data_ptr(),
              C.byref(nc), C.byref(nr))
        out = out[: A.n]
        out.n_colors, out.n_rounds = nc.value, nr.value
        return out
    elif isinstance(A, (BandedBlockBandedMatrix, BlockSkylineMatrix)):
        return torch.from_numpy(A.matrix_colors()).to(torch.device("cuda") if device is None else torch.device(device))
    elif isinstance(A, torch.Tensor):
        n = A.shape[1] if A.dim() == 2 else 1
        return torch.arange(1, n + 1, dtype=torch.int64, device=A.device if A.is_cuda else (device or "cuda"))
    else:
        raise TypeError(f"matrix_colors: unsupported type {type(A)}")
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    out = torch.zeros(max(n, 1), dtype=torch.int64, device=dev)
    _call(dev, (), lib.fdb_matrix_colors_banded, n, l, u, out.data_ptr(), C.c_void_p(_stream(None, dev)))
    return out[:n]


def check_coloring(A: "SparseMatrixCSC | SparseMatrixCSR", colorvec) -> int:
    """Number of (row, colour) collisions of `colorvec` on the CSC or CSR pattern (0 = valid for the decompression)."""
    csr = isinstance(A, SparseMatrixCSR)
    cp, k1 = _index_ptr(A.rowptr if csr else A.colptr)
    rv, k2 = _index_ptr(A.colval if csr else A.rowval)
    cv, k3 = _index_ptr(colorvec)
    out = C.c_int64()
    fn = L.lib().fdb_check_coloring_csr if csr else L.lib().fdb_check_coloring_csc
    L.check(fn(A.m, A.n, cp, rv, cv, C.byref(out)))
    return out.value


# ------------------------------------------------------------------------------------------------ the public call
def _as_fn(f, m, n, device, plan_batch, complex_=False, scalar=False, **kind):
    if isinstance(f, NativeFn):
        return f.address, f.ctx_ptr, None
    w = _PyFn(f, m, n, device, bool(getattr(f, "batched", False)), complex_, scalar, **kind)
    return L.fn_address(w.cfunc), None, w


def finite_difference_jacobian_(J, f, x, cache=None, f_in=None, returntype=None, *, fdtype=None, relstep=None,
                                absstep=None, colorvec=None, sparsity=_DEFAULT, dir=True, stream=None):
    """finite_difference_jacobian!(J, f, x, cache::JacobianCache, f_in=nothing; relstep, absstep, colorvec, sparsity, dir)
    (jacobians.jl:504-514), or — when `cache` is None or an fdtype string — the cache-less form
    finite_difference_jacobian!(J, f, x, fdtype, returntype, f_in; relstep, absstep, colorvec, sparsity) (:446-455).

    J: SparseMatrixCSC | BandedMatrix | Tridiagonal | column-major dense CUDA tensor (zeros_colmajor).
    f: Python callable f(fx, x) on CUDA tensors (set f.batched=True for 2-D batches) or a NativeFn.
    x: float64 CUDA tensor (any shape; flattened like Julia's vec).  Never modified.
    Returns None.
    """
    if isinstance(cache, str) or cache is None:
        # cache-less entry :446-471
        fd = cache if isinstance(cache, str) else (fdtype or "forward")
        if isinstance(f_in, torch.dtype):
            f_in = None
        if sparsity is _DEFAULT:
            sparsity = J if _has_sparsestruct(J) else None                              # :455
        xv = x.reshape(-1)
        m = _shape_of(J)[0]
        if f_in is None and _fdtype_code(fd) == L.FDB_FORWARD:
            fx = torch.zeros_like(xv) if m == xv.numel() else torch.zeros(m, dtype=torch.float64, device=x.device)
            c = JacobianCache(xv, fx, fd)                                                # :456-463 (f(fx,x) runs inside)
            # the reference evaluates f(fx,x) here and passes cache.fx as f_in; the plan does the same evaluation
            # first thing inside fdb_jacobian (same call count, same order)
            return finite_difference_jacobian_(J, f, x, c, None, relstep=relstep, absstep=absstep,
                                               colorvec=range(1, xv.numel() + 1) if colorvec is None else colorvec,
                                               sparsity=sparsity, stream=stream)
        if f_in is None:
            c = JacobianCache(xv, fd)                                                    # :464-465
        else:
            c = JacobianCache(xv, f_in.reshape(-1), fd)                                  # :466-467
        return finite_difference_jacobian_(J, f, x, c, c.fx if f_in is not None else None, relstep=relstep,
                                           absstep=absstep,
                                           colorvec=range(1, xv.numel() + 1) if colorvec is None else colorvec,
                                           sparsity=sparsity, stream=stream)

    if not isinstance(cache, JacobianCache):
        raise TypeError("cache must be a JacobianCache, an fdtype string, or None")
    if not _is_cuda(x) or x.dtype != torch.float64:
        raise TypeError("x must be a float64 CUDA tensor: the GPU path has no CPU implementation")
    fd = _fdtype_code(cache.fdtype)
    colorvec = cache.colorvec if colorvec is None else colorvec                          # :511
    sparsity = cache.sparsity if sparsity is _DEFAULT else sparsity                 # :512
    xv = x.reshape(-1)
    if not xv.is_contiguous():
        xv = xv.contiguous()
    n = xv.numel()
    m, ncols = _shape_of(J)                                                              # :515
    if ncols != n:
        raise ValueError(f"size(J,2)={ncols} != length(x)={n}")
    plan = cache.plan_for(J, sparsity, colorvec, n)
    if isinstance(J, DenseColumnBlock) and plan.dense_range() != (J.col0, J.col0 + J.ncols):
        raise ValueError(f"DenseColumnBlock [{J.col0}, {J.col0 + J.ncols}) is not this rank's column block {plan.dense_range()}")
    jv = _j_values(J)
    if not _is_cuda(jv) or jv.dtype != torch.float64:
        raise TypeError("J's value storage must be a float64 CUDA tensor")
    if cache.fx.numel() != m:
        raise ValueError(f"length(cache.fx)={cache.fx.numel()} != size(J,1)={m} (use the 3-array constructor)")
    addr, ctx, pyfn = _as_fn(f, m, n, x.device, 1, fd == L.FDB_COMPLEX)
    stream = _stream(stream, x.device)
    if fd == L.FDB_COMPLEX:
        # jacobians.jl:623-648: one complex evaluation per colour, J = imag(f(x + im*eps*e_k))/eps, eps = eps(Float64)
        _call(x.device, [pyfn], L.lib().fdb_jacobian_complex, plan.handle, addr, ctx, xv.data_ptr(), jv.data_ptr(),
              C.c_void_p(stream))
        cache._last_plan = plan
        return None
    fin_ptr = None
    if f_in is not None and fd == L.FDB_FORWARD:
        f_in = f_in.reshape(-1)
        if not _is_cuda(f_in) or f_in.dtype != torch.float64 or f_in.numel() != m:
            raise TypeError("f_in must be a float64 CUDA tensor of length size(J,1)")
        fin_ptr = f_in.data_ptr()
    _call(x.device, [pyfn], L.lib().fdb_jacobian, plan.handle, addr, ctx, xv.data_ptr(), jv.data_ptr(), cache.fx.data_ptr(),
          fin_ptr, *_steps(relstep, absstep), float(dir), C.c_void_p(stream))
    cache._last_plan = plan
    return None


finite_difference_jacobian_b = finite_difference_jacobian_  # alias ("bang")


# ------------------------------------------------------------------------------------------------ JVP (src/jvp.jl)
class JVPCache:
    """Mirror of FiniteDiff.JVPCache{X1, FX1, fdtype} (src/jvp.jl:14-17): fields x1, fx1.

        JVPCache(x, fdtype="forward")          allocating: x1 = copy(x), fx1 = copy(x)      (:39-44)
        JVPCache(x, fx1, fdtype="forward")     non-allocating: aliases the arrays passed in (:73-80)
    """

    def __init__(self, x, fx1=None, fdtype="forward"):
        if isinstance(fx1, str):
            fdtype, fx1 = fx1, None
        self.fdtype = fdtype.lstrip(":") if isinstance(fdtype, str) else fdtype
        code = _fdtype_code(self.fdtype)
        if not _is_cuda(x):
            raise TypeError("JVPCache needs CUDA float64 tensors (this path has no CPU implementation)")
        if fx1 is None:
            self.x1, self.fx1 = x.clone(), x.clone()
        else:
            self.x1, self.fx1 = x, fx1
        self._code = code
        self._plan = None

    def plan(self, m: int, n: int) -> "Plan":
        if self._plan is None or self._plan_key != (m, n):
            if self._code == L.FDB_COMPLEX:
                # jvp.jl:248-250
                raise ValueError("finite_difference_jvp doesn't support :complex-mode finite diff")
            o = _opts(self._code, _device_index(self.x1.device))
            self._plan, self._plan_key = Plan(_new_handle("fdb_jvp_plan_create", m, n, C.byref(o)).value), (m, n)
        return self._plan


def finite_difference_jvp_(jvp, f, x, v, cache=None, f_in=None, *, relstep=None, absstep=None, dir=True, stream=None):
    """finite_difference_jvp!(jvp, f, x, v, cache::JVPCache, f_in=nothing; relstep, absstep, dir) (src/jvp.jl:238-274), or
    — when `cache` is None or an fdtype string — the cache-less form (:198-216).
    jvp[m], x[n], v[n]: float64 CUDA tensors; f(fx, x) as for the Jacobian.  Returns None."""
    if isinstance(cache, str) or cache is None:
        fd = cache if isinstance(cache, str) else "forward"
        xv = x.reshape(-1)
        if f_in is not None:
            c = JVPCache(xv.clone(), f_in.reshape(-1).clone(), fd)                      # JVPCache(x, f_in, fdtype)  :209
            return finite_difference_jvp_(jvp, f, x, v, c, c.fx1, relstep=relstep, absstep=absstep, stream=stream)
        c = JVPCache(xv, fd)                                                            # :210-215 (f(fx,x) runs inside)
        if jvp.numel() != xv.numel():
            c.fx1 = torch.zeros(jvp.numel(), dtype=torch.float64, device=x.device)
        return finite_difference_jvp_(jvp, f, x, v, c, None, relstep=relstep, absstep=absstep, stream=stream)
    if not isinstance(cache, JVPCache):
        raise TypeError("cache must be a JVPCache, an fdtype string, or None")
    for t in (jvp, x, v):
        if not _is_cuda(t) or t.dtype != torch.float64:
            raise TypeError("jvp, x, v must be float64 CUDA tensors: the GPU path has no CPU implementation")
    xv, vv, jv = x.reshape(-1), v.reshape(-1), jvp.reshape(-1)
    if not (xv.is_contiguous() and vv.is_contiguous() and jv.is_contiguous()):
        raise ValueError("jvp, x, v must be contiguous")
    n, m = xv.numel(), jv.numel()
    if vv.numel() != n:
        raise ValueError("length(v) != length(x)")
    # The device reads and writes n / m contiguous doubles from each buffer's first element: a strided view, a float32
    # or short array, or memory on another device would be read past its end or written outside the view.
    x1v, fx1v = _flat_f64(cache.x1, "cache.x1"), _flat_f64(cache.fx1, "cache.fx1")
    if x1v.numel() != n or fx1v.numel() != m:
        raise ValueError("JVPCache arrays do not match length(x) / length(jvp)")
    fin_ptr = None
    if f_in is not None and cache._code == L.FDB_FORWARD:                              # f_in is only read forward :257-258
        finv = _flat_f64(f_in, "f_in")
        if finv.numel() != m:
            raise ValueError("length(f_in) != length(jvp)")
        fin_ptr = _fx_ptr(finv)                 # an empty f_in is still given: f(fx1, x) must not run
    for t in (x1v, fx1v) + (() if fin_ptr is None else (finv,)):
        if t.device != x.device:
            raise ValueError("JVPCache arrays and f_in must be on x's device")
    plan = cache.plan(m, n)
    addr, ctx, pyfn = _as_fn(f, m, n, x.device, 1)
    _call(x.device, [pyfn], L.lib().fdb_jvp, plan.handle, addr, ctx, jv.data_ptr(), xv.data_ptr(), vv.data_ptr(),
          x1v.data_ptr(), fx1v.data_ptr(), fin_ptr, *_steps(relstep, absstep), float(dir),
          C.c_void_p(_stream(stream, x.device)))
    cache._last_plan = plan
    return None


# ------------------------------------------------------------------------------------------------ out-of-place forms
def _native_call(f: "NativeFn", fx: torch.Tensor, x: torch.Tensor, stream):
    """Evaluate a native fdb_fn once, f(fx, x), on `stream` (the cache-less out-of-place form's f(x))."""
    fn = L.FDB_FN(f.address)
    rc = fn(f.ctx_ptr, fx.data_ptr() if fx.numel() else None, x.data_ptr() if x.numel() else None, 1,
            max(fx.numel(), 1), max(x.numel(), 1), C.c_void_p(stream))
    if rc != 0:
        raise L.FdbError(L.FDB_ERR_CALLBACK, f"user f! returned {rc}")


def _oop_band(sparsity):
    """(l, u) of a band sparsity the out-of-place Jacobian takes in closed form (BandedMatrix with l, u >= 0, Diagonal,
    Bidiagonal, SymTridiagonal), else None."""
    if isinstance(sparsity, (BandedMatrix,) + _LA_BANDED) and sparsity.l >= 0 and sparsity.u >= 0:
        return int(sparsity.l), int(sparsity.u)
    return None


def _oop_block(sparsity):
    """("block_banded", (l, u, lam, mu)) or ("block_dense", (l, u)) for a block sparsity the out-of-place Jacobian takes
    in closed form (a BandedBlockBandedMatrix, BlockBandedMatrix included, or a BlockSkylineMatrix, with square blocks and
    non-negative bandwidths), else None.  Its result is sparse only."""
    if isinstance(sparsity, BandedBlockBandedMatrix) and min(sparsity.l, sparsity.u, sparsity.lam, sparsity.mu) >= 0 \
            and sparsity.rb == sparsity.cb:
        return "block_banded", (sparsity.l, sparsity.u, sparsity.lam, sparsity.mu)
    if isinstance(sparsity, BlockSkylineMatrix) and min(sparsity.l, sparsity.u) >= 0 and sparsity.rb == sparsity.cb:
        return "block_dense", (sparsity.l, sparsity.u)
    return None


def _oop_csr(sparsity, jac_prototype):
    """True when (sparsity, jac_prototype) gives a CSR result: a SparseMatrixCSR prototype with a SparseMatrixCSR or a
    SparseMatrixCSC sparsity (fdb_oop_plan_create_csr).  Every other pairing with a CSR on either side is not built."""
    return isinstance(jac_prototype, SparseMatrixCSR) and isinstance(sparsity, (SparseMatrixCSR, SparseMatrixCSC))


def _oop_kind(sparsity, jac_prototype):
    """(result kind, m, ncols) the pair (sparsity, jac_prototype) gives; m / ncols None where f and colorvec decide."""
    if isinstance(sparsity, SparseMatrixCSR) or isinstance(jac_prototype, SparseMatrixCSR):
        if not _oop_csr(sparsity, jac_prototype):
            raise TypeError(f"not built: a {type(sparsity).__name__} sparsity with a {type(jac_prototype).__name__} "
                            "jac_prototype in the out-of-place Jacobian (a SparseMatrixCSR result takes a "
                            "SparseMatrixCSR or SparseMatrixCSC sparsity and a SparseMatrixCSR jac_prototype)")
        if jac_prototype.shape != sparsity.shape:
            raise ValueError(f"jac_prototype is {jac_prototype.shape[0]}x{jac_prototype.shape[1]} but sparsity is "
                             f"{sparsity.shape[0]}x{sparsity.shape[1]}")
        return L.FDB_OOP_SPARSE, int(jac_prototype.shape[0]), int(jac_prototype.shape[1])
    block = _oop_block(sparsity) is not None and isinstance(jac_prototype, SparseMatrixCSC)
    if sparsity is not None and not isinstance(sparsity, SparseMatrixCSC) and _oop_band(sparsity) is None and not block:
        raise TypeError(f"not built: sparsity of type {type(sparsity).__name__} in the out-of-place Jacobian "
                        "(SparseMatrixCSC, BandedMatrix with l, u >= 0, Diagonal, Bidiagonal, SymTridiagonal or None; "
                        "BandedBlockBandedMatrix and BlockSkylineMatrix with square blocks and a SparseMatrixCSC "
                        "jac_prototype)")
    if jac_prototype is not None:
        if isinstance(jac_prototype, SparseMatrixCSC):
            pm, pn = jac_prototype.shape
        elif isinstance(jac_prototype, torch.Tensor) and jac_prototype.dim() == 2 and \
                (jac_prototype.shape[0] <= 1 or jac_prototype.stride(0) == 1):
            pm, pn = jac_prototype.shape
        else:
            raise TypeError(f"not built: jac_prototype of type {type(jac_prototype).__name__} in the out-of-place "
                            "Jacobian (a dense column-major tensor, a SparseMatrixCSC or None)")
        if sparsity is not None and (pm, pn) != sparsity.shape:
            raise ValueError(f"jac_prototype is {pm}x{pn} but sparsity is {sparsity.shape[0]}x{sparsity.shape[1]}")
        kind = L.FDB_OOP_SPARSE if isinstance(jac_prototype, SparseMatrixCSC) else L.FDB_OOP_DENSE
        return kind, int(pm), int(pn)
    if sparsity is not None:
        return L.FDB_OOP_DENSE, sparsity.shape[0], sparsity.shape[1]
    return L.FDB_OOP_RAW, None, None


def _csr_of_csc(A):
    """(rowptr, colval), Int64 and 1-based on the host: the CSR of a CSC pattern's entry set (scipy's O(nnz) transpose;
    every stored entry kept, rows in order and columns ascending within a row)."""
    import scipy.sparse as sps
    cp = np.asarray(A.colptr.cpu() if isinstance(A.colptr, torch.Tensor) else A.colptr, dtype=np.int64) - 1
    nnz = int(cp[-1]) if len(cp) else 0
    rv = np.asarray(A.rowval.cpu() if isinstance(A.rowval, torch.Tensor) else A.rowval, dtype=np.int64)[:nnz] - 1
    T = sps.csc_matrix((np.ones(nnz, dtype=np.int8), rv, cp), shape=(A.m, A.n)).tocsr()
    return T.indptr.astype(np.int64) + 1, T.indices.astype(np.int64) + 1


def _oop_plan_route(kind, sparsity, colorvec, pn, m, n, csr=False):
    """(suffix, args, keep) of the out-of-place plan for a result of `kind` with m rows and n = length(x): it is made by
    fdb_oop_plan_create_<suffix>(&h, *args, &opts) (or fdb_group_create_oop_<suffix>(&h, n_devices, devices, *args,
    &opts)), and `keep` holds the host arrays the pointers in args point into.  csr: a CSR result (_oop_csr), whose plan
    takes the CSR of the sparsity's entry set."""
    cvp, k0 = _index_ptr(None if _is_identity_colorvec(colorvec, n) else colorvec)
    if csr:
        rowptr, colval = (sparsity.rowptr, sparsity.colval) if isinstance(sparsity, SparseMatrixCSR) else \
            _csr_of_csc(sparsity)
        rp, k1 = _index_ptr(rowptr)
        cv, k2 = _index_ptr(colval)
        return "csr", (m, n, rp, cv, cvp, kind, max(m, 1)), [k0, k1, k2]
    band = _oop_band(sparsity)
    if band is not None:
        return "banded", (m, n, band[0], band[1], cvp, kind, max(m, 1)), [k0]
    block = _oop_block(sparsity)
    if block is not None:
        suffix, bw = block
        blocks = np.asarray(sparsity.rb, dtype=np.int64)
        return suffix, (len(blocks), blocks.ctypes.data if len(blocks) else None, *bw, cvp, kind, max(m, 1)), [k0, blocks]
    if sparsity is not None:
        cp, k1 = _index_ptr(sparsity.colptr)
        rv, k2 = _index_ptr(sparsity.rowval)
        return "csc", (m, n, cp, rv, cvp, kind, max(m, 1)), [k0, k1, k2]
    return "dense", (m, n, cvp, pn or 0, kind, max(m, 1)), [k0]


def _oop_rows(f, x, fd, f_in, m_default, sparsity, pm, n):
    """(f_in, m): the rows of an out-of-place result.  In forward mode a Python f is evaluated at x first — vecfx = _vec(f(x))
    (:299-300), the same call at the same point, still before the colours — and handed on as f_in, so the row count is f's
    own; otherwise those of f_in, else m_default.  A sparsity fixes them, and a prototype must agree."""
    if f_in is None and fd == L.FDB_FORWARD and not isinstance(f, NativeFn):
        f_in = _oop_result(f(x), (-1,))
    if f_in is not None:
        if f_in.is_complex():
            raise TypeError("not built: complex-valued f_in (complex-valued results of the out-of-place path)")
        f_in = f_in.reshape(-1)
    m = f_in.numel() if f_in is not None else m_default
    if sparsity is not None:
        m, sn = sparsity.shape
        if sn != n:
            raise ValueError(f"size(sparsity, 2) = {sn} != length(x) = {n}")
    elif pm is not None and pm != m:
        raise TypeError(f"not built: a {pm}-row jac_prototype for an f with {m} values")
    return f_in, m


def _oop_fin_ptr(f_in, fd, m):
    """Device pointer of f_in as the ABI reads it (forward mode only, :297-298), or None."""
    if f_in is None or fd != L.FDB_FORWARD:
        return None
    finv = _flat_f64(f_in, "f_in")
    if finv.numel() != m:
        raise ValueError("length(f_in) != the rows of the result")
    return _fx_ptr(finv)


class _OopOutput:
    """Device storage of an out-of-place result and the fdb_oop_out naming it.  ncols: the prototype's columns, else
    the quotient columns C = maximum(colorvec) of the whole result (dense branch); a sparse result holds up to m*C
    candidates without a sparsity and nnz(sparsity) = n_entries with one.  csr: a CSR result, whose pointer holds the
    m + 1 row starts and whose stored indices are columns."""

    def __init__(self, kind, sparsity, pn, m, C, n_entries, dev, csr=False):
        self.kind, self.m, self.dev, self.csr = kind, m, dev, csr
        self.ncols = pn if pn is not None else C
        self.out = L.OopOut()
        self.dense = None
        if kind == L.FDB_OOP_SPARSE:
            self.cap = m * C if sparsity is None else n_entries
            self.colptr = torch.empty((m if csr else self.ncols) + 1, dtype=torch.int64, device=dev)
            self.rowval = torch.empty(max(self.cap, 1), dtype=torch.int64, device=dev)
            self.nzval = torch.empty(max(self.cap, 1), dtype=torch.float64, device=dev)
            self.nnz = torch.empty(1, dtype=torch.int64, device=dev)
            o = self.out
            o.colptr, o.rowval, o.nzval, o.cap, o.nnz = (self.colptr.data_ptr(), self.rowval.data_ptr(),
                                                         self.nzval.data_ptr(), self.cap, self.nnz.data_ptr())
        else:
            self.dense = torch.empty((self.ncols, m), dtype=torch.float64, device=dev).t()  # column-major, ldJ = m
            self.out.J = self.dense.data_ptr() if self.dense.numel() else _fx_ptr(self.dense)  # m = 0: nothing is written

    def result(self, stream):
        """The dense tensor, or the SparseMatrixCSC (SparseMatrixCSR) sized to the kept entries (reading that count is the
        one host sync; when most candidates were dropped its stored indices and nzval are copied into storage of their
        own size)."""
        if self.kind != L.FDB_OOP_SPARSE:
            return self.dense
        _call(self.dev, (), L.lib().fdb_stream_sync, C.c_void_p(stream))
        nnz = int(self.nnz.item())
        rowval, nzval = self.rowval[:nnz], self.nzval[:nnz]
        if 2 * nnz < self.cap:
            rowval, nzval = rowval.clone(), nzval.clone()
        if self.csr:
            return SparseMatrixCSR(self.m, self.ncols, self.colptr, rowval, nzval)
        return SparseMatrixCSC(self.m, self.ncols, self.colptr, rowval, nzval)


def finite_difference_jacobian(f, x, cache=None, f_in=None, returntype=None, *, fdtype=None, relstep=None, absstep=None,
                               colorvec=None, sparsity=_DEFAULT, jac_prototype=None, dir=True, stream=None):
    """J = finite_difference_jacobian(f, x, cache::JacobianCache, f_in=nothing; relstep, absstep, colorvec, sparsity,
    jac_prototype, dir) (jacobians.jl:277-429), or - when `cache` is None or an fdtype string - the cache-less form
    (:240-259), which evaluates f(x) once and passes it on as f_in.

    f: an out-of-place Python callable, f(x) -> CUDA tensor of m values (f.batched = True: (batch, n) -> (batch, m);
       complex step: complex128 in and out), or a NativeFn (the in-place fdb_fn; the trampoline is not needed).
    x: float64 CUDA tensor, never modified; cache.x1 receives a copy of it (:293-295).
    The result follows (sparsity, jac_prototype) as the reference's J + Ji does:
        None / None                 dense m x maximum(colorvec) column-major tensor of the raw quotients
        None / dense tensor         dense, column i = 0.0 + dx_i, the other columns +0.0
        None / SparseMatrixCSC      SparseMatrixCSC holding the nonzero entries of each dx_i in column i
        CSC / None or dense         dense size(sparsity): structural slots 0.0 + dx, +0.0 elsewhere (an invalid colouring
                                    raises, as _make_Ji throws)
        CSC / SparseMatrixCSC       SparseMatrixCSC with the structural entries whose value is not +-0.0 (NaN kept)
        band / as for CSC           the same results for a BandedMatrix (l, u >= 0), Diagonal, Bidiagonal or SymTridiagonal
                                    sparsity, whose structural entries are the in-matrix band (l, u): a closed-form plan
                                    (fdb_oop_plan_create_banded) builds no entry list
        block / SparseMatrixCSC     the sparse result for a BandedBlockBandedMatrix (BlockBandedMatrix included) or
                                    BlockSkylineMatrix sparsity with square blocks, whose structural entries are those of
                                    findstructralnz: closed-form plans (fdb_oop_plan_create_block_banded / _block_dense)
                                    build no entry list; a dense result of a block sparsity is not built
        CSR / SparseMatrixCSR       SparseMatrixCSR (fdb_oop_plan_create_csr): the sparsity's stored entries whose value
                                    is not +-0.0 (NaN kept), rows in order and each row in the sparsity's own storage
                                    order; the values are the CSC route's bit for bit
        CSC / SparseMatrixCSR       the same, for the CSR of the CSC's entry set (built on the host in O(nnz))
    A sparse result is sized to the kept entries: reading that count is the call's one host synchronisation (when most
    candidates were dropped its rowval / nzval are copied into storage of their own size).  Other sparsity / prototype
    types (a CSR sparsity with any other prototype, a CSR prototype with any other sparsity) and complex-valued results
    raise TypeError (not built).
    Rows of the result: size(sparsity, 1) or size(jac_prototype, 1) when given; else those of f(x) — forward mode with a
    Python f evaluates it first, as the reference does (:299-300), and passes it on as f_in — or of f_in; else length of
    cache.fx (central and complex mode, and a NativeFn, whose output length the mirror cannot see before the device calls
    it: build the cache as JacobianCache(x, fx) for m != n).  The cache-less form with a NativeFn sizes f(x) the same way,
    from sparsity / prototype or length(x)."""
    if cache is None or isinstance(cache, str):
        fd = cache if isinstance(cache, str) else (fdtype or "forward")
        if not _is_cuda(x) or x.dtype != torch.float64:
            raise TypeError("x must be a float64 CUDA tensor: the GPU path has no CPU implementation")
        xv = x.reshape(-1)
        if f_in is None:                                                                  # :250-251
            stream = _stream(stream, x.device)
            if isinstance(f, NativeFn):
                sp = None if sparsity is _DEFAULT else sparsity
                m = sp.shape[0] if isinstance(sp, (SparseMatrixCSC, SparseMatrixCSR)) or _oop_band(sp) is not None or \
                    _oop_block(sp) is not None else (
                    jac_prototype.shape[0] if jac_prototype is not None else xv.numel())
                xin = xv.to(torch.complex128) if _fdtype_code(fd) == L.FDB_COMPLEX else xv
                fx = torch.empty(m, dtype=xin.dtype, device=x.device)
                with torch.cuda.device(x.device):
                    _native_call(f, fx, xin.contiguous(), stream)
            else:
                fx = f(x)
                if not isinstance(fx, torch.Tensor) or not fx.is_cuda:
                    raise TypeError("an out-of-place f must return a CUDA tensor")
        else:
            fx = f_in                                                                     # :252-253
        if fx.is_complex() and _fdtype_code(fd) != L.FDB_COMPLEX:
            raise TypeError("not built: f returns a complex array (complex-valued results of the out-of-place path)")
        c = JacobianCache(xv, fx.reshape(-1).real.to(torch.float64) if fx.is_complex() else fx.reshape(-1), fd)
        return finite_difference_jacobian(f, x, c, fx.real if fx.is_complex() else fx, relstep=relstep,
                                          absstep=absstep, colorvec=range(1, xv.numel() + 1) if colorvec is None else colorvec,
                                          sparsity=None if sparsity is _DEFAULT else sparsity, jac_prototype=jac_prototype,
                                          dir=dir, stream=stream)                         # :255-258
    if not isinstance(cache, JacobianCache):
        raise TypeError("cache must be a JacobianCache, an fdtype string, or None")
    if not _is_cuda(x) or x.dtype != torch.float64:
        raise TypeError("x must be a float64 CUDA tensor: the GPU path has no CPU implementation")
    fd = _fdtype_code(cache.fdtype)
    colorvec = cache.colorvec if colorvec is None else colorvec                           # :284
    sparsity = cache.sparsity if sparsity is _DEFAULT else sparsity                       # :285
    kind, pm, pn = _oop_kind(sparsity, jac_prototype)
    csr = _oop_csr(sparsity, jac_prototype)
    xv = x.reshape(-1)
    if not xv.is_contiguous():
        xv = xv.contiguous()
    n = xv.numel()
    if cache.x1 is not x:                                                                 # :293-295
        cache.x1.reshape(-1).copy_(xv)
    f_in, m = _oop_rows(f, x, fd, f_in, cache.fx.numel(), sparsity, pm, n)
    dev = x.device
    plan = cache._oop_plan_for(kind, sparsity, colorvec, pn, m, n, dev, csr)
    res = _OopOutput(kind, sparsity, pn, m, plan.dense_range()[1], plan.info()["n_entries"], dev, csr)
    addr, ctx, pyfn = _as_fn(f, m, n, dev, 1, fd == L.FDB_COMPLEX, oop=True)
    stream = _stream(stream, dev)
    fin_ptr = _oop_fin_ptr(f_in, fd, m)
    if fd == L.FDB_COMPLEX:
        _call(dev, [pyfn], L.lib().fdb_jacobian_oop_complex, plan.handle, addr, ctx, xv.data_ptr(), C.byref(res.out),
              C.c_void_p(stream))
    else:
        _call(dev, [pyfn], L.lib().fdb_jacobian_oop, plan.handle, addr, ctx, xv.data_ptr(), C.byref(res.out), None, fin_ptr,
              *_steps(relstep, absstep), float(dir), C.c_void_p(stream))
    cache._last_plan = plan
    return res.result(stream)


def finite_difference_jvp(f, x, v, cache=None, f_in=None, *, relstep=None, absstep=None, dir=True, stream=None):
    """jvp = finite_difference_jvp(f, x, v, cache::JVPCache, f_in=nothing; relstep, absstep, dir) (src/jvp.jl:159-189), or -
    when `cache` is None or an fdtype string - the cache-less form (:133-146), which evaluates f(x) once and passes it on.
    f is out of place as for finite_difference_jacobian.  Central mode evaluates f(x + eps v) before f(x - eps v).  Returns
    a new float64 CUDA tensor of m values; the cache arrays are not written (x1 and fx1 are fresh arrays in the reference).
    m is the length of f(x) in forward mode with a Python f (evaluated first, jvp.jl:175) or of f_in; else length of
    cache.fx1 (central mode, a NativeFn: build the cache as JVPCache(x, fx1) for m != n)."""
    if cache is None or isinstance(cache, str):
        fd = cache if isinstance(cache, str) else "forward"
        if f_in is None:
            if isinstance(f, NativeFn):
                fx = torch.empty(x.numel(), dtype=torch.float64, device=x.device)
                with torch.cuda.device(x.device):
                    _native_call(f, fx, x.reshape(-1).contiguous(), _stream(stream, x.device))
            else:
                fx = f(x)                                                                  # :139-140
        else:
            fx = f_in
        if not isinstance(fx, torch.Tensor) or not fx.is_cuda:
            raise TypeError("an out-of-place f must return a CUDA tensor")
        if fx.is_complex():
            raise TypeError("not built: f returns a complex array (complex-valued results of the out-of-place path)")
        c = JVPCache(x.reshape(-1), fx.reshape(-1), fd)                                   # :144
        return finite_difference_jvp(f, x, v, c, fx, relstep=relstep, absstep=absstep, dir=dir, stream=stream)
    if not isinstance(cache, JVPCache):
        raise TypeError("cache must be a JVPCache, an fdtype string, or None")
    for t in (x, v):
        if not _is_cuda(t) or t.dtype != torch.float64:
            raise TypeError("x, v must be float64 CUDA tensors: the GPU path has no CPU implementation")
    xv, vv = x.reshape(-1).contiguous(), v.reshape(-1).contiguous()
    n = xv.numel()
    if vv.numel() != n:
        raise ValueError("length(v) != length(x)")
    fin_ptr = finv = None
    if f_in is None and cache._code == L.FDB_FORWARD and not isinstance(f, NativeFn):
        f_in = _oop_result(f(x), (-1,))                                                   # fx = f(x)  :175
    if f_in is not None:
        if f_in.is_complex():
            raise TypeError("not built: complex-valued f_in (complex-valued results of the out-of-place path)")
        finv = _flat_f64(f_in, "f_in")
        m = finv.numel()
        if cache._code == L.FDB_FORWARD:                                                  # read forward only :175
            fin_ptr = _fx_ptr(finv)
    else:
        m = cache.fx1.numel()
    plan = cache.plan(m, n)
    jvp = torch.empty(m, dtype=torch.float64, device=x.device)
    x1 = torch.empty(n, dtype=torch.float64, device=x.device)
    fx1 = torch.empty(m, dtype=torch.float64, device=x.device)
    addr, ctx, pyfn = _as_fn(f, m, n, x.device, 1, oop=True)
    _call(x.device, [pyfn], L.lib().fdb_jvp_oop, plan.handle, addr, ctx, _fx_ptr(jvp), xv.data_ptr() if n else None,
          vv.data_ptr() if n else None, _fx_ptr(x1), _fx_ptr(fx1), fin_ptr, *_steps(relstep, absstep), float(dir),
          C.c_void_p(_stream(stream, x.device)))
    cache._last_plan = plan
    return jvp


def _shape_of(J):
    if isinstance(J, (SparseMatrixCSC, SparseMatrixCSR, BandedMatrix, Tridiagonal, BandedBlockBandedMatrix, BlockSkylineMatrix,
                      DenseColumnBlock)
                  + _LA_BANDED):
        return J.shape
    if isinstance(J, torch.Tensor):
        if J.dim() == 1:
            return (J.shape[0], 1)
        return tuple(J.shape)
    raise TypeError(f"unsupported J type {type(J)}")


# ------------------------------------------------------------------------------------------------ Hessian (src/hessians.jl)
def _hessian_fdtype_code(fdtype) -> int:
    """The Hessian's fdtype: "hcentral" (FDB_HCENTRAL); the Jacobian's codes pass through so that the plan rejects them
    the way the reference's @assert does (hessians.jl:206)."""
    if isinstance(fdtype, str) and fdtype.lstrip(":") == "hcentral":
        return L.FDB_HCENTRAL
    if fdtype == L.FDB_HCENTRAL:
        return L.FDB_HCENTRAL
    return _fdtype_code(fdtype)


def _scalar_x(x, what="x"):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise TypeError(f"{what} must be a float64 CUDA tensor: the GPU path has no CPU implementation")
    if x.dtype != torch.float64:
        raise TypeError(f"{what} must be float64 (complex-valued x is not supported)")
    xv = x.reshape(-1)
    return xv if xv.is_contiguous() else xv.contiguous()


class HessianCache:
    """Mirror of FiniteDiff.HessianCache (hessians.jl:1-9, :60-80):

        HessianCache(x, fdtype="hcentral")                   allocating: xpp, xpm, xmp, xmm = copies of x
        HessianCache(xpp, xpm, xmp, xmm, fdtype="hcentral")  non-allocating: aliases the arrays passed in

    The cache arrays are scratch (the reference copies x into them before use, :213-216): a cache built from another x
    changes nothing (issue #185, finitedifftests.jl:608-614).  The GPU path keeps its points in plan-owned memory and
    does not touch them.  Extra keywords (GPU path only): max_batch, scratch_bytes, use_graph, and rank / world: the
    plan then evaluates f(x) and the points of rank's share of the i-blocks only and writes only the entries it owns
    (include/fdjac_b200.h, fdb_hessian_plan_create; distributed.GroupHessian drives all ranks from one process)."""

    def __init__(self, *arrays, fdtype="hcentral", **plan_kw):
        if len(arrays) == 2 and not isinstance(arrays[1], torch.Tensor):     # HessianCache(x, fdtype)
            arrays, fdtype = arrays[:1], arrays[1]
        elif len(arrays) == 5:                                                # HessianCache(xpp, xpm, xmp, xmm, fdtype)
            arrays, fdtype = arrays[:4], arrays[4]
        if len(arrays) == 1:
            x = arrays[0]
            if not _is_cuda(x):
                raise TypeError("HessianCache needs CUDA float64 tensors (this path has no CPU implementation)")
            self.xpp, self.xpm, self.xmp, self.xmm = (x.clone() for _ in range(4))
        elif len(arrays) == 4:
            self.xpp, self.xpm, self.xmp, self.xmm = arrays
        else:
            raise TypeError("HessianCache(x) or HessianCache(xpp, xpm, xmp, xmm)")
        self.fdtype = fdtype.lstrip(":") if isinstance(fdtype, str) else fdtype
        self._plan_kw = plan_kw
        self._plans = {}

    def plan_for(self, n: int, ldH: int, device) -> Plan:
        def create():
            o = _opts(_hessian_fdtype_code(self.fdtype), _device_index(device), **self._plan_kw)
            return Plan(_new_handle("fdb_hessian_plan_create", n, ldH, C.byref(o)).value)
        return _cached_plan(self, (n, ldH, str(device)), create)


def _colmajor_square(H, n):
    if not isinstance(H, torch.Tensor) or not H.is_cuda or H.dtype != torch.float64:
        raise TypeError("H must be a float64 CUDA tensor")
    if H.dim() != 2 or tuple(H.shape) != (n, n):
        raise ValueError(f"H must be {n} x {n}")
    if n > 1 and H.stride(0) != 1:
        raise ValueError("H must be column-major (Julia Matrix layout): use zeros_colmajor(n, n) or X.t()")
    return max(int(H.stride(1)) if n > 1 else n, n, 1)


def finite_difference_hessian_(H, f, x, cache=None, *, relstep=None, absstep=None, fx=None, stream=None):
    """finite_difference_hessian!(H, f, x, cache::HessianCache; relstep, absstep) (hessians.jl:202-292), or — when
    `cache` is None or an fdtype string — the cache-less form (:181-189).

    H: column-major float64 CUDA tensor (n, n), e.g. zeros_colmajor(n, n); both triangles are written (copytri!, :291).
    f: Python callable f(x) -> scalar (a 0-d CUDA tensor needs no host sync; set f.batched=True to receive a (batch, n)
       tensor and return (batch,) values) or a NativeFn (batched fdb_fn with m = 1).
    x: float64 CUDA tensor, never modified.  fx: optional 1-element float64 CUDA tensor that receives f(x).
    Returns None."""
    if cache is None or isinstance(cache, str):
        cache = HessianCache(x, fdtype=cache or "hcentral")
    if not isinstance(cache, HessianCache):
        raise TypeError("cache must be a HessianCache, an fdtype string, or None")
    xv = _scalar_x(x)
    n = xv.numel()
    ldH = _colmajor_square(H, n)
    plan = cache.plan_for(n, ldH, xv.device)
    addr, ctx, pyfn = _as_fn(f, 1, n, xv.device, 1, scalar=True)
    fx_ptr = None
    if fx is not None:
        if not _is_cuda(fx) or fx.dtype != torch.float64 or fx.numel() != 1:
            raise TypeError("fx must be a 1-element float64 CUDA tensor")
        fx_ptr = fx.data_ptr()
    _call(xv.device, [pyfn], L.lib().fdb_hessian, plan.handle, addr, ctx, xv.data_ptr(), H.data_ptr() if n > 0 else None,
          fx_ptr, *_steps(relstep, absstep), C.c_void_p(_stream(stream, xv.device)))
    cache._last_plan = plan
    return None


def finite_difference_hessian(f, x, cache=None, *, relstep=None, absstep=None, stream=None):
    """finite_difference_hessian(f, x[, cache]; relstep, absstep) (hessians.jl:140-167): a new column-major n x n H with
    both triangles filled (the reference returns Symmetric(H), whose entries are the same)."""
    n = x.numel()
    H = zeros_colmajor(n, n, device=x.device)
    finite_difference_hessian_(H, f, x, cache, relstep=relstep, absstep=absstep, stream=stream)
    return H


# ------------------------------------------------------------------------------------------------ gradient (src/gradients.jl)
def _is_number(x) -> bool:
    """x is a scalar input in the reference's sense (x::Number): a Python / numpy number.  (A tensor t is passed to a
    cache built for the scalar -> vector case.)"""
    return isinstance(x, numbers.Number)


class GradientCache:
    """Mirror of FiniteDiff.GradientCache (gradients.jl:1-7) on real Float64 arrays:

        GradientCache(df, x, fdtype="central", returntype=float64)     allocating, fx = nothing   (:19-62)
        GradientCache(fx, c1, c2, c3, fdtype="central", returntype)    non-allocating             (:104-123)

    x an array: the vector -> scalar gradient.  x a number: the scalar -> vector gradient of an in-place
    f(fx, t) (:50-59: c1, c2 = zero(df), complex mode c1 = complex zero(df), c3 = x); the non-allocating form is scalar
    -> vector when c3 is a number.  Its fx, when given, is the m values f(x) and is used in forward mode (:501-502).

    A gradient is the dense column branch of the Jacobian with m = 1 (gradients.jl:408-468 against jacobians.jl:548-557,
    590-598, 625-631): the same steps, points, quotients and call order.  The GPU path therefore runs a dense Jacobian
    plan (m = 1, ldJ = 1) with df as J; a non-None fx (a number or a 1-element CUDA tensor) is used as f(x) in forward
    mode, as :410 does.  c1..c3 are scratch.  Extra keywords (GPU path only): max_batch, scratch_bytes, use_graph."""

    def __init__(self, *arrays, fdtype="central", returntype=torch.float64, **plan_kw):
        arrays = list(arrays)
        if arrays and isinstance(arrays[-1], str):
            fdtype = arrays.pop()
        self.scalar_x = False
        if len(arrays) == 2:
            df, x = arrays
            if _is_number(x):
                # the scalar -> vector case (:50-59)
                _real_input(x)
                if not isinstance(df, torch.Tensor) or not df.is_cuda:
                    raise TypeError("df must be a float64 CUDA tensor: the GPU path has no CPU implementation")
                if df.is_complex() or df.dtype != torch.float64:
                    raise TypeError("df must be real Float64: complex-valued gradients are not supported")
                self.scalar_x = True
                complex_mode = isinstance(fdtype, str) and fdtype.lstrip(":") == "complex" or fdtype == L.FDB_COMPLEX
                if complex_mode:
                    self.fx, self.c1, self.c2 = None, torch.zeros(df.shape, dtype=torch.complex128, device=df.device), None
                else:
                    self.fx, self.c1, self.c2 = None, torch.zeros_like(df), torch.zeros_like(df)
                self.c3 = x
            else:
                for t, name in ((df, "df"), (x, "x")):
                    if not isinstance(t, torch.Tensor):
                        raise TypeError(f"{name} must be a CUDA tensor or x a number")
                    if t.is_complex():
                        raise TypeError(f"{name} must be real Float64: complex-valued gradients are not supported")
                self.fx, self.c1, self.c2, self.c3 = None, None, None, torch.zeros_like(x)
        elif len(arrays) == 4:
            self.fx, self.c1, self.c2, self.c3 = arrays
            self.scalar_x = _is_number(self.c3)
        else:
            raise TypeError("GradientCache(df, x[, fdtype]) or GradientCache(fx, c1, c2, c3[, fdtype])")
        if returntype not in (torch.float64, float, np.float64):
            raise TypeError("only Float64 is supported by the GPU path")
        self.fdtype = fdtype.lstrip(":") if isinstance(fdtype, str) else fdtype
        _fdtype_code(self.fdtype)
        self._plan_kw = plan_kw
        self._plans = {}

    def _plan(self, creator, device, *args) -> Plan:
        o = _opts(_fdtype_code(self.fdtype), _device_index(device), **self._plan_kw)
        return Plan(_new_handle(creator, *args, C.byref(o)).value)

    def plan_for(self, n: int, device) -> Plan:
        return _cached_plan(self, (n, str(device)), lambda: self._plan("fdb_plan_create_dense", device, 1, n, 1))

    def scalar_plan_for(self, m: int, device) -> Plan:
        return _cached_plan(self, ("scalar", m, str(device)),
                            lambda: self._plan("fdb_scalar_gradient_plan_create", device, m))


def finite_difference_gradient_(df, f, x, cache=None, *, relstep=None, absstep=None, dir=True, stream=None):
    """finite_difference_gradient!(df, f, x, cache::GradientCache; relstep, absstep, dir) (gradients.jl:390-473), or —
    when `cache` is None or an fdtype string — the cache-less form (:220-248).

    df, x: float64 CUDA vectors of length n (complex arrays are rejected with TypeError).
    f: Python callable f(x) -> scalar as for finite_difference_hessian_ (complex step: f receives complex128 x and
       returns a complex scalar), or a NativeFn (fdb_fn with m = 1; fdb_fn_c for complex).

    Scalar -> vector (gradients.jl:477-533): x a number (or, with a scalar -> vector cache, a 1-element
    float64 CUDA tensor: the device slot is read by the call, so a captured graph follows t written in place); df the m
    outputs.  f: in-place f(fx, t) with fx a CUDA row of m values and t a 0-d CUDA tensor (float64, complex128 in complex
    mode), or a NativeFn (fdb_fn with n = 1 and m outputs; fdb_fn_c for complex).  A number t is staged into one
    cache-owned device slot on the call's stream.  Returns None."""
    if cache is None or isinstance(cache, str):
        cache = GradientCache(df, x, cache or "central")
    if not isinstance(cache, GradientCache):
        raise TypeError("cache must be a GradientCache, an fdtype string, or None")
    if cache.scalar_x or _is_number(x):
        return _scalar_gradient_(df, f, x, cache, relstep, absstep, dir, stream)
    if not isinstance(x, torch.Tensor) or not isinstance(df, torch.Tensor):
        raise TypeError("x and df must be CUDA tensors (the scalar -> vector form is not supported)")
    xv = _scalar_x(x)
    dv = _scalar_x(df, "df")
    n = xv.numel()
    if dv.numel() != n:
        raise ValueError(f"length(df)={dv.numel()} != length(x)={n}")
    if df.reshape(-1).data_ptr() != dv.data_ptr():
        raise ValueError("df must be contiguous")
    fd = _fdtype_code(cache.fdtype)
    plan = cache.plan_for(n, xv.device)
    addr, ctx, pyfn = _as_fn(f, 1, n, xv.device, 1, fd == L.FDB_COMPLEX, scalar=True)
    stream = _stream(stream, xv.device)
    if fd == L.FDB_COMPLEX:                                                  # :458-469
        _call(xv.device, [pyfn], L.lib().fdb_jacobian_complex, plan.handle, addr, ctx, xv.data_ptr(), dv.data_ptr(),
              C.c_void_p(stream))
    else:
        fin = None
        if fd == L.FDB_FORWARD and cache.fx is not None:                    # fx0 = fx !== nothing ? fx : f(x)   :410
            if isinstance(cache.fx, torch.Tensor):
                fin = cache.fx
                if not fin.is_cuda or fin.dtype != torch.float64 or fin.numel() != 1:
                    raise TypeError("cache.fx must be a number or a 1-element float64 CUDA tensor")
            else:
                fin = _device_slot(cache, "_fin", xv.device, stream, cache.fx)
        # d_fx = NULL: f(x) goes to the plan's own buffer (cache.fx is an input here, never written)
        _call(xv.device, [pyfn], L.lib().fdb_jacobian, plan.handle, addr, ctx, xv.data_ptr(), dv.data_ptr(), None,
              None if fin is None else fin.data_ptr(), *_steps(relstep, absstep), float(dir), C.c_void_p(stream))
    cache._last_plan = plan
    return None


def finite_difference_gradient(f, x, cache=None, *, relstep=None, absstep=None, dir=True, stream=None, fx=None, c1=None,
                               c2=None):
    """finite_difference_gradient(f, x[, cache | fdtype]; relstep, absstep, dir) (gradients.jl:168-218, :250-300): a new
    float64 CUDA vector df.

    Scalar x (a number, or a 1-element tensor with a scalar -> vector cache): the scalar -> vector gradient of an in-place f(fx, t).  With a cache, df has
    the cache's m outputs.  Cache-less, one of fx, c1, c2 (CUDA tensors of m values) must be given to size df (:185-195);
    as in the reference it only sizes df — the cache is built without it, so forward mode still evaluates f(x)."""
    if (isinstance(cache, GradientCache) and cache.scalar_x) or _is_number(x):
        if isinstance(cache, GradientCache):
            proto = cache.c1 if isinstance(cache.c1, torch.Tensor) else cache.fx
            if not isinstance(proto, torch.Tensor):
                raise TypeError("a scalar -> vector GradientCache needs c1 or fx as a CUDA tensor to size df")
        else:
            proto = next((a for a in (c1, fx, c2) if a is not None), None)      # :188-194
            if proto is None:                                                  # :186
                raise TypeError("In the scalar->vector in-place map case, at least one of fx, c1 or c2 must be provided, "
                                "otherwise we cannot infer the return size.")
            if not isinstance(proto, torch.Tensor) or not proto.is_cuda:
                raise TypeError("fx / c1 / c2 must be CUDA tensors: the GPU path has no CPU implementation")
        df = torch.zeros(proto.numel(), dtype=torch.float64, device=proto.device)
        finite_difference_gradient_(df, f, x, cache, relstep=relstep, absstep=absstep, dir=dir, stream=stream)
        return df
    if not isinstance(x, torch.Tensor):
        raise TypeError("x must be a CUDA tensor or a real number")
    df = torch.zeros(x.numel(), dtype=torch.float64, device=x.device)
    finite_difference_gradient_(df, f, x, cache, relstep=relstep, absstep=absstep, dir=dir, stream=stream)
    return df


def _real_input(x):
    if isinstance(x, torch.Tensor):
        if x.is_complex() or x.dtype != torch.float64:
            raise TypeError("x must be real Float64: complex-valued x is not supported")
        if not x.is_cuda:
            raise TypeError("x must be a CUDA tensor or a number: the GPU path has no CPU implementation")
    elif isinstance(x, complex) or not isinstance(x, numbers.Real):
        raise TypeError("x must be a real number: complex-valued x is not supported")


def _flat_f64(t, what):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError(f"{what} must be a float64 CUDA tensor: the GPU path has no CPU implementation")
    if t.is_complex() or t.dtype != torch.float64:
        raise TypeError(f"{what} must be real Float64 (complex-valued arrays are not supported)")
    if not t.is_contiguous():
        raise ValueError(f"{what} must be contiguous")
    return t.reshape(-1)


_SLOTS = {}


def _fx_ptr(fxv):
    """Device pointer of a given cache.fx.  An empty one has no storage (data_ptr 0, which the ABI reads as "not given"),
    so it is passed as a valid one-element slot: nothing is read from it, and f(x) is not evaluated."""
    if fxv.numel():
        return fxv.data_ptr()
    slot = _SLOTS.get(fxv.device)
    if slot is None:
        slot = _SLOTS[fxv.device] = torch.zeros(1, dtype=torch.float64, device=fxv.device)
    return slot.data_ptr()


def _scalar_gradient_(df, f, x, cache, relstep, absstep, dir, stream):
    """finite_difference_gradient!(df, f, x::Number, cache) (gradients.jl:477-533) through fdb_derivative."""
    _real_input(x)
    dv = _flat_f64(df, "df")
    m = dv.numel()
    if isinstance(cache.c1, torch.Tensor) and cache.c1.numel() != m:
        raise ValueError(f"length(df)={m} != the cache's {cache.c1.numel()} outputs")
    dev = dv.device
    fd = _fdtype_code(cache.fdtype)
    if isinstance(x, torch.Tensor):
        if x.numel() != 1 or x.device != dev:
            raise ValueError("a tensor t must hold one float64 value on df's device")
        tv = _flat_f64(x, "x")
    else:
        tv = None
    plan = cache.scalar_plan_for(m, dev)
    addr, ctx, pyfn = _as_fn(f, m, 1, dev, 1, fd == L.FDB_COMPLEX, tvec=True)
    stream = _stream(stream, dev)
    if tv is None:
        tv = _device_slot(cache, "_t", dev, stream, x)
    if fd == L.FDB_COMPLEX:
        _call(dev, [pyfn], L.lib().fdb_derivative_complex, plan.handle, addr, ctx, dv.data_ptr(), tv.data_ptr(),
              C.c_void_p(stream))
    else:
        fx_ptr = None
        if fd == L.FDB_FORWARD and cache.fx is not None:                      # :501-502
            fxv = _flat_f64(cache.fx, "cache.fx")
            if fxv.numel() != m or fxv.device != dev:
                raise ValueError("cache.fx must hold the m values f(x) on df's device")
            fx_ptr = _fx_ptr(fxv)
        _call(dev, [pyfn], L.lib().fdb_derivative, plan.handle, addr, ctx, dv.data_ptr(), tv.data_ptr(), fx_ptr,
              *_steps(relstep, absstep), float(dir), C.c_void_p(stream))
    cache._last_plan = plan
    return None


# ------------------------------------------------------------------------------------------------ derivative (src/derivatives.jl)
class DerivativeCache:
    """Mirror of FiniteDiff.DerivativeCache (derivatives.jl:38-88):

        DerivativeCache(x, fx=None, epsilon=None, fdtype="central", returntype=float64)

    fx (n values f(x)) is kept in forward mode only; otherwise it is dropped with a warning (:67-73).  epsilon is allocated
    (zeros like x) when not given or of another dtype, and dropped with a warning in complex mode (:78-86); the StridedArray
    path never reads or writes it.  Complex mode with a non-real returntype is fdtype_error (:63-65).  Extra keywords (GPU
    path only): max_batch (2: both central points in one f call), use_graph."""

    def __init__(self, x, fx=None, epsilon=None, fdtype="central", returntype=torch.float64, **plan_kw):
        if isinstance(fx, str):
            fdtype, fx = fx, None
        elif isinstance(epsilon, str):
            fdtype, epsilon = epsilon, None
        self.fdtype = fdtype.lstrip(":") if isinstance(fdtype, str) else fdtype
        code = _fdtype_code(self.fdtype)
        if returntype in (torch.complex128, torch.complex64, complex, np.complex128):
            if code == L.FDB_COMPLEX:                                          # :63-65
                raise ValueError(f"Unrecognized fdtype for returntype {returntype}: complex step needs a real return type")
            raise TypeError("complex-valued derivatives are not supported: only Float64")
        if returntype not in (torch.float64, float, np.float64):
            raise TypeError("only Float64 is supported by the GPU path")
        _flat_f64(x, "x")
        if code != L.FDB_FORWARD and fx is not None:                            # :67-70
            warnings.warn("Pre-computed function values are only useful for fdtype==Val(:forward).")
            fx = None
        if epsilon is not None and code == L.FDB_COMPLEX:                       # :78-80
            warnings.warn("Val(:complex) makes the epsilon array redundant.")
            epsilon = None
        elif epsilon is None or not isinstance(epsilon, torch.Tensor) or epsilon.dtype != torch.float64:   # :82-84
            epsilon = torch.zeros_like(x)
        self.fx, self.epsilon = fx, epsilon
        self._code = code
        self._plan_kw = plan_kw
        self._plans = {}

    def plan_for(self, n: int, device) -> Plan:
        def create():
            o = _opts(self._code, _device_index(device), **self._plan_kw)
            return Plan(_new_handle("fdb_derivative_plan_create", n, C.byref(o)).value)
        return _cached_plan(self, (n, str(device)), create)


def finite_difference_derivative_(df, f, x, cache="central", returntype=None, fx=None, epsilon=None, *, relstep=None,
                                  absstep=None, dir=True, stream=None):
    """finite_difference_derivative!(df, f, x::StridedArray, cache::DerivativeCache; relstep, absstep, dir)
    (derivatives.jl:197-233), or — when `cache` is None or an fdtype string — the cache-less form
    finite_difference_derivative!(df, f, x, fdtype, returntype, fx, epsilon; relstep, absstep) (:133-146).

    df, x: contiguous float64 CUDA tensors of the same size; x is never modified.
    f: elementwise scalar function as a Python callable applied to a whole CUDA tensor, returning a tensor of its shape
       (torch.sin works; complex step: complex128 in and out; set f.batched = True to receive a (batch, n) tensor), or a
       NativeFn (fdb_fn with m = n evaluated elementwise; fdb_fn_c for complex).  Returns df."""
    if cache is None or isinstance(cache, str):
        cache = DerivativeCache(x, fx, epsilon, cache or "central", returntype or torch.float64)
    if not isinstance(cache, DerivativeCache):
        raise TypeError("cache must be a DerivativeCache, an fdtype string, or None")
    xv = _flat_f64(x, "x")
    dv = _flat_f64(df, "df")
    n = xv.numel()
    if dv.numel() != n:
        raise ValueError(f"length(df)={dv.numel()} != length(x)={n}")
    if dv.device != xv.device:
        raise ValueError("df and x must be on the same device")
    plan = cache.plan_for(n, xv.device)
    addr, ctx, pyfn = _as_fn(f, n, n, xv.device, 1, cache._code == L.FDB_COMPLEX, elementwise=True)
    stream = _stream(stream, xv.device)
    if cache._code == L.FDB_COMPLEX:
        _call(xv.device, [pyfn], L.lib().fdb_derivative_complex, plan.handle, addr, ctx, dv.data_ptr(), xv.data_ptr(),
              C.c_void_p(stream))
    else:
        fx_ptr = None
        if cache._code == L.FDB_FORWARD and cache.fx is not None:              # :213-214
            fxv = _flat_f64(cache.fx, "cache.fx")
            if fxv.numel() != n or fxv.device != xv.device:
                raise ValueError("cache.fx must hold the n values f(x) on x's device")
            fx_ptr = _fx_ptr(fxv)
        _call(xv.device, [pyfn], L.lib().fdb_derivative, plan.handle, addr, ctx, dv.data_ptr(), xv.data_ptr(), fx_ptr,
              *_steps(relstep, absstep), float(dir), C.c_void_p(stream))
    cache._last_plan = plan
    return df


def finite_difference_derivative(f, x, cache="central", returntype=None, fx=None, epsilon=None, *, relstep=None,
                                 absstep=None, dir=True, stream=None):
    """finite_difference_derivative(f, x::StridedArray[, fdtype | cache, returntype, fx, epsilon]; relstep, absstep)
    (derivatives.jl:104-116): a new float64 CUDA tensor of x's shape."""
    if not isinstance(x, torch.Tensor):
        raise TypeError("x must be a float64 CUDA tensor (the single-point derivative is not provided)")
    df = torch.zeros(x.shape, dtype=torch.float64, device=x.device)
    return finite_difference_derivative_(df, f, x, cache, returntype, fx, epsilon, relstep=relstep, absstep=absstep,
                                         dir=dir, stream=stream)
