"""finitediff.jl_b200 — H100 (sm_90a) drop-in for FiniteDiff.jl's coloured sparse-Jacobian hot path.

Layout (only what the path needs):
    csrc/      hand-written CUDA kernels + the C ABI (libfdjac_b200.so; include/fdjac_b200.h)
    api.py     host-side mirror of the reference interface (JacobianCache / finite_difference_jacobian!, HessianCache /
               finite_difference_hessian!, GradientCache / finite_difference_gradient!, DerivativeCache /
               finite_difference_derivative!, and the out-of-place finite_difference_jacobian / finite_difference_jvp)
    distributed.py  multi-GPU plumbing over the C ABI's fdb_group_* / fdb_sync_* (colour shards, column blocks)
    julia/     the `ccall` wrapper a Julia host would load (not executable in this image: no julia)
    _lib.py    ctypes binding of the C ABI (fails loudly if the .so is missing)
    build.py   nvcc recipe (sm_90a only)

The directory name contains a dot, so it is imported through _bootstrap.py (repository root) under the alias
`finitediff_jl_b200`.
"""
from . import _lib  # noqa: F401
from .api import (BandedBlockBandedMatrix, BandedMatrix, BlockBandedMatrix, BlockSkylineMatrix, DenseColumnBlock, JacobianCache, JVPCache, NativeFn, Plan, SparseMatrixCSC, SparseMatrixCSR, Tridiagonal, compute_epsilon,
                  Diagonal, Bidiagonal, SymTridiagonal,
                  default_relstep, finite_difference_jacobian_, finite_difference_jacobian_b, finite_difference_jvp_,
                  check_coloring, make_plan, matrix_colors, pinned_empty, resize_, zeros_colmajor,
                  HessianCache, finite_difference_hessian_, finite_difference_hessian,
                  GradientCache, finite_difference_gradient_, finite_difference_gradient,
                  DerivativeCache, finite_difference_derivative_, finite_difference_derivative,
                  finite_difference_jacobian, finite_difference_jvp)

__all__ = ["BandedBlockBandedMatrix", "BandedMatrix", "BlockBandedMatrix", "BlockSkylineMatrix", "DenseColumnBlock", "JacobianCache", "JVPCache", "finite_difference_jvp_", "NativeFn", "Plan", "SparseMatrixCSC", "SparseMatrixCSR", "Tridiagonal", "compute_epsilon",
           "Diagonal", "Bidiagonal", "SymTridiagonal",
           "default_relstep", "finite_difference_jacobian_", "finite_difference_jacobian_b", "make_plan", "matrix_colors", "check_coloring",
           "pinned_empty", "resize_", "zeros_colmajor", "HessianCache", "finite_difference_hessian_",
           "finite_difference_hessian", "GradientCache", "finite_difference_gradient_", "finite_difference_gradient",
           "DerivativeCache", "finite_difference_derivative_", "finite_difference_derivative",
           "finite_difference_jacobian", "finite_difference_jvp"]
