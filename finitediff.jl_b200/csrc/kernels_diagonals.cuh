// kernels_diagonals.cuh — the diagonal-storage scatter: LinearAlgebra's Diagonal, Bidiagonal and Tridiagonal storage as
// the Jacobian target of a banded plan with l, u in {0, 1} (FDB_J_DIAGONALS).
//
// Storage: one packed buffer holding the stored diagonals in ascending row-minus-column order — the sub-diagonal
// (r = c+1, n-1 slots, when l = 1), the main diagonal (n slots), the super-diagonal (c = r+1, n-1 slots, when u = 1) —
// each from the top left: [dl; d; du] (Tridiagonal), [dv; ev] (Bidiagonal :U), [ev; dv] (:L), [d] (Diagonal).  These
// slots are exactly the in-matrix band (l, u) that ext/FiniteDiffBandedMatricesExt.jl:13-27 writes, and every one of
// them is a structural entry, so no slot is ever outside the structure.
//
// A launch walks the buffer in storage order, one slot per thread and kDgPer contiguous runs of kThreads slots per tile.
// The diagonal of a slot takes at most two compares, (r, c) follow in closed form, and the column's colour comes from the
// plan's colour source (the cyclic closed form of matrix_colors, or the table).  A launch writes the slots of the columns
// whose colour it holds (the quotient) and, with write_other, those of the columns without a valid colour (+0.0); so the
// launches of one Jacobian write every slot exactly once and J needs no zero fill.  The quotient is fd_quotient, the
// same IEEE sequence as every other scatter.
#pragma once
#include "kernels_scatter.cuh"

namespace fdb {

constexpr int kDgPer = 4;                     // slots per thread and tile
constexpr int kDgTile = kThreads * kDgPer;

struct DiagArgs {
  const double *fx, *Fp, *Fm, *eps;
  const int32_t *local_of;
  double *J;
  int64_t total;               // (l+u+1) n - l - u slots (64-bit: 3n passes 2^32 for n near 2^31)
  int64_t sub_end;             // l (n-1): the sub-diagonal occupies slots [0, sub_end)
  int64_t main_end;            // sub_end + n: the main diagonal occupies [sub_end, main_end), the super-diagonal the rest
  int64_t ldF;
  int32_t C, l0, G;
  int32_t write_other;         // also define the columns without a valid colour (+0.0)
};

template <typename CS, int MODE>
__global__ void __launch_bounds__(kThreads)
diff_scatter_diagonals(const DiagArgs a, const CS cs) {
  extern __shared__ __align__(16) unsigned char smem[];
  double *s_eps = reinterpret_cast<double *>(smem);
  int32_t *s_slab = reinterpret_cast<int32_t *>(smem + sizeof(double) * (a.C <= kSmemTable ? a.C : 0));
  const bool tables = a.C <= kSmemTable;
  if (tables) {
    for (int i = threadIdx.x; i < a.C; i += kThreads) {
      const int32_t lo = a.local_of[i];
      int32_t sl = lo < 0 ? -1 : lo - a.l0;
      if (sl >= a.G) sl = -1;
      s_slab[i] = sl;
      s_eps[i] = a.eps[i];
    }
    __syncthreads();
  }
  const int64_t ntiles = (a.total + kDgTile - 1) / kDgTile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t s0 = tile * kDgTile;
#pragma unroll
    for (int p = 0; p < kDgPer; ++p) {
      const int64_t s = s0 + p * kThreads + threadIdx.x;
      if (s >= a.total) break;
      int64_t r, c;
      if (s < a.sub_end) { c = s; r = s + 1; }                      // sub-diagonal
      else if (s < a.main_end) { c = s - a.sub_end; r = c; }        // main diagonal
      else { r = s - a.main_end; c = r + 1; }                       // super-diagonal
      const uint32_t k = cs.at(c);
      int32_t slab = -1;
      double e = 1.0;
      if (k < (uint32_t)a.C) {
        if (tables) { slab = s_slab[k]; e = s_eps[k]; }
        else {
          const int32_t lo = __ldg(a.local_of + k);
          slab = lo < 0 ? -1 : lo - a.l0;
          if (slab >= a.G) slab = -1;
          e = __ldg(a.eps + k);
        }
        if (slab < 0) continue;                                     // another group's / rank's column
      } else if (!a.write_other) {
        continue;                                                   // no valid colour: defined by the first launch of rank 0
      }
      double v = 0.0;
      if (slab >= 0)
        v = fd_quotient<MODE>(a.Fp + (int64_t)slab * a.ldF, MODE == kCentral ? a.Fm + (int64_t)slab * a.ldF : a.fx, r, e);
      st_stream(a.J + s, v);
    }
  }
}

}  // namespace fdb
