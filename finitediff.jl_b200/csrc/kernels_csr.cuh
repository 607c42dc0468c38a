// kernels_csr.cuh — the CSR scatter: J is the nzval of a CSR matrix with the sparsity's own pattern, the target the
// generic `J[r, c] = v` hook reaches with a row-compressed matrix (ext/FiniteDiffSparseArraysExt.jl:20-28,
// iteration_utils.jl:25-32) — cuSPARSE's, cuDSS's and AMGX's input format.
//
// A launch walks nzval in storage order: kCsrPer runs of kThreads entries per tile.  Entry s of row r reads its column
// c = colval[s] and the colour k of c, and stores the quotient of k's slab at row r.  All the entries of a row gather the
// same slab row and f(x) row, and consecutive rows gather consecutive ones, so the gathers are row-local by construction.
// The row of an entry: the tile's first and last rows (the largest r with rowptr[r] <= s, for the tile's first and last
// entry) are found once by a search of the row pointer.  When the tile spans at most kCsrStage rows their starts are
// staged in shared memory and each entry searches them; otherwise (a tile across thousands of empty rows) the entry
// searches rowptr[rlo..rhi] in global memory.  An empty row shares its start with the next row, so the largest r with
// rowptr[r] <= s is always the row that holds s.
//
// The launch writes the quotient of every entry whose colour it holds and, with write_other, +0.0 for every entry whose
// column has no valid colour, so the launches of one Jacobian write every slot exactly once and J needs no zero fill.
// The quotient is fd_quotient, the same IEEE sequence as every other scatter.
#pragma once
#include "kernels_scatter.cuh"
#include "kernels_plan.cuh"

namespace fdb {

constexpr int kCsrPer = 4;                    // entries per thread and tile
constexpr int kCsrTile = kThreads * kCsrPer;
constexpr int kCsrStage = kCsrTile;           // row starts of a tile staged in shared memory

struct CsrArgs {
  const int32_t *rowptr;       // [m + 1] 0-based: row r holds entries [rowptr[r], rowptr[r+1])
  const int32_t *colval;       // [nnz] 0-based column of every entry
  const double *fx, *Fp, *Fm, *eps;
  const int32_t *local_of;
  double *J;
  int64_t ldF;
  int32_t m, nnz;
  int32_t C, l0, G;
  int32_t full;                // one group on one rank: every valid colour is resident at slab = colour, no ownership test
  int32_t write_other;         // also define the entries of columns without a valid colour (+0.0)
};

// the largest r in [lo, hi] with ptr[r] <= s, given ptr[lo] <= s
__device__ __forceinline__ int32_t csr_row_of(const int32_t *ptr, int32_t lo, int32_t hi, int32_t s) {
  while (lo < hi) {
    const int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi + 1u) >> 1);
    if (ptr[mid] <= s) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <typename CS, int MODE>
__global__ void __launch_bounds__(kThreads)
diff_scatter_csr(const CsrArgs a, const CS cs) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int32_t s_range[2];
  __shared__ int32_t s_ptr[kCsrStage];
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
  }
  const int32_t ntiles = (int32_t)(((int64_t)a.nnz + kCsrTile - 1) / kCsrTile);
  for (int32_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int32_t s0 = tile * kCsrTile;                  // < nnz < 2^31
    __syncthreads();                                     // the previous tile's readers of s_range / s_ptr are done
    if (threadIdx.x < 2) {
      const int32_t s = threadIdx.x == 0 ? s0 : ((int64_t)s0 + kCsrTile < a.nnz ? s0 + kCsrTile - 1 : a.nnz - 1);
      s_range[threadIdx.x] = csr_row_of(a.rowptr, 0, a.m - 1, s);
    }
    __syncthreads();
    const int32_t rlo = s_range[0], rhi = s_range[1];
    const bool staged = rhi - rlo < kCsrStage;
    if (staged)
      for (int t = threadIdx.x; t <= rhi - rlo; t += kThreads) s_ptr[t] = __ldg(a.rowptr + rlo + t);
    __syncthreads();
#pragma unroll
    for (int p = 0; p < kCsrPer; ++p) {
      const int32_t s = s0 + p * kThreads + (int32_t)threadIdx.x;
      if (s >= a.nnz) break;
      const int32_t r = staged ? rlo + csr_row_of(s_ptr, 0, rhi - rlo, s) : csr_row_of(a.rowptr, rlo, rhi, s);
      const uint32_t k = cs.at(__ldcs(a.colval + s));
      int32_t slab = -1;
      double e = 1.0;
      if (k < (uint32_t)a.C) {
        if (a.full) { slab = (int32_t)k; e = tables ? s_eps[k] : __ldg(a.eps + k); }
        else if (tables) { slab = s_slab[k]; e = s_eps[k]; }
        else {
          const int32_t lo = __ldg(a.local_of + k);
          slab = lo < 0 ? -1 : lo - a.l0;
          if (slab >= a.G) slab = -1;
          e = __ldg(a.eps + k);
        }
        if (slab < 0) continue;                          // another group's / rank's column
      } else if (!a.write_other) {
        continue;                                        // no valid colour: defined by the first launch of rank 0
      }
      double v = 0.0;
      if (slab >= 0)
        v = fd_quotient<MODE>(a.Fp + (int64_t)slab * a.ldF, MODE == kCentral ? a.Fm + (int64_t)slab * a.ldF : a.fx, r, e);
      st_stream(a.J + s, v);
    }
  }
}

// Plan pass over the entries: colval32[s] = colval[s] - 1 (kErrColRange outside 1..n) and the entries per colour
// (the LPT weights), counted like expand_csc.
template <typename CT>
__global__ void __launch_bounds__(kThreads)
csr_plan_pass(const int64_t *__restrict__ colval, int64_t n, int64_t nnz, const CT *__restrict__ jcolor, int32_t C,
              int32_t *__restrict__ colval32, unsigned long long *__restrict__ color_count, uint32_t *__restrict__ err) {
  extern __shared__ unsigned int s_hist[];   // [C] when C <= kPlanSmemColors
  unsigned int *s_cnt = count_begin(s_hist, C, color_count);
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int lane = threadIdx.x & 31;
  // warp-uniform trip count: count_color uses full-warp collectives
  for (int64_t p0 = blockIdx.x * (int64_t)kThreads + threadIdx.x - lane; p0 < nnz; p0 += stride) {
    const int64_t p = p0 + lane;
    uint32_t k = 0xffffffffu;
    if (p < nnz) {
      const int64_t c = colval[p];
      if (c < 1 || c > n) { atomicOr(err, kErrColRange); colval32[p] = 0; }
      else { colval32[p] = (int32_t)(c - 1); k = (uint32_t)jcolor[c - 1]; }
    }
    count_color(k, C, s_cnt, color_count);
  }
  count_end(s_cnt, C, color_count);
}

// rowptr32[r] = rowptr[r] - 1 (the plan has validated the row pointer)
__global__ void __launch_bounds__(kThreads)
csr_rowptr32(const int64_t *__restrict__ rowptr, int64_t m, int32_t *__restrict__ rowptr32) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t r = blockIdx.x * (int64_t)kThreads + threadIdx.x; r <= m; r += stride) rowptr32[r] = (int32_t)(rowptr[r] - 1);
}

// Int64 1-based copy of a 0-based int32 index array (CSR -> CSC of the pattern for the colouring entry points)
__global__ void __launch_bounds__(kThreads)
widen_index(const int32_t *__restrict__ src, int64_t count, int64_t *__restrict__ dst) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < count; i += stride) dst[i] = (int64_t)src[i] + 1;
}

}  // namespace fdb
