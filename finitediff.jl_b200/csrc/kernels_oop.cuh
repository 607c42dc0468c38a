// kernels_oop.cuh — the result forms of the out-of-place Jacobian, finite_difference_jacobian(f, x, cache, f_in; …)
// (jacobians.jl:277-429).  The out-of-place form returns `J = J + Ji` summed over the colours, and what that sum leaves
// depends on the type of J (the _make_Ji methods, jacobians.jl:151-187 and ext/FiniteDiffSparseArraysExt.jl:7-17):
//   dense J     every structural slot holds 0.0 + q (a -0.0 quotient becomes +0.0), every other element +0.0;
//   sparse J    sparse `+` is SparseArrays' zero-preserving map, which stores a result only when it is not iszero: the
//               structural entries whose quotient is not ±0.0, in storage order (NaN is kept).
// The points and f! outputs come from the in-place colour loop (perturbation in its out-of-place mode); the dense results'
// quotients from its diff+scatter, which these kernels finish, and the sparse result's from oop_compact itself when every
// f! output is resident.
#pragma once
#include "common.cuh"
#include "kernels_scatter.cuh"

namespace fdb {

// J[dest[e]] += 0.0 over the structural slots of a zero-filled dense J that holds the quotients: J + Ji at the entry's
// colour is (+0.0) + q, and the later colours add +0.0 to a value that is no longer -0.0
__global__ void __launch_bounds__(kThreads)
oop_plus_zero_slots(double *__restrict__ J, const int64_t *__restrict__ dest, int64_t E) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < E; e += stride) {
    const int64_t d = __ldcs(dest + e);
    J[d] = J[d] + 0.0;
  }
}

// Dense J without sparsity, given a dense prototype with `ncols` >= C columns: column c < C holds the quotients and becomes
// 0.0 + q; columns C..ncols-1 are zero(dx) summed over the colours, +0.0.  Tiles of kTile rows, grid-stride over
// (column, row tile).
__global__ void __launch_bounds__(kThreads)
oop_dense_finish(double *__restrict__ J, int64_t ldJ, int64_t m, int64_t C, int64_t ncols) {
  const int64_t rtiles = (m + kTile - 1) / kTile;
  const int64_t total = rtiles * ncols;
  for (int64_t t = blockIdx.x; t < total; t += gridDim.x) {
    const int64_t c = t / rtiles, r0 = (t - c * rtiles) * kTile;
    double *col = J + c * ldJ;
#pragma unroll
    for (int u = 0; u < kTile / kThreads; ++u) {
      const int64_t r = r0 + u * kThreads + threadIdx.x;
      if (r < m) col[r] = c < C ? col[r] + 0.0 : 0.0;
    }
  }
}

// ---- zero-dropping compaction of a CSC result (sparse `+`, SparseArrays' _map_zeropres!) ----
// One pass over the candidate entries in storage order.  With a CSC sparsity whose f! outputs are all resident (MODE =
// kForward / kCentral / kComplex) the pass forms each entry's quotient from them itself — (F_k[r] - f(x)[r]) / eps_k,
// (F_k[r] - Fm_k[r]) / (2 eps_k) or imag(F_k[r]) / eps, the in-place scatter's own operations (fd_quotient) — so the
// candidates are never stored; MODE = kCopy reads candidates already formed (the dense branch's m x C block, or a
// sparsity whose outputs come in several groups). (the column-major, row-sorted order of sparse(I, J, V)): an entry
// is kept when its value is not ±0.0.  Each 1024-entry tile counts its kept entries with warp ballots, publishes the
// count, and finds the number kept before it by a decoupled look-back over the tiles before it (Merrill & Garland,
// "Single-pass Parallel Prefix Scan with Decoupled Look-back", NVIDIA 2016).  Tiles are claimed in order from a counter,
// so every tile a block waits for is held by a block that is running.  The kernel writes 1-based Int64 rowval, nzval,
// colptr for every column that starts in the tile, and the kept count to *nnz.
//   FULL = false: candidates are a CSC pattern's entries (row32[e], colptr32 0-based, ncols columns);
//   FULL = true:  candidates are every element of an m x C column-major block (sparsity === nothing), ncols >= C.
constexpr uint64_t kLbAggregate = 1ull << 62, kLbPrefix = 2ull << 62, kLbValue = (1ull << 62) - 1;

struct CompactArgs {
  const double *vals;        // [E] candidate values in storage order (kCopy)
  const void *ecolor;        // [E] 0-based colour of the entry's column (CT), quotient modes
  const double *Fp, *Fm, *fx, *eps;   // resident f! outputs [C][ldF], central minus outputs, f(x), step sizes [C]
  int64_t ldF;               // doubles between two colours' outputs
  int32_t ncolors;
  const int32_t *row32;      // [E] 0-based rows (FULL = false)
  const int32_t *colptr32;   // [ncols + 1] 0-based column starts (FULL = false)
  int64_t E, m, C, ncols;
  int64_t *colptr, *rowval;  // outputs: [ncols + 1], [<= E]  (1-based)
  double *nzval;             // [<= E]
  int64_t *nnz;              // kept count
  unsigned long long *state; // [ntiles] look-back words, zeroed before the launch
  unsigned long long *claim; // tile counter, zeroed before the launch
  const int32_t *tile_col;   // [ntiles] first column starting at or after the tile's first entry (FULL = false)
};

template <bool FULL>
__device__ __forceinline__ int64_t compact_col_start(const CompactArgs &a, int64_t c) {
  if (FULL) return (c < a.C ? c : a.C) * a.m;
  return c < a.ncols ? (int64_t)__ldg(a.colptr32 + c) : a.E;
}

// Plan time (the pattern is fixed): per tile, the first column whose start is at or after the tile's first entry, so that
// the compaction reads it instead of searching colptr on every call
__global__ void __launch_bounds__(kThreads)
oop_tile_first_col(const int32_t *__restrict__ colptr32, int64_t ncols, int64_t ntiles, int32_t *__restrict__ tile_col) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t t = blockIdx.x * (int64_t)kThreads + threadIdx.x; t < ntiles; t += stride) {
    const int64_t t0 = t * kTile;
    int64_t lo = 0, hi = ncols;                    // column ncols "starts" at E >= t0
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (colptr32[mid] < t0) lo = mid + 1; else hi = mid;
    }
    tile_col[t] = (int32_t)lo;
  }
}

template <bool FULL, int MODE, typename CT>
__global__ void __launch_bounds__(kThreads)
oop_compact(const CompactArgs a) {
  constexpr int kWarps = kThreads / 32, kRounds = kTile / kThreads;
  __shared__ uint32_t s_mask[kRounds * kWarps];
  __shared__ uint32_t s_pre[kRounds * kWarps + 1];
  __shared__ int64_t s_tile, s_base;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t ntiles = (a.E + kTile - 1) / kTile;
  if (ntiles == 0) {   // no candidates: every column is empty
    if (blockIdx.x == 0) {
      for (int64_t c = threadIdx.x; c <= a.ncols; c += kThreads) a.colptr[c] = 1;
      if (threadIdx.x == 0) *a.nnz = 0;
    }
    return;
  }
  for (;;) {
    if (threadIdx.x == 0) s_tile = (int64_t)atomicAdd(a.claim, 1ull);
    __syncthreads();
    const int64_t tile = s_tile;
    if (tile >= ntiles) return;
    const int64_t t0 = tile * kTile;
    // element (round u, warp w, lane) = t0 + u*kThreads + w*32 + lane: (u, w, lane) order is storage order
    double v[kRounds];
    int32_t r[kRounds];
#pragma unroll
    for (int u = 0; u < kRounds; ++u) {
      const int64_t e = t0 + u * kThreads + threadIdx.x;
      const bool in = e < a.E;
      if (FULL) r[u] = in ? (int32_t)(e % a.m) : 0;
      else r[u] = in ? __ldcs(a.row32 + e) : 0;
      if (MODE == kCopy) {
        v[u] = in ? __ldcs(a.vals + e) : 0.0;
      } else {
        const uint32_t k = in ? (uint32_t)reinterpret_cast<const CT *>(a.ecolor)[e] : 0xFFFFFFFFu;
        // a column without a valid colour is never perturbed: its entries are 0 and dropped
        v[u] = k < (uint32_t)a.ncolors
                   ? fd_quotient<MODE>(a.Fp + (int64_t)k * a.ldF, MODE == kCentral ? a.Fm + (int64_t)k * a.ldF : a.fx, r[u],
                                       __ldg(a.eps + k))
                   : 0.0;
      }
      const uint32_t mk = __ballot_sync(0xffffffffu, v[u] != 0.0);   // NaN != 0.0 is true: NaN is kept
      if (lane == 0) s_mask[u * kWarps + w] = mk;
    }
    __syncthreads();
    if (w == 0) {
      // exclusive scan of the 32 (round, warp) counts
      const uint32_t cnt = __popc(s_mask[lane]);
      uint32_t inc = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
      }
      s_pre[lane] = inc - cnt;
      const uint64_t total = __shfl_sync(0xffffffffu, inc, 31);
      if (lane == 31) s_pre[32] = inc;
      // decoupled look-back, a window of 32 predecessors per step (lane j reads tile p - j).  Every tile before one that
      // published its inclusive prefix has published too, so a window with an unpublished tile is re-read (spin) and a
      // window with a prefix ends the walk at its nearest one.
      volatile unsigned long long *st = a.state;
      int64_t base = 0;
      if (tile == 0) {
        if (lane == 0) st[0] = kLbPrefix | total;
      } else {
        if (lane == 0) st[tile] = kLbAggregate | total;
        __threadfence();
        for (int64_t p = tile - 1;;) {
          const int64_t q = p - lane;
          const unsigned long long sv = q >= 0 ? st[q] : kLbPrefix;       // before tile 0: a prefix of 0
          const uint32_t flag = (uint32_t)(sv >> 62);
          if (__any_sync(0xffffffffu, flag == 0)) continue;
          const uint32_t pre = __ballot_sync(0xffffffffu, flag == 2);
          const int first = pre ? __ffs(pre) - 1 : 31;
          int64_t val = lane <= first ? (int64_t)(sv & kLbValue) : 0;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) val += __shfl_xor_sync(0xffffffffu, val, o);
          base += val;
          if (pre) break;
          p -= 32;
        }
        __threadfence();
        if (lane == 0) st[tile] = kLbPrefix | (uint64_t)(base + (int64_t)total);
      }
      if (lane == 0) s_base = base;
    }
    __syncthreads();
    const int64_t base = s_base;
#pragma unroll
    for (int u = 0; u < kRounds; ++u) {
      const uint32_t mk = s_mask[u * kWarps + w];
      if (mk >> lane & 1u) {
        const int64_t o = base + s_pre[u * kWarps + w] + __popc(mk & ((1u << lane) - 1u));
        a.rowval[o] = (int64_t)r[u] + 1;
        a.nzval[o] = v[u];
      }
    }
    // colptr of the columns that start inside this tile (the last tile also takes the columns that start at E)
    const bool last = tile == ntiles - 1;
    const int64_t t1 = last ? a.E + 1 : t0 + kTile;
    // first column that starts at or after t0 (FULL: ceil(t0 / m), at most C since t0 < E = C*m)
    const int64_t clo = FULL ? (t0 + a.m - 1) / a.m : (int64_t)__ldg(a.tile_col + tile);
    for (int64_t c = clo + threadIdx.x; c <= a.ncols; c += kThreads) {
      const int64_t p = compact_col_start<FULL>(a, c);
      if (p >= t1) break;
      const int64_t q = p - t0;                      // position inside the tile, 0..1024
      int64_t before;
      if (q >= kTile || p >= a.E) before = s_pre[32];
      else {
        const int i = (int)(q / 32);                 // (round, warp) slot of position q
        before = s_pre[i] + __popc(s_mask[i] & ((1u << (q & 31)) - 1u));
      }
      a.colptr[c] = base + before + 1;
    }
    if (last && threadIdx.x == 0) *a.nnz = base + (int64_t)s_pre[32];
    __syncthreads();
  }
}

}  // namespace fdb
