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
#include "kernels_blockband.cuh"
#include "kernels_csr.cuh"

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
// FORM is the structure of the candidates:
//   kFormCsc:  a CSC pattern's entries (row32[e], colptr32 0-based, ncols columns);
//   kFormFull: every element of an m x C column-major block (sparsity === nothing), ncols >= C;
//   kFormBand: the in-matrix band (l, u) of an m x n matrix, column-major and row-sorted, in closed form (BandShape): no
//              row, colour-per-entry or column-start stream.  kCopy reads the candidates in band-data layout (slot u + r - c
//              of column c, stride l + u + 1), as the in-place band scatter writes them.
//   kFormBlockBand / kFormBlockDense: the entry set of a BandedBlockBandedMatrix / BlockSkylineMatrix with square blocks,
//              in closed form from the block offsets (BlockShape, BlockBandForm, BlockDenseForm below).
//   kFormCsr:  a CSR pattern's entries in row order (CsrForm below): candidate e is slot e, row32[e] its 0-based column
//              (the stored minor index), colptr32 the 0-based row pointer and ncols = m, so the pointer pass below writes
//              the row starts.  Only the quotient modes use it: kCopy has no use for the row, and the kFormCsc pass over
//              (colval, rowptr) is already the CSR copy.
constexpr uint64_t kLbAggregate = 1ull << 62, kLbPrefix = 2ull << 62, kLbValue = (1ull << 62) - 1;
enum { kFormCsc = 0, kFormFull = 1, kFormBand = 2, kFormBlockBand = 3, kFormBlockDense = 4, kFormCsr = 5 };

// The in-matrix band E(m, n, l, u) = {(r, c) : -u <= r - c <= l, 0 <= r < m, 0 <= c < n} (0-based), l, u >= 0, clamped to
// l <= m - 1, u <= n - 1 (the same set).  Column c holds rows max(0, c - u) .. min(m - 1, c + l); columns c >= m + u are
// empty.  The interior columns [ca, cb) hold w = l + u + 1 rows each and start at sa + (c - ca) w.
struct BandShape {
  int64_t m, n, l, u, w;
  int64_t ca, cb, sa, sb, E;
  FastDiv wdiv;
};

// entries in the columns before c, 0 <= c <= n: sum over j < c of min(m-1, j+l) - max(0, j-u) + 1
__host__ __device__ __forceinline__ int64_t band_col_start(int64_t m, int64_t l, int64_t u, int64_t c) {
  if (m <= 0) return 0;
  const int64_t k = c < m + u ? c : m + u;                         // non-empty columns before c
  const int64_t K = m - 1;
  int64_t t = K - l + 1;                                           // columns j < k with j + l <= K
  t = t < 0 ? 0 : (t > k ? k : t);
  const int64_t A = t * l + t * (t - 1) / 2 + (k - t) * K;         // sum of min(K, j + l)
  const int64_t s = k - u - 1 > 0 ? k - u - 1 : 0;                 // columns j < k with j > u
  return k + A - s * (s + 1) / 2;                                  // - sum of max(0, j - u)
}

inline BandShape make_band_shape(int64_t m, int64_t n, int64_t l, int64_t u) {
  BandShape b{};
  b.m = m; b.n = n; b.l = l; b.u = u; b.w = l + u + 1;
  b.ca = u < n ? u : n;
  b.cb = m - l < n ? m - l : n;
  if (b.cb < b.ca) b.cb = b.ca;
  b.sa = band_col_start(m, l, u, b.ca);
  b.sb = band_col_start(m, l, u, b.cb);
  b.E = band_col_start(m, l, u, n);
  b.wdiv = make_fastdiv((uint32_t)b.w);
  return b;
}

__device__ __forceinline__ int64_t band_start(const BandShape &b, int64_t c) {
  if (c >= b.ca && c <= b.cb) return b.sa + (c - b.ca) * b.w;
  return band_col_start(b.m, b.l, b.u, c);
}

// the column c and row r of candidate e, 0 <= e < E: division in the interior, a search over the closed-form column
// starts in the head and tail columns
__device__ __forceinline__ void band_locate(const BandShape &b, int64_t e, int64_t &c, int64_t &r) {
  if (e >= b.sa && e < b.sb) {
    const int64_t q = e - b.sa;
    const int64_t d = q < (int64_t)0xFFFFFFFFll ? (int64_t)b.wdiv.div((uint32_t)q) : q / b.w;
    c = b.ca + d;
    r = c - b.u + (q - d * b.w);
    return;
  }
  int64_t lo = 0, hi = b.n - 1;                                    // the last column starting at or before e
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (band_col_start(b.m, b.l, b.u, mid) <= e) lo = mid; else hi = mid - 1;
  }
  c = lo;
  r = (c - b.u > 0 ? c - b.u : 0) + (e - band_col_start(b.m, b.l, b.u, c));
}

// the first column that starts at or after candidate t0 < E (columns between the interior and E are never empty)
__device__ __forceinline__ int64_t band_first_col(const BandShape &b, int64_t t0) {
  int64_t c, r;
  band_locate(b, t0, c, r);
  return band_start(b, c) < t0 ? c + 1 : c;
}

struct CompactArgs {
  const double *vals;        // [E] candidate values in storage order (kCopy)
  const void *ecolor;        // [E] 0-based colour of the entry's column (CT), quotient modes
  const double *Fp, *Fm, *fx, *eps;   // resident f! outputs [C][ldF], central minus outputs, f(x), step sizes [C]
  int64_t ldF;               // doubles between two colours' outputs
  int32_t ncolors;
  const int32_t *row32;      // [E] 0-based rows (kFormCsc; kFormCsr: columns)
  const int32_t *colptr32;   // [ncols + 1] 0-based column starts (kFormCsc; kFormCsr: row starts, ncols = m)
  int64_t E, m, C, ncols;
  int64_t *colptr, *rowval;  // outputs: [ncols + 1], [<= E]  (1-based)
  double *nzval;             // [<= E]
  int64_t *nnz;              // kept count
  unsigned long long *state; // [ntiles] look-back words, zeroed before the launch
  unsigned long long *claim; // tile counter, zeroed before the launch
  const int32_t *tile_col;   // [ntiles] first column (kFormCsr: row) starting at or after the tile's first entry
  BandShape band;            // kFormBand
};

template <int FORM>
__device__ __forceinline__ int64_t compact_col_start(const CompactArgs &a, int64_t c) {
  if (FORM == kFormFull) return (c < a.C ? c : a.C) * a.m;
  if (FORM == kFormBand) return c < a.ncols ? band_start(a.band, c) : a.E;
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

// The compaction over candidates of structure FORM.  CS: the colour source, of the entry (kFormCsc: TableColors over
// ecolor) or of the column (kFormBand); unused by kCopy.  The block forms pass their form object (BlockBandForm,
// BlockDenseForm), which stages each tile's block geometry and gives every candidate its row, source slot and colour.
template <int FORM, int MODE, typename CS>
__device__ __forceinline__ void compact_tiles(const CompactArgs &a, const CS &cs) {
  constexpr bool kBlock = FORM == kFormBlockBand || FORM == kFormBlockDense;
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
    if constexpr (kBlock) cs.begin_tile(a.E, t0);   // (synchronises the block)
    if constexpr (FORM == kFormCsr) cs.begin_tile(a, t0);
    // element (round u, warp w, lane) = t0 + u*kThreads + w*32 + lane: (u, w, lane) order is storage order
    double v[kRounds];
    int32_t r[kRounds];
#pragma unroll
    for (int u = 0; u < kRounds; ++u) {
      const int64_t e = t0 + u * kThreads + threadIdx.x;
      const bool in = e < a.E;
      if constexpr (kBlock) {
        // the form gives the row, the slot of the candidate buffer (kCopy) and the colour of the column (quotients)
        int32_t row = 0;
        int64_t src = e;
        uint32_t k = 0xFFFFFFFFu;
        if (in) cs.template locate<MODE != kCopy>(e, row, src, k);
        r[u] = row;
        if (MODE == kCopy) v[u] = in ? __ldcs(a.vals + src) : 0.0;
        else
          v[u] = k < (uint32_t)a.ncolors
                     ? fd_quotient<MODE>(a.Fp + (int64_t)k * a.ldF, MODE == kCentral ? a.Fm + (int64_t)k * a.ldF : a.fx,
                                         row, __ldg(a.eps + k))
                     : 0.0;
      } else if constexpr (FORM == kFormCsr) {
        // the stored index is the column; the quotient is read at the entry's row
        int32_t row = 0, c = 0;
        uint32_t k = 0xFFFFFFFFu;
        if (in) {
          c = __ldcs(a.row32 + e);
          row = cs.row_of(a, (int32_t)e);
          k = cs.colors.at(c);
        }
        r[u] = c;
        v[u] = k < (uint32_t)a.ncolors
                   ? fd_quotient<MODE>(a.Fp + (int64_t)k * a.ldF, MODE == kCentral ? a.Fm + (int64_t)k * a.ldF : a.fx, row,
                                       __ldg(a.eps + k))
                   : 0.0;
      } else {
        int64_t bc = 0, br = 0;                      // kFormBand: the candidate's column and row
        if (FORM == kFormBand) {
          if (in) band_locate(a.band, e, bc, br);
          r[u] = (int32_t)br;
        } else if (FORM == kFormFull) {
          r[u] = in ? (int32_t)(e % a.m) : 0;
        } else {
          r[u] = in ? __ldcs(a.row32 + e) : 0;
        }
        if (MODE == kCopy) {
          const int64_t src = FORM == kFormBand ? bc * a.band.w + a.band.u + br - bc : e;
          v[u] = in ? __ldcs(a.vals + src) : 0.0;
        } else {
          uint32_t k = 0xFFFFFFFFu;
          if constexpr (FORM == kFormBand) { if (in) k = cs.at(bc); }
          else if (in) k = (uint32_t)cs.p[e];
          // a column without a valid colour is never perturbed: its entries are 0 and dropped
          v[u] = k < (uint32_t)a.ncolors
                     ? fd_quotient<MODE>(a.Fp + (int64_t)k * a.ldF, MODE == kCentral ? a.Fm + (int64_t)k * a.ldF : a.fx, r[u],
                                         __ldg(a.eps + k))
                     : 0.0;
        }
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
    // first column that starts at or after t0 (kFormFull: ceil(t0 / m), at most C since t0 < E = C*m)
    int64_t clo;
    if constexpr (kBlock) clo = cs.first_col(t0);
    else clo = FORM == kFormFull   ? (t0 + a.m - 1) / a.m
               : FORM == kFormBand ? band_first_col(a.band, t0)
                                   : (int64_t)__ldg(a.tile_col + tile);
    for (int64_t c = clo + threadIdx.x; c <= a.ncols; c += kThreads) {
      int64_t p;
      if constexpr (kBlock) p = cs.col_start(a.E, c);
      else p = compact_col_start<FORM>(a, c);
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

// FULL = false: a CSC pattern's entries (kFormCsc, per-entry colours of type CT); FULL = true: the m x C block
template <bool FULL, int MODE, typename CT>
__global__ void __launch_bounds__(kThreads)
oop_compact(const CompactArgs a) {
  compact_tiles<FULL ? kFormFull : kFormCsc, MODE>(a, TableColors<CT>{reinterpret_cast<const CT *>(a.ecolor)});
}

// the in-matrix band (kFormBand), per-column colours from CS
template <int MODE, typename CS>
__global__ void __launch_bounds__(kThreads)
oop_compact_band(const CompactArgs a, const CS cs) {
  compact_tiles<kFormBand, MODE>(a, cs);
}

// ---- the block forms ----
// The entry set E of a block structure with square blocks (block K has rows and columns boff[K] .. boff[K+1] - 1), in
// column-major, row-sorted order.  Column j of block column J holds, for every block row K in K0(J) = max(0, J-u) ..
// K1(J) = min(N-1, J+l) in turn:
//   kFormBlockBand  (BandedBlockBandedMatrix) the sub-band rows max(0, j-mu) .. min(m_K-1, j+lam) of block (K, J).  The
//                   entries of block (K, J) in its columns before j number band_col_start(m_K, lam, mu, j), so column j
//                   starts at start[J] + sum_K band_col_start(m_K, lam, mu, j);
//   kFormBlockDense (BlockSkylineMatrix) every row of those blocks, one contiguous range of height h_J: the slab storage
//                   order of the in-place block-dense plan is this order, and candidate e is slot e.
// start[J] is the first entry of block column J (nblocks + 1 values: the only table besides the block offsets).  Every
// column holds at least its diagonal entry, so a tile of kTile candidates spans at most kTile columns.
struct BlockShape {
  const int32_t *boff;         // [nblocks + 1] first row / column of every block, 0-based
  const int64_t *start;        // [nblocks + 1] first entry of every block column
  const void *jcolor;          // [n] colour of column c (CT); not read with block_cyclic
  int64_t n, lam, mu, u_full;  // u_full: the block upper bandwidth as given (band-data slot of kCopy)
  int64_t w;                   // kFormBlockBand: band-data slots per column, (l+u+1)(lam+mu+1)
  int32_t nblocks, l, u;       // l, u clamped to nblocks (the same structure)
  int32_t bs;                  // kFormBlockDense with block_cyclic: the uniform block size
  int32_t block_cyclic;        // the colour is the block-cyclic closed form of matrix_colors: no colour stream
  FastDiv bw, sw;              // l+u+1 and lam+mu+1 as given (the cyclic colour's periods)
};

// entries of E in columns 0 .. j-1 of block column J (kFormBlockBand): at most l+u+1 closed forms
__host__ __device__ __forceinline__ int64_t bb_col_offset(const int32_t *boff, int32_t nblocks, int32_t l, int32_t u,
                                                          int64_t lam, int64_t mu, int32_t J, int64_t j) {
  const int32_t K0 = J - u > 0 ? J - u : 0, K1 = J + l < nblocks - 1 ? J + l : nblocks - 1;
  int64_t s = 0;
  for (int32_t K = K0; K <= K1; ++K) s += band_col_start((int64_t)boff[K + 1] - boff[K], lam, mu, j);
  return s;
}

// the block column holding candidate e: the largest J with start[J] <= e (an empty block column shares its start with
// the next one)
__device__ __forceinline__ int32_t blk_column_of(const BlockShape &b, int32_t lo, int32_t hi, int64_t e) {
  while (lo < hi) {
    const int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi + 1u) >> 1);
    if (__ldg(b.start + mid) <= e) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <typename CT>
__device__ __forceinline__ uint32_t blk_table_color(const BlockShape &b, int64_t c) {
  return (uint32_t)__ldg(reinterpret_cast<const CT *>(b.jcolor) + c);
}

// Block-banded: each tile stages the starts of the columns it spans (c_lo .. c_lo + nc, the last one the start of the
// column after the tile's last), found once per tile from the closed form; a candidate then finds its column by a search
// of that table in shared memory and its block and row by walking the blocks of the column.
struct BlockBandTile {
  int64_t cs[kTile + 1];       // start of column c_lo + i
  int32_t cj[kTile + 1];       // its block column
  int64_t c_lo, c_hi;          // the columns of the tile's first and last candidates (at most kTile columns)
  int32_t jlo, jhi;            // their block columns
  __device__ __forceinline__ int32_t nc() const { return (int32_t)(c_hi - c_lo) + 1; }
};

template <typename CT>
struct BlockBandForm {
  BlockShape b;
  BlockBandTile *t;

  // column of candidate e and its block column: a search over the block-column starts, then over the closed form
  __device__ __forceinline__ void column_of(int64_t e, int64_t &c, int32_t &J) const {
    J = blk_column_of(b, 0, b.nblocks - 1, e);
    const int64_t rel = e - __ldg(b.start + J);
    int64_t lo = 0, hi = (int64_t)__ldg(b.boff + J + 1) - __ldg(b.boff + J) - 1;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (bb_col_offset(b.boff, b.nblocks, b.l, b.u, b.lam, b.mu, J, mid) <= rel) lo = mid;
      else hi = mid - 1;
    }
    c = __ldg(b.boff + J) + lo;
  }

  __device__ __forceinline__ void begin_tile(int64_t E, int64_t t0) const {
    if (threadIdx.x < 2) {
      int64_t c;
      int32_t J;
      column_of(threadIdx.x == 0 ? t0 : (t0 + kTile < E ? t0 + kTile : E) - 1, c, J);
      if (threadIdx.x == 0) { t->c_lo = c; t->jlo = J; }
      else { t->c_hi = c; t->jhi = J; }
    }
    __syncthreads();
    const int64_t c_lo = t->c_lo;
    const int32_t nc = t->nc(), jlo = t->jlo, jhi = t->jhi;
    for (int i = threadIdx.x; i <= nc; i += kThreads) {
      const int64_t c = c_lo + i;
      int64_t s = E;
      int32_t J = jhi;
      if (c < b.n) {
        J = i < nc ? bb_block_of(b.boff, jlo, jhi, (int32_t)c) : bb_block_of(b.boff, jhi, b.nblocks - 1, (int32_t)c);
        s = __ldg(b.start + J) + bb_col_offset(b.boff, b.nblocks, b.l, b.u, b.lam, b.mu, J, c - __ldg(b.boff + J));
      }
      t->cs[i] = s;
      t->cj[i] = J;
    }
    __syncthreads();
  }

  template <bool COLOR>
  __device__ __forceinline__ void locate(int64_t e, int32_t &row, int64_t &src, uint32_t &k) const {
    int32_t lo = 0, hi = t->nc() - 1;                   // the last staged column starting at or before e
    while (lo < hi) {
      const int32_t mid = (lo + hi + 1) >> 1;
      if (t->cs[mid] <= e) lo = mid;
      else hi = mid - 1;
    }
    const int64_t c = t->c_lo + lo;
    const int32_t J = t->cj[lo];
    const int64_t j = c - __ldg(b.boff + J);
    int64_t q = e - t->cs[lo];                          // position inside the column
    const int32_t K0 = J - b.u > 0 ? J - b.u : 0, K1 = J + b.l < b.nblocks - 1 ? J + b.l : b.nblocks - 1;
    const int64_t rlo = j - b.mu > 0 ? j - b.mu : 0;    // first sub-band row of column j in every block
    int32_t K = K0;
    for (;; ++K) {                                      // the block row of the q-th entry of the column
      const int64_t rK = __ldg(b.boff + K), mK = (int64_t)__ldg(b.boff + K + 1) - rK;
      const int64_t rhi = j + b.lam < mK - 1 ? j + b.lam : mK - 1;
      const int64_t cnt = rhi >= rlo ? rhi - rlo + 1 : 0;
      if (q < cnt || K == K1) { row = (int32_t)(rK + rlo + q); break; }
      q -= cnt;
    }
    // entry (k, j) of block (K, J), k = rlo + q: slot (K - J + u)(lam + mu + 1) + (mu + k - j) of column c
    src = c * b.w + ((int64_t)K - J + b.u_full) * (b.lam + b.mu + 1) + (b.mu + rlo + q - j);
    if (COLOR)
      k = b.block_cyclic ? b.bw.mod((uint32_t)J) * b.sw.d + b.sw.mod((uint32_t)j) : blk_table_color<CT>(b, c);
  }

  // the first column that starts at or after t0, and the start of column c >= it (every column the tile's colptr pass
  // reaches is staged: a later one starts after the tile)
  __device__ __forceinline__ int64_t first_col(int64_t t0) const { return t->cs[0] == t0 ? t->c_lo : t->c_lo + 1; }
  __device__ __forceinline__ int64_t col_start(int64_t E, int64_t c) const {
    const int64_t i = c - t->c_lo;
    return i <= t->nc() ? t->cs[i] : E;
  }
};

// Block-dense: the staging of diff_scatter_block_dense (the tile's first and last block columns, and the geometry of
// up to kBdStage block columns between them in shared memory); candidate e is slot e, and its column and row come from
// (e - start_J) / h_J.
struct BlockDenseTile {
  int64_t start[kBdStage];
  int32_t h[kBdStage], row0[kBdStage], col0[kBdStage];
  int32_t jlo, jhi;
};

template <typename CT>
struct BlockDenseForm {
  BlockShape b;
  BlockDenseTile *t;

  __device__ __forceinline__ void slab(int32_t J, int32_t &h, int32_t &row0) const {
    const int32_t K0 = J - b.u > 0 ? J - b.u : 0, K1 = J + b.l < b.nblocks - 1 ? J + b.l : b.nblocks - 1;
    row0 = __ldg(b.boff + K0);
    h = __ldg(b.boff + K1 + 1) - row0;
  }

  __device__ __forceinline__ void begin_tile(int64_t E, int64_t t0) const {
    if (threadIdx.x < 2) {
      const int64_t s = threadIdx.x == 0 ? t0 : (t0 + kTile < E ? t0 + kTile : E) - 1;
      const int32_t J = blk_column_of(b, 0, b.nblocks - 1, s);
      if (threadIdx.x == 0) t->jlo = J;
      else t->jhi = J;
    }
    __syncthreads();
    const int32_t jlo = t->jlo, jhi = t->jhi;
    if (jhi - jlo < kBdStage && threadIdx.x <= jhi - jlo) {
      const int32_t J = jlo + threadIdx.x;
      t->start[threadIdx.x] = __ldg(b.start + J);
      slab(J, t->h[threadIdx.x], t->row0[threadIdx.x]);
      t->col0[threadIdx.x] = __ldg(b.boff + J);
    }
    __syncthreads();
  }

  // block column, its start, height, first row and first column of candidate e
  __device__ __forceinline__ void geometry(int64_t e, int32_t &J, int64_t &st, int32_t &h, int32_t &row0,
                                           int32_t &col0) const {
    const int32_t jlo = t->jlo, jhi = t->jhi;
    if (jhi - jlo < kBdStage) {
      const int32_t i = bd_column_of(t->start, 0, jhi - jlo, e);
      J = jlo + i; st = t->start[i]; h = t->h[i]; row0 = t->row0[i]; col0 = t->col0[i];
    } else {
      J = blk_column_of(b, jlo, jhi, e);
      st = __ldg(b.start + J);
      slab(J, h, row0);
      col0 = __ldg(b.boff + J);
    }
  }

  template <bool COLOR>
  __device__ __forceinline__ void locate(int64_t e, int32_t &row, int64_t &src, uint32_t &k) const {
    int32_t J, h, row0, col0;
    int64_t st;
    geometry(e, J, st, h, row0, col0);
    const uint32_t rel = (uint32_t)(e - st);           // < h cb[J] <= 2^32 (the plan refuses larger slabs)
    const uint32_t j = rel / (uint32_t)h;
    row = row0 + (int32_t)(rel - j * (uint32_t)h);
    src = e;
    if (COLOR) k = b.block_cyclic ? b.bw.mod((uint32_t)J) * (uint32_t)b.bs + j : blk_table_color<CT>(b, col0 + (int64_t)j);
  }

  __device__ __forceinline__ int64_t first_col(int64_t t0) const {
    int32_t J, h, row0, col0;
    int64_t st;
    geometry(t0, J, st, h, row0, col0);
    const uint32_t rel = (uint32_t)(t0 - st), j = rel / (uint32_t)h;
    return col0 + (int64_t)j + (rel == j * (uint32_t)h ? 0 : 1);
  }
  // column c >= first_col(t0): in block columns jlo .. jhi, or after the tile (its start is at least start[jhi + 1])
  __device__ __forceinline__ int64_t col_start(int64_t E, int64_t c) const {
    if (c >= b.n) return E;
    const int32_t jhi = t->jhi;
    if (c >= __ldg(b.boff + jhi + 1)) return __ldg(b.start + jhi + 1);
    const int32_t J = bb_block_of(b.boff, t->jlo, jhi, (int32_t)c);
    int32_t h, row0;
    slab(J, h, row0);
    return __ldg(b.start + J) + (c - __ldg(b.boff + J)) * (int64_t)h;
  }
};

// BandedBlockBandedMatrix (kFormBlockBand) and BlockSkylineMatrix (kFormBlockDense) entry sets; colours of type CT
template <int MODE, typename CT>
__global__ void __launch_bounds__(kThreads)
oop_compact_block_band(const CompactArgs a, const BlockShape b) {
  __shared__ BlockBandTile s_t;
  compact_tiles<kFormBlockBand, MODE>(a, BlockBandForm<CT>{b, &s_t});
}

template <int MODE, typename CT>
__global__ void __launch_bounds__(kThreads)
oop_compact_block_dense(const CompactArgs a, const BlockShape b) {
  __shared__ BlockDenseTile s_t;
  compact_tiles<kFormBlockDense, MODE>(a, BlockDenseForm<CT>{b, &s_t});
}

// ---- the CSR form ----
// A CSR pattern's entries in storage order (row order; columns within a row, repeats included, as stored).  The row of a
// candidate is found as diff_scatter_csr finds it: the tile's first and last rows by a search of the row pointer, once;
// their starts staged in shared memory when the tile spans at most kTile rows, and searched there; otherwise (long runs
// of empty rows) rowptr[rlo..rhi] is searched in global memory.
struct CsrTile {
  int32_t ptr[kTile];          // row starts rowptr[rlo .. rhi], staged
  int32_t rlo, rhi;
};

template <typename CS>
struct CsrForm {
  CS colors;                   // the colour of a column: the cyclic closed form or the table
  CsrTile *t;

  __device__ __forceinline__ void begin_tile(const CompactArgs &a, int64_t t0) const {
    if (threadIdx.x < 2) {
      const int64_t s = threadIdx.x == 0 ? t0 : (t0 + kTile < a.E ? t0 + kTile : a.E) - 1;
      const int32_t r = csr_row_of(a.colptr32, 0, (int32_t)a.ncols - 1, (int32_t)s);
      if (threadIdx.x == 0) t->rlo = r;
      else t->rhi = r;
    }
    __syncthreads();
    const int32_t rlo = t->rlo, rhi = t->rhi;
    if (rhi - rlo < kTile)
      for (int i = threadIdx.x; i <= rhi - rlo; i += kThreads) t->ptr[i] = __ldg(a.colptr32 + rlo + i);
    __syncthreads();
  }

  __device__ __forceinline__ int32_t row_of(const CompactArgs &a, int32_t e) const {
    const int32_t rlo = t->rlo, rhi = t->rhi;
    return rhi - rlo < kTile ? rlo + csr_row_of(t->ptr, 0, rhi - rlo, e) : csr_row_of(a.colptr32, rlo, rhi, e);
  }
};

// A CSR pattern (kFormCsr), per-column colours from CS; quotient modes only
template <int MODE, typename CS>
__global__ void __launch_bounds__(kThreads)
oop_compact_csr(const CompactArgs a, const CS cs) {
  static_assert(MODE != kCopy, "the CSR copy is oop_compact<false, kCopy> over (colval, rowptr)");
  __shared__ CsrTile s_t;
  compact_tiles<kFormCsr, MODE>(a, CsrForm<CS>{cs, &s_t});
}

// Plan time, block-banded result: the entries of E in every block column, sum_K band_col_start(m_K, lam, mu, cb[J])
__global__ void __launch_bounds__(kThreads)
block_band_col_counts(const int32_t *__restrict__ boff, int32_t nblocks, int32_t l, int32_t u, int64_t lam, int64_t mu,
                      int64_t *__restrict__ cnt) {
  for (int32_t J = blockIdx.x * kThreads + threadIdx.x; J < nblocks; J += gridDim.x * kThreads)
    cnt[J] = bb_col_offset(boff, nblocks, l, u, lam, mu, J, (int64_t)boff[J + 1] - boff[J]);
}

// J[r + c ldJ] += 0.0 over the band entries of the columns whose colour this rank owns, for a zero-filled dense J that
// holds their quotients: the closed-form counterpart of oop_plus_zero_slots (no destination list)
template <typename CS>
__global__ void __launch_bounds__(kThreads)
oop_band_plus_zero(double *__restrict__ J, int64_t ldJ, const BandShape b, const CS cs, const int32_t *__restrict__ local_of,
                   int32_t C) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < b.E; e += stride) {
    int64_t c, r;
    band_locate(b, e, c, r);
    const uint32_t k = cs.at(c);
    if (k >= (uint32_t)C || __ldg(local_of + k) < 0) continue;
    double *p = J + c * ldJ + r;
    *p = *p + 0.0;
  }
}

// Plan time, dense result: the (row, colour) collisions of count_color_conflicts in closed form.  Columns c1 < c2 share
// rows only when c2 - c1 <= l + u, and then exactly min(m-1, c1+l) - max(0, c2-u) + 1 of them when that is positive; each
// shared row of two columns of one valid colour is one collision.
template <typename CS>
__global__ void __launch_bounds__(kThreads)
count_band_conflicts(const BandShape b, const CS cs, int32_t C, unsigned long long *__restrict__ conflicts) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  unsigned long long bad = 0;
  for (int64_t c1 = blockIdx.x * (int64_t)kThreads + threadIdx.x; c1 < b.n; c1 += stride) {
    const uint32_t k = cs.at(c1);
    if (k >= (uint32_t)C) continue;
    const int64_t hi1 = c1 + b.l < b.m - 1 ? c1 + b.l : b.m - 1;
    const int64_t last = c1 + b.l + b.u < b.n - 1 ? c1 + b.l + b.u : b.n - 1;
    for (int64_t c2 = c1 + 1; c2 <= last; ++c2) {
      const int64_t lo2 = c2 - b.u > 0 ? c2 - b.u : 0;
      if (lo2 > hi1) break;
      if (cs.at(c2) == k) bad += (unsigned long long)(hi1 - lo2 + 1);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) bad += __shfl_xor_sync(0xffffffffu, bad, o);
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(conflicts, bad);
}

}  // namespace fdb
