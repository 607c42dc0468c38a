// kernels_blockband.cuh — the block-banded scatter: BandedBlockBandedMatrix band data as the Jacobian target
// (ext/FiniteDiffBlockBandedMatricesExt.jl:16-42), with square blocks.
//
// Storage: w = (l+u+1)(lam+mu+1) slots per matrix column, column-major.  Slot t = b*(lam+mu+1) + d of column c (block J,
// local column j) holds entry (k, j) of block (K, J) with K = J + b - u and k = j + d - mu, when 0 <= K < nblocks and
// 0 <= k < size(K); every other slot is outside the structure (or the matrix) and holds +0.0.  The structure is a closed
// form of (block sizes, l, u, lam, mu): no index stream is read, and the plan keeps only the block offsets.
//
// A launch walks the band data in storage order, one slot per thread and kBbPer contiguous runs of kThreads slots per
// tile, and writes every slot of the columns it defines: the columns whose colour this launch holds (the quotient, or
// +0.0 outside the structure) and, with write_other, the columns without a valid colour (+0.0).  So the launches of one
// Jacobian write every slot exactly once and J needs no zero fill.  The quotient is fd_quotient, the same IEEE sequence
// as every other scatter.
#pragma once
#include "kernels_scatter.cuh"

namespace fdb {

constexpr int kBbPer = 4;                     // slots per thread and tile
constexpr int kBbTile = kThreads * kBbPer;

struct BlockBandArgs {
  const void *jcolor;          // [n] colour of column c (CT); not read with block_cyclic
  const int32_t *boff;         // [nblocks + 1] first column of every block, 0-based
  const double *fx, *Fp, *Fm, *eps;
  const int32_t *local_of;
  double *J;
  int64_t total;               // w * n slots
  int64_t ldF;
  int32_t C, l0, G;
  int32_t write_other;         // also define the columns without a valid colour (+0.0)
  int32_t nblocks, u, mu;
  int32_t uniform;             // every block has bs.d columns: the block of a column is c / bs
  int32_t block_cyclic;        // colour of (J, j) is (J mod (l+u+1))(lam+mu+1) + (j mod (lam+mu+1)): no colour stream
  FastDiv w, sw, bs, bw;       // slots per column, lam+mu+1, uniform block size, l+u+1
};

// the largest J in [lo, hi] with off[J] <= c, given off[lo] <= c (empty blocks share their offset with the next block,
// so the result is the block that holds column c)
__device__ __forceinline__ int32_t bb_block_of(const int32_t *__restrict__ off, int32_t lo, int32_t hi, int32_t c) {
  while (lo < hi) {
    const int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi + 1u) >> 1);
    if (__ldg(off + mid) <= c) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

template <typename CT, int MODE>
__global__ void __launch_bounds__(kThreads)
diff_scatter_block_band(const BlockBandArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int32_t s_range[2];
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
  const CT *__restrict__ jcolor = reinterpret_cast<const CT *>(a.jcolor);
  const int64_t wl = a.w.d;
  const int64_t ntiles = (a.total + kBbTile - 1) / kBbTile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t s0 = tile * kBbTile;
    const int64_t c0 = s0 / wl;                          // first column of the tile (64-bit: w*n may pass 2^32)
    const uint32_t r0 = (uint32_t)(s0 - c0 * wl);        // its first slot's offset in that column (< w < 2^31)
    int32_t jlo = 0, jhi = 0;
    if (!a.uniform) {
      // the blocks of the tile's first and last columns bound every per-slot search
      __syncthreads();                                   // the previous tile's readers of s_range are done
      if (threadIdx.x < 2) {
        int64_t last = s0 + kBbTile < a.total ? s0 + kBbTile - 1 : a.total - 1;
        const int64_t c = threadIdx.x == 0 ? c0 : last / wl;
        s_range[threadIdx.x] = bb_block_of(a.boff, 0, a.nblocks - 1, (int32_t)c);
      }
      __syncthreads();
      jlo = s_range[0];
      jhi = s_range[1];
    }
#pragma unroll
    for (int p = 0; p < kBbPer; ++p) {
      const int i = p * kThreads + threadIdx.x;
      if (s0 + i >= a.total) break;
      const uint32_t q = r0 + (uint32_t)i;
      const uint32_t cc = a.w.div(q);
      const uint32_t t = q - cc * a.w.d;
      const int32_t c = (int32_t)(c0 + cc);
      const uint32_t b = a.sw.div(t);
      const int32_t d = (int32_t)(t - b * a.sw.d);
      int32_t Jb, cj;                                    // block of column c, its first column
      if (a.uniform) { Jb = (int32_t)a.bs.div((uint32_t)c); cj = Jb * (int32_t)a.bs.d; }
      else { Jb = bb_block_of(a.boff, jlo, jhi, c); cj = __ldg(a.boff + Jb); }
      const int32_t j = c - cj;
      const uint32_t k = a.block_cyclic ? a.bw.mod((uint32_t)Jb) * a.sw.d + a.sw.mod((uint32_t)j)
                                        : (uint32_t)__ldg(jcolor + c);
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
        if (slab < 0) continue;                          // another group's / rank's column
      } else if (!a.write_other) {
        continue;                                        // no valid colour: defined by the first launch of rank 0
      }
      double v = 0.0;
      if (slab >= 0) {
        const int32_t K = Jb + (int32_t)b - a.u;
        if (K >= 0 && K < a.nblocks) {
          int32_t rK, szK;                               // first row and size of block row K
          if (a.uniform) { rK = K * (int32_t)a.bs.d; szK = (int32_t)a.bs.d; }
          else { rK = __ldg(a.boff + K); szK = __ldg(a.boff + K + 1) - rK; }
          const int32_t kk = j + d - a.mu;
          if (kk >= 0 && kk < szK)
            v = fd_quotient<MODE>(a.Fp + (int64_t)slab * a.ldF, MODE == kCentral ? a.Fm + (int64_t)slab * a.ldF : a.fx,
                                  rK + kk, e);
        }
      }
      st_stream(a.J + s0 + i, v);
    }
  }
}

// Plan pass, one thread per column: the structural entries of the column, summed per colour into cnt[colour]
// (cnt[C]: the columns without a valid colour) — the LPT weights and n_entries — and whether the colouring is the
// block-cyclic closed form (*not_cyclic stays 0).
template <typename CT>
__global__ void __launch_bounds__(kThreads)
block_band_plan_pass(const CT *__restrict__ jcolor, const int32_t *__restrict__ boff, int32_t nblocks, int32_t n, int64_t l,
                     int64_t u, int64_t lam, int64_t mu, int32_t C, unsigned long long *cnt, uint32_t *not_cyclic) {
  const int64_t bw = l + u + 1, sw = lam + mu + 1;
  for (int32_t c = blockIdx.x * kThreads + threadIdx.x; c < n; c += gridDim.x * kThreads) {
    const int32_t Jb = bb_block_of(boff, 0, nblocks - 1, c);
    const int64_t j = c - boff[Jb];
    const int64_t K0 = Jb - u > 0 ? Jb - u : 0, K1 = Jb + l < nblocks - 1 ? Jb + l : nblocks - 1;
    unsigned long long entries = 0;
    for (int64_t K = K0; K <= K1; ++K) {
      const int64_t sz = boff[K + 1] - boff[K];
      const int64_t lo = j - mu > 0 ? j - mu : 0, hi = j + lam < sz - 1 ? j + lam : sz - 1;
      if (hi >= lo) entries += (unsigned long long)(hi - lo + 1);
    }
    const uint32_t k = (uint32_t)jcolor[c];
    atomicAdd(cnt + (k < (uint32_t)C ? k : (uint32_t)C), entries);
    if ((int64_t)k != (Jb % bw) * sw + j % sw) atomicOr(not_cyclic, 1u);
  }
}

// ------------------------------------------------------------------------------------------------ block-dense storage
// The block-dense scatter: BlockBandedMatrices' BlockBandedMatrix (a BlockSkylineMatrix with constant block bandwidths)
// as the Jacobian target (ext/FiniteDiffBlockBandedMatricesExt.jl:44-68), with square blocks.
//
// Storage, as that package lays it out: block column J (0-based, width cb[J]) covers block rows K0(J) = max(0, J-u) ..
// K1(J) = min(N-1, J+l), and its data is one column-major slab of height h_J = rows of those blocks, starting at slot
// start_J = sum_{J' < J} h_J' cb[J'].  Slot start_J + j h_J + r holds entry (row0_J + r, col0_J + j), where row0_J is the
// first row of block row K0(J) and col0_J the first column of block J: the rows of a slab are contiguous rows of the
// matrix.  Every slot is a structural entry.
//
// A launch walks the slabs in storage order like diff_scatter_block_band: one slot per thread, kBbPer runs of kThreads
// slots per tile.  The tile's first and last block columns are found once by a search of the start table; their
// (start, h, row0, col0) are staged in shared memory (kBdStage of them; a tile spanning more, i.e. slabs shorter than
// kBbTile / kBdStage slots, searches the table in global memory instead).  Each slot then finds its block column among
// them and its column and row from (slot - start_J) / h_J.  It writes the quotient for a column whose colour the launch
// holds and, with write_other, +0.0 for a column without a valid colour, so the launches of one Jacobian write every
// slot exactly once and J needs no zero fill.
constexpr int kBdStage = kThreads;            // block columns of a tile staged in shared memory

struct BlockDenseArgs {
  const void *jcolor;          // [n] colour of column c (CT); not read with block_cyclic
  const int32_t *boff;         // [nblocks + 1] first row / column of every block, 0-based
  const int64_t *start;        // [nblocks + 1] first slot of every block column's slab
  const double *fx, *Fp, *Fm, *eps;
  const int32_t *local_of;
  double *J;
  int64_t total;               // slots: start[nblocks]
  int64_t ldF;
  int32_t C, l0, G;
  int32_t write_other;         // also define the columns without a valid colour (+0.0)
  int32_t nblocks, l, u;
  int32_t bs;                  // block_cyclic: the uniform block size
  int32_t block_cyclic;        // colour of (J, j) is (J mod (l+u+1)) bs + j: no colour stream
  FastDiv bw;                  // l+u+1
};

// the largest J in [lo, hi] with st[J] <= s, given st[lo] <= s (an empty slab shares its start with the next one, so
// the result is the block column whose slab holds slot s)
__device__ __forceinline__ int32_t bd_column_of(const int64_t *st, int32_t lo, int32_t hi, int64_t s) {
  while (lo < hi) {
    const int32_t mid = (int32_t)(((uint32_t)lo + (uint32_t)hi + 1u) >> 1);
    if (st[mid] <= s) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// slab geometry of block column J: its height and its first row
__device__ __forceinline__ void bd_slab(const BlockDenseArgs &a, int32_t J, int32_t &h, int32_t &row0) {
  const int32_t K0 = J - a.u > 0 ? J - a.u : 0, K1 = J + a.l < a.nblocks - 1 ? J + a.l : a.nblocks - 1;
  row0 = __ldg(a.boff + K0);
  h = __ldg(a.boff + K1 + 1) - row0;
}

template <typename CT, int MODE>
__global__ void __launch_bounds__(kThreads)
diff_scatter_block_dense(const BlockDenseArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int32_t s_range[2];
  __shared__ int64_t s_start[kBdStage];
  __shared__ int32_t s_h[kBdStage], s_row0[kBdStage], s_col0[kBdStage];
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
  const CT *__restrict__ jcolor = reinterpret_cast<const CT *>(a.jcolor);
  const int64_t ntiles = (a.total + kBbTile - 1) / kBbTile;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t s0 = tile * kBbTile;
    __syncthreads();                                     // the previous tile's readers of the staged table are done
    if (threadIdx.x < 2) {
      const int64_t s = threadIdx.x == 0 ? s0 : (s0 + kBbTile < a.total ? s0 + kBbTile - 1 : a.total - 1);
      s_range[threadIdx.x] = bd_column_of(a.start, 0, a.nblocks - 1, s);
    }
    __syncthreads();
    const int32_t jlo = s_range[0], jhi = s_range[1];
    const bool staged = jhi - jlo < kBdStage;
    if (staged && threadIdx.x <= jhi - jlo) {
      const int32_t J = jlo + threadIdx.x;
      s_start[threadIdx.x] = __ldg(a.start + J);
      bd_slab(a, J, s_h[threadIdx.x], s_row0[threadIdx.x]);
      s_col0[threadIdx.x] = __ldg(a.boff + J);
    }
    __syncthreads();
#pragma unroll
    for (int p = 0; p < kBbPer; ++p) {
      const int i = p * kThreads + threadIdx.x;
      const int64_t s = s0 + i;
      if (s >= a.total) break;
      int32_t Jb, h, row0, col0;
      int64_t st;
      if (staged) {
        const int32_t t = bd_column_of(s_start, 0, jhi - jlo, s);
        Jb = jlo + t; st = s_start[t]; h = s_h[t]; row0 = s_row0[t]; col0 = s_col0[t];
      } else {
        Jb = bd_column_of(a.start, jlo, jhi, s);
        st = __ldg(a.start + Jb);
        bd_slab(a, Jb, h, row0);
        col0 = __ldg(a.boff + Jb);
      }
      const uint32_t rel = (uint32_t)(s - st);         // < h cb[J] < 2^32 (the plan refuses larger slabs)
      const uint32_t j = rel / (uint32_t)h;
      const int32_t r = (int32_t)(rel - j * (uint32_t)h);
      const int32_t c = col0 + (int32_t)j;
      const uint32_t k = a.block_cyclic ? a.bw.mod((uint32_t)Jb) * (uint32_t)a.bs + j : (uint32_t)__ldg(jcolor + c);
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
        if (slab < 0) continue;                          // another group's / rank's column
      } else if (!a.write_other) {
        continue;                                        // no valid colour: defined by the first launch of rank 0
      }
      double v = 0.0;
      if (slab >= 0)
        v = fd_quotient<MODE>(a.Fp + (int64_t)slab * a.ldF, MODE == kCentral ? a.Fm + (int64_t)slab * a.ldF : a.fx,
                              row0 + r, e);
      st_stream(a.J + s, v);
    }
  }
}

// Plan pass, one thread per column: the column's structural entries (its slab height), summed per colour into
// cnt[colour] (cnt[C]: the columns without a valid colour) — the LPT weights and n_entries — and whether the colouring is
// the block-cyclic closed form for uniform blocks of bs columns (*not_cyclic stays 0; bs = 0: never).
template <typename CT>
__global__ void __launch_bounds__(kThreads)
block_dense_plan_pass(const CT *__restrict__ jcolor, const int32_t *__restrict__ boff, int32_t nblocks, int32_t n,
                      int64_t l, int64_t u, int32_t bs, int32_t C, unsigned long long *cnt, uint32_t *not_cyclic) {
  const int64_t bw = l + u + 1;
  for (int32_t c = blockIdx.x * kThreads + threadIdx.x; c < n; c += gridDim.x * kThreads) {
    const int32_t Jb = bb_block_of(boff, 0, nblocks - 1, c);
    const int64_t j = c - boff[Jb];
    const int64_t K0 = Jb - u > 0 ? Jb - u : 0, K1 = Jb + l < nblocks - 1 ? Jb + l : nblocks - 1;
    const unsigned long long entries = (unsigned long long)(boff[K1 + 1] - boff[K0]);
    const uint32_t k = (uint32_t)jcolor[c];
    atomicAdd(cnt + (k < (uint32_t)C ? k : (uint32_t)C), entries);
    if (bs == 0 || (int64_t)k != (Jb % bw) * bs + j) atomicOr(not_cyclic, 1u);
  }
}

}  // namespace fdb
