// kernels_staged.cuh — K5s: the graded diff+scatter kernel with its slab gathers staged through shared memory by TMA.
//
// Same arithmetic as diff_scatter_ident<FULL> (kernels_scatter.cuh):  nzval[p] = (F[color(p)][row(p)] - fx[row(p)]) / eps
// walked in J's storage order — but for ROW-LOCAL patterns (tridiagonal, banded, stencil CSC: the rows of 1024 consecutive
// entries span a few hundred rows) the per-entry dependent gathers `row -> F[k][row]` are replaced by
//   * one bulk copy per resident slab and tile (`cp.async.bulk` global -> shared, completion on an mbarrier), issued
//     two tiles ahead by one thread: every slab row crosses the memory system exactly once, fully coalesced, and the
//     loads do not wait for the row indices;
//   * 16-bit row offsets relative to the tile's window (row16[e] = row[e] - tile_w0[tile]) instead of int32 rows:
//     2 bytes less per entry on the index stream.
// The gather form is a latency-limited dependent gather; here the only global loads a warp waits for are its own
// coalesced index pairs.  cp.async.bulk and mbarrier transaction counts are Hopper (sm_90) instructions.
// Compulsory bytes per Jacobian: E*(2 + |colour| + 8) + 8*m*(slabs + 1)  (C2 forward: 650 MB; gather form: 710 MB).
// For an exact clipped band (C2's tridiagonal) the band form reads no per-entry stream at all: E*8 + 8*m*(slabs + 1)
// (+ n colour bytes unless the colouring is cyclic; C2 forward: 560 MB).
#pragma once
#include "common.cuh"
#include "kernels_scatter.cuh"

namespace fdb {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void bulk_g2s(void *sdst, const void *gsrc, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(sdst)),
               "l"(__cvta_generic_to_global(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

constexpr int kStageMaxWin = 8;        // windows per tile: C + 1 (forward: slabs + fx) or 2C (central: plus / minus slabs)
constexpr int kStagesMax = 3;          // tiles in flight per block (2 by default: 8 blocks/SM; 3 leaves 6)
constexpr int kStageMaxSmem = 46 * 1024;
// shared memory behind the staged windows: full / empty mbarriers and two phases of walk positions per stage
constexpr size_t kStageCtlBytes = 4 * kStagesMax * 8;

struct StagedArgs {
  const uint16_t *row16;     // [E] row - tile_w0[tile]                        (indexed form)
  const int32_t *tile_w0;    // [E / kTile] even first row of every full tile's window
  const int32_t *row32;      // [E] (the partial last tile of the indexed form)
  const double *fx, *Fp, *Fm, *eps;
  double *J;
  int32_t C, W;              // colours (slab == colour), window length in rows (even)
  int32_t stages;            // 2 or 3
  int64_t ldF, src_len;      // slab stride; readable doubles behind fx / every slab (even)
  int64_t E;
  int32_t j_aligned;
  unsigned long long *claim; // walk positions claimed past each block's first `stages` (0 between launches)
  int32_t reverse;           // walk the full tiles from the end of J's storage towards its start: the rows the last f! wrote
                             // most recently (the tail of the last slab) are read while they are still in L2
  // band form: the pattern is exactly the clipped band, column c holding rows max(0, c-l) .. min(m-1, c+u) in order
  const int32_t *colptr32;   // [n+1] (only the clipped head / tail columns are searched)
  int32_t l, n;
  int32_t col_a, col_b;      // interior columns [col_a, col_b): all w = l+u+1 rows present
  int32_t e_a, e_b;          // their entries [e_a, e_b) = colptr32[col_a], colptr32[col_b]
  FastDiv w;
};

// band form: column and row of entry e.  Interior entries in closed form; the few clipped head / tail columns by a
// binary search of colptr32 over their own range (head: l columns; tail: the columns after the interior)
__device__ __forceinline__ void band_locate(const StagedArgs &a, uint32_t e, uint32_t &c, uint32_t &r) {
  if (e >= (uint32_t)a.e_a && e < (uint32_t)a.e_b) {
    const uint32_t q = a.w.div(e - a.e_a);
    c = a.col_a + q;
    r = c - a.l + (e - a.e_a - q * a.w.d);
    return;
  }
  int32_t lo = e < (uint32_t)a.e_a ? 0 : a.col_b, hi = e < (uint32_t)a.e_a ? a.col_a : a.n;   // colptr32[lo] <= e
  while (hi - lo > 1) {
    const int32_t mid = (lo + hi) >> 1;
    if ((uint32_t)__ldg(a.colptr32 + mid) <= e) lo = mid; else hi = mid;
  }
  c = (uint32_t)lo;
  r = (uint32_t)max(0, lo - a.l) + (e - (uint32_t)__ldg(a.colptr32 + lo));
}

// plan time: window start (even) of every full tile, 16-bit offsets, largest span
template <typename CT>
__global__ void __launch_bounds__(kThreads)
stage_prepare(const int32_t *__restrict__ row32, int64_t ntiles, int32_t *__restrict__ tile_w0, uint16_t *__restrict__ row16,
              unsigned int *__restrict__ max_span, const CT *__restrict__ ecolor /* non-null: pack the colour into bits 12..15 */,
              int32_t C) {
  __shared__ int32_t s_min[kThreads / 32], s_max[kThreads / 32];
  __shared__ int32_t s_w0;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int32_t *rt = row32 + tile * kTile;
    int32_t r[kTile / kThreads];
    int32_t mn = INT_MAX, mx = INT_MIN;
#pragma unroll
    for (int u = 0; u < kTile / kThreads; ++u) {
      r[u] = rt[u * kThreads + threadIdx.x];
      mn = min(mn, r[u]);
      mx = max(mx, r[u]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
      mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) { s_min[threadIdx.x >> 5] = mn; s_max[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
      int32_t a = s_min[0], b = s_max[0];
      for (int w = 1; w < kThreads / 32; ++w) { a = min(a, s_min[w]); b = max(b, s_max[w]); }
      a &= ~1;
      s_w0 = a;
      tile_w0[tile] = a;
      atomicMax(max_span, (unsigned int)(b - a + 1));
    }
    __syncthreads();
    const int32_t w0 = s_w0;
#pragma unroll
    for (int u = 0; u < kTile / kThreads; ++u) {
      int32_t d = r[u] - w0;
      d = d > 65535 ? 65535 : d;
      if (ecolor) {                                      // packed form: offset < 4096 in bits 0..11, colour (15 = none) above
        uint32_t k = (uint32_t)ecolor[tile * kTile + u * kThreads + threadIdx.x];
        if (k >= (uint32_t)C) k = 15u;
        d = (d & 0xFFF) | (int32_t)(k << 12);
      }
      row16[tile * kTile + u * kThreads + threadIdx.x] = (uint16_t)d;
    }
    __syncthreads();
  }
}

// CS: colour source (common.cuh).  Indexed form: TableColors over the per-entry colours (unless PACKED); band form: the
// colour of the entry's column (the per-column table or the cyclic closed form)
// MINB: resident blocks per SM the register budget is cut for (8 -> 32 registers, 6 -> 40: no spill of the prefetched
// index registers; with TMA doing the wide loads the kernel needs fewer resident warps than the gather form)
// PACKED: few colours and short windows (C <= 14, W <= 4096): the entry's colour rides in the top 4 bits of its 16-bit row
// offset — the per-entry colour stream is not read at all (2 index bytes per entry instead of 2 + |colour|)
// EMPTYBAR: a stage is handed back to the producer through a second mbarrier (one arrival per warp) instead of a block-wide
// __syncthreads(): warps that finished a tile go straight on to the next one (A/B variant, see DESIGN.md §4)
// BAND: the pattern is an exact clipped band — every entry's row and column follow from its position (band_locate), no
// per-entry index stream is read: the kernel streams the staged windows in and J out
template <typename CS, int MODE, int MINB, bool PREFETCH, bool PACKED, bool EMPTYBAR = false, bool BAND = false>
__global__ void __launch_bounds__(kThreads, MINB)
diff_scatter_staged(const StagedArgs a, const CS colors) {
  static_assert(MODE == kForward || MODE == kCentral, "staged scatter: forward / central");
  static_assert(!(BAND && (PACKED || PREFETCH)), "band form: no index stream to pack or prefetch");
  static_assert(!(PREFETCH && EMPTYBAR), "index prefetch reads the next walk position behind the block barrier");
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int C = a.C, W = a.W;
  const int nwin = MODE == kCentral ? 2 * C : C + 1;
  const int stage_elems = nwin * W;
  const int kStages = a.stages;
  double *buf = reinterpret_cast<double *>(smem_raw);                       // [stages][nwin][W]
  uint64_t *full = reinterpret_cast<uint64_t *>(buf + kStages * stage_elems);
  uint64_t *empty = full + kStagesMax;
  int64_t *s_pos = reinterpret_cast<int64_t *>(empty + kStagesMax);         // [2][kStagesMax] walk positions
  double *s_eps = reinterpret_cast<double *>(s_pos + 2 * kStagesMax);       // [C]
  const int64_t nfull = a.E / kTile;
  constexpr int kHalf = kTile / 2;
  const int tid2 = 2 * threadIdx.x;
  // position in the walk -> tile of J's storage (the walk order is free: every tile is independent)
  auto phys = [&](int64_t t) -> int64_t { return a.reverse ? nfull - 1 - t : t; };

  // one thread feeds the pipeline: nwin bulk copies per tile, all completing on the stage's mbarrier.  A position past
  // the walk fills nothing: the bare arrival completes the stage's phase and the block reads the end of its walk there.
  auto issue = [&](int64_t pos, int s) {
    if (pos >= nfull) { mbar_arrive(full + s); return; }
    const int64_t tile = phys(pos);
    const int32_t w0 = __ldg(a.tile_w0 + tile);
    int64_t len = a.src_len - w0;
    if (len > W) len = W;
    const uint32_t bytes = (uint32_t)len * 8u;
    double *dst = buf + s * stage_elems;
    mbar_arrive_expect_tx(full + s, bytes * (uint32_t)nwin);
    for (int k = 0; k < C; ++k) bulk_g2s(dst + k * W, a.Fp + (int64_t)k * a.ldF + w0, bytes, full + s);
    if (MODE == kCentral) {
      for (int k = 0; k < C; ++k) bulk_g2s(dst + (C + k) * W, a.Fm + (int64_t)k * a.ldF + w0, bytes, full + s);
    } else {
      bulk_g2s(dst + C * W, a.fx + w0, bytes, full + s);
    }
  };
  // Walk positions: each block starts on blockIdx.x + s * gridDim.x (s < stages); every later position is claimed from
  // the counter *a.claim when a stage is refilled, `stages` iterations ahead, so a block that falls behind takes fewer
  // tiles and the blocks end together.  The position of the iteration on stage s in phase parity p sits in
  // s_pos[p * kStagesMax + s]: written by the producer before the block barrier (or the empty-stage wait) of the
  // iteration `stages` earlier, so it is read after that barrier, or after the full-stage wait that the producer's
  // arrival releases; its previous value was read before that iteration's barrier.
  // Every iteration that takes a tile claims once, so a launch makes exactly nfull claims: the one that draws nfull - 1
  // is the last, and re-arms the counter for the next launch (graph replays included) with no host step.
  auto claim = [&]() -> int64_t {
    const unsigned long long v = atomicAdd(a.claim, 1ull);
    if (v == (unsigned long long)nfull - 1) atomicExch(a.claim, 0ull);
    return (int64_t)kStages * gridDim.x + (int64_t)v;
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, kThreads / 32); }
    fence_mbar_init();
    for (int s = 0; s < kStages; ++s) s_pos[s] = min((int64_t)blockIdx.x + (int64_t)s * gridDim.x, nfull);
  }
  // everything above reads nothing the kernel before this one writes (programmatic dependent launch)
  cudaGridDependencySynchronize();
  for (int i = threadIdx.x; i < C; i += kThreads) s_eps[i] = a.eps[i];
  __syncthreads();
  if (threadIdx.x == 0)
    for (int s = 0; s < kStages; ++s) issue(s_pos[s], s);

  auto value = [&](const double *__restrict__ win, uint32_t r, uint32_t k) -> double {
    if (k >= (uint32_t)C) return 0.0;                    // column without a valid colour: stays 0 (fill_matrix!)
    const double e = s_eps[k];
    const double hi = win[k * W + r];
    const double lo = MODE == kCentral ? win[(C + k) * W + r] : win[C * W + r];
    const double d = hi - lo;                            // jacobians.jl:565 / :607 — same IEEE operations
    return d / (MODE == kCentral ? 2 * e : e);
  };

  // window offsets and colours of the lane's two entry pairs.  Indexed form: coalesced index pairs, independent of the
  // staged data (with PREFETCH loaded ONE TILE AHEAD, so their latency overlaps the previous tile's wait + arithmetic).
  // Band form: derived from the tile's position; an interior tile (all its columns complete) takes one division per pair.
  struct Idx { ushort2 ra, rb; uint32_t ka0, ka1, kb0, kb1; };
  auto load_idx = [&](int64_t tile) {
    Idx x;
    if constexpr (BAND) {
      const uint32_t e0 = (uint32_t)(tile * kTile), w0 = (uint32_t)__ldg(a.tile_w0 + tile);
      const bool interior = e0 >= (uint32_t)a.e_a && e0 + kTile <= (uint32_t)a.e_b;
      auto pair = [&](uint32_t e, ushort2 &rr, uint32_t &k0, uint32_t &k1) {
        uint32_t c, r, c1, r1;
        if (interior) {
          const uint32_t v = e - a.e_a, q = a.w.div(v), o = v - q * a.w.d;
          c = a.col_a + q;
          r = c - a.l + o;
          const bool wrap = o + 1 == a.w.d;                  // the pair's second entry starts the next column
          c1 = wrap ? c + 1 : c;
          r1 = wrap ? c1 - a.l : r + 1;
        } else {
          band_locate(a, e, c, r);
          band_locate(a, e + 1, c1, r1);
        }
        rr.x = (unsigned short)(r - w0);
        rr.y = (unsigned short)(r1 - w0);
        k0 = colors.at(c);
        k1 = c1 == c ? k0 : colors.at(c1);
      };
      pair(e0 + tid2, x.ra, x.ka0, x.ka1);
      pair(e0 + kHalf + tid2, x.rb, x.kb0, x.kb1);
    } else {
      const uint16_t *__restrict__ rt = a.row16 + tile * kTile;
      x.ra = __ldcs(reinterpret_cast<const ushort2 *>(rt + tid2));
      x.rb = __ldcs(reinterpret_cast<const ushort2 *>(rt + kHalf + tid2));
      if (PACKED) {
        x.ka0 = x.ra.x >> 12; x.ka1 = x.ra.y >> 12; x.kb0 = x.rb.x >> 12; x.kb1 = x.rb.y >> 12;
        x.ra.x &= 0xFFF; x.ra.y &= 0xFFF; x.rb.x &= 0xFFF; x.rb.y &= 0xFFF;
      } else {
        colors.tile(tile * kTile, tid2, x.ka0, x.ka1, x.kb0, x.kb1);
      }
    }
    return x;
  };
  int s = 0;
  uint32_t parity = 0;
  Idx nx{};
  if (PREFETCH && s_pos[0] < nfull) nx = load_idx(phys(s_pos[0]));
  for (;;) {
    int64_t pos;
    if (EMPTYBAR) {                                       // the position is released with the stage
      while (!mbar_try_wait(full + s, parity)) {}
      pos = s_pos[parity * kStagesMax + s];
      if (pos >= nfull) break;
    } else {                                              // written behind an earlier block barrier
      pos = s_pos[parity * kStagesMax + s];
      if (pos >= nfull) break;
    }
    const int64_t tile = phys(pos);
    double *__restrict__ Jt = a.J + tile * kTile;
    const Idx cur = PREFETCH ? nx : load_idx(tile);
    if (PREFETCH) {                                       // the next iteration's position: stage s + 1, or stage 0 of the next phase
      const int64_t pn = s + 1 == kStages ? s_pos[(parity ^ 1u) * kStagesMax] : s_pos[parity * kStagesMax + s + 1];
      if (pn < nfull) nx = load_idx(phys(pn));
    }
    const ushort2 ra = cur.ra, rb = cur.rb;
    const uint32_t ka0 = cur.ka0, ka1 = cur.ka1, kb0 = cur.kb0, kb1 = cur.kb1;
    // the position this stage is refilled with (the iteration `stages` later): claimed while the tile is computed
    int64_t *refill = s_pos + (parity ^ 1u) * kStagesMax + s;
    if (threadIdx.x == 0) *refill = claim();
    if (!EMPTYBAR) while (!mbar_try_wait(full + s, parity)) {}
    const double *__restrict__ win = buf + s * stage_elems;
    const double va0 = value(win, ra.x, ka0), va1 = value(win, ra.y, ka1);
    const double vb0 = value(win, rb.x, kb0), vb1 = value(win, rb.y, kb1);
    if (a.j_aligned) {
      st_stream2(Jt + tid2, va0, va1);
      st_stream2(Jt + kHalf + tid2, vb0, vb1);
    } else {
      Jt[tid2] = va0; Jt[tid2 + 1] = va1; Jt[kHalf + tid2] = vb0; Jt[kHalf + tid2 + 1] = vb1;
    }
    if (EMPTYBAR) {
      __syncwarp();
      if ((threadIdx.x & 31) == 0) mbar_arrive(empty + s);              // this warp is done with stage s
      if (threadIdx.x == 0) {
        while (!mbar_try_wait(empty + s, parity)) {}                     // ... and so are the other seven: refill it
        issue(*refill, s);
      }
    } else {
      __syncthreads();                                    // every lane is done with stage s: refill it
      if (threadIdx.x == 0) issue(*refill, s);
    }
    if (++s == kStages) { s = 0; parity ^= 1u; }
  }
  // the last, partial tile (E % kTile entries): gather form, one block
  const int64_t rem0 = nfull * kTile;
  if (rem0 < a.E && blockIdx.x == (unsigned)(nfull % gridDim.x)) {
    for (int64_t e = rem0 + threadIdx.x; e < a.E; e += kThreads) {
      uint32_t k, r;
      if constexpr (BAND) {
        uint32_t c;
        band_locate(a, (uint32_t)e, c, r);
        k = colors.at(c);
      } else {
        k = colors.at(e);
        r = (uint32_t)a.row32[e];
      }
      double v = 0.0;
      if (k < (uint32_t)C)
        v = fd_quotient<MODE>(a.Fp + (int64_t)k * a.ldF, MODE == kCentral ? a.Fm + (int64_t)k * a.ldF : a.fx, r, s_eps[k]);
      a.J[e] = v;
    }
  }
}

}  // namespace fdb
