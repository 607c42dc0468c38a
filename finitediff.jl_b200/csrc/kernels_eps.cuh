// kernels_eps.cuh — K2: step size per colour, on device, no host sync.
//
// Reference (per colour k, jacobians.jl:559-561 / :600-602):
//     @. x2 = x1 * (_color == k);  tmp = norm(x2);  eps = compute_epsilon(Val(fd), sqrt(tmp), relstep, absstep, dir)
// i.e. eps_k = max(relstep*|sqrt(||x[color==k]||_2)|, absstep) [*dir forward] (epsilons.jl:26-29,50-53).
// The colour-k components of x1 are still pristine when colour k is processed (every component belongs to
// exactly one colour), so all C sums of squares come from ONE pass over (x, colour) instead of C passes.
//
// Determinism: fixed block ranges, fixed in-block order, fixed cross-block order — no floating-point atomics.
#pragma once
#include "common.cuh"

namespace fdb {

constexpr int kEpsRegColors = 8;     // register path when C <= 8
constexpr int kEpsWindow = 512;      // colours per pass on the shared-memory path
constexpr int kEpsWarps = kThreads / 32;
constexpr int kEpsBatch = 4;        // 32-wide steps whose loads are in flight together on the window path

struct EpsParams {
  int fdtype_central;
  double relstep, absstep, dir;
};

// the step-size formula from a colour's norm
__device__ __forceinline__ double eps_from_norm(double tmp, const EpsParams &p) {
  const double a = p.relstep * fabs(sqrt(tmp));       // relstep*abs(sqrt(tmp))       :561 + epsilons.jl:28
  double e = max_julia(a, p.absstep);                 // max(.., absstep)
  if (!p.fdtype_central) e = e * p.dir;               // *dir (forward only)          epsilons.jl:28 vs :52
  return e;
}

// ... and from its fp64 sum of squares
__device__ __forceinline__ double eps_from_sumsq(double ss, const EpsParams &p) {
  return eps_from_norm(sqrt(ss), p);                  // norm(x2)                     jacobians.jl:560
}

// ---- sums of squares outside the fp64 range ----
// The reference's norm(x2) is OpenBLAS dnrm2 for n >= 32, an x87 80-bit sum that neither overflows nor underflows for
// any double, and stdlib generic_norm2 for n < 32.  A plain fp64 sum gives Inf once |x| >~ 1.34e154, and below ~1e-154
// every square is rounded to a subnormal grid of absolute step 2^-1074: n such roundings put the sum about
// n*2^-1075 / sum off, even when the sum itself is a normal number.  Below 2^-900 that loss can exceed the parity bar for
// plausible n; above it, it is under n*2^-175.
//   n >= 32: the norm is rescued when the sum is +Inf or below 2^-900.
//   n < 32:  generic_norm2 sums unscaled (as lossily as a plain fp64 sum: subnormal squares add exactly) unless
//            maxabs^2 == 0 or n*maxabs^2 overflows.  maxabs^2 == 0 is a zero sum; an overflowing n*maxabs^2 with a
//            finite sum leaves both sums accurate; so the rescue runs when the sum is 0 or +Inf.
// A NaN sum is never rescued (the step is NaN either way).  Small sums need no rescue when max(relstep*sqrt(tmp),
// absstep) is absstep for every tmp <= 2^-448 (the default absstep = relstep is such a case).  The check is made per
// colour where the step size is formed; in-range colours take no other instruction.
constexpr double kSumsqRescueBelow = 0x1p-900;

// Warp-uniform when ss is (every lane holds the same warp_sum result).
__device__ __forceinline__ bool sumsq_out_of_range(double ss, int64_t n, const EpsParams &p) {
  if (ss == INFINITY) return true;
  if (!(n < 32 ? ss == 0.0 : ss < kSumsqRescueBelow)) return false;
  return !(fabs(p.relstep) * 0x1p-224 < p.absstep);
}

// eps of a colour whose fp64 sum of squares `ss` is out of range, from its norm re-read from x (nothing writes the
// caller's x while the step sizes are computed).  Called by all 32 lanes of a warp; `value(i)` is the colour's i-th component for
// i in [0, count), or 0.0 for an index outside the colour.  The components are scaled by 2^-600 (sum +Inf) or 2^600
// (sum small): exact, and the square of every finite scaled double is then a finite normal number.  Lane-strided
// partial sums and a fixed shuffle tree: the value depends only on the colour's components in the order `value` gives.
// Not inlined, and it stores eps itself so that little is live across the call: the callers' register counts stay what
// their in-range code needs.
template <class Value>
__device__ __noinline__ void store_rescued_eps(Value value, int64_t count, double ss, EpsParams prm, double *eps_k) {
  const bool big = ss == INFINITY;
  const double down = big ? 0x1p-600 : 0x1p600;
  double acc = 0.0;
  for (int64_t i = threadIdx.x & 31; i < count; i += 32) {
    const double v = value(i) * down;
    acc += v * v;
  }
  const double e = eps_from_norm(sqrt(warp_sum(acc)) * (big ? 0x1p600 : 0x1p-600), prm);
  if ((threadIdx.x & 31) == 0) *eps_k = e;
}

// colour k's components of x in index order, through a colour source (register path) or a colour table (window path)
template <typename CS> struct ColourOfSource {
  const double *x;
  CS colors;
  uint32_t k;
  __device__ __forceinline__ double operator()(int64_t j) const { return colors.at(j) == k ? x[j] : 0.0; }
};
// colour k's components through its column list (list path): ascending, as the plan sorted them
struct ColourOfList {
  const double *x;
  const int32_t *cols;
  __device__ __forceinline__ double operator()(int64_t i) const { return x[cols[i]]; }
};

// C <= 8: per-thread register accumulators (NC = 4 or 8 of them) over the block's tiles (fixed tile -> block -> lane
// mapping; colours from a colour source, common.cuh), shuffle tree, fixed warp order; the LAST block to finish (atomic ticket) reduces the block partials in
// fixed order and applies the step-size formula — one launch, no host involvement, bit-reproducible for a given grid.
template <int NC>
__device__ __forceinline__ void sumsq_accumulate(double (&acc)[NC], double v, uint32_t c) {
  const double sq = v * v;
  // predicated adds (ISETP + @P DADD): an element belongs to exactly one colour, the other accumulators are untouched
  // — same values as adding 0.0, half the instructions of a select+add (the kernel is issue-bound)
#pragma unroll
  for (int k = 0; k < NC; ++k)
    if (c == (uint32_t)k) acc[k] += sq;
}

template <typename CS, int NC, int DEPTH = 1>
__global__ void __launch_bounds__(kThreads)
color_sumsq_reg(const double *__restrict__ x, const CS colors, int64_t n, int x_aligned, int32_t C,
                EpsParams prm, double *__restrict__ partial /* [gridDim.x][kEpsRegColors] */,
                unsigned int *__restrict__ ticket, double *__restrict__ eps, double *__restrict__ sumsq) {
  double acc[NC];
#pragma unroll
  for (int k = 0; k < NC; ++k) acc[k] = 0.0;
  constexpr int kHalf = kTile / 2;
  const int64_t nfull = x_aligned ? n / kTile : 0;
  const int tid2 = 2 * threadIdx.x;
  int64_t tile = blockIdx.x;
  if (DEPTH == 2) {
    // two tiles' loads in flight; accumulated in the same order as the one-tile loop (tile, then tile + gridDim.x)
    for (; tile + gridDim.x < nfull; tile += 2 * (int64_t)gridDim.x) {
      const double *__restrict__ xa = x + tile * kTile, *__restrict__ xb = xa + (int64_t)gridDim.x * kTile;
      const double2 a0 = ld_stream2(xa + tid2), a1 = ld_stream2(xa + kHalf + tid2);
      const double2 b0 = ld_stream2(xb + tid2), b1 = ld_stream2(xb + kHalf + tid2);
      uint32_t p0, p1, p2, p3, q0, q1, q2, q3;
      colors.tile(tile * kTile, tid2, p0, p1, p2, p3);
      colors.tile((tile + gridDim.x) * kTile, tid2, q0, q1, q2, q3);
      sumsq_accumulate<NC>(acc, a0.x, p0);
      sumsq_accumulate<NC>(acc, a0.y, p1);
      sumsq_accumulate<NC>(acc, a1.x, p2);
      sumsq_accumulate<NC>(acc, a1.y, p3);
      sumsq_accumulate<NC>(acc, b0.x, q0);
      sumsq_accumulate<NC>(acc, b0.y, q1);
      sumsq_accumulate<NC>(acc, b1.x, q2);
      sumsq_accumulate<NC>(acc, b1.y, q3);
    }
  }
  for (; tile < nfull; tile += gridDim.x) {
    const double *__restrict__ xt = x + tile * kTile;
    const double2 va = ld_stream2(xt + tid2);
    const double2 vb = ld_stream2(xt + kHalf + tid2);
    uint32_t ca0, ca1, cb0, cb1;
    colors.tile(tile * kTile, tid2, ca0, ca1, cb0, cb1);
    sumsq_accumulate<NC>(acc, va.x, ca0);
    sumsq_accumulate<NC>(acc, va.y, ca1);
    sumsq_accumulate<NC>(acc, vb.x, cb0);
    sumsq_accumulate<NC>(acc, vb.y, cb1);
  }
  // remainder (or everything, when x is not 16-byte aligned): scalar, same lane order
  {
    const int64_t rem0 = nfull * kTile;
    const int64_t ntail = (n - rem0 + kTile - 1) / kTile;
    for (int64_t tt = blockIdx.x; tt < ntail; tt += gridDim.x) {
      const int64_t base = rem0 + tt * kTile;
#pragma unroll
      for (int u = 0; u < kPairsPerThread; ++u) {
        const int64_t j = base + u * kHalf + tid2;
        if (j < n) sumsq_accumulate<NC>(acc, ld_stream(x + j), colors.at(j));
        if (j + 1 < n) sumsq_accumulate<NC>(acc, ld_stream(x + j + 1), colors.at(j + 1));
      }
    }
  }
  __shared__ double s[kEpsWarps][kEpsRegColors];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NC; ++k) {
    const double t = warp_sum(acc[k]);
    if (lane == 0) s[w][k] = t;
  }
  __syncthreads();
  if (threadIdx.x < NC) {
    double t = 0.0;
#pragma unroll
    for (int ww = 0; ww < kEpsWarps; ++ww) t += s[ww][threadIdx.x];
    __stcg(partial + (int64_t)blockIdx.x * kEpsRegColors + threadIdx.x, t);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  // last block: warp w reduces colour w over the blocks (lanes stride the blocks, then a shuffle tree)
  static_assert(kEpsWarps == kEpsRegColors, "one warp per register colour");
  if (w < C) {
    double t0 = 0.0, t1 = 0.0, t2 = 0.0, t3 = 0.0;   // 4 independent chains (fixed order): loads overlap
    int b = lane;
    for (; b + 96 < (int)gridDim.x; b += 128) {
      t0 += __ldcg(partial + (int64_t)b * kEpsRegColors + w);
      t1 += __ldcg(partial + (int64_t)(b + 32) * kEpsRegColors + w);
      t2 += __ldcg(partial + (int64_t)(b + 64) * kEpsRegColors + w);
      t3 += __ldcg(partial + (int64_t)(b + 96) * kEpsRegColors + w);
    }
    for (; b < (int)gridDim.x; b += 32) t0 += __ldcg(partial + (int64_t)b * kEpsRegColors + w);
    double t = warp_sum((t0 + t1) + (t2 + t3));
    if (lane == 0 && sumsq) sumsq[w] = t;
    if (sumsq_out_of_range(t, n, prm)) store_rescued_eps(ColourOfSource<CS>{x, colors, (uint32_t)w}, n, t, prm, eps + w);
    else if (lane == 0) eps[w] = eps_from_sumsq(t, prm);
  }
  if (threadIdx.x == 0) *ticket = 0u;   // re-arm for the next call (stream-ordered)
}

// General C: colours [k0, k0+W) per pass; every warp owns a private W-entry accumulator in shared memory and walks
// the block's range in aligned 32-column steps.  `group` (plan time, color_lane_conflicts) is the largest lane-group
// size whose aligned groups never repeat a colour: the 32/group groups of a step update the accumulators one after the
// other, lanes of a group all at once — plain shared-memory read-modify-writes, no collectives (a match.any
// version is bound by the MIO queue).  group < 4 (arbitrary colourings) falls back to combining equal
// colours with match.any in ascending lane order.  Accumulation order is fixed either way.
template <typename CT>
__global__ void __launch_bounds__(kThreads)
color_sumsq_win(const double *__restrict__ x, const CT *__restrict__ jcolor, int64_t n, int64_t chunk, int32_t k0,
                int32_t W, int32_t group, double *__restrict__ partial /* [gridDim.x][W] */) {
  extern __shared__ double sacc[];  // kEpsWarps * W
  for (int i = threadIdx.x; i < kEpsWarps * W; i += kThreads) sacc[i] = 0.0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double *acc = sacc + (size_t)w * W;
  const int64_t start = (int64_t)blockIdx.x * chunk;     // chunk is a multiple of 32: steps are aligned column groups
  int64_t end = start + chunk;
  if (end > n) end = n;
  // warp w takes the steps [start + (t*kEpsWarps + w)*32, +32); the loads of kEpsBatch steps are issued before the
  // first one is accumulated
  constexpr int64_t kStep = (int64_t)kEpsWarps * 32;
  const int my_group = lane / (group > 0 ? group : 1);
  for (int64_t base = start + (int64_t)w * 32; base < end; base += kStep * kEpsBatch) {
    double v[kEpsBatch];
    int32_t cc[kEpsBatch];
#pragma unroll
    for (int u = 0; u < kEpsBatch; ++u) {
      const int64_t j = base + u * kStep + lane;
      v[u] = 0.0;
      cc[u] = -1;
      if (j < end) {
        v[u] = ld_stream(x + j);
        cc[u] = (int32_t)(uint32_t)jcolor[j] - k0;
      }
    }
#pragma unroll
    for (int u = 0; u < kEpsBatch; ++u) {
      const int32_t c = (cc[u] >= 0 && cc[u] < W) ? cc[u] : -1;
      const double sq = v[u] * v[u];
      if (group == 32) {
        if (c >= 0) acc[c] += sq;
        __syncwarp();
      } else if (group >= 4) {
        for (int ph = 0; ph < 32 / group; ++ph) {
          if (c >= 0 && my_group == ph) acc[c] += sq;
          __syncwarp();
        }
      } else {
        const unsigned act = __ballot_sync(0xffffffffu, c >= 0);
        if (c >= 0) {
          const unsigned peers = __match_any_sync(act, c);
          double s = 0.0;
          unsigned mm = peers;
          while (mm) {
            const int l = __ffs(mm) - 1;
            mm &= mm - 1;
            s += __shfl_sync(peers, sq, l);
          }
          if (lane == __ffs(peers) - 1) acc[c] += s;
        }
        __syncwarp();
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < W; i += kThreads) {
    double t = 0.0;
#pragma unroll
    for (int ww = 0; ww < kEpsWarps; ++ww) t += sacc[(size_t)ww * W + i];
    partial[(int64_t)blockIdx.x * W + i] = t;
  }
}

// ---- many colours, CSC plans: sums of squares from the per-colour column lists ----
// The plan holds every colour's columns as one sorted list (cols_by_color, ascending inside a colour).  Colour k's sum is
// computed from ITS list alone: chunks of kEpsListChunk columns, one block per chunk (fixed lane -> element mapping, fixed
// reduction tree), then one warp per colour adds the chunk partials in order.  The value of eps_k therefore depends only
// on (x, the colour's column set) — not on the number of GPUs, the launch geometry or the other colours — and the pass
// reads 4 + 8 bytes per column instead of streaming x once per 512-colour window with shared-memory read-modify-writes
// (color_sumsq_win is slower on C4's 64 colours; it stays for plans without column lists).
constexpr int kEpsListChunk = 4096;

__global__ void __launch_bounds__(kThreads)
color_sumsq_lists(const double *__restrict__ x, const int32_t *__restrict__ cols_by_color,
                  const int64_t *__restrict__ bucket_start /* [C+1] */, const int64_t *__restrict__ chunk_base /* [C+1] */,
                  int32_t C, double *__restrict__ partial) {
  __shared__ double s[kEpsWarps];
  for (int32_t k = blockIdx.y; k < C; k += gridDim.y) {
    const int64_t b0 = bucket_start[k], len = bucket_start[k + 1] - b0;
    const int64_t nchunks = (len + kEpsListChunk - 1) / kEpsListChunk;
    for (int64_t ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
      const int64_t c0 = b0 + ch * kEpsListChunk;
      int64_t c1 = c0 + kEpsListChunk;
      if (c1 > b0 + len) c1 = b0 + len;
      double v[kEpsListChunk / kThreads];
#pragma unroll
      for (int u = 0; u < kEpsListChunk / kThreads; ++u) {          // all gathers of the chunk in flight together
        const int64_t i = c0 + u * kThreads + threadIdx.x;
        v[u] = i < c1 ? __ldg(x + __ldcs(cols_by_color + i)) : 0.0;
      }
      double acc = 0.0;
#pragma unroll
      for (int u = 0; u < kEpsListChunk / kThreads; ++u) acc += v[u] * v[u];
      acc = warp_sum(acc);
      if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
      __syncthreads();
      if (threadIdx.x == 0) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < kEpsWarps; ++w) t += s[w];
        partial[chunk_base[k] + ch] = t;
      }
      __syncthreads();
    }
  }
}

// one warp per colour: chunk partials in fixed order, then the step-size formula
__global__ void __launch_bounds__(kThreads)
finalize_eps_lists(const double *__restrict__ partial, const int64_t *__restrict__ chunk_base, int32_t C, EpsParams prm,
                   double *__restrict__ eps, double *__restrict__ sumsq, const double *__restrict__ x,
                   const int32_t *__restrict__ cols_by_color, const int64_t *__restrict__ bucket_start, int64_t n) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)kThreads + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * kThreads) >> 5;
  for (int64_t k = warp; k < C; k += nwarps) {
    const int64_t p0 = chunk_base[k], p1 = chunk_base[k + 1];
    double t = 0.0;
    for (int64_t p = p0 + lane; p < p1; p += 32) t += partial[p];
    t = warp_sum(t);
    if (lane == 0 && sumsq) sumsq[k] = t;
    if (sumsq_out_of_range(t, n, prm)) {
      const int64_t b0 = bucket_start[k];
      store_rescued_eps(ColourOfList{x, cols_by_color + b0}, bucket_start[k + 1] - b0, t, prm, eps + k);
    } else if (lane == 0) {
      eps[k] = eps_from_sumsq(t, prm);
    }
  }
}

// One warp per colour: fixed-order reduction over the block partials, then the step-size formula.
template <typename CT>
__global__ void __launch_bounds__(kThreads)
finalize_eps(const double *__restrict__ partial, int32_t nblocks, int32_t stride /* colours per partial row */,
             int32_t k0, int32_t ncolors_here, EpsParams prm, double *__restrict__ eps /* [C] */,
             double *__restrict__ sumsq /* [C] or null */, const double *__restrict__ x, const CT *__restrict__ jcolor,
             int64_t n) {
  const int lane = threadIdx.x & 31;
  const int c = (int)((blockIdx.x * (int64_t)kThreads + threadIdx.x) >> 5);
  if (c >= ncolors_here) return;
  double t = 0.0;
  for (int b = lane; b < nblocks; b += 32) t += partial[(int64_t)b * stride + c];
  t = warp_sum(t);
  if (lane == 0 && sumsq) sumsq[k0 + c] = t;
  if (sumsq_out_of_range(t, n, prm))
    store_rescued_eps(ColourOfSource<TableColors<CT>>{x, {jcolor}, (uint32_t)(k0 + c)}, n, t, prm, eps + k0 + c);
  else if (lane == 0)
    eps[k0 + c] = eps_from_sumsq(t, prm);
}

// Dense-column branch: per-COMPONENT step (jacobians.jl:550,592): eps_i = compute_epsilon(fd, x_i, relstep, absstep, dir)
__global__ void __launch_bounds__(kThreads)
component_eps(const double *__restrict__ x, int64_t c0, int64_t ncols, int fdtype_central, double relstep,
              double absstep, double dir, double *__restrict__ eps) {
  const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  if (i >= ncols) return;
  const double a = relstep * fabs(x[c0 + i]);
  double e = max_julia(a, absstep);
  if (!fdtype_central) e = e * dir;
  eps[i] = e;
}

}  // namespace fdb
