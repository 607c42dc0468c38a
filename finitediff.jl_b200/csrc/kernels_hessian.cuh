// kernels_hessian.cuh — the dense Hessian of a scalar f: finite_difference_hessian!(H, f, x, cache) (src/hessians.jl:202-292).
//
// The reference evaluates f at 2n^2 + 1 points, in one global sequence:
//     p = 0                 f(x)
//     i-block i (0-based)   x + eps_i e_i, x - eps_i e_i                                   (:229-233)
//                           then for j > i: (+,+), (+,-), (-,+), (-,-) on components (i, j)  (:265-269)
// i-block i starts at S(i) = 1 + 2i + 4(i(n-1) - i(i-1)/2) and holds 2 + 4(n-1-i) points.  Every point differs from x in
// at most two components, so the B batch rows stay resident: per batch the patch kernel restores the <= 2 components the
// previous batch changed on each row and writes the new ones (O(B) bytes).  f writes its scalars (ldfx = 1) into the value
// buffer V; whole i-blocks fill one chunk of V, and the assembly kernel turns a chunk into H's entries.
//
// A rank plan (world > 1) owns the i-blocks [i_r, i_{r+1}) and evaluates f(x) followed by its own points, so its local
// sequence is {0} u [S(i_r), S(i_{r+1})): local index q is global point q == 0 ? 0 : q + off with off = S(i_r) - 1 (0 on
// one device, where the map is the identity).
#pragma once
#include "common.cuh"

namespace fdb {

// first point of i-block i (i in [0, n]; S(n) = 2n^2 + 1 is the end of the sequence)
__host__ __device__ __forceinline__ int64_t hess_block_start(int64_t i, int64_t n) {
  return 1 + 2 * i + 4 * (i * (n - 1) - i * (i - 1) / 2);
}

// point p of the sequence -> (i, j, signs): j < 0 for the diagonal pair (one component changed), s_i / s_j = +1 or -1.
// p = 0 (f(x)) gives i < 0: no component changes.
__device__ __forceinline__ void hess_decode(int64_t p, int64_t n, int64_t &i, int64_t &j, int &si, int &sj) {
  j = -1;
  si = sj = 1;
  if (p <= 0) { i = -1; return; }
  // largest i with S(i) <= p (integer binary search: S is strictly increasing on [0, n])
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (hess_block_start(mid, n) <= p) lo = mid; else hi = mid - 1;
  }
  i = lo;
  const int64_t r = p - hess_block_start(lo, n);
  if (r < 2) { si = r == 0 ? 1 : -1; return; }
  const int64_t q = r - 2;
  j = i + 1 + (q >> 2);
  const int pat = (int)(q & 3);          // 0 (+,+)  1 (+,-)  2 (-,+)  3 (-,-)
  si = pat < 2 ? 1 : -1;
  sj = (pat & 1) ? -1 : 1;
}

__device__ __forceinline__ double step_from(double xv, double e, int sign) {
  return sign > 0 ? __dadd_rn(xv, e) : __dsub_rn(xv, e);
}

// local index q of a rank's sequence -> global point
__device__ __forceinline__ int64_t hess_global(int64_t q, int64_t off) { return q == 0 ? 0 : q + off; }

// Batch of `cnt` points starting at local index p0 on rows 0..cnt-1 of X; the previous batch (prev_p0, prev_cnt) left
// its components on rows 0..prev_cnt-1.  Restores exactly (the reference writes the saved x_j / x_i back, :272-289).
__global__ void __launch_bounds__(kThreads)
hess_patch(const double *__restrict__ x, const double *__restrict__ eps, int64_t n, int64_t ldx, int64_t off, int64_t p0,
           int32_t cnt, int64_t prev_p0, int32_t prev_cnt, double *__restrict__ X) {
  for (int b = blockIdx.x * kThreads + threadIdx.x; b < max(cnt, prev_cnt); b += gridDim.x * kThreads) {
    double *row = X + (int64_t)b * ldx;
    int64_t i, j;
    int si, sj;
    if (b < prev_cnt) {
      hess_decode(hess_global(prev_p0 + b, off), n, i, j, si, sj);
      if (i >= 0) row[i] = x[i];
      if (j >= 0) row[j] = x[j];
    }
    if (b < cnt) {
      hess_decode(hess_global(p0 + b, off), n, i, j, si, sj);
      if (i >= 0) row[i] = step_from(x[i], eps[i], si);
      if (j >= 0) row[j] = step_from(x[j], eps[j], sj);
    }
  }
}

// Assembly of the i-blocks [i0, i1) held in V (V[0] = f(x); point p of the chunk at V[p - S(i0) + 1]).  Tiles of 32 x 32
// entries (i = column tile, j >= i = row tile): the lower triangle H[j, i] (column i contiguous) is stored directly, the
// upper H[i, j] through a shared-memory transpose, so both stores are coalesced; diagonal tiles write each entry once.
// Only rows [0, n) of each column are written.
//   H[i,i] = ((fpp - 2 fx) + fmm) / (eps_i * eps_i)                              (:233, epsilon^2 = epsilon*epsilon)
//   H[i,j] = (((fpp - fpm) - fmp) + fmm) / ((4 eps_i) * eps_j)                  (:268-269)
constexpr int kHT = 32;
__global__ void __launch_bounds__(kThreads)
hess_assemble(const double *__restrict__ V, const double *__restrict__ eps, int64_t n, int64_t i0, int64_t i1,
              int64_t n_tiles, double *__restrict__ H, int64_t ldH) {
  __shared__ double s[kHT][kHT + 1];
  const int64_t nt = (n + kHT - 1) / kHT;
  const int64_t ta = i0 / kHT;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const double fx2 = __dmul_rn(2.0, V[0]);
  const int64_t cs = hess_block_start(i0, n);
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    // column tile ti: tiles before it (from ta) = sum_{k=ta}^{ti-1} (nt - k)
    int64_t lo = ta, hi = (i1 - 1) / kHT;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      const int64_t before = (mid - ta) * nt - (mid * (mid - 1) / 2 - ta * (ta - 1) / 2);
      if (before <= t) lo = mid; else hi = mid - 1;
    }
    const int64_t ti = lo;
    const int64_t tj = ti + (t - ((ti - ta) * nt - (ti * (ti - 1) / 2 - ta * (ta - 1) / 2)));
    const int64_t ib = max(i0, ti * kHT), ie = min(i1, ti * kHT + kHT);
    // lower triangle + diagonal: thread tx walks the rows j of column i
    const int64_t j = tj * kHT + tx;
    for (int il = ty; il < kHT; il += kThreads / 32) {
      const int64_t i = ti * kHT + il;
      if (i < ib || i >= ie || j >= n || j < i) continue;
      const int64_t base = hess_block_start(i, n) - cs + 1;
      const double ei = eps[i];
      double v;
      if (j == i) {
        v = __ddiv_rn(__dadd_rn(__dsub_rn(V[base], fx2), V[base + 1]), __dmul_rn(ei, ei));
      } else {
        const double *q = V + base + 2 + 4 * (j - i - 1);
        v = __ddiv_rn(__dadd_rn(__dsub_rn(__dsub_rn(q[0], q[1]), q[2]), q[3]), __dmul_rn(__dmul_rn(4.0, ei), eps[j]));
      }
      H[j + i * ldH] = v;
      s[il][tx] = v;
    }
    __syncthreads();
    // upper triangle (copytri!(H, 'U'), :291): thread tx walks the rows i of column j
    const int64_t i = ti * kHT + tx;
    for (int jl = ty; jl < kHT; jl += kThreads / 32) {
      const int64_t jj = tj * kHT + jl;
      if (i >= ib && i < ie && jj < n && jj > i) H[i + jj * ldH] = s[tx][jl];
    }
    __syncthreads();
  }
}

// number of assembly tiles of the chunk [i0, i1)
inline int64_t hess_tiles(int64_t n, int64_t i0, int64_t i1) {
  if (i1 <= i0) return 0;
  const int64_t nt = (n + kHT - 1) / kHT, ta = i0 / kHT, tb = (i1 - 1) / kHT + 1;
  return (tb - ta) * nt - (tb * (tb - 1) / 2 - ta * (ta - 1) / 2);
}

}  // namespace fdb
