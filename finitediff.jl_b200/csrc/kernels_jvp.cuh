// kernels_jvp.cuh — Jacobian-vector product (SURVEY.md §8f rank 2): finite_difference_jvp!(jvp, f, x, v, cache, f_in)
// src/jvp.jl:238-274.  The matrix-free sibling of the coloured Jacobian: one (forward) or two (central) f! calls,
//     tmp = sqrt(abs(dot(x, v)));  eps = compute_epsilon(fdtype, tmp, relstep, absstep, dir)        (:252-253)
//     forward: f(fx1, x);  x1 = x + eps*v;  f(jvp, x1);  jvp = (jvp - fx1)/eps                        (:254-262)
//     central: x1 = x - eps*v; f(fx1, x1);  x1 = x + eps*v; f(jvp, x1);  jvp = (jvp - fx1)/(2 eps)    (:263-268)
// Three streaming kernels; eps is produced and consumed on the device (no host sync).
#pragma once
#include "common.cuh"
#include "kernels_eps.cuh"

namespace fdb {

// dot(x, v) with a fixed reduction order (tile -> lane -> warp tree -> block -> last-block-done over blocks), then eps
__global__ void __launch_bounds__(kThreads)
jvp_dot_eps(const double *__restrict__ x, const double *__restrict__ v, int64_t n, int aligned, EpsParams prm,
            double *__restrict__ partial, unsigned int *__restrict__ ticket, double *__restrict__ eps,
            double *__restrict__ dot_out) {
  double acc = 0.0;
  constexpr int kHalf = kTile / 2;
  const int tid2 = 2 * threadIdx.x;
  const int64_t nfull = aligned ? n / kTile : 0;
  for (int64_t tile = blockIdx.x; tile < nfull; tile += gridDim.x) {
    const double2 xa = ld_stream2(x + tile * kTile + tid2), va = ld_stream2(v + tile * kTile + tid2);
    const double2 xb = ld_stream2(x + tile * kTile + kHalf + tid2), vb = ld_stream2(v + tile * kTile + kHalf + tid2);
    acc += xa.x * va.x;
    acc += xa.y * va.y;
    acc += xb.x * vb.x;
    acc += xb.y * vb.y;
  }
  const int64_t rem0 = nfull * kTile;
  const int64_t ntail = (n - rem0 + kTile - 1) / kTile;
  for (int64_t tt = blockIdx.x; tt < ntail; tt += gridDim.x) {
    const int64_t base = rem0 + tt * kTile;
#pragma unroll
    for (int u = 0; u < kPairsPerThread; ++u) {
      const int64_t j = base + u * kHalf + tid2;
      if (j < n) acc += ld_stream(x + j) * ld_stream(v + j);
      if (j + 1 < n) acc += ld_stream(x + j + 1) * ld_stream(v + j + 1);
    }
  }
  __shared__ double s[kThreads / 32];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const double t = warp_sum(acc);
  if (lane == 0) s[w] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double b = 0.0;
#pragma unroll
    for (int ww = 0; ww < kThreads / 32; ++ww) b += s[ww];
    __stcg(partial + blockIdx.x, b);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s_last) return;
  if (w == 0) {
    double d = 0.0;
    for (int b = lane; b < (int)gridDim.x; b += 32) d += __ldcg(partial + b);
    d = warp_sum(d);
    if (lane == 0) {
      const double tmp = sqrt(fabs(d));                       // sqrt(abs(dot(x, v)))          jvp.jl:252
      const double a = prm.relstep * fabs(tmp);                // compute_epsilon               epsilons.jl:26-29 / :50-53
      double e = max_julia(a, prm.absstep);
      if (!prm.fdtype_central) e = e * prm.dir;
      eps[0] = e;
      if (dot_out) dot_out[0] = d;
      *ticket = 0u;
    }
  }
}

// x1 = x + eps*v  (minus = 0)   or   x1 = x - eps*v  (minus = 1)     jvp.jl:260,264,266
__global__ void __launch_bounds__(kThreads)
jvp_point(const double *__restrict__ x, const double *__restrict__ v, const double *__restrict__ eps, int minus,
          double *__restrict__ x1, int64_t n, int aligned) {
  const double e = __ldg(eps);
  constexpr int kHalf = kTile / 2;
  const int tid2 = 2 * threadIdx.x;
  const int64_t nfull = aligned ? n / kTile : 0;
  for (int64_t tile = blockIdx.x; tile < nfull; tile += gridDim.x) {
    const int64_t base = tile * kTile;
    const double2 xa = ld_stream2(x + base + tid2), va = ld_stream2(v + base + tid2);
    const double2 xb = ld_stream2(x + base + kHalf + tid2), vb = ld_stream2(v + base + kHalf + tid2);
    if (minus) {
      st_stream2(x1 + base + tid2, xa.x - e * va.x, xa.y - e * va.y);
      st_stream2(x1 + base + kHalf + tid2, xb.x - e * vb.x, xb.y - e * vb.y);
    } else {
      st_stream2(x1 + base + tid2, xa.x + e * va.x, xa.y + e * va.y);
      st_stream2(x1 + base + kHalf + tid2, xb.x + e * vb.x, xb.y + e * vb.y);
    }
  }
  const int64_t rem0 = nfull * kTile;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = rem0 + blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride) {
    const double t = e * v[j];
    x1[j] = minus ? x[j] - t : x[j] + t;
  }
}

// jvp = (jvp - fx1) / eps   or   / (2 eps)                                jvp.jl:262,268
__global__ void __launch_bounds__(kThreads)
jvp_quotient(double *__restrict__ jvp, const double *__restrict__ fx1, const double *__restrict__ eps, int central,
             int64_t m) {
  const double e = __ldg(eps);
  const double denom = central ? 2 * e : e;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < m; i += stride) jvp[i] = (jvp[i] - fx1[i]) / denom;
}

}  // namespace fdb
