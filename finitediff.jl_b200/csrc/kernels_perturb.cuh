// kernels_perturb.cuh — K3: build the perturbed point(s) of one or several colours.
//
// Reference, forward (jacobians.jl:562,584):  x1 .+= eps_k*(color==k);  f!(fx1,x1);  x1 .-= eps_k*(color==k)
// central (:603-604,:619-620) additionally  x .-= eps_k*(color==k) ... x .+= eps_k*(color==k)  on the caller's x.
// The reference never restores exactly: after colour c has been processed its components hold (x+eps_c)-eps_c
// (and (x-eps_c)+eps_c in the caller's x), and every LATER colour's f! sees those drifted values.  Because a
// component belongs to one colour only, the state of x1 at colour k has the closed form
//        x1_k[j] = c(j) <  k : (x[j]+eps_c)-eps_c      (drift replay, `drift` != 0)
//                  c(j) == k :  x[j]+eps_k
//                  else      :  x[j]
// which needs no sequential dependence between colours — any GPU can build the point of any colour from the
// pristine x and the eps table.  The caller's x is never written.
//
// Memory shape: one streaming pass, x read once (16-byte loads), every output written once (16-byte stores); the
// colour ids come as one narrow load per pair, or from the closed form of a cyclic colouring (no colour stream); the eps
// table sits in shared memory.
#pragma once
#include "common.cuh"

namespace fdb {

constexpr int kPerturbSmemColors = 1024;   // eps table staged in shared memory up to this many colours
constexpr int kPerturbMaxPoints = 4;       // colours (points) built per launch; larger batches loop on the host

struct PerturbArgs {
  const double *x;
  const double *eps;
  double *xp, *xm;
  int64_t n, ldx;
  int32_t C, drift, kcount;
  int32_t k[kPerturbMaxPoints];   // global colour id of each point
  int32_t aligned;                // x, xp, xm 16-byte aligned and ldx even
  int32_t reverse;                // walk the full tiles from the end of x to its start (the tail of x is what the pass
                                  // before left in L2; the heads of the points are what the first f! reads first)
};

template <bool CENTRAL>
__device__ __forceinline__ void perturb_one(double v, uint32_t c, bool valid, double e, int drift, uint32_t k,
                                            double &p, double &q) {
  // plus point
  p = v;
  q = v;
  if (valid) {
    if (c == k) { p = v + e; if (CENTRAL) q = v - e; }
    else if (c < k && drift) { p = (v + e) - e; if (CENTRAL) q = (v - e) + e; }
  }
}

// NP = compile-time bound on the points built per launch (1: the usual one-colour-per-callback case; kPerturbMaxPoints:
// batched callbacks).  Full tiles take the unchecked 16-byte path; the last partial tile (or unaligned buffers) the scalar one.
template <typename CS, bool CENTRAL, int NP>
__global__ void __launch_bounds__(kThreads)
perturb_colors(const PerturbArgs a, const CS colors) {
  extern __shared__ double s_eps[];
  const bool use_smem = a.C <= kPerturbSmemColors;
  if (use_smem) {
    for (int i = threadIdx.x; i < a.C; i += kThreads) s_eps[i] = a.eps[i];
    __syncthreads();
  }
  constexpr int kHalf = kTile / 2;
  const int tid2 = 2 * threadIdx.x;
  const int64_t nfull = a.aligned ? a.n / kTile : 0;
  auto eps_of = [&](uint32_t c) -> double {
    return c < (uint32_t)a.C ? (use_smem ? s_eps[c] : __ldg(a.eps + c)) : 0.0;
  };
  for (int64_t pos = blockIdx.x; pos < nfull; pos += gridDim.x) {
    const int64_t base = (a.reverse ? nfull - 1 - pos : pos) * kTile;
    const double2 va = ld_stream2(a.x + base + tid2);
    const double2 vb = ld_stream2(a.x + base + kHalf + tid2);
    uint32_t ca0, ca1, cb0, cb1;
    colors.tile(base, tid2, ca0, ca1, cb0, cb1);
    const double ea0 = eps_of(ca0), ea1 = eps_of(ca1), eb0 = eps_of(cb0), eb1 = eps_of(cb1);
    const bool ya0 = ca0 < (uint32_t)a.C, ya1 = ca1 < (uint32_t)a.C, yb0 = cb0 < (uint32_t)a.C, yb1 = cb1 < (uint32_t)a.C;
#pragma unroll
    for (int b = 0; b < NP; ++b) {
      if (NP > 1 && b >= a.kcount) break;
      const uint32_t k = (uint32_t)a.k[b];
      double p0, q0, p1, q1;
      perturb_one<CENTRAL>(va.x, ca0, ya0, ea0, a.drift, k, p0, q0);
      perturb_one<CENTRAL>(va.y, ca1, ya1, ea1, a.drift, k, p1, q1);
      st_stream2(a.xp + (int64_t)b * a.ldx + base + tid2, p0, p1);
      if (CENTRAL) st_stream2(a.xm + (int64_t)b * a.ldx + base + tid2, q0, q1);
      perturb_one<CENTRAL>(vb.x, cb0, yb0, eb0, a.drift, k, p0, q0);
      perturb_one<CENTRAL>(vb.y, cb1, yb1, eb1, a.drift, k, p1, q1);
      st_stream2(a.xp + (int64_t)b * a.ldx + base + kHalf + tid2, p0, p1);
      if (CENTRAL) st_stream2(a.xm + (int64_t)b * a.ldx + base + kHalf + tid2, q0, q1);
    }
  }
  // remainder (or everything when a buffer is not 16-byte aligned): scalar, bounds-checked
  const int64_t rem0 = nfull * kTile;
  const int64_t ntail = (a.n - rem0 + kTile - 1) / kTile;
  for (int64_t tt = blockIdx.x; tt < ntail; tt += gridDim.x) {
    for (int64_t j = rem0 + tt * kTile + threadIdx.x; j < a.n && j < rem0 + (tt + 1) * kTile; j += kThreads) {
      const double v = ld_stream(a.x + j);
      const uint32_t c = colors.at(j);
      const bool y = c < (uint32_t)a.C;
      const double e = eps_of(c);
#pragma unroll
      for (int b = 0; b < NP; ++b) {
        if (NP > 1 && b >= a.kcount) break;
        double p, q;
        perturb_one<CENTRAL>(v, c, y, e, a.drift, (uint32_t)a.k[b], p, q);
        a.xp[(int64_t)b * a.ldx + j] = p;
        if (CENTRAL) a.xm[(int64_t)b * a.ldx + j] = q;
      }
    }
  }
}

// ---- complex step (jacobians.jl:634,644):  x1 = x + im*eps*(color==k)  ...  x1 = x1 - im*eps*(color==k) ----
// The point is complex128 (re, im interleaved): re = x, im = eps on the colour's columns, 0 elsewhere.  No drift: the
// imaginary part returns to exactly 0 ((0+eps)-eps) and the real part is never touched.  xp is addressed in DOUBLES:
// point b starts at xp + b*ldx with ldx = 2 * (complex elements per point).
template <typename CS, int NP>
__global__ void __launch_bounds__(kThreads)
perturb_complex(const PerturbArgs a, const CS colors) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < a.n; j += stride) {
    const double v = ld_stream(a.x + j);
    const uint32_t c = colors.at(j);
    const double e = c < (uint32_t)a.C ? __ldg(a.eps + c) : 0.0;
#pragma unroll
    for (int b = 0; b < NP; ++b) {
      if (NP > 1 && b >= a.kcount) break;
      st_stream2(a.xp + (int64_t)b * a.ldx + 2 * j, v, c == (uint32_t)a.k[b] ? e : 0.0);
    }
  }
}

// dense complex branch (jacobians.jl:627-631): X[b] = complex(x), then only the imaginary part of one component per copy
__global__ void __launch_bounds__(kThreads)
replicate_x_complex(const double *__restrict__ x, int64_t n, int64_t ldx /* doubles */, int32_t B, double *__restrict__ X) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride) {
    const double v = x[j];
    for (int32_t b = 0; b < B; ++b) st_stream2(X + (int64_t)b * ldx + 2 * j, v, 0.0);
  }
}

__global__ void __launch_bounds__(kThreads)
set_components_complex(const double *__restrict__ eps_local, int64_t col0_local, int64_t c0, int64_t prev_c0, int32_t B,
                       int32_t prevB, int64_t ldx /* doubles */, double *__restrict__ X) {
  const int b = blockIdx.x * kThreads + threadIdx.x;
  if (b < prevB) X[(int64_t)b * ldx + 2 * (prev_c0 + b) + 1] = 0.0;                      // x1[i] = x1_save   :631
  if (b < B) X[(int64_t)b * ldx + 2 * (c0 + b) + 1] = eps_local[col0_local + b];          // x1_save + im*eps :628
}

__global__ void __launch_bounds__(kThreads)
fill_value(double *__restrict__ p, int64_t n, double v) {
  const int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x;
  if (i < n) p[i] = v;
}

// ---- dense-column branch (jacobians.jl:548-557, :590-598) ----
// The batch buffer X[b] (b < B) holds B copies of x; per batch only the one perturbed component per copy changes.

// X[b][:] = x  for b < B
__global__ void __launch_bounds__(kThreads)
replicate_x(const double *__restrict__ x, int64_t n, int64_t ldx, int32_t B, double *__restrict__ X) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride) {
    const double v = x[j];
    for (int32_t b = 0; b < B; ++b) X[(int64_t)b * ldx + j] = v;
  }
}

// batch starting at column c0 (global index): restore the previous batch's component (exact restore, as the
// reference writes the saved value back :557,:598) and set X[b][c0+b] = x[c0+b] + sign*eps[b_local].
__global__ void __launch_bounds__(kThreads)
set_components(const double *__restrict__ x, const double *__restrict__ eps_local /* indexed by local column */,
               int64_t col0_local, int64_t c0, int64_t prev_c0, int32_t B, int32_t prevB, int64_t ldx, double sign,
               double *__restrict__ X) {
  const int b = blockIdx.x * kThreads + threadIdx.x;
  if (b < prevB) {
    const int64_t pc = prev_c0 + b;
    X[(int64_t)b * ldx + pc] = x[pc];
  }
  if (b < B) {
    const int64_t c = c0 + b;
    X[(int64_t)b * ldx + c] = x[c] + sign * eps_local[col0_local + b];
  }
}

}  // namespace fdb
