// kernels_derivative.cuh — derivatives with a scalar input per step size:
//   finite_difference_derivative!(df, f, x::StridedArray, cache::DerivativeCache)   src/derivatives.jl:197-233
//   finite_difference_gradient!(df, f, x::Number, cache::GradientCache)            src/gradients.jl:477-533
// Both form one step size per scalar input and one quotient per output:
//   eps = compute_epsilon(fdtype, x, relstep, absstep, dir)   forward max(relstep*|x|, absstep)*dir, central without dir
//   forward  (f(x+eps) - f(x)) / eps          (f(x) or the cache's fx)
//   central  (f(x+eps) - f(x-eps)) * (1/(2eps))   derivative, derivatives.jl:220-222: the reciprocal is rounded first
//            (f(x+eps) - f(x-eps)) / (2eps)       scalar gradient, gradients.jl:520
//   complex  imag(f(x + im*eps)) / eps with eps = eps(Float64) = 2^-52; the point's real part is x + 0.0 (im*eps is
//            Complex(false*eps, eps) and false*eps is a strong +0.0), so a -0.0 component reads +0.0
// The derivative takes eps_i from x_i (x stride 1); the scalar gradient takes one eps from its single x for every output.
// Neither pass stores eps: the quotient pass recomputes it from x (8 B per component) instead of writing and re-reading
// a step array (16 B).  Every rounding is explicit (__dadd_rn / __dmul_rn / __ddiv_rn): the contraction
// fma(max(..), dir, x) of the forward point would change its last bit.
#pragma once
#include "common.cuh"

namespace fdb {

struct DerivSteps {
  double relstep, absstep, dir;
};

// compute_epsilon(Val(:forward) / Val(:central), x, relstep, absstep, dir)   epsilons.jl:26-29 / :50-53
template <int MODE>
__device__ __forceinline__ double deriv_eps(double v, const DerivSteps &s) {
  const double e = max_julia(__dmul_rn(s.relstep, fabs(v)), s.absstep);
  return MODE == 0 ? __dmul_rn(e, s.dir) : e;
}

constexpr double kComplexStep = 0x1p-52;   // eps(Float64)

// Perturbed points of n components into xp (plan scratch, 16-byte aligned, ldx even):
//   MODE 0 forward   xp[j] = x_j + eps_j
//   MODE 1 central   xp[j] = x_j + eps_j,  xp[ldx + j] = x_j - eps_j   (two rows: one batched f call takes both)
//   MODE 2 complex   xp is complex128: xp[j] = (x_j + 0.0, 2^-52)
// x is read once.  aligned: x is 16-byte aligned (full tiles take 16-byte loads and stores; the rest is scalar).
// The complex pass stores one element per lane: in the pair layout of the real modes (each lane storing two adjacent
// complex128 values) it ran at 80 % of its read:write mix's streaming ceiling at n = 10^8 (scripts/derivative_bench.py,
// H100 80GB HBM3 at 700 W), one element per lane at 100 %.
template <int MODE>
__global__ void __launch_bounds__(kThreads)
deriv_points(const double *__restrict__ x, int64_t n, int64_t ldx, double *__restrict__ xp, DerivSteps s, int aligned) {
  constexpr int kHalf = kTile / 2;
  const int tid2 = 2 * threadIdx.x;
  // complex: one element per lane and step, so that each warp stores one contiguous 512-byte run of complex128 (x is read
  // with 8-byte loads, which need no alignment, so the full tiles need no aligned x)
  const int64_t nfull = (aligned || MODE == 2) ? n / kTile : 0;
  for (int64_t t = blockIdx.x; t < nfull; t += gridDim.x) {
    if constexpr (MODE == 2) {
#pragma unroll
      for (int u = 0; u < kTile / kThreads; ++u) {
        const int64_t j = t * kTile + u * kThreads + threadIdx.x;
        st_stream2(xp + 2 * j, __dadd_rn(ld_stream(x + j), 0.0), kComplexStep);
      }
    } else {
#pragma unroll
      for (int u = 0; u < kPairsPerThread; ++u) {
        const int64_t j = t * kTile + u * kHalf + tid2;
        const double2 v = ld_stream2(x + j);
        const double e0 = deriv_eps<MODE>(v.x, s), e1 = deriv_eps<MODE>(v.y, s);
        st_stream2(xp + j, __dadd_rn(v.x, e0), __dadd_rn(v.y, e1));
        if (MODE == 1) st_stream2(xp + ldx + j, __dsub_rn(v.x, e0), __dsub_rn(v.y, e1));
      }
    }
  }
  const int64_t rem0 = nfull * kTile;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = rem0 + blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride) {
    const double v = ld_stream(x + j);
    if (MODE == 2) {
      st_stream2(xp + 2 * j, __dadd_rn(v, 0.0), kComplexStep);
    } else {
      const double e = deriv_eps<MODE>(v, s);
      xp[j] = __dadd_rn(v, e);
      if (MODE == 1) xp[ldx + j] = __dsub_rn(v, e);
    }
  }
}

template <int MODE, bool ELEM>
__device__ __forceinline__ double deriv_q(double p, double b, double v, const DerivSteps &s) {
  if (MODE == 2) return __ddiv_rn(p, kComplexStep);                       // imag(f) / epsilon_complex
  const double e = deriv_eps<MODE>(v, s);
  if (MODE == 0) return __ddiv_rn(__dsub_rn(p, b), e);                   // (f(x+eps) - f(x)) / eps
  if (ELEM) return __dmul_rn(__dsub_rn(p, b), __ddiv_rn(1.0, __dmul_rn(2.0, e)));   // derivatives.jl:220-222
  return __ddiv_rn(__dsub_rn(p, b), __dmul_rn(2.0, e));                  // gradients.jl:520
}

// df[i] from the f outputs, i < m.  fp: f at the plus point (MODE 2: complex128, imaginary part read); fb: the base row,
// f(x) / cache.fx (forward) or f at the minus point (central).  ELEM: eps_i from x[i] (derivative; central multiplies by
// the rounded reciprocal of 2eps); otherwise eps from x[0] for every output (scalar gradient; central divides by 2eps).
// aligned: fp, fb, df and (ELEM) x 16-byte aligned.
template <int MODE, bool ELEM>
__global__ void __launch_bounds__(kThreads)
deriv_quotient(const double *__restrict__ fp, const double *__restrict__ fb, const double *__restrict__ x,
               double *__restrict__ df, int64_t m, DerivSteps s, int aligned) {
  constexpr int kHalf = kTile / 2;
  const int tid2 = 2 * threadIdx.x;
  const double x0 = ELEM ? 0.0 : __ldg(x);
  const int64_t nfull = aligned ? m / kTile : 0;
  for (int64_t t = blockIdx.x; t < nfull; t += gridDim.x) {
#pragma unroll
    for (int u = 0; u < kPairsPerThread; ++u) {
      const int64_t j = t * kTile + u * kHalf + tid2;
      double2 p, b = make_double2(0.0, 0.0), v = make_double2(x0, x0);
      if (MODE == 2) {
        p = make_double2(ld_stream2(fp + 2 * j).y, ld_stream2(fp + 2 * j + 2).y);
      } else {
        p = ld_stream2(fp + j);
        b = ld_stream2(fb + j);
        if (ELEM) v = ld_stream2(x + j);
      }
      st_stream2(df + j, deriv_q<MODE, ELEM>(p.x, b.x, v.x, s), deriv_q<MODE, ELEM>(p.y, b.y, v.y, s));
    }
  }
  const int64_t rem0 = nfull * kTile;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = rem0 + blockIdx.x * (int64_t)kThreads + threadIdx.x; j < m; j += stride) {
    if (MODE == 2) df[j] = deriv_q<MODE, ELEM>(ld_stream(fp + 2 * j + 1), 0.0, 0.0, s);
    else df[j] = deriv_q<MODE, ELEM>(ld_stream(fp + j), ld_stream(fb + j), ELEM ? ld_stream(x + j) : x0, s);
  }
}

}  // namespace fdb
