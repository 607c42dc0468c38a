// synth_fns.cu — libfdjac_synth.so: synthetic f!(dx, x) device functions for the bench / parity harness
// (include/fdjac_synth.h).  Bit-identical to oracle/synth_fns.c: explicit __dadd_rn/__dmul_rn, same evaluation order.
#include "../../include/fdjac_synth.h"

#include <cuda_runtime.h>
#include <cstdint>

namespace {
constexpr int kT = 256;

__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }

// dx[i] = (x[i-1] - 2*x[i]) + x[i+1];  dx[0] = -2*x[0] + x[1];  dx[n-1] = x[n-2] - 2*x[n-1]
__global__ void __launch_bounds__(kT) k_tridiag(double *__restrict__ fx, const double *__restrict__ x, int64_t n,
                                                int64_t ldfx, int64_t ldx) {
  const double *xb = x + (int64_t)blockIdx.y * ldx;
  double *fb = fx + (int64_t)blockIdx.y * ldfx;
  const int64_t stride = (int64_t)gridDim.x * kT * 2;
  for (int64_t i0 = (blockIdx.x * (int64_t)kT + threadIdx.x) * 2; i0 < n; i0 += stride) {
    // two rows per thread: one 16-byte load of (x[i0], x[i0+1]) plus the two neighbours
    if (i0 + 1 < n) {
      const double2 c = *reinterpret_cast<const double2 *>(xb + i0);
      const double lft = i0 > 0 ? __ldg(xb + i0 - 1) : 0.0;
      const double rgt = i0 + 2 < n ? __ldg(xb + i0 + 2) : 0.0;
      double a, b;
      if (i0 == 0) a = add(mul(-2.0, c.x), c.y);
      else a = add(sub(lft, mul(2.0, c.x)), c.y);
      if (i0 + 1 == n - 1) b = sub(c.x, mul(2.0, c.y));
      else b = add(sub(c.x, mul(2.0, c.y)), rgt);
      __stcs(reinterpret_cast<double2 *>(fb + i0), make_double2(a, b));
    } else {
      // last row of an odd-length vector
      const double c = xb[i0];
      fb[i0] = n == 1 ? mul(-2.0, c) : sub(__ldg(xb + i0 - 1), mul(2.0, c));
    }
  }
}

__global__ void __launch_bounds__(kT) k_lap5(double *__restrict__ out, const double *__restrict__ x, int64_t g,
                                             int64_t ldfx, int64_t ldx) {
  const double *xb = x + (int64_t)blockIdx.z * ldx;
  double *ob = out + (int64_t)blockIdx.z * ldfx;
  const int64_t j = blockIdx.y;  // grid column
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < g; i += (int64_t)gridDim.x * kT) {
    const int64_t im = i > 0 ? i - 1 : 0, ip = i + 1 < g ? i + 1 : g - 1;
    const int64_t jm = j > 0 ? j - 1 : 0, jp = j + 1 < g ? j + 1 : g - 1;
    double s = xb[i + j * g];
    s = add(s, xb[im + j * g]);
    s = add(s, xb[ip + j * g]);
    s = add(s, xb[i + jm * g]);
    s = add(s, xb[i + jp * g]);
    ob[i + j * g] = s;
  }
}

// ELL layout [K][m]: entry p of row i at p*m + i -> the index / coefficient streams are read fully coalesced
__global__ void __launch_bounds__(kT) k_ellrows(double *__restrict__ fx, const double *__restrict__ x, int64_t m, int K,
                                                const int32_t *__restrict__ cols, const double *__restrict__ coef,
                                                int64_t ldfx, int64_t ldx) {
  const double *xb = x + (int64_t)blockIdx.y * ldx;
  double *fb = fx + (int64_t)blockIdx.y * ldfx;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < m; i += (int64_t)gridDim.x * kT) {
    const double x0 = __ldg(xb + __ldcs(cols + i));
    double s = mul(__ldcs(coef + i), x0);
    for (int p = 1; p < K; ++p) s = add(s, mul(__ldcs(coef + (int64_t)p * m + i), __ldg(xb + __ldcs(cols + (int64_t)p * m + i))));
    s = add(s, mul(0.1, mul(x0, x0)));
    fb[i] = s;
  }
}

// blocked sum: blocks of 1024 summed sequentially (one thread each — tiny), then block sums sequentially
__global__ void __launch_bounds__(kT) k_block_sums(const double *__restrict__ x, int64_t n, int64_t ldx,
                                                   double *__restrict__ bs, int64_t nblk) {
  // one warp per 1024-block: lane l sums x[b + l + 32 j] (j ascending, coalesced), xor butterfly — the order of
  // oracle/synth_fns.c:synth_blocked_sum
  const double *xb = x + (int64_t)blockIdx.y * ldx;
  const int lane = threadIdx.x & 31;
  for (int64_t b = blockIdx.x * (int64_t)(kT / 32) + (threadIdx.x >> 5); b < nblk; b += (int64_t)gridDim.x * (kT / 32)) {
    const int64_t s0 = b * 1024;
    double s = 0.0;
#pragma unroll 8
    for (int j = 0; j < 32; ++j) {
      const int64_t idx = s0 + lane + 32 * j;
      s = add(s, idx < n ? xb[idx] : 0.0);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = add(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) bs[(int64_t)blockIdx.y * nblk + b] = s;
  }
}

// S[p] = (block sums of point p added in block order) / n, left in bs[p*nblk] (only thread p touches row p)
__global__ void __launch_bounds__(kT) k_point_sums(double *__restrict__ bs, int64_t nblk, int64_t n, int64_t batch) {
  const int64_t p = blockIdx.x * (int64_t)kT + threadIdx.x;
  if (p >= batch) return;
  double t = 0.0;
  for (int64_t b = 0; b < nblk; ++b) t = add(t, bs[p * nblk + b]);
  bs[p * nblk] = __ddiv_rn(t, (double)n);
}

__global__ void __launch_bounds__(kT) k_rank1(double *__restrict__ fx, const double *__restrict__ x, int64_t n,
                                              const double *__restrict__ w, const double *__restrict__ bs, int64_t nblk,
                                              int64_t ldfx, int64_t ldx, int vec_ok) {
  const double *xb = x + (int64_t)blockIdx.y * ldx;
  double *fb = fx + (int64_t)blockIdx.y * ldfx;
  const double s = __ldg(bs + (int64_t)blockIdx.y * nblk);
  const int64_t stride = (int64_t)gridDim.x * kT;
  if (vec_ok) {
    // two rows per lane, two independent 16-byte loads of x in flight; x and f are read / written once (streaming), w is
    // shared by every point of the batch (cacheable)
    const int64_t n2 = n >> 1;
    const double2 *x2 = reinterpret_cast<const double2 *>(xb), *w2 = reinterpret_cast<const double2 *>(w);
    double2 *f2 = reinterpret_cast<double2 *>(fb);
    int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x;
    for (; i + stride < n2; i += 2 * stride) {
      const double2 a = __ldcs(x2 + i), b = __ldcs(x2 + i + stride);
      const double2 wa = __ldg(w2 + i), wb = __ldg(w2 + i + stride);
      __stcs(f2 + i, make_double2(add(mul(a.x, a.x), mul(wa.x, s)), add(mul(a.y, a.y), mul(wa.y, s))));
      __stcs(f2 + i + stride, make_double2(add(mul(b.x, b.x), mul(wb.x, s)), add(mul(b.y, b.y), mul(wb.y, s))));
    }
    for (; i < n2; i += stride) {
      const double2 a = __ldcs(x2 + i), wa = __ldg(w2 + i);
      __stcs(f2 + i, make_double2(add(mul(a.x, a.x), mul(wa.x, s)), add(mul(a.y, a.y), mul(wa.y, s))));
    }
    if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) { const double v = xb[n - 1]; fb[n - 1] = add(mul(v, v), mul(w[n - 1], s)); }
    return;
  }
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < n; i += stride) {
    const double v = xb[i];
    fb[i] = add(mul(v, v), mul(w[i], s));
  }
}

// Slice-aware tridiagonal stencil (column-block sharded runs): rows [row0, row0+nrows) of the n-row problem, reading a
// slice of x whose element 0 is global component x0.  Same expression per row as k_tridiag => bit-identical values.
__global__ void __launch_bounds__(kT) k_tridiag_rows(double *__restrict__ fx, const double *__restrict__ x, int64_t n,
                                                     int64_t row0, int64_t nrows, int64_t x0, int64_t ldfx, int64_t ldx) {
  const double *xb = x + (int64_t)blockIdx.y * ldx - x0;     // xb[global index]
  double *fb = fx + (int64_t)blockIdx.y * ldfx;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < nrows; i += (int64_t)gridDim.x * kT) {
    const int64_t r = row0 + i;
    const double c = xb[r];
    double o;
    if (n == 1) o = mul(-2.0, c);
    else if (r == 0) o = add(mul(-2.0, c), xb[1]);
    else if (r == n - 1) o = sub(xb[r - 1], mul(2.0, c));
    else o = add(sub(xb[r - 1], mul(2.0, c)), xb[r + 1]);
    fb[i] = o;
  }
}

// complex twin of k_tridiag (complex-step path): complex128 arrays as double2; the stencil on re and im separately
__global__ void __launch_bounds__(kT) k_tridiag_c(double2 *__restrict__ fx, const double2 *__restrict__ x, int64_t n,
                                                  int64_t ldfx, int64_t ldx) {
  const double2 *xb = x + (int64_t)blockIdx.y * ldx;
  double2 *fb = fx + (int64_t)blockIdx.y * ldfx;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kT) {
    const double2 c = xb[i];
    double2 o;
    if (n == 1) { o.x = mul(-2.0, c.x); o.y = mul(-2.0, c.y); }
    else if (i == 0) { const double2 r = xb[1]; o.x = add(mul(-2.0, c.x), r.x); o.y = add(mul(-2.0, c.y), r.y); }
    else if (i == n - 1) { const double2 l = xb[i - 1]; o.x = sub(l.x, mul(2.0, c.x)); o.y = sub(l.y, mul(2.0, c.y)); }
    else {
      const double2 l = xb[i - 1], r = xb[i + 1];
      o.x = add(sub(l.x, mul(2.0, c.x)), r.x);
      o.y = add(sub(l.y, mul(2.0, c.y)), r.y);
    }
    fb[i] = o;
  }
}

// complex twin of k_ellrows (complex-step path): the same sum with complex x, written out on (re, im):
// coef*(a+ib) = coef*a + i*coef*b;  x0^2 = (a*a - b*b) + i*(a*b + a*b)
__global__ void __launch_bounds__(kT) k_ellrows_c(double2 *__restrict__ fx, const double2 *__restrict__ x, int64_t m, int K,
                                                  const int32_t *__restrict__ cols, const double *__restrict__ coef,
                                                  int64_t ldfx, int64_t ldx) {
  const double2 *xb = x + (int64_t)blockIdx.y * ldx;
  double2 *fb = fx + (int64_t)blockIdx.y * ldfx;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < m; i += (int64_t)gridDim.x * kT) {
    const double2 x0 = xb[cols[i]];
    const double c0 = coef[i];
    double re = mul(c0, x0.x), im = mul(c0, x0.y);
    for (int p = 1; p < K; ++p) {
      const double c = coef[(int64_t)p * m + i];
      const double2 v = xb[cols[(int64_t)p * m + i]];
      re = add(re, mul(c, v.x));
      im = add(im, mul(c, v.y));
    }
    re = add(re, mul(0.1, sub(mul(x0.x, x0.x), mul(x0.y, x0.y))));
    im = add(im, mul(0.1, add(mul(x0.x, x0.y), mul(x0.x, x0.y))));
    fb[i] = make_double2(re, im);
  }
}

// ---- scalar functions f: R^n -> R (Hessian / gradient harness), one point per block.  Blocked order of k_block_sums:
// 1024-element blocks, lane l of a warp sums the terms of elements l, l+32, ..., l+992 of its block ascending, an xor
// butterfly adds the lanes, then thread 0 adds the block sums in block order.  Twins: scalar_oracle/synth_scalar.c.
//   KIND 0 (quartic): f = sum_i (a_i x_i^4 + x_i x_{i+1}) + (sum_i w_i x_i)^2 / (2n)
//   KIND 1 (sumsq):   f = sum_i x_i^2  (sum(abs2, x))
//   KIND 2 (guarded): f = sum_i (g(a_i x_i^4, 1/4) + g(x_i x_{i+1}, -1/2) + z_i) + s^2 / (2n),
//                     s = g(sum_i g(w_i x_i, 3/4), 3/2),  z_i = (!isnan(x_i) && signbit(x_i)) ? w_i : 0,
//                     g(t, c) = (isfinite(t) && |t| <= 2^500) ? t : c
//                     finite for every input; depends on the sign of a zero, never on a NaN's sign or payload
__device__ __forceinline__ double butterfly(double s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s = add(s, __shfl_xor_sync(0xffffffffu, s, o));
  return s;
}

__device__ __forceinline__ double guard(double t, double c) { return (isfinite(t) && fabs(t) <= 0x1p500) ? t : c; }

template <int KIND>
__global__ void k_scalar(double *__restrict__ fx, const double *__restrict__ x, int64_t n, const double *__restrict__ a,
                         const double *__restrict__ w, int64_t ldfx, int64_t ldx) {
  extern __shared__ double sh[];   // [2][nblk] block sums
  const double *xb = x + (int64_t)blockIdx.x * ldx;
  const int64_t nblk = (n + 1023) / 1024;
  const int lane = threadIdx.x & 31;
  for (int64_t b = threadIdx.x >> 5; b < nblk; b += blockDim.x >> 5) {
    double s1 = 0.0, s2 = 0.0;
    for (int j = 0; j < 32; ++j) {
      const int64_t i = b * 1024 + lane + 32 * j;
      double t1 = 0.0, t2 = 0.0;
      if (i < n) {
        const double v = xb[i];
        if (KIND == 0) {
          const double q = mul(v, v);
          t1 = mul(a[i], mul(q, q));
          if (i + 1 < n) t1 = add(t1, mul(v, xb[i + 1]));
          t2 = mul(w[i], v);
        } else if (KIND == 2) {
          const double q = mul(v, v);
          t1 = guard(mul(a[i], mul(q, q)), 0.25);
          if (i + 1 < n) t1 = add(t1, guard(mul(v, xb[i + 1]), -0.5));
          t1 = add(t1, (!isnan(v) && signbit(v)) ? w[i] : 0.0);
          t2 = guard(mul(w[i], v), 0.75);
        } else {
          t1 = mul(v, v);
        }
      }
      s1 = add(s1, t1);
      s2 = add(s2, t2);
    }
    s1 = butterfly(s1);
    s2 = butterfly(s2);
    if (lane == 0) { sh[b] = s1; sh[nblk + b] = s2; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S1 = 0.0, S2 = 0.0;
    for (int64_t b = 0; b < nblk; ++b) { S1 = add(S1, sh[b]); S2 = add(S2, sh[nblk + b]); }
    if (KIND == 2) {
      const double s = guard(S2, 1.5);
      fx[(int64_t)blockIdx.x * ldfx] = n > 0 ? add(S1, __ddiv_rn(mul(s, s), (double)(2 * n))) : S1;
    } else {
      fx[(int64_t)blockIdx.x * ldfx] = (KIND == 0 && n > 0) ? add(S1, __ddiv_rn(mul(S2, S2), (double)(2 * n))) : S1;
    }
  }
}

// complex128 twin of the quartic (complex-step gradients): the same sums on (re, im) with Julia's complex product
// z*w = (zr*wr - zi*wi) + i(zr*wi + zi*wr); a_i, w_i and 2n are real
__device__ __forceinline__ double2 cmul(double2 z, double2 v) {
  return make_double2(sub(mul(z.x, v.x), mul(z.y, v.y)), add(mul(z.x, v.y), mul(z.y, v.x)));
}

__global__ void k_scalar_c(double2 *__restrict__ fx, const double2 *__restrict__ x, int64_t n, const double *__restrict__ a,
                           const double *__restrict__ w, int64_t ldfx, int64_t ldx) {
  extern __shared__ double sh[];   // [4][nblk]
  const double2 *xb = x + (int64_t)blockIdx.x * ldx;
  const int64_t nblk = (n + 1023) / 1024;
  const int lane = threadIdx.x & 31;
  for (int64_t b = threadIdx.x >> 5; b < nblk; b += blockDim.x >> 5) {
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int j = 0; j < 32; ++j) {
      const int64_t i = b * 1024 + lane + 32 * j;
      double t[4] = {0.0, 0.0, 0.0, 0.0};
      if (i < n) {
        const double2 v = xb[i];
        const double2 q = cmul(v, v), q2 = cmul(q, q);
        double2 t1 = make_double2(mul(a[i], q2.x), mul(a[i], q2.y));
        if (i + 1 < n) { const double2 u = cmul(v, xb[i + 1]); t1 = make_double2(add(t1.x, u.x), add(t1.y, u.y)); }
        t[0] = t1.x; t[1] = t1.y; t[2] = mul(w[i], v.x); t[3] = mul(w[i], v.y);
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) s[k] = add(s[k], t[k]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] = butterfly(s[k]);
    if (lane == 0) for (int k = 0; k < 4; ++k) sh[k * nblk + b] = s[k];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S[4] = {0.0, 0.0, 0.0, 0.0};
    for (int64_t b = 0; b < nblk; ++b) for (int k = 0; k < 4; ++k) S[k] = add(S[k], sh[k * nblk + b]);
    double2 f = make_double2(S[0], S[1]);
    if (n > 0) {
      const double2 sq = cmul(make_double2(S[2], S[3]), make_double2(S[2], S[3]));
      const double d = (double)(2 * n);
      f = make_double2(add(f.x, __ddiv_rn(sq.x, d)), add(f.y, __ddiv_rn(sq.y, d)));
    }
    fx[(int64_t)blockIdx.x * ldfx] = f;
  }
}

// ---- elementwise and scalar-input functions (derivative / scalar -> vector gradient harness), one output per thread.
// Output i of point b:  p_i(v) = (a_i (v^2 v) + w_i v^2) + v  with v = x[b*ldx + i] (SCALAR = false: elementwise, for
// finite_difference_derivative!) or v = x[b*ldx] (SCALAR = true: m outputs of one scalar t, for the scalar -> vector
// gradient).  GUARD: every term through guard(), plus z = (!isnan(v) && signbit(v)) ? w_i : 0, so p_i is finite for every
// v and sees the sign of a zero.  Twins: scalar_oracle/synth_scalar.c.
template <bool GUARD>
__device__ __forceinline__ double poly_at(double v, double a, double w) {
  const double q = mul(v, v), c = mul(q, v);
  if (!GUARD) return add(add(mul(a, c), mul(w, q)), v);
  const double t = add(add(guard(mul(a, c), 0.25), guard(mul(w, q), -0.5)), guard(v, 0.75));
  return add(t, (!isnan(v) && signbit(v)) ? w : 0.0);
}

template <bool GUARD, bool SCALAR>
__global__ void __launch_bounds__(kT) k_poly(double *__restrict__ fx, const double *__restrict__ x, int64_t n,
                                             const double *__restrict__ a, const double *__restrict__ w, int64_t ldfx,
                                             int64_t ldx) {
  const double *xb = x + (int64_t)blockIdx.y * ldx;
  double *fb = fx + (int64_t)blockIdx.y * ldfx;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kT)
    fb[i] = poly_at<GUARD>(SCALAR ? xb[0] : xb[i], a[i], w[i]);
}

// complex128 twin: the same terms with Julia's complex product; a_i, w_i real.  GUARD: guard() on the real and the
// imaginary part of each term, and z (from the sign of the real part) added to the IMAGINARY part, the one a complex step
// reads.
template <bool GUARD>
__device__ __forceinline__ double2 poly_at_c(double2 v, double a, double w) {
  const double2 q = cmul(v, v), c = cmul(q, v);
  double2 t1 = make_double2(mul(a, c.x), mul(a, c.y)), t2 = make_double2(mul(w, q.x), mul(w, q.y)), t3 = v;
  if (GUARD) {
    t1 = make_double2(guard(t1.x, 0.25), guard(t1.y, 0.25));
    t2 = make_double2(guard(t2.x, -0.5), guard(t2.y, -0.5));
    t3 = make_double2(guard(t3.x, 0.75), guard(t3.y, 0.75));
  }
  double2 r = make_double2(add(add(t1.x, t2.x), t3.x), add(add(t1.y, t2.y), t3.y));
  if (GUARD) r.y = add(r.y, (!isnan(v.x) && signbit(v.x)) ? w : 0.0);
  return r;
}

template <bool GUARD, bool SCALAR>
__global__ void __launch_bounds__(kT) k_poly_c(double2 *__restrict__ fx, const double2 *__restrict__ x, int64_t n,
                                               const double *__restrict__ a, const double *__restrict__ w, int64_t ldfx,
                                               int64_t ldx) {
  const double2 *xb = x + (int64_t)blockIdx.y * ldx;
  double2 *fb = fx + (int64_t)blockIdx.y * ldfx;
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kT)
    fb[i] = poly_at_c<GUARD>(SCALAR ? xb[0] : xb[i], a[i], w[i]);
}

__device__ __forceinline__ uint64_t splitmix64_at(uint64_t seed, uint64_t i) {
  uint64_t z = seed + (i + 1) * 0x9E3779B97F4A7C15ULL;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

__global__ void __launch_bounds__(kT) k_fill_x(double *__restrict__ x, int64_t n, uint64_t seed) {
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kT)
    x[i] = __dadd_rn(0.5, __dmul_rn((double)(splitmix64_at(seed, (uint64_t)i) >> 11), 1.0 / 9007199254740992.0));
}

__global__ void __launch_bounds__(kT) k_flush(double *__restrict__ p, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)kT + threadIdx.x; i < n; i += (int64_t)gridDim.x * kT) p[i] = 0.0;
}

inline int blocks_for(int64_t items, int64_t cap = 132 * 8) {
  int64_t b = (items + kT - 1) / kT;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}
}  // namespace

// Store-only bandwidth probe: n doubles written once with 16-byte streaming stores, grid-stride in address order.
// mode 0: one constant; mode 1: a different value per element (rules out constant-data effects in the memory system)
__global__ void __launch_bounds__(kT) k_store_probe(double *__restrict__ out, int64_t n, int mode) {
  const int64_t stride = (int64_t)gridDim.x * kT * 2;
  for (int64_t i = (blockIdx.x * (int64_t)kT + threadIdx.x) * 2; i + 1 < n; i += stride) {
    const double v0 = mode ? (double)i * 1.0000001 + 0.5 : 1.0;
    const double v1 = mode ? (double)(i + 1) * 1.0000001 + 0.5 : 1.0;
    __stcs(reinterpret_cast<double2 *>(out + i), make_double2(v0, v1));
  }
}

// Streaming bandwidth probe for a traffic mix: R source vectors read, W destination vectors written, n doubles each,
// 16-byte streaming loads and stores, grid-stride in address order.  With W = 0 the sum of the loads goes to sink[0]
// only if it is a NaN (never for finite sources), so the loads are not dead code.
template <int R, int W>
__global__ void __launch_bounds__(kT) k_stream_probe(const double *__restrict__ src, int64_t lds, double *__restrict__ dst,
                                                     int64_t ldd, int64_t n, double *__restrict__ sink) {
  const int64_t stride = (int64_t)gridDim.x * kT * 2;
  double acc = 0.0;
  for (int64_t i = (blockIdx.x * (int64_t)kT + threadIdx.x) * 2; i + 1 < n; i += stride) {
    double2 v[R];
#pragma unroll
    for (int r = 0; r < R; ++r) v[r] = __ldcs(reinterpret_cast<const double2 *>(src + r * lds + i));
    double a = v[0].x, b = v[0].y;
#pragma unroll
    for (int r = 1; r < R; ++r) { a += v[r].x; b += v[r].y; }
#pragma unroll
    for (int w = 0; w < W; ++w) __stcs(reinterpret_cast<double2 *>(dst + w * ldd + i), make_double2(a + w, b + w));
    if (W == 0) acc += a + b;
  }
  if (W == 0 && acc != acc) sink[0] = acc;
}

extern "C" {

int fdbs_stream_probe(const double *d_src, int64_t lds, int reads, double *d_dst, int64_t ldd, int writes, int64_t n,
                      int blocks, double *d_sink, void *stream) {
  if (n <= 0 || blocks <= 0 || ((uintptr_t)d_src & 15) || ((uintptr_t)d_dst & 15) || (lds & 1) || (ldd & 1)) return 1;
  cudaStream_t s = (cudaStream_t)stream;
  if (reads == 1 && writes == 0) k_stream_probe<1, 0><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else if (reads == 1 && writes == 3) k_stream_probe<1, 3><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else if (reads == 4 && writes == 3) k_stream_probe<4, 3><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else if (reads == 1 && writes == 1) k_stream_probe<1, 1><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else if (reads == 1 && writes == 2) k_stream_probe<1, 2><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else if (reads == 2 && writes == 1) k_stream_probe<2, 1><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else if (reads == 3 && writes == 1) k_stream_probe<3, 1><<<blocks, kT, 0, s>>>(d_src, lds, d_dst, ldd, n, d_sink);
  else return 2;
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_tridiag(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_tridiag_ctx *c = (fdbs_tridiag_ctx *)vctx;
  if (!c || batch < 1 || batch > 65535) return 1;
  c->calls += batch;
  if (c->n <= 0) return 0;
  // the 16-byte path needs 16-byte aligned rows (plan buffers are; ldx/ldfx are even)
  if (((uintptr_t)d_x & 15) || ((uintptr_t)d_fx & 15) || (ldx & 1) || (ldfx & 1)) return 2;
  dim3 grid((unsigned)blocks_for((c->n + 1) / 2), (unsigned)batch);
  k_tridiag<<<grid, kT, 0, (cudaStream_t)stream>>>(d_fx, d_x, c->n, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_tridiag_rows(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_tridiag_rows_ctx *c = (fdbs_tridiag_rows_ctx *)vctx;
  if (!c || batch < 1 || batch > 65535) return 1;
  c->calls += batch;
  if (c->nrows <= 0) return 0;
  dim3 grid((unsigned)blocks_for(c->nrows), (unsigned)batch);
  k_tridiag_rows<<<grid, kT, 0, (cudaStream_t)stream>>>(d_fx, d_x, c->n, c->row0, c->nrows, c->x0, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_tridiag_c(void *vctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_tridiag_ctx *c = (fdbs_tridiag_ctx *)vctx;
  if (!c || batch < 1 || batch > 65535) return 1;
  c->calls += batch;
  if (c->n <= 0) return 0;
  dim3 grid((unsigned)blocks_for(c->n), (unsigned)batch);
  k_tridiag_c<<<grid, kT, 0, (cudaStream_t)stream>>>((double2 *)d_fx, (const double2 *)d_x, c->n, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_lap5(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_lap5_ctx *c = (fdbs_lap5_ctx *)vctx;
  if (!c || batch < 1 || batch > 65535 || c->g > 65535) return 1;
  c->calls += batch;
  if (c->g <= 0) return 0;
  dim3 grid((unsigned)blocks_for(c->g, 8), (unsigned)c->g, (unsigned)batch);
  k_lap5<<<grid, kT, 0, (cudaStream_t)stream>>>(d_fx, d_x, c->g, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_ellrows(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_ell_ctx *c = (fdbs_ell_ctx *)vctx;
  if (!c || batch < 1 || batch > 65535) return 1;
  c->calls += batch;
  if (c->m <= 0) return 0;
  dim3 grid((unsigned)blocks_for(c->m, 132 * 16), (unsigned)batch);
  k_ellrows<<<grid, kT, 0, (cudaStream_t)stream>>>(d_fx, d_x, c->m, (int)c->K, c->d_cols, c->d_coef, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_ellrows_c(void *vctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_ell_ctx *c = (fdbs_ell_ctx *)vctx;
  if (!c || batch < 1 || batch > 65535) return 1;
  c->calls += batch;
  if (c->m <= 0) return 0;
  dim3 grid((unsigned)blocks_for(c->m, 132 * 16), (unsigned)batch);
  k_ellrows_c<<<grid, kT, 0, (cudaStream_t)stream>>>((double2 *)d_fx, (const double2 *)d_x, c->m, (int)c->K, c->d_cols,
                                                     c->d_coef, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_rank1(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_rank1_ctx *c = (fdbs_rank1_ctx *)vctx;
  if (!c || batch < 1 || batch > c->max_batch || batch > 65535) return 1;
  c->calls += batch;
  if (c->n <= 0) return 0;
  const int64_t nblk = (c->n + 1023) / 1024;
  dim3 g1((unsigned)blocks_for(nblk * 32, 64), (unsigned)batch);   // one warp per 1024-block
  k_block_sums<<<g1, kT, 0, (cudaStream_t)stream>>>(d_x, c->n, ldx, c->d_block_sums, nblk);
  k_point_sums<<<(unsigned)((batch + kT - 1) / kT), kT, 0, (cudaStream_t)stream>>>(c->d_block_sums, nblk, c->n, batch);
  // 16-byte path: every point / output / w base 16-byte aligned (even leading dimensions)
  const int vec_ok = (((uintptr_t)d_x | (uintptr_t)d_fx | (uintptr_t)c->d_w) & 15) == 0 && (ldx & 1) == 0 && (ldfx & 1) == 0;
  dim3 g2((unsigned)blocks_for((c->n + 3) / 4, 128), (unsigned)batch);
  k_rank1<<<g2, kT, 0, (cudaStream_t)stream>>>(d_fx, d_x, c->n, c->d_w, c->d_block_sums, nblk, ldfx, ldx, vec_ok);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

// one block per point: a warp per 1024-block, up to 8 warps; the block sums stay in shared memory
static int scalar_launch(const fdbs_scalar_ctx *c, int64_t batch, int words, unsigned *threads, size_t *smem) {
  const int64_t nblk = (c->n + 1023) / 1024;
  if (nblk * words * 8 > 48 * 1024) return 1;
  *threads = 32u * (unsigned)(nblk < 1 ? 1 : (nblk > 8 ? 8 : nblk));
  *smem = (size_t)(nblk * words * 8);
  return batch < 1 || batch > 2147483647 ? 1 : 0;
}

int fdbs_quartic(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_scalar_ctx *c = (fdbs_scalar_ctx *)vctx;
  unsigned threads;
  size_t smem;
  if (!c || c->n < 0 || (c->n > 0 && (!c->d_a || !c->d_w)) || scalar_launch(c, batch, 2, &threads, &smem)) return 1;
  c->calls += batch;
  k_scalar<0><<<(unsigned)batch, threads, smem, (cudaStream_t)stream>>>(d_fx, d_x, c->n, c->d_a, c->d_w, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_sumsq(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_scalar_ctx *c = (fdbs_scalar_ctx *)vctx;
  unsigned threads;
  size_t smem;
  if (!c || c->n < 0 || scalar_launch(c, batch, 2, &threads, &smem)) return 1;
  c->calls += batch;
  k_scalar<1><<<(unsigned)batch, threads, smem, (cudaStream_t)stream>>>(d_fx, d_x, c->n, nullptr, nullptr, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_guarded(void *vctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_scalar_ctx *c = (fdbs_scalar_ctx *)vctx;
  unsigned threads;
  size_t smem;
  if (!c || c->n < 0 || (c->n > 0 && (!c->d_a || !c->d_w)) || scalar_launch(c, batch, 2, &threads, &smem)) return 1;
  c->calls += batch;
  k_scalar<2><<<(unsigned)batch, threads, smem, (cudaStream_t)stream>>>(d_fx, d_x, c->n, c->d_a, c->d_w, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_quartic_c(void *vctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream) {
  fdbs_scalar_ctx *c = (fdbs_scalar_ctx *)vctx;
  unsigned threads;
  size_t smem;
  if (!c || c->n < 0 || (c->n > 0 && (!c->d_a || !c->d_w)) || scalar_launch(c, batch, 4, &threads, &smem)) return 1;
  c->calls += batch;
  k_scalar_c<<<(unsigned)batch, threads, smem, (cudaStream_t)stream>>>((double2 *)d_fx, (const double2 *)d_x, c->n, c->d_a,
                                                                       c->d_w, ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

}  // extern "C"

template <bool GUARD, bool SCALAR>
static int poly_launch(void *vctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream,
                       bool complex_) {
  fdbs_scalar_ctx *c = (fdbs_scalar_ctx *)vctx;
  if (!c || c->n < 0 || (c->n > 0 && (!c->d_a || !c->d_w)) || batch < 1 || batch > 65535) return 1;
  c->calls += batch;
  if (c->n == 0) return 0;
  dim3 grid((unsigned)blocks_for(c->n), (unsigned)batch);
  if (complex_)
    k_poly_c<GUARD, SCALAR><<<grid, kT, 0, (cudaStream_t)stream>>>((double2 *)d_fx, (const double2 *)d_x, c->n, c->d_a,
                                                                    c->d_w, ldfx, ldx);
  else
    k_poly<GUARD, SCALAR><<<grid, kT, 0, (cudaStream_t)stream>>>((double *)d_fx, (const double *)d_x, c->n, c->d_a, c->d_w,
                                                                  ldfx, ldx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

extern "C" {

int fdbs_poly(void *c, double *fx, const double *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<false, false>(c, fx, x, b, lf, lx, s, false);
}
int fdbs_poly_guarded(void *c, double *fx, const double *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<true, false>(c, fx, x, b, lf, lx, s, false);
}
int fdbs_poly_c(void *c, void *fx, const void *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<false, false>(c, fx, x, b, lf, lx, s, true);
}
int fdbs_poly_guarded_c(void *c, void *fx, const void *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<true, false>(c, fx, x, b, lf, lx, s, true);
}
int fdbs_tpoly(void *c, double *fx, const double *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<false, true>(c, fx, x, b, lf, lx, s, false);
}
int fdbs_tpoly_guarded(void *c, double *fx, const double *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<true, true>(c, fx, x, b, lf, lx, s, false);
}
int fdbs_tpoly_c(void *c, void *fx, const void *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<false, true>(c, fx, x, b, lf, lx, s, true);
}
int fdbs_tpoly_guarded_c(void *c, void *fx, const void *x, int64_t b, int64_t lf, int64_t lx, void *s) {
  return poly_launch<true, true>(c, fx, x, b, lf, lx, s, true);
}

int fdbs_fail(void *, double *, const double *, int64_t, int64_t, int64_t, void *) { return 42; }

int fdbs_fill_x(double *d_x, int64_t n, uint64_t seed, void *stream) {
  if (n <= 0) return 0;
  k_fill_x<<<blocks_for(n), kT, 0, (cudaStream_t)stream>>>(d_x, n, seed);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_store_probe(double *d_out, int64_t n, int mode, int blocks, void *stream) {
  if (n <= 0 || blocks <= 0) return 1;
  k_store_probe<<<blocks, kT, 0, (cudaStream_t)stream>>>(d_out, n, mode);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

int fdbs_flush_l2(void *d_buf, int64_t bytes, void *stream) {
  if (bytes <= 0) return 0;
  k_flush<<<blocks_for(bytes / 8), kT, 0, (cudaStream_t)stream>>>((double *)d_buf, bytes / 8);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

}  // extern "C"
