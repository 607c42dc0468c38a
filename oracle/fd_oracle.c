/*
 * fd_oracle.c — CPU ORACLE (test infrastructure; see fd_oracle.h for the header
 * statement, scope and parity pinning).  Plain C restatement of FiniteDiff.jl's
 * cached coloured Jacobian driver.  Every block cites the reference file:line it
 * follows.  Build: gcc -O2 -fno-fast-math -ffp-contract=off [-fopenmp].
 */
#include "fd_oracle.h"
#include <complex.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <float.h>

#define PAR_FOR _Pragma("omp parallel for schedule(static) if(nt > 1) num_threads(nt)")

/* src/epsilons.jl:134-144  default_relstep: sqrt(eps) forward, cbrt(eps) central */
double fdo_default_relstep(int fdtype) {
  if (fdtype == FDO_FORWARD) return sqrt(DBL_EPSILON);
  if (fdtype == FDO_CENTRAL) return cbrt(DBL_EPSILON);
  return 1.0;
}

/* Julia Base max(x::Float64, y::Float64): NaN if either argument is NaN (it returns x - y then), otherwise the larger
 * one, with +0.0 counted larger than -0.0.  A NaN in x (a diverging Newton or ODE step) therefore gives a NaN step. */
static inline double max_julia(double a, double b) {
  if (isnan(a) || isnan(b)) return a - b;
  return signbit(a - b) ? b : a;
}

/* src/epsilons.jl:26-29 (forward: max(relstep*abs(x),absstep)*dir)
 * src/epsilons.jl:50-53 (central: max(relstep*abs(x),absstep), dir ignored) */
double fdo_compute_epsilon(int fdtype, double x, double relstep, double absstep, double dir) {
  double a = relstep * fabs(x);
  double e = max_julia(a, absstep);
  if (fdtype == FDO_FORWARD) return e * dir;
  return e;
}

/* `maximum(colorvec)` jacobians.jl:547; colorvec===NULL means the default 1:n */
int64_t fdo_max_color(const int64_t *colorvec, int64_t n) {
  if (!colorvec) return n;
  int64_t mx = (n > 0) ? colorvec[0] : 0;
  for (int64_t j = 1; j < n; ++j)
    if (colorvec[j] > mx) mx = colorvec[j];
  return mx;
}

/* src/jacobians.jl:473-488 */
int64_t fdo_findstructralnz_dense(const double *A, int64_t m, int64_t n, int64_t *rows, int64_t *cols) {
  int64_t idx = 0;
  for (int64_t j = 0; j < n; ++j)
    for (int64_t i = 0; i < m; ++i)
      if (A[j * m + i] != 0.0) {
        if (rows) rows[idx] = i + 1;
        if (cols) cols[idx] = j + 1;
        ++idx;
      }
  return idx;
}

static inline int64_t color_of(const int64_t *colorvec, int64_t j0 /*0-based*/) {
  return colorvec ? colorvec[j0] : j0 + 1;
}

/* Julia Bool*Float64: x*true = x, x*false = copysign(0.0, x) (a "strong zero") */
static inline double mul_bool(double v, int b) { return b ? v : copysign(0.0, v); }

/* J[row,col] = v for the (row,col)-addressed storages */
static inline void setindex_rc(const fdo_problem *P, double *J, int64_t r /*1-based*/, int64_t c, double v) {
  if (P->j_kind == FDO_J_DENSE) {
    J[(c - 1) * P->ldJ + (r - 1)] = v;
  } else { /* FDO_J_BAND: data[u+r-c+1, c], data is (l+u+1) x n column-major (ext/Banded..:22) */
    int64_t w = P->l + P->u + 1;
    J[(c - 1) * w + (P->u + r - c)] = v;
  }
}

/* One call of the decompression hook for colour `color_i` with vfx = divided differences. */
static void colorediteration(const fdo_problem *P, double *J, const double *vfx,
                             const int64_t *colorvec, int64_t color_i, int nt) {
  const int64_t n = P->n, m = P->m;
  switch (P->sp_kind) {
  case FDO_SP_CSC_SAME: {
    /* ext/FiniteDiffSparseArraysExt.jl:38-47 — nzval[spidx] = vfx[rowval[spidx]] */
    PAR_FOR
    for (int64_t c = 0; c < n; ++c) {
      if (color_of(colorvec, c) == color_i) {
        for (int64_t p = P->colptr[c]; p <= P->colptr[c + 1] - 1; ++p) {
          int64_t r = P->rowval[p - 1];
          J[p - 1] = vfx[r - 1];
        }
      }
    }
  } break;
  case FDO_SP_CSC: {
    /* ext/FiniteDiffSparseArraysExt.jl:20-28 — J[row,col] = vfx[row] */
    PAR_FOR
    for (int64_t c = 0; c < n; ++c) {
      if (color_of(colorvec, c) == color_i) {
        for (int64_t p = P->colptr[c]; p <= P->colptr[c + 1] - 1; ++p) {
          int64_t r = P->rowval[p - 1];
          setindex_rc(P, J, r, c + 1, vfx[r - 1]);
        }
      }
    }
  } break;
  case FDO_SP_COO: {
    /* src/iteration_utils.jl:25-32 — loop over ALL structural nz, colour test per nz */
    PAR_FOR
    for (int64_t i = 0; i < P->nnz; ++i) {
      int64_t c = P->cols_index[i], r = P->rows_index[i];
      if (color_of(colorvec, c - 1) == color_i) {
        if (P->j_kind == FDO_J_SLOTS) J[P->slots[i] - 1] = vfx[r - 1];
        else setindex_rc(P, J, r, c, vfx[r - 1]);
      }
    }
  } break;
  case FDO_SP_BANDED: {
    /* ext/FiniteDiffBandedMatricesExt.jl:13-27 — whole in-band column range */
    int64_t c_lo = (1 - P->l > 1) ? 1 - P->l : 1;        /* max(1,1-l) */
    int64_t c_hi = (n + P->u < n) ? n + P->u : n;        /* min(ncols,ncols+u) */
    PAR_FOR
    for (int64_t c = c_lo; c <= c_hi; ++c) {
      if (color_of(colorvec, c - 1) == color_i) {
        int64_t r_lo = (c - P->u > 1) ? c - P->u : 1;    /* max(1,col-u) */
        int64_t r_hi = (c + P->l < m) ? c + P->l : m;    /* min(nrows,col+l) */
        for (int64_t r = r_lo; r <= r_hi; ++r) setindex_rc(P, J, r, c, vfx[r - 1]);
      }
    }
  } break;
  default: break;
  }
}

/*
 * LinearAlgebra.norm(x2)  (jacobians.jl:560,601) for a Vector{Float64} — third-party arithmetic that is NOT under
 * the reference package (Julia stdlib LinearAlgebra, Project.toml:30 julia >= 1.10, and its BLAS, OpenBLAS):
 *   norm(x) = norm2(x);   norm2(x::StridedVector{Float64}) = length(x) < 32 ? generic_norm2(x) : BLAS.nrm2(x)
 *
 * (a) generic_norm2 (n < 32; stdlib generic.jl): maxabs = normInf(x); 0 / Inf returned as is; when n*maxabs^2 is finite
 *     and maxabs^2 != 0 the squares are added one by one IN ORDER in Float64 and the result is sqrt(sum); otherwise the
 *     elements are divided by maxabs first and the result is maxabs*sqrt(sum).
 * (b) BLAS.nrm2 -> OpenBLAS dnrm2, x86-64 kernel kernel/x86_64/nrm2.S: x87 code — every element is squared and added in
 *     80-bit extended precision into FOUR interleaved accumulators (element i -> accumulator i mod 4 over the unrolled
 *     body, the last n mod 8 elements one by one), the accumulators are added, fsqrt in extended precision, and the
 *     result is rounded to double once, on the store.  No scaling (the 15-bit exponent makes it unnecessary).
 *     `long double` is that x87 format with gcc on x86-64, so the loop below IS that computation.
 *
 * Pinning: (b) is compared BIT FOR BIT with OpenBLAS's own dnrm2 binary (the scipy wheel's libscipy_openblas, 0.3.31, the
 * same kernel file Julia's bundled OpenBLAS builds) — committed vectors tests/golden/dnrm2_openblas.json (made by
 * tests/golden/make_dnrm2_golden.py) and, where scipy is importable, live (tests/test_oracle_norm.py): 2..12 million
 * element vectors included, 0 mismatches.  The extended-precision sum is insensitive to how the accumulators are
 * combined (every plausible variant gives the same double on all of those vectors).  (a) follows the stdlib source as
 * published; it cannot be executed here.
 */
static double generic_norm2(const double *v, int64_t n) {
  double maxabs = 0.0;                                   /* normInf: NaN-propagating maximum of abs */
  for (int64_t i = 0; i < n; ++i) {
    const double a = fabs(v[i]);
    if (i == 0) maxabs = a;
    else maxabs = (isnan(maxabs) || maxabs > a) ? maxabs : a;
  }
  if (maxabs == 0.0 || isinf(maxabs)) return maxabs;
  if (isfinite((double)n * maxabs * maxabs) && maxabs * maxabs != 0.0) {
    double sum = v[0] * v[0];
    for (int64_t i = 1; i < n; ++i) sum += v[i] * v[i];
    return sqrt(sum);
  }
  double t = fabs(v[0]) / maxabs;
  double sum = t * t;
  for (int64_t i = 1; i < n; ++i) { t = fabs(v[i]) / maxabs; sum += t * t; }
  return maxabs * sqrt(sum);
}

#if LDBL_MANT_DIG != 64
#warning "long double is not the x87 80-bit format here: fdo_norm2 will not reproduce OpenBLAS's x86-64 dnrm2 bit for bit (tests/test_oracle_norm.py will say so)"
#endif
static double openblas_dnrm2_x87(const double *v, int64_t n) {
  long double a0 = 0.0L, a1 = 0.0L, a2 = 0.0L, a3 = 0.0L;
  const int64_t body = n & ~(int64_t)7;
  for (int64_t i = 0; i < body; i += 4) {
    const long double v0 = v[i], v1 = v[i + 1], v2 = v[i + 2], v3 = v[i + 3];
    a0 += v0 * v0; a1 += v1 * v1; a2 += v2 * v2; a3 += v3 * v3;
  }
  for (int64_t i = body; i < n; ++i) { const long double t = v[i]; a0 += t * t; }
  return (double)sqrtl((a0 + a1) + (a2 + a3));
}

double fdo_norm2(const double *v, int64_t n) {
  if (n <= 0) return 0.0;                                /* norm of an empty vector: float(norm(zero(T))) */
  return n < 32 ? generic_norm2(v, n) : openblas_dnrm2_x87(v, n);
}

static double norm2(const double *v, int64_t n, int nt) {
  /* nt > 1 is the all-host-threads timing variant (bench.py --impl reference): an OpenMP reduction, whose value
   * differs from the reference's single-threaded norm by reduction-order accuracy; parity runs use nt == 1 */
  if (nt > 1) {
    double s = 0.0;
#pragma omp parallel for reduction(+ : s) schedule(static) num_threads(nt)
    for (int64_t i = 0; i < n; ++i) s += v[i] * v[i];
    return sqrt(s);
  }
  return fdo_norm2(v, n);
}

int fdo_finite_difference_jacobian(const fdo_problem *P, double *J, fdo_fn f, void *ctx,
                                   double *x, fdo_cache *cache, fdo_opts *o) {
  if (!P || !J || !f || !x || !cache || !o) return 1;
  const int64_t m = P->m, n = P->n;                     /* jacobians.jl:515 */
  const int64_t *colorvec = o->colorvec;                /* :516 (_color = reshape(colorvec,...)) */
  const int nt = o->nthreads > 1 ? o->nthreads : 1;
  const int fdtype = o->fdtype;
  if (fdtype != FDO_FORWARD && fdtype != FDO_CENTRAL) return 2; /* fdtype_error, epsilons.jl:159-167 */
  /* NaN = keyword not given; any other value (0 included) is used as passed, like the reference's keywords */
  double relstep = isnan(o->relstep) ? fdo_default_relstep(fdtype) : o->relstep; /* :508 */
  double absstep = isnan(o->absstep) ? relstep : o->absstep;                     /* :509 */
  double dir = o->dir;
  double *x1 = cache->x1, *x2 = cache->x2, *fx = cache->fx, *fx1 = cache->fx1; /* :518 */
  o->fcalls = 0;

  /* copyto!(x1, x)  :519 */
  memcpy(x1, x, (size_t)n * sizeof(double));
  const double *vfx = fx; /* :520 */

  /* :522-528 rows_index/cols_index come precomputed in P (findstructralnz /
   * _findstructralnz); nothing for CSC / banded (their ext sets _use_findstructralnz=false). */

  /* fill_matrix!(J,false) when sparsity !== nothing  :530-532; ext/Sparse..:30 fills nzval */
  if (P->sp_kind != FDO_SP_NONE) memset(J, 0, (size_t)P->j_len * sizeof(double));

  const int64_t maxcolor = fdo_max_color(colorvec, n); /* maximum(colorvec) :547/:589 */

  if (fdtype == FDO_FORWARD) {
    /* :540-545 */
    if (!o->f_in) { f(ctx, fx, x); o->fcalls++; vfx = fx; }
    else vfx = o->f_in;

    for (int64_t color_i = 1; color_i <= maxcolor; ++color_i) { /* :547 */
      if (P->sp_kind == FDO_SP_NONE) {
        /* dense column branch :548-557 */
        double x1_save = x1[color_i - 1];
        double eps = o->eps_override ? o->eps_override[color_i - 1]
                                     : fdo_compute_epsilon(FDO_FORWARD, x1_save, relstep, absstep, dir);
        if (o->eps_out) o->eps_out[color_i - 1] = eps;
        x1[color_i - 1] = x1_save + eps;
        f(ctx, fx1, x1); o->fcalls++;
        double *Jc = J + (color_i - 1) * P->ldJ;
        PAR_FOR
        for (int64_t i = 0; i < m; ++i) Jc[i] = (fx1[i] - vfx[i]) / eps; /* :555 */
        x1[color_i - 1] = x1_save;                                       /* :557 */
      } else {
        /* coloured branch :558-585 */
        PAR_FOR
        for (int64_t j = 0; j < n; ++j) x2[j] = mul_bool(x1[j], color_of(colorvec, j) == color_i); /* :559 */
        double tmp = norm2(x2, n, nt);                                                           /* :560 */
        double eps = o->eps_override ? o->eps_override[color_i - 1]
                                     : fdo_compute_epsilon(FDO_FORWARD, sqrt(tmp), relstep, absstep, dir); /* :561 */
        if (o->eps_out) o->eps_out[color_i - 1] = eps;
        PAR_FOR
        for (int64_t j = 0; j < n; ++j) x1[j] = x1[j] + mul_bool(eps, color_of(colorvec, j) == color_i);   /* :562 */
        f(ctx, fx1, x1); o->fcalls++;                                                                     /* :563 */
        PAR_FOR
        for (int64_t i = 0; i < m; ++i) fx1[i] = (fx1[i] - vfx[i]) / eps;                                 /* :565 in place */
        colorediteration(P, J, fx1, colorvec, color_i, nt);                                               /* :566-572 */
        if (o->no_drift) {
          /* exact restore of the colour's components; the others get :584 as written (x1 - copysign(0, eps), which
           * only changes the sign of a zero) */
          PAR_FOR
          for (int64_t j = 0; j < n; ++j) x1[j] = color_of(colorvec, j) == color_i ? x[j] : x1[j] - mul_bool(eps, 0);
        } else {
          PAR_FOR
          for (int64_t j = 0; j < n; ++j) x1[j] = x1[j] - mul_bool(eps, color_of(colorvec, j) == color_i); /* :584 */
        }
      }
    }
  } else { /* FDO_CENTRAL :587-622 */
    for (int64_t color_i = 1; color_i <= maxcolor; ++color_i) { /* :589 */
      if (P->sp_kind == FDO_SP_NONE) {
        /* :590-598 */
        double x_save = x[color_i - 1];
        double eps = o->eps_override ? o->eps_override[color_i - 1]
                                     : fdo_compute_epsilon(FDO_CENTRAL, x_save, relstep, absstep, dir);
        if (o->eps_out) o->eps_out[color_i - 1] = eps;
        x1[color_i - 1] = x_save + eps;
        f(ctx, fx1, x1); o->fcalls++;
        x1[color_i - 1] = x_save - eps;
        f(ctx, fx, x1); o->fcalls++;
        double *Jc = J + (color_i - 1) * P->ldJ;
        const double two_eps = 2 * eps;
        PAR_FOR
        for (int64_t i = 0; i < m; ++i) Jc[i] = (fx1[i] - fx[i]) / two_eps; /* :597 */
        x1[color_i - 1] = x_save;
      } else {
        /* :599-621 */
        PAR_FOR
        for (int64_t j = 0; j < n; ++j) x2[j] = mul_bool(x1[j], color_of(colorvec, j) == color_i); /* :600 */
        double tmp = norm2(x2, n, nt);                                                           /* :601 */
        double eps = o->eps_override ? o->eps_override[color_i - 1]
                                     : fdo_compute_epsilon(FDO_CENTRAL, sqrt(tmp), relstep, absstep, dir); /* :602 */
        if (o->eps_out) o->eps_out[color_i - 1] = eps;
        PAR_FOR
        for (int64_t j = 0; j < n; ++j) {
          int b = color_of(colorvec, j) == color_i;
          x1[j] = x1[j] + mul_bool(eps, b); /* :603 */
          x[j] = x[j] - mul_bool(eps, b);   /* :604 caller's x perturbed in place */
        }
        f(ctx, fx1, x1); o->fcalls++; /* :605 */
        f(ctx, fx, x); o->fcalls++;   /* :606 */
        const double two_eps = 2 * eps;
        PAR_FOR
        for (int64_t i = 0; i < m; ++i) fx1[i] = (fx1[i] - fx[i]) / two_eps; /* :607 */
        colorediteration(P, J, fx1, colorvec, color_i, nt);                 /* :608-614 */
        if (o->no_drift) {
          /* exact restore (not what the reference does; used to compare with drift-free runs).  x2 still holds this
           * colour's components as they were before :603-604, and with exact restores those are the caller's values:
           * (x - eps) + eps and (x1 + eps) - eps would replay the drift whenever the rounding does not cancel. */
          PAR_FOR
          for (int64_t j = 0; j < n; ++j) {
            if (color_of(colorvec, j) == color_i) { x[j] = x2[j]; x1[j] = x2[j]; }
            else { x1[j] = x1[j] - mul_bool(eps, 0); x[j] = x[j] + mul_bool(eps, 0); }   /* :619-620 as written */
          }
        } else {
          PAR_FOR
          for (int64_t j = 0; j < n; ++j) {
            int b = color_of(colorvec, j) == color_i;
            x1[j] = x1[j] - mul_bool(eps, b); /* :619 */
            x[j] = x[j] + mul_bool(eps, b);   /* :620 */
          }
        }
      }
    }
  }
  return 0; /* nothing  :652 */
}

int fdo_finite_difference_jacobian_cacheless(const fdo_problem *P, double *J, fdo_fn f, void *ctx,
                                             double *x, fdo_opts *o) {
  /* jacobians.jl:446-471 */
  if (!P || !J || !f || !x || !o) return 1;
  const int64_t m = P->m, n = P->n;
  fdo_cache c;
  c.x1 = (double *)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
  c.x2 = (double *)calloc((size_t)(n > 0 ? n : 1), sizeof(double));
  c.fx = (double *)calloc((size_t)(m > 0 ? m : 1), sizeof(double));
  c.fx1 = (double *)calloc((size_t)(m > 0 ? m : 1), sizeof(double));
  if (!c.x1 || !c.x2 || !c.fx || !c.fx1) { free(c.x1); free(c.x2); free(c.fx); free(c.fx1); return 3; }
  int64_t pre_calls = 0;
  fdo_opts oo = *o;
  double *fin_copy = NULL;
  if (!o->f_in && o->fdtype == FDO_FORWARD) {
    /* :456-463: fx = zero(x) | zeros(returntype,size(J,1)); f(fx,x); cache = JacobianCache(x,fx,...) */
    f(ctx, c.fx, x); pre_calls = 1;
    memcpy(c.fx1, c.fx, sizeof(double) * (size_t)m); /* JacobianCache(x,fx): _fx1 = copy(fx) :72 */
    oo.f_in = c.fx;                                   /* :469 passes cache.fx as f_in */
  } else if (o->f_in) {
    /* :466 cache = JacobianCache(x, f_in, ...): fx = copy(f_in); then f_in := cache.fx (:469) */
    fin_copy = c.fx;
    memcpy(c.fx, o->f_in, sizeof(double) * (size_t)m);
    memcpy(c.fx1, o->f_in, sizeof(double) * (size_t)m);
    oo.f_in = (o->fdtype == FDO_FORWARD) ? c.fx : NULL;
  }
  (void)fin_copy;
  int rc = fdo_finite_difference_jacobian(P, J, f, ctx, x, &c, &oo);
  o->fcalls = oo.fcalls + pre_calls;
  free(c.x1); free(c.x2); free(c.fx); free(c.fx1);
  return rc;
}

/* ---------------------------------------------------------------------------------------------------------------
 * Complex-step colour loop — src/jacobians.jl:623-648 (fdtype == Val(:complex) && returntype <: Real), with the
 * cache of the complex constructors (:20-32, :60-76, :105-117: x1 and fx are complex, fx1 === nothing) after
 * copyto!(x1, x) (:519).  epsilon = eps(eltype(x)) (:624); J[r,c] = imag(f(x + im*eps*e_k))[r] / eps.
 * --------------------------------------------------------------------------------------------------------------- */
int fdo_finite_difference_jacobian_complex(const fdo_problem *P, double *J, fdo_fn_c f, void *ctx, const double *x,
                                           const int64_t *colorvec, int nthreads, int64_t *fcalls) {
  if (!P || !J || !f || !x) return 1;
  const int64_t m = P->m, n = P->n;
  const int nt = nthreads > 1 ? nthreads : 1;
  double _Complex *x1 = (double _Complex *)malloc(sizeof(double _Complex) * (size_t)(n > 0 ? n : 1));
  double _Complex *fx = (double _Complex *)calloc((size_t)(m > 0 ? m : 1), sizeof(double _Complex));
  double *vre = (double *)malloc(sizeof(double) * (size_t)(m > 0 ? m : 1));
  if (!x1 || !fx || !vre) { free(x1); free(fx); free(vre); return 3; }
  for (int64_t j = 0; j < n; ++j) x1[j] = x[j];                 /* copyto!(x1, x)  :519 */
  if (P->sp_kind != FDO_SP_NONE) memset(J, 0, (size_t)P->j_len * sizeof(double)); /* fill_matrix! :530-532 */
  const double epsilon = DBL_EPSILON;                            /* eps(eltype(x))  :624 */
  const int64_t maxcolor = fdo_max_color(colorvec, n);
  int64_t calls = 0;
  for (int64_t color_i = 1; color_i <= maxcolor; ++color_i) {    /* :625 */
    if (P->sp_kind == FDO_SP_NONE) {
      /* :626-631 */
      double _Complex x1_save = x1[color_i - 1];
      x1[color_i - 1] = x1_save + epsilon * _Complex_I;
      f(ctx, fx, x1); calls++;
      double *Jc = J + (color_i - 1) * P->ldJ;
      for (int64_t i = 0; i < m; ++i) Jc[i] = cimag(fx[i]) / epsilon;   /* :630 */
      x1[color_i - 1] = x1_save;
    } else {
      /* :632-645.  im*epsilon is Complex(epsilon*false, epsilon*true) = (+0.0, eps), and times (color == k) it is
       * (+0.0, eps) or, by the strong-zero rule of mul_bool applied to each part, (+0.0, +0.0).  So :634 adds +0.0 to
       * the real part of EVERY component (a -0.0 becomes +0.0 from the first colour on) and :644 subtracts +0.0 (the
       * identity).  The adds are written out per part: C's complex `+` on these operands is the same two IEEE adds. */
      PAR_FOR
      for (int64_t j = 0; j < n; ++j) {
        const int b = color_of(colorvec, j) == color_i;
        x1[j] = CMPLX(creal(x1[j]) + 0.0, cimag(x1[j]) + mul_bool(epsilon, b));              /* :634 */
      }
      f(ctx, fx, x1); calls++;                                                               /* :635 */
      PAR_FOR
      for (int64_t i = 0; i < m; ++i) { vre[i] = cimag(fx[i]) / epsilon; fx[i] = vre[i]; }     /* :636 vfx = imag(vfx)/eps */
      colorediteration(P, J, vre, colorvec, color_i, nt);                                    /* :637-643 */
      PAR_FOR
      for (int64_t j = 0; j < n; ++j) {
        const int b = color_of(colorvec, j) == color_i;
        x1[j] = CMPLX(creal(x1[j]) - 0.0, cimag(x1[j]) - mul_bool(epsilon, b));              /* :644 */
      }
    }
  }
  if (fcalls) *fcalls = calls;
  free(x1); free(fx); free(vre);
  return 0;
}

/* ---------------------------------------------------------------------------------------------------------------
 * Jacobian-vector product — src/jvp.jl:238-274, cached in-place form finite_difference_jvp!(jvp, f, x, v, cache, f_in).
 * cache = (x1[n], fx1[m]).  dot(x, v) is BLAS ddot in Julia: restated as a sequential sum (bit-level eps unpinned,
 * like norm in the Jacobian driver; `eps_override` lets a test pin it).
 * --------------------------------------------------------------------------------------------------------------- */
int fdo_finite_difference_jvp(double *jvp, fdo_fn f, void *ctx, const double *x, const double *v, int64_t m, int64_t n,
                              double *x1, double *fx1, const double *f_in, int fdtype, double relstep, double absstep,
                              double dir, const double *eps_override, double *eps_out, int64_t *fcalls) {
  if (!jvp || !f || !x || !v || !x1 || !fx1) return 1;
  if (fdtype != FDO_FORWARD && fdtype != FDO_CENTRAL) return 2;   /* :248-250 complex rejected; fdtype_error :270 */
  if (isnan(relstep)) relstep = fdo_default_relstep(fdtype);      /* :245 */
  if (isnan(absstep)) absstep = relstep;                          /* :246 */
  double d = 0.0;
  for (int64_t j = 0; j < n; ++j) d += x[j] * v[j];
  const double tmp = sqrt(fabs(d));                               /* :252 */
  double epsilon = eps_override ? *eps_override : fdo_compute_epsilon(fdtype, tmp, relstep, absstep, dir); /* :253 */
  if (eps_out) *eps_out = epsilon;
  int64_t calls = 0;
  if (fdtype == FDO_FORWARD) {
    const double *base = fx1;
    if (!f_in) { f(ctx, fx1, x); calls++; }                       /* :255 */
    else base = f_in;                                             /* :257-258 */
    for (int64_t j = 0; j < n; ++j) x1[j] = x[j] + epsilon * v[j]; /* :260 */
    f(ctx, jvp, x1); calls++;                                      /* :261 */
    for (int64_t i = 0; i < m; ++i) jvp[i] = (jvp[i] - base[i]) / epsilon; /* :262 */
  } else {
    for (int64_t j = 0; j < n; ++j) x1[j] = x[j] - epsilon * v[j]; /* :264 */
    f(ctx, fx1, x1); calls++;                                      /* :265 */
    for (int64_t j = 0; j < n; ++j) x1[j] = x[j] + epsilon * v[j]; /* :266 */
    f(ctx, jvp, x1); calls++;                                      /* :267 */
    const double two_eps = 2 * epsilon;
    for (int64_t i = 0; i < m; ++i) jvp[i] = (jvp[i] - fx1[i]) / two_eps; /* :268 */
  }
  if (fcalls) *fcalls = calls;
  return 0;
}
