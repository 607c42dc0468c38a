/* fd_oop_oracle.c — C restatement of the reference's OUT-OF-PLACE forms (test infrastructure, gcc -ffp-contract=off):
 *   finite_difference_jacobian(f, x, cache, f_in; relstep, absstep, colorvec, sparsity, jac_prototype, dir)
 *                                                    src/jacobians.jl:277-429
 *   _make_Ji (dense and SparseMatrixCSC methods)    src/jacobians.jl:151-187, ext/FiniteDiffSparseArraysExt.jl:7-17
 *   J + Ji on SparseMatrixCSC                        SparseArrays' zero-preserving map: a result is stored only when it is
 *                                                    not iszero (restated from the stdlib; parity unpinned at source level)
 *   finite_difference_jvp(f, x, v, cache, f_in; …)   src/jvp.jl:159-189
 * Written from the reference source independently of the device code and of tests/_literal_oop.py.  f is evaluated through
 * a callback (real: fdoo_fn, complex: fdoo_fn_c on interleaved complex128), so callers can log every point. */
#include <complex.h>
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef void (*fdoo_fn)(void *ctx, double *fx, const double *x);
typedef void (*fdoo_fn_c)(void *ctx, double _Complex *fx, const double _Complex *x);

enum { FDOO_FORWARD = 0, FDOO_CENTRAL = 1, FDOO_COMPLEX = 2 };
enum { FDOO_RAW = 0, FDOO_DENSE = 1, FDOO_SPARSE = 2 };
enum { FDOO_OK = 0, FDOO_THROWS = 1, FDOO_BAD = 2 };

/* Julia max on Float64 (NaN if either is NaN; +0.0 above -0.0) */
static double jmax(double a, double b) {
  if (isnan(a) || isnan(b)) return a - b;
  return signbit(a - b) ? b : a;
}
/* compute_epsilon(Val(:forward), x, relstep, absstep, dir) = max(relstep*abs(x), absstep)*dir    epsilons.jl:26-29 */
static double eps_fwd(double x, double relstep, double absstep, double dir) { return jmax(relstep * fabs(x), absstep) * dir; }
/* compute_epsilon(Val(:central), x, relstep, absstep) = max(relstep*abs(x), absstep)             epsilons.jl:50-53 */
static double eps_cen(double x, double relstep, double absstep) { return jmax(relstep * fabs(x), absstep); }
/* e * (c == k): Julia's Bool product is a strong zero, e*false = copysign(0, e) */
static double bmul(double e, int b) { return b ? e : copysign(0.0, e); }

double fdoo_default_relstep(int fdtype) {                                         /* epsilons.jl:134-144 */
  return fdtype == FDOO_FORWARD ? sqrt(DBL_EPSILON) : (fdtype == FDOO_CENTRAL ? cbrt(DBL_EPSILON) : 1.0);
}

typedef struct {
  int64_t m, n;
  int32_t fdtype, kind;        /* FDOO_* */
  int64_t ncols;               /* columns of the prototype (dense / sparse kinds); raw: maximum(colorvec) on return */
  const int64_t *colorvec;     /* n, 1-based */
  const int64_t *colptr, *rowval; /* sparsity (1-based CSC) or NULL (sparsity === nothing) */
  const double *f_in;          /* nullable */
  double relstep, absstep, dir;
  const double *eps_override;  /* nullable: per colour of the coloured branch */
  double *J;                   /* dense result, m x ncols column-major */
  int64_t *out_colptr, *out_rowval; double *out_nzval;   /* sparse result (capacity: nnz of sparsity, or m*ncols) */
  int64_t nnz, fcalls;
  double *eps_out;             /* nullable: the step of each colour / column */
} fdoo_args;

/* one colour's dx (length m): the coloured branch (sparsity given)       jacobians.jl:338-344, 378-387, 415-418 */
static void colour_dx(fdoo_args *a, const double *x, const double *vecfx, int64_t k, fdoo_fn f, fdoo_fn_c fc, void *ctx,
                      double *dx, double *p1, double *p2, double _Complex *pc, double _Complex *fcv) {
  const int64_t n = a->n, m = a->m;
  if (a->fdtype == FDOO_COMPLEX) {
    const double e = DBL_EPSILON;                                               /* :395 */
    for (int64_t j = 0; j < n; ++j)                                             /* vecx + im*eps*(colorvec == k)  :415 */
      pc[j] = CMPLX(x[j] + 0.0, a->colorvec[j] == k ? e : 0.0);
    fc(ctx, fcv, pc); a->fcalls++;                                              /* :417 */
    for (int64_t r = 0; r < m; ++r) dx[r] = cimag(fcv[r]) / e;                  /* :418 */
    if (a->eps_out) a->eps_out[k - 1] = e;
    return;
  }
  double e;
  if (a->eps_override) e = a->eps_override[k - 1];
  else {
    double s = 0.0;                                                             /* norm(vecx .* (colorvec .== k)) :338 */
    for (int64_t j = 0; j < n; ++j) if (a->colorvec[j] == k) s += x[j] * x[j];
    e = eps_fwd(sqrt(sqrt(s)), a->relstep, a->absstep, a->dir);                 /* Val(:forward), sqrt(tmp)  :339-340 */
  }
  if (a->eps_out) a->eps_out[k - 1] = e;
  for (int64_t j = 0; j < n; ++j) p1[j] = x[j] + bmul(e, a->colorvec[j] == k);  /* :341 / :381 */
  if (a->fdtype == FDOO_FORWARD) {
    f(ctx, dx, p1); a->fcalls++;                                                /* :343 */
    for (int64_t r = 0; r < m; ++r) dx[r] = (dx[r] - vecfx[r]) / e;             /* :344 */
    return;
  }
  for (int64_t j = 0; j < n; ++j) p2[j] = x[j] - bmul(e, a->colorvec[j] == k);  /* :382 */
  double *f2 = (double *)fcv;
  f(ctx, dx, p1); a->fcalls++;                                                  /* :385 */
  f(ctx, f2, p2); a->fcalls++;                                                  /* :386 */
  for (int64_t r = 0; r < m; ++r) dx[r] = (dx[r] - f2[r]) / (2 * e);            /* :387 */
}

/* calculate_Ji_forward / _central / _complex (i)          jacobians.jl:319-327, 356-367, 397-404 */
static void column_dx(fdoo_args *a, const double *x, const double *vecfx, int64_t i, fdoo_fn f, fdoo_fn_c fc, void *ctx,
                      double *dx, double *p1, double *p2, double _Complex *pc, double _Complex *fcv) {
  const int64_t n = a->n, m = a->m;
  const double xs = x[i - 1];
  if (a->fdtype == FDOO_COMPLEX) {
    const double e = DBL_EPSILON;
    for (int64_t j = 0; j < n; ++j) pc[j] = CMPLX(x[j], 0.0);                  /* complex.(vecx) */
    pc[i - 1] = CMPLX(xs + 0.0, e);                                             /* x_save + im*epsilon   :399 */
    fc(ctx, fcv, pc); a->fcalls++;
    for (int64_t r = 0; r < m; ++r) dx[r] = cimag(fcv[r]) / e;                  /* :402 */
    if (a->eps_out) a->eps_out[i - 1] = e;
    return;
  }
  const double e = eps_fwd(xs, a->relstep, a->absstep, a->dir);                 /* :321 / :358 (Val(:forward)) */
  if (a->eps_out) a->eps_out[i - 1] = e;
  memcpy(p1, x, (size_t)n * 8);
  p1[i - 1] = xs + e;                                                           /* setindex  :322 / :359 */
  if (a->fdtype == FDOO_FORWARD) {
    f(ctx, dx, p1); a->fcalls++;
    for (int64_t r = 0; r < m; ++r) dx[r] = (dx[r] - vecfx[r]) / e;             /* :325 */
    return;
  }
  memcpy(p2, x, (size_t)n * 8);
  p2[i - 1] = xs - e;                                                           /* :360 */
  double *f2 = (double *)fcv;
  f(ctx, dx, p1); a->fcalls++;                                                  /* :363 */
  f(ctx, f2, p2); a->fcalls++;                                                  /* :364 */
  for (int64_t r = 0; r < m; ++r) dx[r] = (dx[r] - f2[r]) / (2 * e);            /* :365 */
}

int fdoo_jacobian_oop(fdoo_args *a, const double *x, fdoo_fn f, fdoo_fn_c fc, void *ctx) {
  const int64_t n = a->n, m = a->m;
  a->fcalls = 0; a->nnz = 0;
  if (n <= 0) return FDOO_BAD;                                                  /* maximum of an empty colorvec */
  int64_t C = a->colorvec[0];
  for (int64_t j = 1; j < n; ++j) if (a->colorvec[j] > C) C = a->colorvec[j];   /* maximum(colorvec) */
  if (a->relstep != a->relstep) a->relstep = fdoo_default_relstep(a->fdtype);   /* :282 (NaN: keyword not given) */
  if (a->absstep != a->absstep) a->absstep = a->relstep;                        /* :283 */
  const int dense_branch = a->colptr == NULL;
  if (a->kind == FDOO_RAW && !dense_branch) return FDOO_BAD;
  if (dense_branch && (C > n || (a->kind == FDOO_RAW && C < 1))) return FDOO_BAD;   /* BoundsError / empty mapreduce */
  if (a->kind == FDOO_RAW) a->ncols = C;
  const int64_t ncols = a->ncols;
  int rc = FDOO_OK;
  double *vecfx = NULL;
  double *dx = malloc((size_t)(m > 0 ? m : 1) * 8), *p1 = malloc((size_t)n * 8), *p2 = malloc((size_t)n * 8);
  double _Complex *pc = malloc((size_t)n * 16), *fcv = malloc((size_t)(m > 0 ? m : 1) * 16);
  double *Jv = NULL; unsigned char *st = NULL;
  int64_t E = dense_branch ? 0 : a->colptr[n] - 1;
  int64_t *ecol = NULL;
  if (a->fdtype == FDOO_FORWARD) {                                              /* :297-300 */
    vecfx = malloc((size_t)(m > 0 ? m : 1) * 8);
    if (a->f_in) memcpy(vecfx, a->f_in, (size_t)m * 8);
    else { f(ctx, vecfx, x); a->fcalls++; }
  }
  if (!dense_branch) {
    ecol = malloc((size_t)(E > 0 ? E : 1) * 8);                                 /* findstructralnz  :313-315 */
    for (int64_t c = 0; c < n; ++c)
      for (int64_t p = a->colptr[c] - 1; p < a->colptr[c + 1] - 1; ++p) ecol[p] = c + 1;
  }
  if (a->kind == FDOO_DENSE) {                                                  /* J = zero(...)  :307-309 */
    memset(a->J, 0, (size_t)(m * ncols) * 8);
  } else if (a->kind == FDOO_SPARSE) {
    const int64_t cap = dense_branch ? m * ncols : E;
    Jv = calloc((size_t)(cap > 0 ? cap : 1), 8); st = calloc((size_t)(cap > 0 ? cap : 1), 1);
  }
  for (int64_t k = 1; k <= C && rc == FDOO_OK; ++k) {
    if (dense_branch) {
      column_dx(a, x, vecfx, k, f, fc, ctx, dx, p1, p2, pc, fcv);
      if (a->kind == FDOO_RAW) { memcpy(a->J + (k - 1) * m, dx, (size_t)m * 8); continue; }   /* mapreduce hcat :330 */
      if (a->kind == FDOO_DENSE) {                                              /* J = J + _make_Ji(...)  :184-187, :336 */
        for (int64_t c = 0; c < ncols; ++c)
          for (int64_t r = 0; r < m; ++r) a->J[c * m + r] = a->J[c * m + r] + (c == k - 1 ? dx[r] : 0.0);
      } else {                                                                  /* sparse(1:nrows, fill(k), dx, ..) */
        if (k > ncols) { rc = FDOO_THROWS; break; }
        for (int64_t c = 0; c < ncols; ++c)
          for (int64_t r = 0; r < m; ++r) {
            const int64_t q = c * m + r;
            const int inj = c == k - 1;
            if (!st[q] && !inj) continue;
            const double v = (st[q] ? Jv[q] : 0.0) + (inj ? dx[r] : 0.0);
            st[q] = v != 0.0 || isnan(v);
            Jv[q] = v;
          }
      }
      continue;
    }
    colour_dx(a, x, vecfx, k, f, fc, ctx, dx, p1, p2, pc, fcv);
    if (a->kind == FDOO_DENSE) {
      /* _make_Ji(::AbstractArray, rows_index, cols_index, dx, colorvec, k, nrows, ncols)  :151-162: the picked entries'
       * rows must be distinct (a repeated row makes the comprehension index past the padded vector: it throws);
       * Ji[r, c] = dx[r] on them, `false` (0.0) elsewhere; J = J + Ji */
      int64_t *owner = malloc((size_t)(m > 0 ? m : 1) * 8);
      for (int64_t r = 0; r < m; ++r) owner[r] = -1;
      for (int64_t p = 0; p < E && rc == FDOO_OK; ++p) {
        if (a->colorvec[ecol[p] - 1] != k) continue;
        const int64_t r = a->rowval[p] - 1;
        if (owner[r] >= 0) rc = FDOO_THROWS;
        owner[r] = ecol[p] - 1;
      }
      if (rc == FDOO_OK)
        for (int64_t c = 0; c < ncols; ++c)
          for (int64_t r = 0; r < m; ++r) a->J[c * m + r] = a->J[c * m + r] + (owner[r] == c ? dx[r] : 0.0);
      free(owner);
    } else {
      /* ext/FiniteDiffSparseArraysExt.jl:7-13: sparse(rows_c, cols_c, dx[rows_c], ..) keeps explicit values; J + Ji
       * stores a result only when it is not iszero.  Both patterns are subsets of the sparsity's entries. */
      for (int64_t p = 0; p < E; ++p) {
        const int inj = a->colorvec[ecol[p] - 1] == k;
        if (!st[p] && !inj) continue;
        const double v = (st[p] ? Jv[p] : 0.0) + (inj ? dx[a->rowval[p] - 1] : 0.0);
        st[p] = v != 0.0 || isnan(v);
        Jv[p] = v;
      }
    }
  }
  if (rc == FDOO_OK && a->kind == FDOO_SPARSE) {                                /* the CSC, column-major, rows sorted */
    int64_t o = 0;
    a->out_colptr[0] = 1;
    for (int64_t c = 0; c < ncols; ++c) {
      if (dense_branch) {
        for (int64_t r = 0; r < m; ++r)
          if (st[c * m + r]) { a->out_rowval[o] = r + 1; a->out_nzval[o] = Jv[c * m + r]; ++o; }
      } else if (c < n) {
        for (int64_t p = a->colptr[c] - 1; p < a->colptr[c + 1] - 1; ++p)
          if (st[p]) { a->out_rowval[o] = a->rowval[p]; a->out_nzval[o] = Jv[p]; ++o; }
      }
      a->out_colptr[c + 1] = o + 1;
    }
    a->nnz = o;
  }
  free(dx); free(p1); free(p2); free(pc); free(fcv); free(vecfx); free(Jv); free(st); free(ecol);
  return rc;
}

/* finite_difference_jvp(f, x, v, cache, f_in; relstep, absstep, dir)   jvp.jl:159-189 */
int fdoo_jvp_oop(int64_t m, int64_t n, int fdtype, const double *x, const double *v, const double *f_in, double relstep,
                 double absstep, double dir, const double *eps_override, fdoo_fn f, void *ctx, double *jvp, double *eps_out,
                 int64_t *fcalls) {
  if (fdtype != FDOO_FORWARD && fdtype != FDOO_CENTRAL) return FDOO_BAD;
  if (relstep != relstep) relstep = fdoo_default_relstep(fdtype);
  if (absstep != absstep) absstep = relstep;
  double e;
  if (eps_override) e = *eps_override;
  else {
    double d = 0.0;
    for (int64_t j = 0; j < n; ++j) d += x[j] * v[j];                           /* dot(_vec(x), _vec(v))  :172 */
    const double tmp = sqrt(fabs(d));
    e = fdtype == FDOO_FORWARD ? eps_fwd(tmp, relstep, absstep, dir) : eps_cen(tmp, relstep, absstep);   /* :173 */
  }
  *eps_out = e;
  *fcalls = 0;
  double *x1 = malloc((size_t)(n > 0 ? n : 1) * 8), *fx = malloc((size_t)(m > 0 ? m : 1) * 8);
  if (fdtype == FDOO_FORWARD) {
    if (f_in) memcpy(fx, f_in, (size_t)m * 8);
    else { f(ctx, fx, x); ++*fcalls; }                                          /* :175 */
    for (int64_t j = 0; j < n; ++j) x1[j] = x[j] + e * v[j];                    /* :176 */
    f(ctx, jvp, x1); ++*fcalls;                                                 /* :177 */
    for (int64_t r = 0; r < m; ++r) jvp[r] = (jvp[r] - fx[r]) / e;              /* :178 */
  } else {
    for (int64_t j = 0; j < n; ++j) x1[j] = x[j] + e * v[j];                    /* :180 */
    f(ctx, jvp, x1); ++*fcalls;                                                 /* :181 */
    for (int64_t j = 0; j < n; ++j) x1[j] = x[j] - e * v[j];                    /* :182 */
    f(ctx, fx, x1); ++*fcalls;                                                  /* :183 */
    for (int64_t r = 0; r < m; ++r) jvp[r] = (jvp[r] - fx[r]) / (2 * e);        /* :184 */
  }
  free(x1); free(fx);
  return FDOO_OK;
}
