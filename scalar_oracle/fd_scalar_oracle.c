/* fd_scalar_oracle.c — see fd_scalar_oracle.h.  Each statement cites the reference line it restates. */
#include "fd_scalar_oracle.h"

#include <float.h>
#include <math.h>
#include <string.h>

/* Julia Base.max on Float64: NaN if either is NaN, +0.0 > -0.0 */
static double max_julia(double a, double b) {
  if (isnan(a) || isnan(b)) return a - b;
  return signbit(a - b) ? b : a;
}

double fdso_default_relstep(int fdtype) {
  if (fdtype == 0) return sqrt(DBL_EPSILON);      /* :forward   epsilons.jl:137 */
  if (fdtype == 1) return cbrt(DBL_EPSILON);      /* :central   :139 */
  if (fdtype == 3) return pow(DBL_EPSILON, 0.25); /* :hcentral  :141  eps(T)^(1/4) */
  return 1.0;
}

static void steps(int fdtype, double *relstep, double *absstep) {
  if (isnan(*relstep)) *relstep = fdso_default_relstep(fdtype);
  if (isnan(*absstep)) *absstep = *relstep;
}

static double call(fdso_fn f, void *ctx, const double *x, int64_t n, fdso_log_fn log, void *log_ctx, int64_t *fcalls) {
  if (log) log(log_ctx, x, n);
  *fcalls += 1;
  return f(ctx, x);
}

int fdso_hessian(double *H, int64_t ldH, fdso_fn f, void *ctx, const double *x, int64_t n, double relstep, double absstep,
                 double *xpp, double *xpm, double *xmp, double *xmm, double *fx_out, fdso_log_fn log, void *log_ctx,
                 int64_t *fcalls) {
  if (ldH < n) return 1;
  steps(3, &relstep, &absstep);                                            /* :204-205 */
  *fcalls = 0;
  const double fx = call(f, ctx, x, n, log, log_ctx, fcalls);             /* :209 fx = f(x) */
  if (fx_out) *fx_out = fx;
  memcpy(xpp, x, (size_t)n * 8);                                           /* :213-216 copyto! */
  memcpy(xpm, x, (size_t)n * 8);
  memcpy(xmp, x, (size_t)n * 8);
  memcpy(xmm, x, (size_t)n * 8);
  for (int64_t i = 0; i < n; ++i) {                                        /* :221 */
    const double xi = x[i];                                                /* :222 */
    const double epsilon = max_julia(relstep * fabs(xi), absstep);         /* :223 compute_epsilon(Val(:hcentral), ...) */
    xpp[i] = xi + epsilon;                                                 /* :226 */
    xmm[i] = xi - epsilon;                                                 /* :227 */
    const double fpp = call(f, ctx, xpp, n, log, log_ctx, fcalls);         /* :233 f(_xpp) - 2*fx + f(_xmm), left to right */
    const double fmm = call(f, ctx, xmm, n, log, log_ctx, fcalls);
    H[i + i * ldH] = (fpp - 2 * fx + fmm) / (epsilon * epsilon);           /* epsilon^2 = literal_pow = epsilon*epsilon */
    const double epsiloni = max_julia(relstep * fabs(xi), absstep);        /* :234 compute_epsilon(Val(:central), ...) */
    const double xp = xi + epsiloni;                                       /* :235 */
    const double xm = xi - epsiloni;                                       /* :236 */
    xpp[i] = xp;                                                           /* :239-242 */
    xpm[i] = xp;
    xmp[i] = xm;
    xmm[i] = xm;
    for (int64_t j = i + 1; j < n; ++j) {                                  /* :250 */
      const double xj = x[j];                                              /* :251 */
      const double epsilonj = max_julia(relstep * fabs(xj), absstep);      /* :252 */
      const double xpj = xj + epsilonj;                                    /* :253 */
      const double xmj = xj - epsilonj;                                    /* :254 */
      xpp[j] = xpj;                                                        /* :257-260 */
      xpm[j] = xmj;
      xmp[j] = xpj;
      xmm[j] = xmj;
      const double a = call(f, ctx, xpp, n, log, log_ctx, fcalls);         /* :268-269 f(_xpp) - f(_xpm) - f(_xmp) + f(_xmm) */
      const double b = call(f, ctx, xpm, n, log, log_ctx, fcalls);
      const double c = call(f, ctx, xmp, n, log, log_ctx, fcalls);
      const double d = call(f, ctx, xmm, n, log, log_ctx, fcalls);
      H[i + j * ldH] = (a - b - c + d) / (4 * epsiloni * epsilonj);
      xpp[j] = xj;                                                         /* :272-275 */
      xpm[j] = xj;
      xmp[j] = xj;
      xmm[j] = xj;
    }
    xpp[i] = xi;                                                           /* :285-288 */
    xpm[i] = xi;
    xmp[i] = xi;
    xmm[i] = xi;
  }
  for (int64_t i = 0; i < n; ++i)                                          /* :291 copytri!(H, 'U') */
    for (int64_t j = i + 1; j < n; ++j) H[j + i * ldH] = H[i + j * ldH];
  return 0;
}

int fdso_gradient(double *df, fdso_fn f, void *ctx, const double *x, int64_t n, int fdtype, const double *fx,
                  double relstep, double absstep, double dir, double *c3, fdso_log_fn log, void *log_ctx, int64_t *fcalls) {
  if (fdtype != 0 && fdtype != 1) return 1;                                /* :470 fdtype_error */
  steps(fdtype, &relstep, &absstep);                                       /* :396-397 */
  *fcalls = 0;
  memcpy(c3, x, (size_t)n * 8);                                            /* :408 copyto!(c3, x) */
  if (fdtype == 0) {
    const double fx0 = fx ? *fx : call(f, ctx, x, n, log, log_ctx, fcalls);   /* :410 */
    for (int64_t i = 0; i < n; ++i) {                                      /* :411 */
      const double epsilon = max_julia(relstep * fabs(x[i]), absstep) * dir;   /* :412 compute_epsilon(Val(:forward), ...) */
      const double x_old = x[i];                                           /* :413 */
      c3[i] += epsilon;                                                    /* :414 */
      const double dfi = (call(f, ctx, c3, n, log, log_ctx, fcalls) - fx0) / epsilon;   /* :415 */
      c3[i] = x_old;                                                       /* :416 */
      df[i] = dfi;                                                         /* :418 real(dfi) */
    }
  } else {
    for (int64_t i = 0; i < n; ++i) {                                      /* :433 */
      const double epsilon = max_julia(relstep * fabs(x[i]), absstep);     /* :434 compute_epsilon(Val(:central), ...) */
      const double x_old = x[i];                                           /* :435 */
      c3[i] += epsilon;                                                    /* :436 */
      double dfi = call(f, ctx, c3, n, log, log_ctx, fcalls);              /* :437 */
      c3[i] = x_old - epsilon;                                             /* :438 */
      dfi -= call(f, ctx, c3, n, log, log_ctx, fcalls);                    /* :439 */
      c3[i] = x_old;                                                       /* :440 */
      df[i] = dfi / (2 * epsilon);                                         /* :441 real(dfi / (2 * epsilon)) */
    }
  }
  return 0;
}

int fdso_gradient_complex(double *df, fdso_fn_c f, void *ctx, const double *x, int64_t n, double *c1, fdso_log_fn log,
                          void *log_ctx, int64_t *fcalls) {
  *fcalls = 0;
  for (int64_t i = 0; i < n; ++i) { c1[2 * i] = x[i]; c1[2 * i + 1] = 0.0; }   /* :460 copyto!(c1, x) */
  const double epsilon_complex = DBL_EPSILON;                              /* :461 eps(real(eltype(x))) */
  for (int64_t i = 0; i < n; ++i) {                                        /* :463 */
    const double re_old = c1[2 * i], im_old = c1[2 * i + 1];               /* :464 c1_old = c1[i] */
    c1[2 * i] = re_old + 0.0;                                              /* :465 c1[i] += im * epsilon_complex: */
    c1[2 * i + 1] = im_old + epsilon_complex;                              /*      im*eps = Complex(0.0, eps) */
    double out[2];
    if (log) log(log_ctx, c1, 2 * n);
    *fcalls += 1;
    f(ctx, c1, out);
    df[i] = out[1] / epsilon_complex;                                      /* :466 imag(f(c1)) / epsilon_complex */
    c1[2 * i] = re_old;                                                    /* :467 */
    c1[2 * i + 1] = im_old;
  }
  return 0;
}

static double epsilon_of(int fdtype, double x, double relstep, double absstep, double dir) {
  const double e = max_julia(relstep * fabs(x), absstep);                 /* epsilons.jl:28 / :52 */
  return fdtype == 0 ? e * dir : e;
}

int fdso_derivative(double *df, fdso_efn f, void *ctx, const double *x, int64_t n, int fdtype, const double *fx,
                    double relstep, double absstep, double dir, fdso_log_fn log, void *log_ctx, int64_t *fcalls) {
  if (fdtype != 0 && fdtype != 1) return 1;                                /* :229-230 fdtype_error */
  steps(fdtype, &relstep, &absstep);                                       /* :202-203 */
  *fcalls = 0;
  for (int64_t i = 0; i < n; ++i) {                                        /* :208 / :218 */
    const double epsilon = epsilon_of(fdtype, x[i], relstep, absstep, dir);   /* :209 / :219 */
    if (fdtype == 0) {
      const double x_plus = x[i] + epsilon;                                /* :210 */
      if (log) log(log_ctx, &x_plus, 1);
      *fcalls += 1;
      const double fp = f(ctx, i, x_plus);                                 /* :212 f(x_plus) - f(x[i]), left to right */
      double fb;
      if (fx) {
        fb = fx[i];                                                        /* :214 */
      } else {
        if (log) log(log_ctx, &x[i], 1);
        *fcalls += 1;
        fb = f(ctx, i, x[i]);
      }
      df[i] = (fp - fb) / epsilon;
    } else {
      const double epsilon_double_inv = 1.0 / (2 * epsilon);               /* :220 */
      const double x_plus = x[i] + epsilon, x_minus = x[i] - epsilon;      /* :221 */
      if (log) log(log_ctx, &x_plus, 1);
      *fcalls += 1;
      const double fp = f(ctx, i, x_plus);                                 /* :222 */
      if (log) log(log_ctx, &x_minus, 1);
      *fcalls += 1;
      const double fm = f(ctx, i, x_minus);
      df[i] = (fp - fm) * epsilon_double_inv;
    }
  }
  return 0;
}

int fdso_derivative_complex(double *df, fdso_efn_c f, void *ctx, const double *x, int64_t n, fdso_log_fn log,
                            void *log_ctx, int64_t *fcalls) {
  *fcalls = 0;
  const double epsilon_complex = DBL_EPSILON;                              /* :225 eps(eltype(x)) */
  for (int64_t i = 0; i < n; ++i) {                                        /* :226 */
    const double z[2] = {x[i] + 0.0, epsilon_complex};                     /* :227 x[i] + im*eps: im*eps = (false*eps, eps) */
    double out[2];
    if (log) log(log_ctx, z, 2);
    *fcalls += 1;
    f(ctx, i, z, out);
    df[i] = out[1] / epsilon_complex;                                      /* imag(f(..)) / epsilon_complex */
  }
  return 0;
}

int fdso_scalar_gradient(double *df, fdso_vfn f, void *ctx, double x, int64_t m, int fdtype, const double *fx,
                         double relstep, double absstep, double dir, double *c1, double *c2, fdso_log_fn log,
                         void *log_ctx, int64_t *fcalls) {
  if (fdtype != 0 && fdtype != 1) return 1;                                /* :530 fdtype_error */
  steps(fdtype, &relstep, &absstep);                                       /* :482-483 */
  *fcalls = 0;
  const double epsilon = epsilon_of(fdtype, x, relstep, absstep, dir);     /* :495 / :512 */
  const double xp = x + epsilon;
  if (log) log(log_ctx, &xp, 1);
  *fcalls += 1;
  f(ctx, c1, xp);                                                          /* :497 / :514 f(c1, x + epsilon) */
  if (fdtype == 0) {
    if (fx) {
      for (int64_t i = 0; i < m; ++i) df[i] = (c1[i] - fx[i]) / epsilon;   /* :502 */
    } else {
      if (log) log(log_ctx, &x, 1);
      *fcalls += 1;
      f(ctx, c2, x);                                                       /* :505 f(c2, x) */
      for (int64_t i = 0; i < m; ++i) df[i] = (c1[i] - c2[i]) / epsilon;   /* :509 */
    }
  } else {
    const double xm = x - epsilon;
    if (log) log(log_ctx, &xm, 1);
    *fcalls += 1;
    f(ctx, c2, xm);                                                        /* :515 f(c2, x - epsilon) */
    for (int64_t i = 0; i < m; ++i) df[i] = (c1[i] - c2[i]) / (2 * epsilon);   /* :520 */
  }
  return 0;
}

int fdso_scalar_gradient_complex(double *df, fdso_vfn_c f, void *ctx, double x, int64_t m, double *c1, fdso_log_fn log,
                                 void *log_ctx, int64_t *fcalls) {
  *fcalls = 0;
  const double epsilon_complex = DBL_EPSILON;                              /* :522 eps(real(eltype(x))) */
  const double z[2] = {x + 0.0, epsilon_complex};                          /* :524 x + im*epsilon_complex */
  if (log) log(log_ctx, z, 2);
  *fcalls += 1;
  f(ctx, c1, z);                                                           /* :524 f(c1, ..) */
  for (int64_t i = 0; i < m; ++i) df[i] = c1[2 * i + 1] / epsilon_complex;   /* :528 imag(c1) / epsilon_complex */
  return 0;
}
