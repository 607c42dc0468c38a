/*
 * fd_scalar_oracle.h — plain-C restatement of the reference's vector->scalar entry points (TEST INFRASTRUCTURE: only
 * tests/ and scripts/ load it; the product library never does).  Written line by line after
 *   finite_difference_hessian!(H, f, x, cache::HessianCache; relstep, absstep)          src/hessians.jl:202-292
 *   finite_difference_gradient!(df, f, x, cache::GradientCache; relstep, absstep, dir)   src/gradients.jl:390-473
 * and of the scalar-input entry points
 *   finite_difference_derivative!(df, f, x::StridedArray, cache::DerivativeCache)          src/derivatives.jl:197-233
 *   finite_difference_gradient!(df, f, x::Number, cache::GradientCache)                    src/gradients.jl:477-533
 * separately from the Jacobian oracle in oracle/, so that "the gradient is the dense Jacobian with m = 1" is a tested
 * claim.  Compiled with -ffp-contract=off: every operation rounds once, in the order the Julia source writes it.
 * relstep / absstep: NaN = keyword not given (default_relstep(fdtype), absstep = relstep), any other value as passed.
 */
#ifndef FD_SCALAR_ORACLE_H
#define FD_SCALAR_ORACLE_H
#include <stdint.h>

/* scalar f(x) of a real vector of n doubles */
typedef double (*fdso_fn)(void *ctx, const double *x);
/* complex-valued f of a complex vector: x and out are complex128 as interleaved (re, im) doubles; out is one value */
typedef void (*fdso_fn_c)(void *ctx, const double *x, double *out);
/* f-call log: called with the argument of every f call, in call order, just before the call (count doubles) */
typedef void (*fdso_log_fn)(void *log_ctx, const double *x, int64_t count);

/* src/hessians.jl:202-292.  H column-major, leading dimension ldH >= n (rows >= n untouched).  xpp..xmm: the cache (n
 * doubles each; contents are scratch, overwritten before use).  fx_out (nullable) receives f(x). */
int fdso_hessian(double *H, int64_t ldH, fdso_fn f, void *ctx, const double *x, int64_t n, double relstep, double absstep,
                 double *xpp, double *xpm, double *xmp, double *xmm, double *fx_out, fdso_log_fn log, void *log_ctx,
                 int64_t *fcalls);

/* src/gradients.jl:390-457, real x and df: fdtype 0 forward (fx: cache.fx or NULL => f(x) is evaluated first, :410) or
 * 1 central; c3: n doubles of scratch.  Returns nonzero for another fdtype. */
int fdso_gradient(double *df, fdso_fn f, void *ctx, const double *x, int64_t n, int fdtype, const double *fx,
                  double relstep, double absstep, double dir, double *c3, fdso_log_fn log, void *log_ctx, int64_t *fcalls);

/* src/gradients.jl:458-469: complex step with real x, df and return type; c1: 2n doubles of scratch (complex(x)). */
int fdso_gradient_complex(double *df, fdso_fn_c f, void *ctx, const double *x, int64_t n, double *c1, fdso_log_fn log,
                          void *log_ctx, int64_t *fcalls);

/* Scalar-input entry points.  The reference calls f on one scalar at a time; these restatements do the same.
 *   fdso_efn   f of component i (the index lets a synthetic f carry per-component coefficients; the reference's f has none)
 *   fdso_efn_c its complex128 form: x and out are one (re, im) pair
 *   fdso_vfn   the in-place scalar -> vector f(fx, t): fills m doubles
 *   fdso_vfn_c its complex form: t one (re, im) pair, fx m complex128 values */
typedef double (*fdso_efn)(void *ctx, int64_t i, double x);
typedef void (*fdso_efn_c)(void *ctx, int64_t i, const double *x, double *out);
typedef void (*fdso_vfn)(void *ctx, double *fx, double t);
typedef void (*fdso_vfn_c)(void *ctx, double *fx, const double *t);

/* src/derivatives.jl:197-223, StridedArray x and df: fdtype 0 forward (fx: cache.fx, n values, or NULL => f(x[i]) after
 * f(x[i] + eps)) or 1 central.  Returns nonzero for another fdtype.  The log sees every scalar argument. */
int fdso_derivative(double *df, fdso_efn f, void *ctx, const double *x, int64_t n, int fdtype, const double *fx,
                    double relstep, double absstep, double dir, fdso_log_fn log, void *log_ctx, int64_t *fcalls);
/* src/derivatives.jl:224-228: complex step, real x and df (the log sees each complex argument as 2 doubles) */
int fdso_derivative_complex(double *df, fdso_efn_c f, void *ctx, const double *x, int64_t n, fdso_log_fn log,
                            void *log_ctx, int64_t *fcalls);
/* src/gradients.jl:477-520, scalar x, m outputs: fdtype 0 forward (fx: cache.fx, m values, or NULL => f(c2, x) after
 * f(c1, x + eps)) or 1 central; c1, c2: m doubles of scratch. */
int fdso_scalar_gradient(double *df, fdso_vfn f, void *ctx, double x, int64_t m, int fdtype, const double *fx,
                         double relstep, double absstep, double dir, double *c1, double *c2, fdso_log_fn log,
                         void *log_ctx, int64_t *fcalls);
/* src/gradients.jl:521-528: complex step; c1: 2m doubles (m complex128 values) */
int fdso_scalar_gradient_complex(double *df, fdso_vfn_c f, void *ctx, double x, int64_t m, double *c1, fdso_log_fn log,
                                 void *log_ctx, int64_t *fcalls);

double fdso_default_relstep(int fdtype);   /* epsilons.jl:134-144; fdtype 3 = hcentral */

/* CPU twins of the device scalar functions of include/fdjac_synth.h (same operations, same blocked order, same bits) */
typedef struct { int64_t n; const double *a; const double *w; } synth_scalar_ctx;
double synth_quartic(void *ctx, const double *x);
double synth_sumsq(void *ctx, const double *x);
double synth_guarded(void *ctx, const double *x);
void synth_quartic_c(void *ctx, const double *x, double *out);
/* twins of fdbs_poly[_guarded][_c] (elementwise, component i) and fdbs_tpoly[_guarded][_c] (n outputs of one t) */
double synth_poly(void *ctx, int64_t i, double v);
double synth_poly_guarded(void *ctx, int64_t i, double v);
void synth_poly_c(void *ctx, int64_t i, const double *v, double *out);
void synth_poly_guarded_c(void *ctx, int64_t i, const double *v, double *out);
void synth_tpoly(void *ctx, double *fx, double t);
void synth_tpoly_guarded(void *ctx, double *fx, double t);
void synth_tpoly_c(void *ctx, double *fx, const double *t);
void synth_tpoly_guarded_c(void *ctx, double *fx, const double *t);

#endif
