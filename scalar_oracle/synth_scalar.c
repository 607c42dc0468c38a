/* synth_scalar.c — CPU twins of the device scalar functions (finitediff.jl_b200/csrc/synth_fns.cu: k_scalar,
 * k_scalar_c): the same operations in the same blocked order — 1024-element blocks; lane l (of 32) sums the terms of
 * elements l, l+32, ..., l+992 ascending; the lanes are combined by the xor butterfly s[l] = s[l] + s[l^o] for
 * o = 16, 8, 4, 2, 1; block sums are added in block order.  -ffp-contract=off keeps every operation a single rounding. */
#include "fd_scalar_oracle.h"

#include <math.h>
#include <stddef.h>

static void butterfly(double s[32]) {
  for (int o = 16; o > 0; o >>= 1) {
    double t[32];
    for (int l = 0; l < 32; ++l) t[l] = s[l] + s[l ^ o];
    for (int l = 0; l < 32; ++l) s[l] = t[l];
  }
}

/* the K per-element terms of element i (K = 1, 2 or 4) */
typedef void (*term_fn)(const synth_scalar_ctx *c, const double *x, int64_t i, double *t);

static void blocked(const synth_scalar_ctx *c, const double *x, int K, term_fn term, double *S) {
  const int64_t n = c->n, nblk = (n + 1023) / 1024;
  for (int k = 0; k < K; ++k) S[k] = 0.0;
  for (int64_t b = 0; b < nblk; ++b) {
    double s[4][32];
    for (int l = 0; l < 32; ++l) {
      for (int k = 0; k < K; ++k) s[k][l] = 0.0;
      for (int j = 0; j < 32; ++j) {
        const int64_t i = b * 1024 + l + 32 * j;
        double t[4] = {0.0, 0.0, 0.0, 0.0};
        if (i < n) term(c, x, i, t);
        for (int k = 0; k < K; ++k) s[k][l] = s[k][l] + t[k];
      }
    }
    for (int k = 0; k < K; ++k) {
      butterfly(s[k]);
      S[k] = S[k] + s[k][0];
    }
  }
}

static void quartic_terms(const synth_scalar_ctx *c, const double *x, int64_t i, double *t) {
  const double v = x[i], q = v * v;
  t[0] = c->a[i] * (q * q);
  if (i + 1 < c->n) t[0] = t[0] + v * x[i + 1];
  t[1] = c->w[i] * v;
}

/* g(t, c) of fdbs_guarded: a term that is not finite or exceeds 2^500 in magnitude is replaced by c */
static double guard(double t, double c) { return (isfinite(t) && fabs(t) <= 0x1p500) ? t : c; }

static void guarded_terms(const synth_scalar_ctx *c, const double *x, int64_t i, double *t) {
  const double v = x[i], q = v * v;
  t[0] = guard(c->a[i] * (q * q), 0.25);
  if (i + 1 < c->n) t[0] = t[0] + guard(v * x[i + 1], -0.5);
  t[0] = t[0] + ((!isnan(v) && signbit(v)) ? c->w[i] : 0.0);
  t[1] = guard(c->w[i] * v, 0.75);
}

static void sumsq_terms(const synth_scalar_ctx *c, const double *x, int64_t i, double *t) {
  (void)c;
  t[0] = x[i] * x[i];
}

/* Julia's complex product (zr*wr - zi*wi) + i(zr*wi + zi*wr) */
static void cmul(double zr, double zi, double wr, double wi, double *r, double *i) {
  *r = zr * wr - zi * wi;
  *i = zr * wi + zi * wr;
}

static void quartic_terms_c(const synth_scalar_ctx *c, const double *x, int64_t i, double *t) {
  const double vr = x[2 * i], vi = x[2 * i + 1];
  double qr, qi, q2r, q2i;
  cmul(vr, vi, vr, vi, &qr, &qi);
  cmul(qr, qi, qr, qi, &q2r, &q2i);
  t[0] = c->a[i] * q2r;
  t[1] = c->a[i] * q2i;
  if (i + 1 < c->n) {
    double ur, ui;
    cmul(vr, vi, x[2 * i + 2], x[2 * i + 3], &ur, &ui);
    t[0] = t[0] + ur;
    t[1] = t[1] + ui;
  }
  t[2] = c->w[i] * vr;
  t[3] = c->w[i] * vi;
}

double synth_quartic(void *ctx, const double *x) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  double S[2];
  blocked(c, x, 2, quartic_terms, S);
  return c->n > 0 ? S[0] + (S[1] * S[1]) / (double)(2 * c->n) : S[0];
}

double synth_guarded(void *ctx, const double *x) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  double S[2];
  blocked(c, x, 2, guarded_terms, S);
  const double s = guard(S[1], 1.5);
  return c->n > 0 ? S[0] + (s * s) / (double)(2 * c->n) : S[0];
}

double synth_sumsq(void *ctx, const double *x) {
  double S[1];
  blocked((const synth_scalar_ctx *)ctx, x, 1, sumsq_terms, S);
  return S[0];
}

void synth_quartic_c(void *ctx, const double *x, double *out) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  double S[4];
  blocked(c, x, 4, quartic_terms_c, S);
  out[0] = S[0];
  out[1] = S[1];
  if (c->n > 0) {
    double sr, si;
    cmul(S[2], S[3], S[2], S[3], &sr, &si);
    const double d = (double)(2 * c->n);
    out[0] = out[0] + sr / d;
    out[1] = out[1] + si / d;
  }
}

/* p_i(v) of fdbs_poly / fdbs_tpoly (synth_fns.cu: poly_at, poly_at_c) */
static double poly_at(const synth_scalar_ctx *c, int64_t i, double v, int g) {
  const double q = v * v, cu = q * v;
  if (!g) return (c->a[i] * cu + c->w[i] * q) + v;
  const double t = (guard(c->a[i] * cu, 0.25) + guard(c->w[i] * q, -0.5)) + guard(v, 0.75);
  return t + ((!isnan(v) && signbit(v)) ? c->w[i] : 0.0);
}

static void poly_at_c(const synth_scalar_ctx *c, int64_t i, const double *v, double *out, int g) {
  double qr, qi, cr, ci;
  cmul(v[0], v[1], v[0], v[1], &qr, &qi);
  cmul(qr, qi, v[0], v[1], &cr, &ci);
  double t1r = c->a[i] * cr, t1i = c->a[i] * ci, t2r = c->w[i] * qr, t2i = c->w[i] * qi, t3r = v[0], t3i = v[1];
  if (g) {
    t1r = guard(t1r, 0.25); t1i = guard(t1i, 0.25);
    t2r = guard(t2r, -0.5); t2i = guard(t2i, -0.5);
    t3r = guard(t3r, 0.75); t3i = guard(t3i, 0.75);
  }
  out[0] = (t1r + t2r) + t3r;
  out[1] = (t1i + t2i) + t3i;
  if (g) out[1] = out[1] + ((!isnan(v[0]) && signbit(v[0])) ? c->w[i] : 0.0);
}

double synth_poly(void *ctx, int64_t i, double v) { return poly_at((const synth_scalar_ctx *)ctx, i, v, 0); }
double synth_poly_guarded(void *ctx, int64_t i, double v) { return poly_at((const synth_scalar_ctx *)ctx, i, v, 1); }
void synth_poly_c(void *ctx, int64_t i, const double *v, double *out) { poly_at_c((const synth_scalar_ctx *)ctx, i, v, out, 0); }
void synth_poly_guarded_c(void *ctx, int64_t i, const double *v, double *out) {
  poly_at_c((const synth_scalar_ctx *)ctx, i, v, out, 1);
}
void synth_tpoly(void *ctx, double *fx, double t) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  for (int64_t i = 0; i < c->n; ++i) fx[i] = poly_at(c, i, t, 0);
}
void synth_tpoly_guarded(void *ctx, double *fx, double t) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  for (int64_t i = 0; i < c->n; ++i) fx[i] = poly_at(c, i, t, 1);
}
void synth_tpoly_c(void *ctx, double *fx, const double *t) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  for (int64_t i = 0; i < c->n; ++i) poly_at_c(c, i, t, fx + 2 * i, 0);
}
void synth_tpoly_guarded_c(void *ctx, double *fx, const double *t) {
  const synth_scalar_ctx *c = (const synth_scalar_ctx *)ctx;
  for (int64_t i = 0; i < c->n; ++i) poly_at_c(c, i, t, fx + 2 * i, 1);
}
