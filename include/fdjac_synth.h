/*
 * fdjac_synth.h — libfdjac_synth.so: device implementations of the SYNTHETIC f!(dx, x) functions the benchmark
 * and the parity tests differentiate (bench/test harness, not part of the product ABI).  Each is an fdb_fn
 * (include/fdjac_b200.h): batched, enqueue-only on the given stream.  Arithmetic is written with explicit
 * __dadd_rn/__dmul_rn so it is bit-identical to the CPU twins in oracle/synth_fns.c.
 *
 *   fdbs_tridiag : test/coloring_tests.jl:5-13    dx[i] = x[i-1] - 2x[i] + x[i+1]
 *   fdbs_tridiag_rows : the same stencil for a row range of the problem, reading a slice of x (column-block shards)
 *   fdbs_lap5    : test/coloring_tests.jl:99-108  clamped 5-point stencil on a g x g grid (column-major)
 *   fdbs_ellrows : dx[i] = sum_p coef[p,i]*x[cols[p,i]] + 0.1*x[cols[0,i]]^2, ELL layout [K][m]   (SURVEY.md §8d config C4)
 *   fdbs_rank1   : dx[i] = x[i]^2 + w[i]*S, S = blocked-sum(x)/n                (SURVEY.md §8d config C5 variant)
 *
 * Scalar functions f: R^n -> R (m = 1: one value per point at d_fx[b*ldfx]) for Hessians and gradients, summed in the
 * blocked order of fdbs_rank1's block sums; CPU twins in scalar_oracle/synth_scalar.c:
 *   fdbs_quartic : f = sum_i (a[i] x[i]^4 + x[i] x[i+1]) + (sum_i w[i] x[i])^2 / (2n)
 *                  Hessian diag(12 a[i] x[i]^2) + (1 on the first sub- and super-diagonal) + w w^T / n
 *   fdbs_quartic_c : its complex128 twin (an fdb_fn_c), for complex-step gradients
 *   fdbs_sumsq   : f = sum(abs2, x)
 *   fdbs_guarded : the quartic with every term guarded, g(t, c) = (isfinite(t) && |t| <= 2^500) ? t : c, plus a
 *                  signed-zero term: f = sum_i (g(a[i] x[i]^4, 1/4) + g(x[i] x[i+1], -1/2) + z[i]) + s^2 / (2n),
 *                  s = g(sum_i g(w[i] x[i], 3/4), 3/2), z[i] = (!isnan(x[i]) && signbit(x[i])) ? w[i] : 0.
 *                  Finite for every double x, so an IEEE edge value in x[k] leaves the entries of H that do not
 *                  involve k finite; sees the sign of a zero but never the sign or payload of a NaN.
 *
 * Elementwise and scalar-input functions (fdbs_scalar_ctx, n = number of outputs), for derivatives and scalar -> vector
 * gradients; CPU twins in scalar_oracle/synth_scalar.c.  Output i of a point:
 *   p_i(v) = (a[i] (v^2 v) + w[i] v^2) + v
 *   fdbs_poly / fdbs_poly_c       : v = x[i] (elementwise: d_fx[b*ldfx + i] = p_i(d_x[b*ldx + i]))
 *   fdbs_tpoly / fdbs_tpoly_c     : v = x[0] (m outputs of one scalar t: d_fx[b*ldfx + i] = p_i(d_x[b*ldx]))
 *   *_guarded                     : every term through g(., c) (c = 1/4, -1/2, 3/4) plus z = (!isnan(v) && signbit(v)) ?
 *                                   w[i] : 0 — finite for every v, sees the sign of a zero.  The complex twins guard the
 *                                   real and imaginary part of each term and add z (from the real part) to the imaginary
 *                                   part, the one a complex step reads.
 */
#ifndef FDJAC_SYNTH_H
#define FDJAC_SYNTH_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int64_t n; int64_t calls; } fdbs_tridiag_ctx;
/* slice-aware variant: rows [row0, row0+nrows) of the n-row stencil; d_x[0] is global component x0 */
typedef struct { int64_t n; int64_t row0; int64_t nrows; int64_t x0; int64_t calls; } fdbs_tridiag_rows_ctx;
typedef struct { int64_t g; int64_t calls; } fdbs_lap5_ctx;
typedef struct { int64_t m; int64_t K; const int32_t *d_cols; const double *d_coef; int64_t calls; } fdbs_ell_ctx;
typedef struct { int64_t n; const double *d_w; double *d_block_sums; int64_t max_batch; int64_t calls; } fdbs_rank1_ctx;
/* scalar functions: d_a / d_w are n doubles (device; unused by fdbs_sumsq); n <= 3 * 2^20 (3 * 2^19 for the complex twin) */
typedef struct { int64_t n; const double *d_a; const double *d_w; int64_t calls; } fdbs_scalar_ctx;

int fdbs_tridiag(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_tridiag_rows(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
/* complex128 twin of fdbs_tridiag (an fdb_fn_c): the stencil on real and imaginary parts, for the complex-step path */
int fdbs_tridiag_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_lap5(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_ellrows(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
/* complex128 twin of fdbs_ellrows (an fdb_fn_c): the same sum on complex x, x0^2 as a complex square; ld* count
 * complex elements */
int fdbs_ellrows_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_rank1(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_quartic(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_quartic_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_sumsq(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_guarded(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_poly(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_poly_guarded(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_poly_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_poly_guarded_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_tpoly(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_tpoly_guarded(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_tpoly_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
int fdbs_tpoly_guarded_c(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);
/* a callback that always fails (error-path tests) */
int fdbs_fail(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);

/* x[i] = 0.5 + u_i, u_i from splitmix64(seed, i): same generator as oracle/synth_fns.c:synth_fill_x */
int fdbs_fill_x(double *d_x, int64_t n, uint64_t seed, void *stream);
/* write a buffer larger than L2 (flushes L2 between timed iterations) */
/* store-only bandwidth probe: mode 0 constant data, mode 1 a distinct value per element */
int fdbs_store_probe(double *d_out, int64_t n, int mode, int blocks, void *stream);
/* read / write mix probe: `reads` vectors of n doubles from d_src (stride lds) read, `writes` vectors written to d_dst
 * (stride ldd), 16-byte streaming accesses; mixes (1, 0), (1, 1), (1, 2), (1, 3), (2, 1), (3, 1), (4, 3); d_sink: one double, written only on a NaN sum */
int fdbs_stream_probe(const double *d_src, int64_t lds, int reads, double *d_dst, int64_t ldd, int writes, int64_t n,
                      int blocks, double *d_sink, void *stream);
int fdbs_flush_l2(void *d_buf, int64_t bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif
