// fdjac_oop.cuh — the out-of-place Jacobian and JVP (include/fdjac_b200.h, "Out-of-place Jacobian").  Included at the end
// of fdjac_abi.cu: an out-of-place plan is an in-place colour-loop plan with `oop` set (pristine points, the forward step
// rule in central mode) whose J target is the result (dense kinds).  A sparse result is formed by oop_compact: from the
// resident f! outputs directly (the in-place scatter is skipped), or, when they come in several groups, from the
// candidates the in-place scatter wrote to a plan-owned buffer.
#include "kernels_oop.cuh"

static fdb_status oop_alloc_sparse(fdb_plan *P, int64_t candidates) {
  TRY(P->alloc_t(&P->oop_vals, (size_t)std::max<int64_t>(candidates, 2)));
  const int64_t ntiles = (candidates + kTile - 1) / kTile;
  TRY(P->alloc_t(&P->oop_state, (size_t)ntiles + 1));
  return FDB_OK;
}

static fdb_plan_opts oop_opts(const fdb_plan_opts *opts) {
  fdb_plan_opts o{};
  if (opts) o = *opts;
  else o.use_current_device = 1;
  return o;
}

extern "C" {

fdb_status fdb_oop_plan_create_csc(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval,
                                   const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (result_kind != FDB_OOP_DENSE && result_kind != FDB_OOP_SPARSE)
    return fail(FDB_ERR_INVALID, "a CSC sparsity gives a dense (FDB_OOP_DENSE) or a sparse (FDB_OOP_SPARSE) result");
  if (n == 0) return fail(FDB_ERR_INVALID, "maximum(colorvec) of an empty colorvec: the reference throws");
  if (opts && opts->world > 1) return fail(FDB_ERR_UNSUPPORTED, "out-of-place plans run on one device (world <= 1)");
  if (result_kind == FDB_OOP_DENSE && m > 0) {
    int64_t conflicts = 0;   // _make_Ji (jacobians.jl:151-162) throws when two columns of one colour share a row
    TRY(fdb_check_coloring_csc(m, n, colptr, rowval, colorvec, &conflicts));
    if (conflicts > 0)
      return fail(FDB_ERR_INVALID, "invalid colouring: %lld (row, colour) collisions; the dense out-of-place result is "
                                   "undefined for it (the reference throws in _make_Ji)", (long long)conflicts);
  }
  fdb_plan_opts o = oop_opts(opts);
  o.strategy = 1;   // one fused pass over the sparsity's storage order (explicit destinations for a dense J)
  fdb_plan *raw = nullptr;
  TRY(fdb_plan_create_csc(&raw, m, n, colptr, rowval, result_kind == FDB_OOP_DENSE ? FDB_J_DENSE : FDB_J_CSC_NZVAL,
                          nullptr, nullptr, ldJ, colorvec, &o));
  PlanPtr owner(raw);
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->oop = 1;
  P->oop_kind = result_kind;
  P->oop_ncols = n;
  if (result_kind == FDB_OOP_SPARSE) {
    TRY(oop_alloc_sparse(P, P->E));
    // one group of resident f! outputs on one rank: the compaction forms the quotients itself, no candidate is stored
    P->oop_fused = P->n_groups <= 1 && P->world == 1;
    const int64_t ntiles = (P->E + kTile - 1) / kTile;
    TRY(P->alloc_t(&P->oop_tile_col, (size_t)std::max<int64_t>(ntiles, 1)));
    if (ntiles > 0) {
      oop_tile_first_col<<<P->grid(ntiles), kThreads>>>(P->colptr32, n, ntiles, P->oop_tile_col);
      CU(cudaGetLastError());
      CU(cudaDeviceSynchronize());
    }
  }
  *plan = owner.release();
  return FDB_OK;
}

fdb_status fdb_oop_plan_create_dense(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colorvec, int64_t ncols_out,
                                     int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (result_kind != FDB_OOP_RAW && result_kind != FDB_OOP_DENSE && result_kind != FDB_OOP_SPARSE)
    return fail(FDB_ERR_INVALID, "result_kind must be FDB_OOP_RAW, FDB_OOP_DENSE or FDB_OOP_SPARSE");
  if (n <= 0 || m < 0) return fail(FDB_ERR_INVALID, "n = %lld: maximum(colorvec) of an empty colorvec throws", (long long)n);
  if (opts && opts->world > 1) return fail(FDB_ERR_UNSUPPORTED, "out-of-place plans run on one device (world <= 1)");
  int dev = 0;
  TRY(check_device(opts, &dev));
  long long C = n;
  {
    DeviceGuard g(dev);
    I64View cv;
    TRY(view_i64(colorvec, n, cv));
    long long mn = 1;
    if (cv.d) TRY(color_range(cv.d, n, &C, &mn));
  }
  if (C < 1) return fail(FDB_ERR_INVALID, "maximum(colorvec) = %lld: the dense out-of-place branch has no column", C);
  if (C > n) return fail(FDB_ERR_INVALID, "maximum(colorvec) = %lld > length(x) = %lld (BoundsError in the reference)", C, (long long)n);
  if (result_kind == FDB_OOP_RAW) ncols_out = C;
  if (result_kind == FDB_OOP_DENSE && ncols_out < C)
    return fail(FDB_ERR_UNSUPPORTED, "not built: a dense prototype with fewer columns (%lld) than colours (%lld)",
                (long long)ncols_out, C);
  if (result_kind == FDB_OOP_SPARSE && ncols_out < C)
    return fail(FDB_ERR_INVALID, "a sparse prototype with %lld columns cannot hold colour %lld (sparse() throws)",
                (long long)ncols_out, C);
  if (result_kind != FDB_OOP_SPARSE && ldJ < m) return fail(FDB_ERR_INVALID, "ldJ < m");
  fdb_plan_opts o = oop_opts(opts);
  fdb_plan *raw = nullptr;
  TRY(create_dense(&raw, m, n, result_kind == FDB_OOP_SPARSE ? std::max<int64_t>(m, 1) : ldJ, C, &o));
  PlanPtr owner(raw);
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->oop = 1;
  P->oop_kind = result_kind;
  P->oop_ncols = ncols_out;
  if (result_kind == FDB_OOP_SPARSE) TRY(oop_alloc_sparse(P, m * C));
  *plan = owner.release();
  return FDB_OK;
}

static fdb_status jacobian_oop_run(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, const fdb_oop_out *out, double *d_fx,
                                   const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  if (!P || !f || !out) return fail(FDB_ERR_INVALID, "NULL plan, f or out");
  if (!P->oop) return fail(FDB_ERR_INVALID, "not an out-of-place plan (fdb_oop_plan_create_csc / _dense)");
  const bool sparse = P->oop_kind == FDB_OOP_SPARSE;
  const bool full = P->sp_kind == SP_NONE;
  const int64_t qcols = P->col_end - P->col_begin;   // dense branch: columns holding quotients, maximum(colorvec)
  const int64_t candidates = full ? P->m * qcols : P->E;
  if (sparse) {
    if (!out->colptr || !out->nnz || (candidates > 0 && (!out->rowval || !out->nzval)))
      return fail(FDB_ERR_INVALID, "NULL colptr, rowval, nzval or nnz");
    if (out->cap < candidates)
      return fail(FDB_ERR_INVALID, "rowval / nzval capacity %lld < %lld candidate entries", (long long)out->cap,
                  (long long)candidates);
  }
  double *J = sparse ? P->oop_vals : out->J;
  P->oop_entry = true;
  const fdb_status st = fdb_jacobian(P, f, ctx, d_x, J, d_fx, d_f_in, relstep, absstep, dir, stream);
  P->oop_entry = false;
  TRY(st);
  DeviceGuard g(P->device);
  cudaStream_t s = (cudaStream_t)stream;
  if (P->oop_kind == FDB_OOP_DENSE) {
    if (!full && P->E > 0) {
      oop_plus_zero_slots<<<P->grid(P->E), kThreads, 0, s>>>(J, P->dest, P->E);
      P->cnt.kernel_launches += 1;
    } else if (full && P->m > 0) {
      const int64_t work = ((P->m + kTile - 1) / kTile) * P->oop_ncols;
      const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(work, (int64_t)P->sm_count * 16));
      oop_dense_finish<<<grid, kThreads, 0, s>>>(J, P->ldJ, P->m, qcols, P->oop_ncols);
      P->cnt.kernel_launches += 1;
    }
  } else if (sparse) {
    const int64_t ntiles = (candidates + kTile - 1) / kTile;
    CU(cudaMemsetAsync(P->oop_state, 0, (size_t)(ntiles + 1) * 8, s));
    CompactArgs a{};
    a.vals = P->oop_vals; a.row32 = P->row32; a.colptr32 = P->colptr32;
    a.ecolor = P->ecolor; a.Fp = P->Fp; a.Fm = P->Fm; a.eps = P->eps; a.ncolors = P->C;
    a.fx = d_f_in ? d_f_in : (d_fx ? d_fx : P->fx_own);
    a.ldF = P->fdtype == FDB_COMPLEX ? 2 * P->ldF : P->ldF;
    a.E = candidates; a.m = P->m; a.C = qcols; a.ncols = P->oop_ncols;
    a.colptr = out->colptr; a.rowval = out->rowval; a.nzval = out->nzval; a.nnz = out->nnz;
    a.state = P->oop_state; a.claim = P->oop_state + ntiles; a.tile_col = P->oop_tile_col;
    auto go = [&](auto kern) { kern<<<resident_grid(P, kern, 0, std::max<int64_t>(ntiles, 1)), kThreads, 0, s>>>(a); };
    if (full) go(oop_compact<true, kCopy, uint8_t>);
    else if (!P->oop_fused) go(oop_compact<false, kCopy, uint8_t>);
    else TRY(dispatch_ct(P->color_bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      if (P->fdtype == FDB_CENTRAL) go(oop_compact<false, kCentral, CT>);
      else if (P->fdtype == FDB_COMPLEX) go(oop_compact<false, kComplex, CT>);
      else go(oop_compact<false, kForward, CT>);
      return FDB_OK;
    }));
    P->cnt.kernel_launches += 1;
  }
  CU(cudaGetLastError());
  return FDB_OK;
}

fdb_status fdb_jacobian_oop(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, const fdb_oop_out *out, double *d_fx,
                            const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  if (P && P->fdtype == FDB_COMPLEX)
    return fail(FDB_ERR_INVALID, "this plan is a complex-step plan: call fdb_jacobian_oop_complex with a complex128 callback");
  return jacobian_oop_run(P, f, ctx, d_x, out, d_fx, d_f_in, relstep, absstep, dir, stream);
}

fdb_status fdb_jacobian_oop_complex(fdb_plan *P, fdb_fn_c f, void *ctx, const double *d_x, const fdb_oop_out *out,
                                    void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  if (P->fdtype != FDB_COMPLEX) return fail(FDB_ERR_INVALID, "fdb_jacobian_oop_complex needs a plan created with fdtype = FDB_COMPLEX");
  P->complex_entry = true;
  const fdb_status st = jacobian_oop_run(P, reinterpret_cast<fdb_fn>(f), ctx, d_x, out, nullptr, nullptr, FDB_STEP_DEFAULT,
                                         FDB_STEP_DEFAULT, 1.0, stream);
  P->complex_entry = false;
  return st;
}

fdb_status fdb_jvp_oop(fdb_plan *P, fdb_fn f, void *ctx, double *d_jvp, const double *d_x, const double *d_v, double *d_x1,
                       double *d_fx1, const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  return jvp_run(P, f, ctx, d_jvp, d_x, d_v, d_x1, d_fx1, d_f_in, relstep, absstep, dir, stream, true);
}

}  // extern "C"
