// fdjac_oop.cuh — the out-of-place Jacobian and JVP (include/fdjac_b200.h, "Out-of-place Jacobian").  Included at the end
// of fdjac_abi.cu: an out-of-place plan is an in-place colour-loop plan with `oop.on` set (pristine points, the forward step
// rule in central mode) whose J target is the result (dense kinds).  A sparse result is formed by oop_compact: from the
// resident f! outputs directly (the in-place scatter is skipped), or, when they come in several groups or several ranks,
// from the candidates the in-place scatter wrote to a plan-owned buffer (the root's, for a group).
//
// Rank plans (opts.world > 1) evaluate only their own colours (dense branch: their column block).  Every colour's point
// starts from the caller's x, so a colour's quotients depend on x and its own step alone and the ranks need no exchange:
// each writes exactly its own slots (oop_member), and only a sparse result has a root-only step, the compaction over
// every candidate (oop_root_finish) once every member has finished.
#include "kernels_oop.cuh"

// `vals`: doubles of the candidate buffer the colour loop writes (the band data of a band sparsity)
static fdb_status oop_alloc_sparse(fdb_plan *P, int64_t candidates, int64_t vals) {
  TRY(P->alloc_t(&P->oop.vals, (size_t)std::max<int64_t>(vals, 2)));
  const int64_t ntiles = (candidates + kTile - 1) / kTile;
  TRY(P->alloc_t(&P->oop.state, (size_t)ntiles + 1));
  return FDB_OK;
}

static fdb_plan_opts oop_opts(const fdb_plan_opts *opts) {
  fdb_plan_opts o{};
  if (opts) o = *opts;
  else o.use_current_device = 1;
  return o;
}

// the slots of a dense result (CSC sparsity) whose `+ 0.0` this rank applies: those of the colours it owns.  One rank
// owns them all, and `dest` itself is used.
static fdb_status oop_own_slots(fdb_plan *P) {
  if (P->world == 1) {
    P->oop.dest = P->entries.dest;
    P->oop.dest_n = P->colors.E;
    return FDB_OK;
  }
  const int64_t E = P->colors.E;
  const size_t cb = (size_t)P->colors.bits / 8;
  std::vector<int64_t> dest((size_t)E), own;
  std::vector<uint8_t> ec((size_t)E * cb);
  if (E > 0) {
    TRY(read_back(dest.data(), P->entries.dest, (size_t)E, "reading the dense result's slots"));
    TRY(read_back(ec.data(), (const uint8_t *)P->entries.ecolor, (size_t)E * cb, "reading the entry colours"));
  }
  for (int64_t e = 0; e < E; ++e) {
    const uint8_t *p = ec.data() + (size_t)e * cb;
    const uint32_t k = cb == 1 ? *p : (cb == 2 ? *reinterpret_cast<const uint16_t *>(p) : *reinterpret_cast<const uint32_t *>(p));
    if (k < (uint32_t)P->colors.C && P->colors.owner[k] == P->rank) own.push_back(dest[(size_t)e]);
  }
  int64_t *d = nullptr;
  TRY(P->alloc_t(&d, std::max<size_t>(own.size(), 1)));
  if (!own.empty()) CU(cudaMemcpy(d, own.data(), own.size() * 8, cudaMemcpyHostToDevice));
  P->oop.dest = d;
  P->oop.dest_n = (int64_t)own.size();
  return FDB_OK;
}

// candidates of the whole result: nnz of the sparsity, or m x maximum(colorvec) on the dense branch
static int64_t oop_candidates(const fdb_plan *P) {
  if (P->sp_kind == SP_BANDED) return P->oop.band_nnz;
  return P->sp_kind == SP_NONE ? P->m * P->oop.qcols : P->colors.E;
}

// the entry set of a band plan (its bandwidths are clamped to the matrix at creation)
static BandShape oop_band_shape(const fdb_plan *P) { return make_band_shape(P->m, P->n, P->band.l, P->band.u); }

// the entry set of a block-banded or block-dense plan (kernels_oop.cuh, BlockShape)
static BlockShape oop_block_shape(const fdb_plan *P) {
  const auto &bb = P->block_band;
  BlockShape b{};
  b.boff = bb.off;
  b.start = P->jkind == FDB_J_BLOCK_DENSE ? bb.start : P->oop.block_start;
  b.jcolor = P->colors.jcolor;
  b.n = P->n; b.lam = bb.lam; b.mu = bb.mu; b.u_full = P->band.u; b.w = bb.w;
  b.nblocks = bb.nblocks;
  b.l = (int32_t)std::min<int64_t>(P->band.l, bb.nblocks);
  b.u = (int32_t)std::min<int64_t>(P->band.u, bb.nblocks);
  b.bs = bb.bs;
  b.block_cyclic = bb.cyclic ? 1 : 0;
  b.bw = make_fastdiv((uint32_t)(P->band.l + P->band.u + 1));
  b.sw = make_fastdiv((uint32_t)(bb.lam + bb.mu + 1));
  return b;
}

// A block or CSR sparsity gives the sparse result only: a dense one would cost the m x n zero fill that the CSC route's
// entry list already undercuts at any size where it fits
static fdb_status oop_block_result(int result_kind, const char *what) {
  if (result_kind == FDB_OOP_DENSE)
    return fail(FDB_ERR_UNSUPPORTED, "not built: a dense out-of-place result of a %s sparsity (give a sparse prototype, "
                                     "or a CSC sparsity)", what);
  if (result_kind != FDB_OOP_SPARSE)
    return fail(FDB_ERR_INVALID, "a %s sparsity gives a sparse (FDB_OOP_SPARSE) result", what);
  return FDB_OK;
}

// The out-of-place form of an in-place block or CSR plan: the sparse result over its |E| = colors.E candidates
static fdb_status oop_block_finish(PlanPtr &owner, fdb_plan **plan) {
  fdb_plan *P = owner.get();
  P->oop.on = 1;
  P->oop.kind = FDB_OOP_SPARSE;
  P->oop.ncols = P->n;
  // many colours: the step sizes from the per-colour column lists, in the CSC plan's summation order
  if (P->colors.C > kEpsRegColors) TRY(build_color_lists(P));
  if (P->rank == 0) {
    // one group of resident f! outputs on one rank: the compaction forms the quotients itself; otherwise the colour loop's
    // block scatter writes the candidates in the in-place layout (every rank into the root's buffer)
    P->oop.fused = P->scratch.n_groups <= 1 && P->world == 1;
    TRY(oop_alloc_sparse(P, P->colors.E, P->oop.fused ? 0 : P->j_len));
  }
  *plan = owner.release();
  return FDB_OK;
}

extern "C" {

fdb_status fdb_oop_plan_create_csc(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval,
                                   const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (result_kind != FDB_OOP_DENSE && result_kind != FDB_OOP_SPARSE)
    return fail(FDB_ERR_INVALID, "a CSC sparsity gives a dense (FDB_OOP_DENSE) or a sparse (FDB_OOP_SPARSE) result");
  if (n == 0) return fail(FDB_ERR_INVALID, "maximum(colorvec) of an empty colorvec: the reference throws");
  if (opts && opts->world > 64) return fail(FDB_ERR_INVALID, "out-of-place plans take world <= 64");
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
  P->oop.on = 1;
  P->oop.kind = result_kind;
  P->oop.ncols = n;
  if (result_kind == FDB_OOP_DENSE) TRY(oop_own_slots(P));
  if (result_kind == FDB_OOP_SPARSE && P->rank == 0) {   // the candidate buffer and the compaction are the root's
    TRY(oop_alloc_sparse(P, P->colors.E, P->colors.E));
    // one group of resident f! outputs on one rank: the compaction forms the quotients itself, no candidate is stored
    P->oop.fused = P->scratch.n_groups <= 1 && P->world == 1;
    const int64_t ntiles = (P->colors.E + kTile - 1) / kTile;
    TRY(P->alloc_t(&P->oop.tile_col, (size_t)std::max<int64_t>(ntiles, 1)));
    if (ntiles > 0) {
      oop_tile_first_col<<<P->grid(ntiles), kThreads>>>(P->entries.colptr32, n, ntiles, P->oop.tile_col);
      CU(cudaGetLastError());
      CU(cudaDeviceSynchronize());
    }
  }
  *plan = owner.release();
  return FDB_OK;
}

fdb_status fdb_oop_plan_create_banded(fdb_plan **plan, int64_t m, int64_t n, int64_t l, int64_t u, const int64_t *colorvec,
                                      int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (result_kind != FDB_OOP_DENSE && result_kind != FDB_OOP_SPARSE)
    return fail(FDB_ERR_INVALID, "a banded sparsity gives a dense (FDB_OOP_DENSE) or a sparse (FDB_OOP_SPARSE) result");
  if (n == 0) return fail(FDB_ERR_INVALID, "maximum(colorvec) of an empty colorvec: the reference throws");
  if (m < 0 || n < 0) return fail(FDB_ERR_INVALID, "negative dimensions m=%lld n=%lld", (long long)m, (long long)n);
  if (l < 0 || u < 0)
    return fail(FDB_ERR_UNSUPPORTED, "not built: negative bandwidths (l, u) = (%lld, %lld) in the out-of-place Jacobian",
                (long long)l, (long long)u);
  if (opts && opts->world > 64) return fail(FDB_ERR_INVALID, "out-of-place plans take world <= 64");
  // bandwidths beyond the matrix give the same entry set as the matrix's own: the candidates and band data use those
  const int64_t lc = std::min<int64_t>(l, std::max<int64_t>(m - 1, 0)), uc = std::min<int64_t>(u, n - 1);
  if (m > 0x7FFFFFF0LL || n > 0x7FFFFFF0LL || lc + uc + 1 > 0x7FFFFFF0LL)
    return fail(FDB_ERR_UNSUPPORTED, "banded out-of-place plans take m, n and l + u + 1 below 2^31");
  fdb_plan_opts o = oop_opts(opts);
  fdb_plan *raw = nullptr;
  TRY(fdb_plan_create_banded(&raw, m, n, lc, uc, result_kind == FDB_OOP_DENSE ? FDB_J_DENSE : FDB_J_BAND, ldJ, colorvec, &o));
  PlanPtr owner(raw);
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->oop.on = 1;
  P->oop.kind = result_kind;
  P->oop.ncols = n;
  const BandShape b = oop_band_shape(P);
  P->oop.band_nnz = b.E;
  // many colours: the step sizes from the per-colour column lists, in the CSC plan's summation order
  if (P->colors.C > kEpsRegColors && n > 0) TRY(build_color_lists(P));
  // _make_Ji (jacobians.jl:151-162) throws when two columns of one colour share a row.  A cyclic colouring with more
  // colours than l + u gives distinct colours to every pair of columns that can share one.
  if (result_kind == FDB_OOP_DENSE && m > 0 && P->colors.C > 0 && !(P->colors.cyclic && P->colors.C > lc + uc)) {
    DevBuf<unsigned long long> d_c;
    TRY(d_c.alloc(1));
    CU(cudaMemset(d_c.get(), 0, 8));
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) {
      return dispatch_colors<decltype(tag)>(P, [&](auto cs) -> fdb_status {
        count_band_conflicts<<<P->grid(n), kThreads>>>(b, cs, P->colors.C, d_c.get());
        CU(cudaGetLastError());
        return FDB_OK;
      });
    }));
    unsigned long long conflicts = 0;
    TRY(read_back(&conflicts, d_c.get(), 1, "conflict count"));
    if (conflicts > 0)
      return fail(FDB_ERR_INVALID, "invalid colouring: %lld (row, colour) collisions; the dense out-of-place result is "
                                   "undefined for it (the reference throws in _make_Ji)", (long long)conflicts);
  }
  if (result_kind == FDB_OOP_SPARSE && P->rank == 0) {
    // one group of resident f! outputs on one rank: the compaction forms the quotients itself; otherwise the colour loop's
    // band scatter writes the candidates in band-data layout (every rank into the root's buffer)
    P->oop.fused = P->scratch.n_groups <= 1 && P->world == 1;
    TRY(oop_alloc_sparse(P, b.E, P->oop.fused ? 0 : P->j_len));
  }
  *plan = owner.release();
  return FDB_OK;
}

// BandedBlockBandedMatrix with square blocks: the in-place block-banded plan (block offsets, cyclic-colour detection)
// plus the entries of E before every block column.  Host work O(nblocks).
fdb_status fdb_oop_plan_create_block_banded(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                            int64_t lam, int64_t mu, const int64_t *colorvec, int result_kind, int64_t ldJ,
                                            const fdb_plan_opts *opts) {
  (void)ldJ;   // a sparse result has no leading dimension
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  TRY(oop_block_result(result_kind, "block-banded"));
  if (opts && opts->world > 64) return fail(FDB_ERR_INVALID, "out-of-place plans take world <= 64");
  fdb_plan_opts o = oop_opts(opts);
  fdb_plan *raw = nullptr;
  // the candidate buffer of a kCopy plan is the in-place band data: ldata is the plan's own
  TRY(fdb_plan_create_block_banded(&raw, nblocks, blocks, l, u, lam, mu, INT64_MAX, colorvec, &o));
  PlanPtr owner(raw);
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (P->n == 0) return fail(FDB_ERR_INVALID, "maximum(colorvec) of an empty colorvec: the reference throws");
  const int32_t N = P->block_band.nblocks;
  std::vector<int64_t> st((size_t)N + 1, 0);
  {
    DevBuf<int64_t> d_cnt;
    TRY(d_cnt.alloc((size_t)N));
    const BlockShape b = oop_block_shape(P);
    block_band_col_counts<<<P->grid(N), kThreads>>>(b.boff, N, b.l, b.u, b.lam, b.mu, d_cnt.get());
    CU(cudaGetLastError());
    TRY(read_back(st.data() + 1, d_cnt.get(), (size_t)N, "block-column entry counts"));
  }
  for (int32_t J = 0; J < N; ++J) st[(size_t)J + 1] += st[(size_t)J];
  TRY(P->alloc_t(&P->oop.block_start, (size_t)N + 1));
  CU(cudaMemcpy(P->oop.block_start, st.data(), ((size_t)N + 1) * 8, cudaMemcpyHostToDevice));
  return oop_block_finish(owner, plan);
}

// BlockSkylineMatrix (BlockBandedMatrices' BlockBandedMatrix) with square blocks: the in-place block-dense plan, whose slab
// starts are the block-column starts of E.  Host work O(nblocks).
fdb_status fdb_oop_plan_create_block_dense(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                           const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  (void)ldJ;
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  TRY(oop_block_result(result_kind, "block-dense"));
  if (opts && opts->world > 64) return fail(FDB_ERR_INVALID, "out-of-place plans take world <= 64");
  fdb_plan_opts o = oop_opts(opts);
  fdb_plan *raw = nullptr;
  TRY(fdb_plan_create_block_dense(&raw, nblocks, blocks, l, u, INT64_MAX, colorvec, &o));
  PlanPtr owner(raw);
  DeviceGuard g(owner->device);
  if (owner->n == 0) return fail(FDB_ERR_INVALID, "maximum(colorvec) of an empty colorvec: the reference throws");
  return oop_block_finish(owner, plan);
}

// A CSR sparsity: the in-place CSR plan (row pointer and columns as 0-based int32) plus, at the root, the first row
// starting in every compaction tile.  The result is a CSR in the sparsity's own storage order.
fdb_status fdb_oop_plan_create_csr(fdb_plan **plan, int64_t m, int64_t n, const int64_t *rowptr, const int64_t *colval,
                                   const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  (void)ldJ;   // a sparse result has no leading dimension
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  TRY(oop_block_result(result_kind, "CSR"));
  if (n == 0) return fail(FDB_ERR_INVALID, "maximum(colorvec) of an empty colorvec: the reference throws");
  if (opts && opts->world > 64) return fail(FDB_ERR_INVALID, "out-of-place plans take world <= 64");
  fdb_plan_opts o = oop_opts(opts);
  fdb_plan *raw = nullptr;
  TRY(fdb_plan_create_csr(&raw, m, n, rowptr, colval, colorvec, &o));
  PlanPtr owner(raw);
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (P->rank == 0) {
    const int64_t ntiles = (P->colors.E + kTile - 1) / kTile;
    TRY(P->alloc_t(&P->oop.tile_col, (size_t)std::max<int64_t>(ntiles, 1)));
    if (ntiles > 0) {
      oop_tile_first_col<<<P->grid(ntiles), kThreads>>>(P->csr.rowptr, m, ntiles, P->oop.tile_col);
      CU(cudaGetLastError());
      CU(cudaDeviceSynchronize());
    }
  }
  return oop_block_finish(owner, plan);
}

fdb_status fdb_oop_plan_create_dense(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colorvec, int64_t ncols_out,
                                     int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (result_kind != FDB_OOP_RAW && result_kind != FDB_OOP_DENSE && result_kind != FDB_OOP_SPARSE)
    return fail(FDB_ERR_INVALID, "result_kind must be FDB_OOP_RAW, FDB_OOP_DENSE or FDB_OOP_SPARSE");
  if (n <= 0 || m < 0) return fail(FDB_ERR_INVALID, "n = %lld: maximum(colorvec) of an empty colorvec throws", (long long)n);
  if (opts && opts->world > 64) return fail(FDB_ERR_INVALID, "out-of-place plans take world <= 64");
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
  // maximum(colorvec) < 1: the reference's colour loop 1:maximum(colorvec) is empty and J = zero(jac_prototype) is returned
  // as it was made (after f(x) in forward mode); without a prototype it sizes J by mapreduce over that empty range, which
  // throws.  C = 0 quotient columns: the finish zero-fills a dense prototype, the compaction of 0 candidates writes colptr 1
  if (C < 1 && result_kind == FDB_OOP_RAW)
    return fail(FDB_ERR_INVALID, "maximum(colorvec) = %lld: the dense out-of-place branch has no column", C);
  if (C < 1) C = 0;
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
  P->oop.on = 1;
  P->oop.kind = result_kind;
  P->oop.ncols = ncols_out;
  P->oop.qcols = C;
  if (result_kind == FDB_OOP_SPARSE && P->rank == 0) TRY(oop_alloc_sparse(P, m * C, m * C));
  *plan = owner.release();
  return FDB_OK;
}

}  // extern "C"

// `out` can take the whole result of P's kind
static fdb_status oop_check_out(const fdb_plan *P, const fdb_oop_out *out) {
  if (P->oop.kind != FDB_OOP_SPARSE) return FDB_OK;
  const int64_t candidates = oop_candidates(P);
  if (!out->colptr || !out->nnz || (candidates > 0 && (!out->rowval || !out->nzval)))
    return fail(FDB_ERR_INVALID, "NULL colptr, rowval, nzval or nnz");
  if (out->cap < candidates)
    return fail(FDB_ERR_INVALID, "rowval / nzval capacity %lld < %lld candidate entries", (long long)out->cap,
                (long long)candidates);
  return FDB_OK;
}

// One rank's share: the colour loop of its colours (dense branch: its column block) and the finish of exactly the slots
// it owns.  `base` is the whole target: the dense result, or the root's candidate buffer of a sparse result.
static fdb_status oop_member(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, double *base, double *d_fx,
                             const double *d_f_in, double relstep, double absstep, double dir, cudaStream_t s) {
  if (oop_idle(P)) return FDB_OK;
  const bool full = P->sp_kind == SP_NONE;
  double *J = base + P->columns.begin * P->ldJ;   // dense branch: this rank's column block
  DeviceGuard g(P->device);
  // a sparse result whose colorvec has no valid colour: nobody scatters, and the candidates are the zeros of rank 0
  // band and block-band data: every column's slots
  const int64_t cand_len = P->sp_kind == SP_BANDED || P->sp_kind == SP_BLOCKBAND ? P->j_len : P->colors.E;
  if (P->oop.kind == FDB_OOP_SPARSE && !full && P->world > 1 && P->colors.local.empty() && cand_len > 0)
    CU(cudaMemsetAsync(J, 0, (size_t)cand_len * 8, s));
  if ((P->n > 0 && !d_x) || (P->j_len > 0 && !J)) return fail(FDB_ERR_INVALID, "NULL x or J");
  TRY(jacobian_run(P, f, ctx, d_x, J, d_fx, d_f_in, relstep, absstep, dir, (void *)s));
  if (P->oop.kind == FDB_OOP_DENSE) {
    if (P->sp_kind == SP_BANDED) {
      // + 0.0 over the band entries of this rank's colours, in closed form
      const BandShape b = oop_band_shape(P);
      if (b.E > 0 && !P->colors.local.empty()) {
        TRY(dispatch_ct(P->colors.bits, [&](auto tag) {
          return dispatch_colors<decltype(tag)>(P, [&](auto cs) -> fdb_status {
            oop_band_plus_zero<<<P->grid(b.E), kThreads, 0, s>>>(J, P->ldJ, b, cs, P->colors.local_of, P->colors.C);
            return FDB_OK;
          });
        }));
        P->cnt.kernel_launches += 1;
      }
    } else if (!full && P->oop.dest_n > 0) {
      oop_plus_zero_slots<<<P->grid(P->oop.dest_n), kThreads, 0, s>>>(J, P->oop.dest, P->oop.dest_n);
      P->cnt.kernel_launches += 1;
    } else if (full && P->m > 0) {
      // column c < C of the block: 0.0 + q; the prototype's columns [C, ncols) are zeros, rank 0's alone
      auto finish = [&](double *Jc, int64_t qcols, int64_t ncols) {
        const int64_t work = ((P->m + kTile - 1) / kTile) * ncols;
        const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(work, (int64_t)P->sm_count * 16));
        oop_dense_finish<<<grid, kThreads, 0, s>>>(Jc, P->ldJ, P->m, qcols, ncols);
        P->cnt.kernel_launches += 1;
      };
      const int64_t ncl = P->columns.end - P->columns.begin;
      const int64_t tail = P->rank == 0 ? P->oop.ncols - P->oop.qcols : 0;
      if (P->columns.end == P->oop.qcols) {
        finish(J, ncl, ncl + tail);
      } else {
        finish(J, ncl, ncl);
        if (tail > 0) finish(base + P->oop.qcols * P->ldJ, 0, tail);
      }
    }
  }
  CU(cudaGetLastError());
  return FDB_OK;
}

// The root-only finish of a sparse result, once every member has written its candidates: the compaction over all of
// them (the full candidate count and maximum(colorvec)), fused with the quotients when one plan holds every f! output.
static fdb_status oop_root_finish(fdb_plan *P, const fdb_oop_out *out, const double *d_fx, const double *d_f_in,
                                  cudaStream_t s) {
  const bool full = P->sp_kind == SP_NONE, band = P->sp_kind == SP_BANDED, block = P->sp_kind == SP_BLOCKBAND;
  const bool csr = P->sp_kind == SP_CSR;
  const int64_t candidates = oop_candidates(P);
  DeviceGuard g(P->device);
  const int64_t ntiles = (candidates + kTile - 1) / kTile;
  CU(cudaMemsetAsync(P->oop.state, 0, (size_t)(ntiles + 1) * 8, s));
  CompactArgs a{};
  a.vals = P->oop.vals; a.row32 = P->entries.row32; a.colptr32 = P->entries.colptr32;
  a.ecolor = P->entries.ecolor; a.Fp = P->scratch.Fp; a.Fm = P->scratch.Fm; a.eps = P->steps.eps; a.ncolors = P->colors.C;
  a.fx = d_f_in ? d_f_in : (d_fx ? d_fx : P->scratch.fx_own);
  a.ldF = P->fdtype == FDB_COMPLEX ? 2 * P->scratch.ldF : P->scratch.ldF;
  a.E = candidates; a.m = P->m; a.C = P->oop.qcols; a.ncols = P->oop.ncols;
  a.colptr = out->colptr; a.rowval = out->rowval; a.nzval = out->nzval; a.nnz = out->nnz;
  a.state = P->oop.state; a.claim = P->oop.state + ntiles; a.tile_col = P->oop.tile_col;
  if (band) a.band = oop_band_shape(P);
  // a CSR result: the columns are the stored index and the row starts the pointer written (out->colptr gets m + 1)
  if (csr) { a.row32 = P->csr.colval; a.colptr32 = P->csr.rowptr; a.ncols = P->m; }
  auto go = [&](auto kern, auto... cs) {
    kern<<<resident_grid(P, kern, 0, std::max<int64_t>(ntiles, 1)), kThreads, 0, s>>>(a, cs...);
  };
  if (full) go(oop_compact<true, kCopy, uint8_t>);
  else if (csr && P->oop.fused) TRY(dispatch_mode(P->fdtype, [&](auto mode) {
    return dispatch_ct(P->colors.bits, [&](auto tag) {
      return dispatch_colors<decltype(tag)>(P, [&](auto cs) -> fdb_status {
        go(oop_compact_csr<decltype(mode)::value, decltype(cs)>, cs);
        return FDB_OK;
      });
    });
  }));
  // the candidates the CSR scatters wrote in slot order: the CSC copy over (colval, rowptr) is the CSR copy
  else if (csr) go(oop_compact<false, kCopy, uint8_t>);
  else if (block) {
    // the candidates from the block scatters' buffer (kCopy), or the quotients from the resident f! outputs
    const BlockShape b = oop_block_shape(P);
    const bool dense = P->jkind == FDB_J_BLOCK_DENSE;
    if (!P->oop.fused) {
      if (dense) go(oop_compact_block_dense<kCopy, uint8_t>, b);
      else go(oop_compact_block_band<kCopy, uint8_t>, b);
    } else {
      TRY(dispatch_mode(P->fdtype, [&](auto mode) {
        return dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
          constexpr int M = decltype(mode)::value;
          if (dense) go(oop_compact_block_dense<M, decltype(tag)>, b);
          else go(oop_compact_block_band<M, decltype(tag)>, b);
          return FDB_OK;
        });
      }));
    }
  }
  else if (band && !P->oop.fused) go(oop_compact_band<kCopy, TableColors<uint8_t>>, TableColors<uint8_t>{nullptr});
  else if (band) TRY(dispatch_mode(P->fdtype, [&](auto mode) {
    return dispatch_ct(P->colors.bits, [&](auto tag) {
      return dispatch_colors<decltype(tag)>(P, [&](auto cs) -> fdb_status {
        go(oop_compact_band<decltype(mode)::value, decltype(cs)>, cs);
        return FDB_OK;
      });
    });
  }));
  else if (!P->oop.fused) go(oop_compact<false, kCopy, uint8_t>);
  else TRY(dispatch_mode(P->fdtype, [&](auto mode) {
    return dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      go(oop_compact<false, decltype(mode)::value, decltype(tag)>);
      return FDB_OK;
    });
  }));
  P->cnt.kernel_launches += 1;
  CU(cudaGetLastError());
  return FDB_OK;
}

// An out-of-place call once check_call has accepted it
static fdb_status jacobian_oop_run(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, const fdb_oop_out *out, double *d_fx,
                                   const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  const bool sparse = P->oop.kind == FDB_OOP_SPARSE;
  if (sparse && P->world > 1)
    return fail(FDB_ERR_INVALID, "a sparse result is compacted over every rank's candidates on one device: run sparse rank "
                                 "plans through fdb_group_create_oop_* / fdb_group_jacobian_oop");
  if (!sparse && P->j_len > 0 && !out->J) return fail(FDB_ERR_INVALID, "NULL x or J");
  TRY(oop_check_out(P, out));
  cudaStream_t s = (cudaStream_t)stream;
  TRY(oop_member(P, f, ctx, d_x, sparse ? P->oop.vals : out->J, d_fx, d_f_in, relstep, absstep, dir, s));
  if (sparse) TRY(oop_root_finish(P, out, d_fx, d_f_in, s));
  return FDB_OK;
}

extern "C" {

fdb_status fdb_jacobian_oop(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, const fdb_oop_out *out, double *d_fx,
                            const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  if (!P || !f || !out) return fail(FDB_ERR_INVALID, "NULL plan, f or out");
  TRY(check_call(P, Call::jacobian_oop));
  return jacobian_oop_run(P, f, ctx, d_x, out, d_fx, d_f_in, relstep, absstep, dir, stream);
}

fdb_status fdb_jacobian_oop_complex(fdb_plan *P, fdb_fn_c f, void *ctx, const double *d_x, const fdb_oop_out *out,
                                    void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::jacobian_oop_complex));
  if (!out) return fail(FDB_ERR_INVALID, "NULL plan, f or out");
  return jacobian_oop_run(P, reinterpret_cast<fdb_fn>(f), ctx, d_x, out, nullptr, nullptr, FDB_STEP_DEFAULT, FDB_STEP_DEFAULT,
                          1.0, stream);
}

fdb_status fdb_jvp_oop(fdb_plan *P, fdb_fn f, void *ctx, double *d_jvp, const double *d_x, const double *d_v, double *d_x1,
                       double *d_fx1, const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  return jvp_run(P, f, ctx, d_jvp, d_x, d_v, d_x1, d_fx1, d_f_in, relstep, absstep, dir, stream, true);
}

// ------------------------------------------------------------------------------------------------ single-process group
fdb_status fdb_group_create_oop_csc(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                    const int64_t *colptr, const int64_t *rowval, const int64_t *colorvec, int result_kind,
                                    int64_t ldJ, const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_oop_plan_create_csc(p, m, n, colptr, rowval, colorvec, result_kind, ldJ, o);
  });
}

fdb_status fdb_group_create_oop_banded(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n, int64_t l,
                                       int64_t u, const int64_t *colorvec, int result_kind, int64_t ldJ,
                                       const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_oop_plan_create_banded(p, m, n, l, u, colorvec, result_kind, ldJ, o);
  });
}

fdb_status fdb_group_create_oop_block_banded(fdb_group **group, int n_devices, const int *devices, int64_t nblocks,
                                            const int64_t *blocks, int64_t l, int64_t u, int64_t lam, int64_t mu,
                                            const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_oop_plan_create_block_banded(p, nblocks, blocks, l, u, lam, mu, colorvec, result_kind, ldJ, o);
  });
}

fdb_status fdb_group_create_oop_block_dense(fdb_group **group, int n_devices, const int *devices, int64_t nblocks,
                                           const int64_t *blocks, int64_t l, int64_t u, const int64_t *colorvec,
                                           int result_kind, int64_t ldJ, const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_oop_plan_create_block_dense(p, nblocks, blocks, l, u, colorvec, result_kind, ldJ, o);
  });
}

fdb_status fdb_group_create_oop_csr(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                    const int64_t *rowptr, const int64_t *colval, const int64_t *colorvec, int result_kind,
                                    int64_t ldJ, const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_oop_plan_create_csr(p, m, n, rowptr, colval, colorvec, result_kind, ldJ, o);
  });
}

fdb_status fdb_group_create_oop_dense(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                      const int64_t *colorvec, int64_t ncols_out, int result_kind, int64_t ldJ,
                                      const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_oop_plan_create_dense(p, m, n, colorvec, ncols_out, result_kind, ldJ, o);
  });
}

fdb_status fdb_group_jacobian_oop(fdb_group *g, fdb_fn f, void *const *ctx, const double *d_x, const fdb_oop_out *out,
                                  double *d_fx, const double *d_f_in, double relstep, double absstep, double dir,
                                  void *stream) {
  if (!g || !f || !out) return fail(FDB_ERR_INVALID, "NULL group, f or out");
  fdb_plan *P0 = g->plans[0];
  TRY(check_call(P0, Call::group_jacobian_oop));
  if (P0->n > 0 && !d_x) return fail(FDB_ERR_INVALID, "NULL x");
  const bool sparse = P0->oop.kind == FDB_OOP_SPARSE;
  if (!sparse && P0->j_len > 0 && !out->J) return fail(FDB_ERR_INVALID, "NULL x or J");
  TRY(oop_check_out(P0, out));
  const int root = g->devices[0];
  cudaStream_t s0 = (cudaStream_t)stream;
  {
    DeviceGuard dg(root);
    if (!dg.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", root);
    // a dense result of a CSC or band sparsity: zero-filled once, by the owner of the buffer, before any member stores
    // into it
    if (g->n > 1 && P0->oop.kind == FDB_OOP_DENSE && (P0->sp_kind == SP_CSC || P0->sp_kind == SP_BANDED) && P0->j_len > 0)
      TRY(zero_J(P0, out->J, s0));
  }
  double *base = sparse ? P0->oop.vals : out->J;
  TRY(group_run(g, d_x, s0, [&](int i, const double *xi, cudaStream_t s) {
    fdb_plan *P = g->plans[i];
    const double *fin_i = d_f_in;
    if (i > 0 && d_f_in && P->fdtype == FDB_FORWARD) TRY(member_replica(g, i, g->fin_rep, d_f_in, g->m, s, &fin_i));
    return oop_member(P, f, ctx ? ctx[i] : nullptr, xi, base, i == 0 ? d_fx : nullptr, fin_i, relstep, absstep, dir, s);
  }, [&](int i) { return oop_idle(g->plans[i]); }));
  if (sparse) {
    DeviceGuard dg(root);
    TRY(oop_root_finish(P0, out, d_fx, d_f_in, s0));
  }
  return FDB_OK;
}

}  // extern "C"
