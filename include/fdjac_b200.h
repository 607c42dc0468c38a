/*
 * fdjac_b200.h — C ABI of libfdjac_b200.so: the H100 (sm_90a) drop-in for ONE path of
 * FiniteDiff.jl — the cached, in-place, graph-coloured Jacobian
 *     finite_difference_jacobian!(J, f!, x, cache::JacobianCache; colorvec, sparsity)
 *     (reference: src/jacobians.jl:504-653 and the hooks it dispatches to).
 *
 * Boundary rules
 *   - plain C, extern "C"; pointers + sizes only; no C++/torch types; never throws.
 *   - every entry point returns an fdb_status; fdb_last_error() gives the thread-local message.
 *   - index arrays cross the ABI exactly as Julia stores them: Int64, 1-BASED
 *     (SparseMatrixCSC{Float64,Int64}.colptr / .rowval, Vector{Int} colorvec), and may live in
 *     HOST or DEVICE memory (detected with cudaPointerGetAttributes) — pointer(J.colptr) can be
 *     passed with no conversion.  The plan keeps private, compressed device copies.
 *   - x, fx, J value buffers are DEVICE pointers (fdb_jacobian) or HOST pointers
 *     (fdb_jacobian_host, which stages H2D/D2H itself).  Caller owns every buffer it passes.
 *   - one in-flight call per plan; calls are stream-ordered and asynchronous (no host sync
 *     inside fdb_jacobian).  Different plans may be used concurrently from different threads.
 *
 * Each entry point cites the reference interface it replaces; the Julia-side binding is in
 * finitediff.jl_b200/julia/FiniteDiffB200.jl and INTEGRATION.md.
 */
#ifndef FDJAC_B200_H
#define FDJAC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FDB_ABI_VERSION 2

/* "keyword not given" for relstep / absstep (jacobians.jl:508-510 defaults: relstep = default_relstep(fdtype, T),
 * absstep = relstep).  Any other value, 0 included, is used as passed: relstep = 0 is a pure absolute step,
 * absstep = 0 a pure relative one, as in the reference. */
#define FDB_STEP_DEFAULT (__builtin_nan(""))

typedef enum {
  FDB_OK = 0,
  FDB_ERR_INVALID = 1,     /* bad argument / inconsistent pattern (the reference would throw / @assert) */
  FDB_ERR_CUDA = 2,        /* a CUDA runtime call failed (message has the cudaError string) */
  FDB_ERR_CALLBACK = 3,    /* user f! returned non-zero: the colour loop was aborted (Julia: exception in f) */
  FDB_ERR_NOMEM = 4,
  FDB_ERR_UNSUPPORTED = 5, /* e.g. fdtype other than forward/central (epsilons.jl:159-167 fdtype_error) */
  FDB_ERR_NO_DEVICE = 6    /* no CUDA device: this library has NO CPU fallback */
} fdb_status;

/* fdtype — the Val(:forward)/Val(:central)/Val(:complex) type parameter of JacobianCache (jacobians.jl:1-9).
 * FDB_COMPLEX is the complex-step colour loop (jacobians.jl:623-648): x + im*eps, J = imag(f)/eps, eps = eps(Float64);
 * plans of that type are driven through fdb_jacobian_complex with a complex128 callback.
 * FDB_HCENTRAL is the Val(:hcentral) of HessianCache (hessians.jl:1-9): Hessian plans only (fdb_hessian_plan_create). */
enum { FDB_FORWARD = 0, FDB_CENTRAL = 1, FDB_COMPLEX = 2, FDB_HCENTRAL = 3 };

/* Where `J[row, col] = v` lands — what the reference decides by dispatch on typeof(J). */
typedef enum {
  FDB_J_CSC_NZVAL = 0, /* J::SparseMatrixCSC with the sparsity's pattern: nzval[p]   (ext/FiniteDiffSparseArraysExt.jl:38-47) */
  FDB_J_DENSE = 1,     /* J::Matrix column-major, leading dimension ldJ              (ext/..SparseArraysExt.jl:20-28, iteration_utils.jl:25-32) */
  FDB_J_BAND = 2,      /* J::BandedMatrix data[(l+u+1) x n], slot [u+r-c+1, c]        (ext/FiniteDiffBandedMatricesExt.jl:13-27) */
  FDB_J_SLOTS = 3,     /* structured J (e.g. Tridiagonal): explicit 1-based slot per structural entry (iteration_utils.jl:25-32) */
  FDB_J_BLOCK_BAND = 4, /* J::BandedBlockBandedMatrix band data, (l+u+1)(lam+mu+1) slots per column (fdb_plan_create_block_banded) */
  FDB_J_DIAGONALS = 5, /* J::Diagonal / Bidiagonal / Tridiagonal storage: the stored diagonals packed in one buffer (fdb_plan_create_banded) */
  FDB_J_BLOCK_DENSE = 6, /* J::BlockBandedMatrix data, one column-major slab per block column (fdb_plan_create_block_dense):
                           entry (r, c) of block (K, J), 0-based, at slot start_J + c*h_J + (rowoff_J(K) + r), where
                           h_J = sum of the sizes of block rows max(0, J-u)..min(N-1, J+l), start_J = sum_{J'<J} h_J'*cb[J']
                           and rowoff_J(K) = the sizes of block rows max(0, J-u)..K-1 */
  FDB_J_CSR = 7         /* J is the nzval of a CSR matrix with the sparsity's own pattern: entry s of row r, column colval[s],
                           at nzval[s] (fdb_plan_create_csr) */
} fdb_jkind;

/*
 * User function f!(fx, x) — replaces the Julia closure called at jacobians.jl:563,605-606.
 * Evaluate `batch` points: for b in [0,batch):  d_fx[b*ldfx .. +m) = f(d_x[b*ldx .. +n)).
 * Must only ENQUEUE work on `stream` (a cudaStream_t) and must not synchronise.  Return 0 on
 * success; any other value aborts the Jacobian and is reported as FDB_ERR_CALLBACK.
 * From Julia: @cfunction(f_trampoline, Cint, (Ptr{Cvoid}, CuPtr{Float64}, CuPtr{Float64}, Int64, Int64, Int64, Ptr{Cvoid})).
 * The plan is created with max_batch = 1 for callbacks that can only do one point per call.
 */
typedef int (*fdb_fn)(void *ctx, double *d_fx, const double *d_x, int64_t batch, int64_t ldfx, int64_t ldx,
                      void *stream);

/* Complex-step variant of the callback (fdtype = FDB_COMPLEX): d_fx / d_x are complex128 arrays (re, im interleaved:
 * cuDoubleComplex / ComplexF64); ldfx / ldx count COMPLEX elements.  Same rules as fdb_fn. */
typedef int (*fdb_fn_c)(void *ctx, void *d_fx, const void *d_x, int64_t batch, int64_t ldfx, int64_t ldx, void *stream);

/* Plan options (all fields have a usable zero default). */
typedef struct {
  int32_t fdtype;          /* FDB_FORWARD (default, as jacobians.jl:13) or FDB_CENTRAL */
  int32_t device;          /* CUDA device ordinal; -1 or 0-initialised+use_current => current device */
  int32_t use_current_device; /* 1: ignore `device`, use cudaGetDevice() */
  int32_t no_drift;        /* 0 (default): replay the reference's (x1+eps)-eps drift of earlier colours bit-exactly
                              (jacobians.jl:562,584); 1: perturb from the pristine x */
  int64_t max_batch;       /* points per f! callback invocation; 0/1 => one point per call */
  int64_t scratch_bytes;   /* budget for the stacked f! outputs; 0 => 8 GiB */
  int32_t rank, world;     /* colour partition over GPUs (one process per GPU): this plan handles the colours
                              owned by `rank` of `world`; world<=1 => all colours */
  int32_t partition;       /* 0: round-robin colours; 1: nnz-balanced (LPT) */
  int32_t strategy;        /* CSC scatter: 0 auto; 1 one fused pass over J's storage order; 2 colour-major entry lists, a
                              launch per group of L2-resident f! outputs, overlapped with the next group's f!; 3 colour-major
                              lists with every f! output resident: one launch at the end (see fdb_plan_info_t.strategy) */
  int32_t use_graph;       /* 1: capture the whole call (library kernels + the callback's launches) into a CUDA graph on
                              first use and replay it while (f, ctx, buffers, scalars) stay the same (the scalars bit for
                              bit: a step of -0.0 is not the step +0.0).  The callback must be capture-safe:
                              enqueue-only on the given stream, no allocation, no host-side state. */
  int32_t shared_j;        /* 1: the J passed to fdb_jacobian is SHARED with other ranks' plans (a peer-mapped pointer to one
                              buffer, e.g. rank 0's): this plan only stores the entries / columns it owns and never zero-fills
                              J — the owner of the buffer zero-fills it (when the scatter is not self-defining) and orders
                              the ranks (fdb_sync_barrier / fdb_group_jacobian do both) */
} fdb_plan_opts;

typedef struct fdb_plan fdb_plan;

typedef struct {
  int64_t m, n;
  int64_t n_entries;       /* structural entries the scatter writes per Jacobian (nnz; in-band slots for banded) */
  int64_t j_len;           /* doubles in J's value storage */
  int64_t n_colors;        /* maximum(colorvec) */
  int64_t n_local_colors;  /* colours this rank evaluates */
  int64_t n_groups;        /* scatter launches per Jacobian (1 => fully fused single pass) */
  int64_t slabs;           /* colours whose f! outputs are resident at once */
  int64_t fcalls_per_jacobian; /* f! evaluations (points) per call: 1+C fwd, 2C central (local colours only) */
  int64_t device_bytes;    /* device memory held by the plan (build scratch is freed when the plan is created) */
  int32_t fdtype, jkind, sp_kind, color_bits;
  int64_t alg_bytes_scatter; /* SURVEY.md §8(d) algorithmic bytes of the diff+scatter per Jacobian */
  int32_t strategy;        /* chosen scatter strategy: 0 fused single pass, 1 per-colour column lists */
  int32_t lanes;           /* lanes per column of the column-list kernel */
  double mean_row_jump;    /* mean |row[e+1]-row[e]| over consecutive entries (gather locality metric) */
  int64_t moved_bytes_scatter; /* COMPULSORY bytes of the shipped diff+scatter formulation per Jacobian (this rank): every
                              index / slab / fx / J byte it must move once — the roofline numerator.  CSC fused pass:
                              E*(4 + |colour| + 8*slabs_read + 8) [+ 8m fx, forward]; colour-major lists: E*(4 + |slot| +
                              8*slabs_read + 8) [+ 8m]; explicit destinations: + 8 per entry; banded / dense: = alg_bytes;
                              TMA-staged fused pass: E*(2 + |colour| + 8) + 8m*(slabs_read*C [+ 1]) */
  int32_t staged;          /* 1: the fused pass runs in its TMA-staged form (row-local pattern: slab windows staged through
                              shared memory by cp.async.bulk, 16-bit row offsets) */
  int32_t lists_resident;  /* 1: colour-major lists with every local colour's f! output resident (one launch) */
} fdb_plan_info_t;

typedef struct {
  int64_t jacobians;       /* completed fdb_jacobian calls */
  int64_t f_points;        /* f! points evaluated */
  int64_t f_invocations;   /* callback invocations */
  int64_t kernel_launches; /* library kernels launched (excludes the user's f!) */
  int64_t scatter_launches;
} fdb_counters_t;

/* ---- library ---- */
int fdb_abi_version(void);
/* thread-local message of the last failing call on this thread */
const char *fdb_last_error(void);
/* number of usable CUDA devices (0 => every compute entry point returns FDB_ERR_NO_DEVICE) */
int fdb_device_count(void);

/* ---- step size: src/epsilons.jl:134-144 / :26-29,50-53 (host-side scalars, for callers and tests) ---- */
double fdb_default_relstep(int fdtype);
double fdb_compute_epsilon(int fdtype, double x, double relstep, double absstep, double dir);

/* ---- plans: the per-(pattern, colorvec, fdtype) state the reference rebuilds on every call
 *      (jacobians.jl:515-535: colour reshape, findstructralnz, same-pattern test) ---- */

/* Which plans each call takes.  Coloured plans: fdb_plan_create_csc / _coo / _banded / _block_banded / _block_dense / _csr; dense plans:
 * fdb_plan_create_dense / _dense_colorvec; out-of-place plans: fdb_oop_plan_create_*.  Any other plan is refused with
 * FDB_ERR_INVALID (FDB_ERR_UNSUPPORTED where noted) before the call allocates, launches or calls f.
 *   fdb_jacobian, fdb_jacobian_host   coloured and dense plans, fdtype forward / central
 *   fdb_jacobian_complex              coloured and dense plans, fdtype complex
 *   fdb_jacobian_oop                  out-of-place plans, fdtype forward / central
 *   fdb_jacobian_oop_complex          out-of-place plans, fdtype complex
 *   fdb_color_eps                     coloured plans (out-of-place CSC, band, block and CSR included) and step-size plans
 *   fdb_plan_set_external_eps         coloured plans (out-of-place CSC, band, block and CSR included)
 *   fdb_plan_set_peers                CSC, COO, JVP and step-size plans (else FDB_ERR_UNSUPPORTED)
 *   fdb_plan_color_owner              every plan but dense, Hessian and derivative plans
 *   fdb_plan_get_eps                  every plan but derivative plans
 *   fdb_jvp, fdb_jvp_oop              JVP plans
 *   fdb_hessian                       Hessian plans
 *   fdb_derivative                    derivative and scalar-gradient plans, fdtype forward / central
 *   fdb_derivative_complex            derivative and scalar-gradient plans, fdtype complex
 *   fdb_group_jacobian                groups of coloured or dense plans, fdtype forward / central (complex:
 *                                     FDB_ERR_UNSUPPORTED)
 *   fdb_group_jacobian_oop            groups of out-of-place plans, fdtype forward / central (complex: FDB_ERR_UNSUPPORTED)
 *   fdb_group_hessian                 groups of Hessian plans */

/* sparsity::SparseMatrixCSC (m x n, colptr[n+1], rowval[nnz]).
 *   jkind = FDB_J_CSC_NZVAL: J is a CSC with pattern (j_colptr, j_rowval); NULL,NULL => same arrays as the sparsity.
 *           Same pattern (ext/..SparseArraysExt.jl:51-52) => fast path nzval[p]; a different pattern is accepted when every
 *           sparsity entry exists in J (the generic J[r,c]= path of :20-28), else FDB_ERR_UNSUPPORTED (would need insertion).
 *   jkind = FDB_J_DENSE: J is a dense column-major matrix with leading dimension ldJ (coloring_tests.jl:51-64).
 * colorvec: n colours, 1-based; NULL => 1:n (jacobians.jl:16). */
fdb_status fdb_plan_create_csc(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval,
                               int jkind, const int64_t *j_colptr, const int64_t *j_rowval, int64_t ldJ,
                               const int64_t *colorvec, const fdb_plan_opts *opts);

/* sparsity given as structural-nonzero lists rows_index/cols_index (ArrayInterface.findstructralnz of a structured
 * matrix, or _findstructralnz of a dense 0/1 prototype, jacobians.jl:473-488,522-528) — generic hook iteration_utils.jl:25-32.
 *   jkind = FDB_J_DENSE (ldJ) or FDB_J_SLOTS (slots[nnz] 1-based into a J value buffer of j_len doubles). */
fdb_status fdb_plan_create_coo(fdb_plan **plan, int64_t m, int64_t n, int64_t nnz, const int64_t *rows_index,
                               const int64_t *cols_index, int jkind, const int64_t *slots, int64_t ldJ_or_jlen,
                               const int64_t *colorvec, const fdb_plan_opts *opts);

/* sparsity::BandedMatrix with bandwidths (l,u): ext/FiniteDiffBandedMatricesExt.jl:13-27 (writes the WHOLE band).
 *   jkind = FDB_J_BAND (J is the (l+u+1) x n band data) or FDB_J_DENSE (ldJ).
 *   jkind = FDB_J_DIAGONALS: LinearAlgebra's Diagonal (l, u) = (0, 0), Bidiagonal :U (0, 1) / :L (1, 0) and Tridiagonal
 *           (1, 1) storage, whose entry set is the in-matrix band (l, u).  Needs m == n and l, u in {0, 1}.  J is one
 *           packed buffer holding the stored diagonals in ascending row-minus-column order: the sub-diagonal (r = c+1,
 *           n-1 values, when l = 1), the main diagonal (n values), the super-diagonal (c = r+1, n-1 values, when u = 1);
 *           entry t of each diagonal is its t-th element from the top left.  So the buffer is [dl; d; du] for
 *           Tridiagonal, [dv; ev] for Bidiagonal :U, [ev; dv] for :L and [d] for Diagonal.  ldJ is the buffer's length in
 *           doubles, at least (l+u+1)*n - l - u (0 for n = 0); slots beyond that are not touched.  Every call writes every
 *           slot exactly once — the quotient for columns with a valid colour, +0.0 for the others — so J is never
 *           zero-filled; a rank plan writes the slots of its own colours' columns (rank 0 also those without a valid
 *           colour), and a rank without colours, or a plan with no colour at all, zero-fills J like FDB_J_BAND.  The column
 *           colours come from the table, or from the closed form when colorvec[j] == j mod C + 1 (matrix_colors).
 *           Any other (m, n, l, u, ldJ): FDB_ERR_INVALID.  fdb_plan_info: jkind FDB_J_DIAGONALS, j_len = that length,
 *           n_entries = the structural entries of columns with a valid colour (j_len when every column has one),
 *           alg_bytes_scatter = 8*j_len + 16*n*C. */
fdb_status fdb_plan_create_banded(fdb_plan **plan, int64_t m, int64_t n, int64_t l, int64_t u, int jkind, int64_t ldJ,
                                  const int64_t *colorvec, const fdb_plan_opts *opts);

/* sparsity::BandedBlockBandedMatrix with square blocks, J the same structure: ext/FiniteDiffBlockBandedMatricesExt.jl:16-42.
 *   blocks: nblocks block sizes (Int64, host or device; the column sizes are the row sizes, as the hook takes them from
 *   axes(Jac, 1)); n = m = sum(blocks).  (l, u) block bandwidths, (lam, mu) sub-block bandwidths, all >= 0.
 *   J is the band data: w = (l+u+1)(lam+mu+1) slots per column, column-major; entry (k, j) of block (K, J) sits at slot
 *   (K-J+u)(lam+mu+1) + (mu+k-j) of its global column (0-based k, j inside the blocks).  ldata >= w*n doubles.
 * The structure is a closed form: plan-time host work is O(nblocks), the plan keeps the block offsets on the device and
 * reads no index stream.  Every call writes every one of the w*n slots exactly once — the quotient on the structural
 * slots of columns with a valid colour, +0.0 everywhere else — with the values of the fill_matrix!-then-scatter of the
 * slot-addressed route (fdb_plan_create_coo with FDB_J_SLOTS on the hook's entry set); slots [w*n, ldata) are not touched.
 * The colouring of ArrayInterface.matrix_colors, (J mod (l+u+1))(lam+mu+1) + (j mod (lam+mu+1)) + 1, is detected and
 * then read in closed form.  opts as for the other coloured plans (forward / central / complex, max_batch, scratch_bytes,
 * no_drift, use_graph, rank / world / partition, fdb_plan_set_external_eps); fdb_plan_set_peers is FDB_ERR_UNSUPPORTED.
 * A rank plan writes the columns of its own colours (rank 0 also those without a valid colour), so the ranks together
 * write every slot once and nobody zero-fills J.  Negative sizes or bandwidths, ldata < w*n, a NULL blocks with
 * nblocks > 0: FDB_ERR_INVALID.  fdb_plan_info: jkind FDB_J_BLOCK_BAND, n_entries = structural entries, j_len = w*n. */
fdb_status fdb_plan_create_block_banded(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                        int64_t lam, int64_t mu, int64_t ldata, const int64_t *colorvec,
                                        const fdb_plan_opts *opts);

/* sparsity::BlockBandedMatrix with square blocks, J the same structure: ext/FiniteDiffBlockBandedMatricesExt.jl:44-68
 * (every row of every block in blockcolrange(J), for every column of the colour).
 *   blocks: nblocks block sizes (Int64, host or device; the column sizes are the row sizes, as the hook takes both from
 *   axes(Jac, 1)); n = m = sum(blocks).  (l, u) block bandwidths, >= 0 (bandwidths of nblocks or more mean nblocks).
 *   J is BlockBandedMatrices' storage of a BlockBandedMatrix (a BlockSkylineMatrix with constant block bandwidths):
 *   FDB_J_BLOCK_DENSE above, j_len = sum_J h_J*cb[J] slots, every one a structural entry.  ldata >= j_len doubles.
 * Plan-time host work is O(nblocks); the plan keeps the block offsets and the slab starts on the device and reads no
 * index stream.  Every call writes every one of the j_len slots exactly once — the quotient in columns with a valid
 * colour, +0.0 in the others — with the values of the slot-addressed route (fdb_plan_create_coo with FDB_J_SLOTS on the
 * hook's entry set); slots [j_len, ldata) are not touched.  For uniform blocks of size b the colouring of
 * ArrayInterface.matrix_colors, (J mod (l+u+1))*b + j + 1 for column j of block J, is detected and then read in closed
 * form.  opts, rank plans and fdb_plan_set_peers (FDB_ERR_UNSUPPORTED) as for fdb_plan_create_block_banded.  Negative
 * sizes or bandwidths, ldata < j_len, a NULL blocks with nblocks > 0: FDB_ERR_INVALID; a block column of more than 2^32
 * slots: FDB_ERR_UNSUPPORTED.  fdb_plan_info: jkind FDB_J_BLOCK_DENSE, n_entries = j_len, alg_bytes_scatter =
 * moved_bytes_scatter = 8*j_len + 16*n*C. */
fdb_status fdb_plan_create_block_dense(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                       int64_t ldata, const int64_t *colorvec, const fdb_plan_opts *opts);

/* sparsity and J: one CSR matrix (m x n, rowptr[m+1], colval[nnz]; Int64, 1-based, host or device), J its nzval — the generic
 * J[r, c] = v hook (ext/FiniteDiffSparseArraysExt.jl:20-28, iteration_utils.jl:25-32) on a row-compressed target, the format
 * GPU sparse solvers take.  Columns within a row may come in any order; a repeated (r, c) is allowed and each of its slots
 * gets the value.  Every call writes every one of the nnz slots exactly once — the quotient of the column's colour, +0.0
 * when the column has no valid colour — so J is never zero-filled; slots past nnz are not touched.  Values, f! calls and
 * f! points are those of the slot route (fdb_plan_create_coo with FDB_J_SLOTS, the CSR's rows and columns and slots 1..nnz)
 * on the same buffer, for any colouring.  opts as for the other coloured plans (forward / central / complex, max_batch,
 * scratch_bytes, no_drift, use_graph, rank / world / partition, shared_j, fdb_color_eps, fdb_plan_set_external_eps);
 * fdb_plan_set_peers is FDB_ERR_UNSUPPORTED.  A rank plan writes the slots of its own colours (rank 0 also those of the
 * columns without a valid colour), so the ranks together write every slot once and nobody zero-fills J.  A NULL rowptr,
 * rowptr[1] != 1, a decreasing rowptr, a column outside 1..n or negative sizes: FDB_ERR_INVALID; nnz >= 2^31:
 * FDB_ERR_UNSUPPORTED; both before any f! call.  fdb_plan_info: jkind FDB_J_CSR, n_entries = j_len = nnz,
 * alg_bytes_scatter = 32*nnz + 16*n + 8 (as for CSC), moved_bytes_scatter = G*(4*nnz + 4*(m+1) + |colour|*n) + E_own*(8*slabs_read
 * + 8) [+ 8m, forward] with G scatter launches (n_groups), |colour| = 0 for a cyclic colouring and E_own the entries of the
 * rank's colours (nnz on one rank). */
fdb_status fdb_plan_create_csr(fdb_plan **plan, int64_t m, int64_t n, const int64_t *rowptr, const int64_t *colval,
                               const int64_t *colorvec, const fdb_plan_opts *opts);

/* sparsity === nothing: dense column branch jacobians.jl:548-557,590-598 (colorvec = 1:n; per-component step).
 * With world>1 the columns are block-partitioned: this rank computes columns [col_begin, col_end) (0-based, see
 * fdb_plan_info) and d_J passed to fdb_jacobian points at THAT column slab (ldJ x ncols_local). */
fdb_status fdb_plan_create_dense(fdb_plan **plan, int64_t m, int64_t n, int64_t ldJ, const fdb_plan_opts *opts);
/* sparsity === nothing WITH a caller-supplied colorvec, as jacobians.jl:547-557 is written: the loop runs color_i in
 * 1:maximum(colorvec), perturbs COMPONENT color_i and writes J[:, color_i] (J is not zero-filled; later columns keep
 * their contents).  maximum(colorvec) > n (BoundsError in the reference) => FDB_ERR_INVALID.  colorvec NULL => 1:n. */
fdb_status fdb_plan_create_dense_colorvec(fdb_plan **plan, int64_t m, int64_t n, int64_t ldJ, const int64_t *colorvec,
                                          const fdb_plan_opts *opts);

fdb_status fdb_plan_destroy(fdb_plan *plan);
fdb_status fdb_plan_info(const fdb_plan *plan, fdb_plan_info_t *info);
fdb_status fdb_plan_counters(const fdb_plan *plan, fdb_counters_t *out);
/* dense plans: the [begin,end) 0-based column range this rank owns; Hessian plans: the rank's i-blocks [i_r, i_{r+1}) */
fdb_status fdb_plan_dense_range(const fdb_plan *plan, int64_t *col_begin, int64_t *col_end);
/* colour ownership (0-based colour index -> owning rank), n_colors entries */
fdb_status fdb_plan_color_owner(const fdb_plan *plan, int32_t *owner_out, int64_t cap);
/* Copy the step sizes used by the most recent call to the host (synchronises `stream`): eps per colour
 * (coloured plans, n_colors entries) or per local column (dense plans).  For tests / diagnostics. */
fdb_status fdb_plan_get_eps(fdb_plan *plan, double *h_eps, int64_t cap, void *stream);
/* Multi-GPU fused gather: besides d_J, the scatter also stores every value it owns into these peer J buffers
 * (device pointers valid on this device: cudaIpcOpenMemHandle / peer-enabled allocations).  n_peers = 0 clears. */
fdb_status fdb_plan_set_peers(fdb_plan *plan, int n_peers, double *const *peer_J);

/* Device-side timing of the diff+scatter launches (CUDA events recorded on the call's stream around every scatter
 * launch).  Off by default.  fdb_plan_read_timing synchronises the recorded events, returns the summed scatter time in
 * milliseconds and the number of launches since the last read, and resets the accumulators. */
fdb_status fdb_plan_enable_timing(fdb_plan *plan, int enable);
fdb_status fdb_plan_read_timing(fdb_plan *plan, double *scatter_ms, int64_t *scatter_launches);

/*
 * The hot path — replaces finite_difference_jacobian!(J, f, x, cache, f_in; relstep, absstep, colorvec, sparsity, dir)
 * (jacobians.jl:504-514) for the plan's (sparsity, colorvec, fdtype).
 *   d_x    : n doubles (device). NEVER modified (the reference perturbs it in place in central mode and restores it,
 *            jacobians.jl:604,620; here the minus points are built in plan-owned scratch).
 *   d_J    : J's value storage (device): nzval / dense / band data / slots buffer.  Fully defined on return
 *            (fill_matrix!(J,0) + scatter semantics of jacobians.jl:530-532,566-572).
 *   d_fx   : m doubles (device) — cache.fx.  Forward mode: receives f(x) unless d_f_in is given.  May be NULL
 *            (plan-owned buffer is used).  Central mode: unused.
 *   d_f_in : forward mode only: precomputed f(x) (`f_in`, jacobians.jl:540-545) or NULL.
 *   relstep, absstep: FDB_STEP_DEFAULT (NaN) => defaults (default_relstep(fdtype); absstep = relstep); other values as passed.
 *   dir    : forward only (epsilons.jl:28); pass 1.0 for the default `dir=true`.
 *   stream : cudaStream_t (NULL = legacy default stream).
 * f!-call count and order match the reference: forward f(x) first (unless f_in) then colours ascending;
 * central f(x+eps e_k) then f(x-eps e_k) per colour; a colour with no columns still triggers its call(s).
 */
fdb_status fdb_jacobian(fdb_plan *plan, fdb_fn f, void *ctx, const double *d_x, double *d_J, double *d_fx,
                        const double *d_f_in, double relstep, double absstep, double dir, void *stream);

/* Complex-step Jacobian (jacobians.jl:623-648) for plans created with fdtype = FDB_COMPLEX: per colour ONE evaluation
 * f(fx, x + im*eps*(color==k)) on complex128 device arrays, J = imag(fx)/eps with eps = eps(Float64); no f(x) baseline,
 * no cancellation (the reference's tests bound the error by 1e-14, finitedifftests.jl:462).  x and J stay real. */
fdb_status fdb_jacobian_complex(fdb_plan *plan, fdb_fn_c f, void *ctx, const double *d_x, double *d_J, void *stream);

/* Same call with HOST buffers (the reference-facing form: Array x, host J storage): copies x to the device, runs
 * fdb_jacobian on an internal stream, copies J's value storage (and fx when h_fx != NULL) back, then synchronises.
 * Pageable memory works; pinned memory (fdb_host_alloc) is what reaches PCIe speed. */
fdb_status fdb_jacobian_host(fdb_plan *plan, fdb_fn f, void *ctx, const double *h_x, double *h_J, double *h_fx,
                             const double *h_f_in, double relstep, double absstep, double dir);

/* ---- Column-block sharding (SURVEY §8f row 4: problems with fewer colours than GPUs) -------------------------------
 * A shard is a plan over a contiguous block of columns of the sparsity (its colptr slice rebased to 1, row indices
 * rebased to the first row the block touches), evaluated on the slice of x that those rows depend on, with a
 * slice-aware f! (the callback's ctx carries the row / x offsets).  The reference takes every colour's step size from
 * the norm over ALL colour-k components of x (jacobians.jl:559-561), so a shard must not derive it from its slice:
 *   fdb_eps_plan_create   plan that only knows (n, colorvec) of the FULL problem,
 *   fdb_color_eps         eps[k] of every colour for a full-length device x (the K2 pass alone), left in the plan
 *                         (fdb_plan_get_eps) and optionally copied to d_eps_out (device, n_colors doubles); also valid
 *                         on any coloured Jacobian plan,
 *   fdb_plan_set_external_eps   makes a Jacobian plan copy its step sizes from d_eps (device, at least the plan's
 *                         n_colors entries, read on the call's stream) instead of running its own K2 pass; NULL
 *                         restores the built-in pass.  With the same eps the shard's values are bit-identical to the
 *                         corresponding segment of the unsharded Jacobian. */
fdb_status fdb_eps_plan_create(fdb_plan **plan, int64_t n, const int64_t *colorvec, const fdb_plan_opts *opts);
fdb_status fdb_color_eps(fdb_plan *plan, const double *d_x, double relstep, double absstep, double dir,
                         double *d_eps_out, void *stream);
fdb_status fdb_plan_set_external_eps(fdb_plan *plan, const double *d_eps);

/* ---- Multi-GPU behind the C ABI (SURVEY §8e) — no NCCL on the data path ---------------------------------------------
 * Colours (dense plans: column blocks) are independent given x: every GPU evaluates its share and its diff+scatter
 * kernel stores the entries it owns straight into ONE Jacobian buffer (the root's) through peer-mapped memory over
 * NVLink — the final gather is the kernel's own store.
 *
 * (1) ONE process, n devices — what a Julia host needs to reach several GPUs from a single
 *     finite_difference_jacobian!(J, f, x, cache) call (jacobians.jl:504-514): fdb_group_create_* builds one plan per
 *     device (rank i of n; devices[0] is the root and owns x, J, fx), enables peer access to the root, and
 *     fdb_group_jacobian pushes x to the members, runs every member's colour loop on its own stream and joins them on
 *     the caller's stream with CUDA events (asynchronous; no host synchronisation).  ctx[i] is the callback context of
 *     member i (f! is invoked with device-i pointers and stream).  Device ordinals may repeat (two members on one GPU).
 *     Dense groups: member i fills its column block of the root's J.  Forward / central plans. */
typedef struct fdb_group fdb_group;
fdb_status fdb_group_create_csc(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                const int64_t *colptr, const int64_t *rowval, int jkind, const int64_t *j_colptr,
                                const int64_t *j_rowval, int64_t ldJ, const int64_t *colorvec, const fdb_plan_opts *opts);
/* banded groups: with FDB_J_BAND or FDB_J_DIAGONALS member i writes every slot of the columns of its own colours straight
 * into the root's buffer, member 0 also the columns without a valid colour; J is zero-filled only when there is no colour. */
fdb_status fdb_group_create_banded(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n, int64_t l,
                                   int64_t u, int jkind, int64_t ldJ, const int64_t *colorvec, const fdb_plan_opts *opts);
/* dense groups: member i owns the contiguous columns [min(n, i*p), min(n, (i+1)*p)), p = ceil(n / n_devices)
 * (fdb_plan_dense_range of its plan); a member left with no column calls f only for f(x) in forward mode without d_f_in,
 * and writes nothing.  With m = 1 and ldJ = 1 this is the gradient of a scalar f (finite_difference_gradient!, df as J):
 * pass f(x), evaluated once at the root, as d_f_in in forward mode, and a call makes 1 + n evaluations as on one device. */
fdb_status fdb_group_create_dense(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n, int64_t ldJ,
                                  const fdb_plan_opts *opts);
/* block-banded groups: member i writes every slot of the columns of its own colours straight into the root's band data,
 * member 0 also the columns without a valid colour; the column sets are disjoint, so J is never zero-filled. */
fdb_status fdb_group_create_block_banded(fdb_group **group, int n_devices, const int *devices, int64_t nblocks,
                                         const int64_t *blocks, int64_t l, int64_t u, int64_t lam, int64_t mu, int64_t ldata,
                                         const int64_t *colorvec, const fdb_plan_opts *opts);
/* block-dense groups: as block-banded groups, into the root's BlockBandedMatrix storage */
fdb_status fdb_group_create_block_dense(fdb_group **group, int n_devices, const int *devices, int64_t nblocks,
                                        const int64_t *blocks, int64_t l, int64_t u, int64_t ldata, const int64_t *colorvec,
                                        const fdb_plan_opts *opts);
/* CSR groups: member i writes the slots of its own colours straight into the root's nzval, member 0 also those of the
 * columns without a valid colour; J is never zero-filled. */
fdb_status fdb_group_create_csr(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                const int64_t *rowptr, const int64_t *colval, const int64_t *colorvec, const fdb_plan_opts *opts);
fdb_status fdb_group_destroy(fdb_group *group);
fdb_status fdb_group_size(const fdb_group *group, int *n_members);
/* member i's plan (owned by the group): fdb_plan_info / fdb_plan_counters / fdb_plan_get_eps / fdb_plan_color_owner */
fdb_status fdb_group_plan(const fdb_group *group, int member, fdb_plan **plan);
/* arguments as fdb_jacobian; d_x, d_J, d_fx, d_f_in live on devices[0], `stream` is a stream of devices[0].  As for
 * fdb_jacobian, d_J may be NULL when no member has a slot of J to write (n = 0). */
fdb_status fdb_group_jacobian(fdb_group *group, fdb_fn f, void *const *ctx, const double *d_x, double *d_J, double *d_fx,
                              const double *d_f_in, double relstep, double absstep, double dir, void *stream);

/* (2) one process per GPU (torchrun / MPI style): create the plan with opts.rank / opts.world and opts.shared_j = 1, map
 *     the root's J with fdb_ipc_open and pass THAT pointer as d_J (or keep a private J and name the root's buffer with
 *     fdb_plan_set_peers).  fdb_sync is the device-side barrier that orders the ranks: a flag block per rank in peer
 *     memory, fdb_sync_barrier enqueues one tiny kernel that signals every peer (st.release.sys) and waits for every
 *     peer's signal (ld.acquire.sys) — stream-ordered, no host involvement, replayable inside a CUDA graph.
 *     Typical call:  barrier (root finished reading J, and zero-filled it if needed)  ->  fdb_jacobian  ->  barrier.
 *       fdb_sync_flags      this rank's flag block (a dedicated allocation: export it with fdb_ipc_get_handle)
 *       fdb_sync_set_peers  every rank's flag block as mapped on this device (fdb_ipc_open), indexed by rank */
typedef struct fdb_sync fdb_sync;
fdb_status fdb_sync_create(fdb_sync **sync, int rank, int world, int device /* -1: current */);
fdb_status fdb_sync_flags(fdb_sync *sync, void **d_flags);
fdb_status fdb_sync_set_peers(fdb_sync *sync, void *const *d_flags_by_rank);
fdb_status fdb_sync_barrier(fdb_sync *sync, void *stream);
fdb_status fdb_sync_destroy(fdb_sync *sync);

/* ---- Colouring on the device: the ArrayInterface.matrix_colors(A) step callers run before this path
 *      (test/coloring_tests.jl:112,117).  d_colorvec is a caller-owned DEVICE array of n Int64 (1-based colours), ready to
 *      be passed to fdb_plan_create_* — a solver that resize!s its problem can recolour and re-plan without a host round
 *      trip of the pattern.
 *        banded   closed form ArrayInterface uses for BandedMatrix / Tridiagonal (l=u=1) / Bidiagonal: cycle 1:(l+u+1)
 *        csc      a valid distance-2 colouring of the columns (no two columns of one colour share a row) by a
 *                 deterministic Jones-Plassmann sweep; the result depends on the pattern alone.  colptr / rowval: Int64,
 *                 1-based, host or device.  n_colors / n_rounds (host, nullable) receive maximum(colorvec) / sweeps.
 *        check    number of (row, colour) collisions of a colouring (0 = valid for this path's decompression).
 *        csr      the same two operations on a CSR pattern (rowptr[m+1], colval[nnz]; Int64, 1-based, host or device): the
 *                 column -> rows adjacency is built on the device, and the colorvec equals fdb_matrix_colors_csc's on the
 *                 same matrix element for element. */
fdb_status fdb_matrix_colors_banded(int64_t n, int64_t l, int64_t u, int64_t *d_colorvec, void *stream);
fdb_status fdb_matrix_colors_csc(int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval, int64_t *d_colorvec,
                                 int64_t *n_colors, int64_t *n_rounds);
fdb_status fdb_check_coloring_csc(int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval, const int64_t *colorvec,
                                  int64_t *n_conflicts);
fdb_status fdb_matrix_colors_csr(int64_t m, int64_t n, const int64_t *rowptr, const int64_t *colval, int64_t *d_colorvec,
                                 int64_t *n_colors, int64_t *n_rounds);
fdb_status fdb_check_coloring_csr(int64_t m, int64_t n, const int64_t *rowptr, const int64_t *colval, const int64_t *colorvec,
                                  int64_t *n_conflicts);

/* ---- Jacobian-vector product: finite_difference_jvp!(jvp, f, x, v, cache::JVPCache, f_in; relstep, absstep, dir)
 *      src/jvp.jl:238-274 — eps from sqrt(abs(dot(x, v))) (computed on the device), forward: f(fx1,x), f(jvp,x+eps v);
 *      central: f(fx1, x-eps v) then f(jvp, x+eps v).  opts->fdtype selects forward/central (complex is rejected like
 *      in the reference).  d_x1 / d_fx1 are the JVPCache arrays (n / m doubles; NULL => plan-owned scratch);
 *      d_f_in: forward only, precomputed f(x). ---- */
fdb_status fdb_jvp_plan_create(fdb_plan **plan, int64_t m, int64_t n, const fdb_plan_opts *opts);
fdb_status fdb_jvp(fdb_plan *plan, fdb_fn f, void *ctx, double *d_jvp, const double *d_x, const double *d_v, double *d_x1,
                   double *d_fx1, const double *d_f_in, double relstep, double absstep, double dir, void *stream);

/* ---- Hessian of a scalar f: finite_difference_hessian!(H, f, x, cache::HessianCache; relstep, absstep)
 *      src/hessians.jl:202-292.  opts->fdtype must be FDB_HCENTRAL (else FDB_ERR_UNSUPPORTED, the reference's
 *      @assert fdtype == Val(:hcentral), :206); H is dense column-major with leading dimension ldH >= n (else
 *      FDB_ERR_INVALID).  max_batch: points per f call (at most 4096); scratch_bytes: one budget (0 => 8 GiB) for the point
 *      rows (at most half of it) and the stacked f values (the rest, filled by whole i-blocks; at least one i-block, 8(4n-1)
 *      bytes, whatever the budget); use_graph as for fdb_jacobian; rank / world split the work over devices (below).
 *
 *      fdb_hessian evaluates f (the batched fdb_fn with m = 1: point b at d_x + b*ldx, its scalar to d_fx[b*ldfx]) at the
 *      reference's 2n^2 + 1 points in the reference's order — f(x); then per i the pair x +- eps_i e_i and, per j > i,
 *      (+,+), (+,-), (-,+), (-,-) on (i, j) — with eps_i = max(relstep*|x_i|, absstep) (:223,234,252), and writes
 *        H[i,i] = ((f++ - 2 f(x)) + f--) / (eps_i*eps_i),  H[i,j] = H[j,i] = (((f++ - f+-) - f-+) + f--) / ((4 eps_i)*eps_j)
 *      to rows [0, n) of every column (padding rows are not touched).  d_x is never modified; d_fx (nullable, one double)
 *      receives f(x).  relstep / absstep: FDB_STEP_DEFAULT => eps(Float64)^(1/4) and absstep = relstep.
 *      Stream-ordered, no host synchronisation.  fdb_plan_info: n_entries = n^2, fcalls_per_jacobian = 2n^2 + 1,
 *      alg_bytes / moved_bytes the library's bytes per Hessian (values read back, H, point replication, patches).
 *
 *      Rank plans (opts.world in 2..64, opts.rank in 0..world-1).  i-block i (the points that change component i and no
 *      smaller one) starts at S(i) = 1 + 2i + 4(i(n-1) - i(i-1)/2) and holds 2 + 4(n-1-i) points; T = 2n^2.  Rank r owns
 *      the i-blocks [i_r, i_{r+1}) with i_0 = 0, i_world = n and, for 0 < r < world, i_r = the i in [i_{r-1}, n] whose
 *      S(i) - 1 is nearest to r*T/world (ties: the smaller i), so each rank's point count is within one block
 *      (2 + 4(n-1)) of T/world; ranges may be empty (e.g. n < world).  fdb_plan_dense_range reports [i_r, i_{r+1}).
 *      A rank evaluates f(x) first (its own, the diagonal needs it), then its points in the reference's order; rank 0
 *      always evaluates f(x) (n = 0 included), a rank > 0 with an empty range calls nothing, launches nothing and leaves
 *      d_fx untouched.  It writes exactly the entries it owns — column i rows [i, n) and row i columns (i, n) for i in its
 *      range — into the d_H it is given, so the ranks together write rows [0, n) of every column once, bit-identical to
 *      one plan; H is never zero-filled and shared_j has no effect.  d_H may be another device's H mapped into this one
 *      (a group member storing into the root's H, or an fdb_ipc_open mapping with one process per GPU); the ordering is
 *      then the Jacobian's: fdb_sync_barrier, fdb_hessian, fdb_sync_barrier.  fdb_plan_info per rank: fcalls_per_jacobian
 *      = 1 + the rank's points (0 for an empty rank > 0), n_entries = sum over its i of 2(n-i) - 1, byte model the
 *      rank's own; summed over the ranks they give the whole Hessian's figures plus one f(x) per non-empty rank > 0. ---- */
fdb_status fdb_hessian_plan_create(fdb_plan **plan, int64_t n, int64_t ldH, const fdb_plan_opts *opts);
fdb_status fdb_hessian(fdb_plan *plan, fdb_fn f, void *ctx, const double *d_x, double *d_H, double *d_fx, double relstep,
                       double absstep, void *stream);
/* One process, n devices: the group form of the rank plans above (fdb_group_create_* / fdb_group_plan / fdb_group_destroy
 * as for Jacobians).  Member i runs rank i of n_devices on its own stream with ctx[i]; d_x, d_H and d_fx live on
 * devices[0] (the root), x is replicated to members on other devices, every member stores its entries straight into the
 * root's H, the root writes f(x) to d_fx, and the members are joined on `stream` (a stream of devices[0]) with events —
 * no host synchronisation.  Device ordinals may repeat.  opts->fdtype must be FDB_HCENTRAL (else FDB_ERR_UNSUPPORTED).
 * fdb_group_hessian on a Jacobian group and fdb_group_jacobian on a Hessian group return FDB_ERR_INVALID before any
 * launch.  f is evaluated once per non-empty member at x; H is bit-identical to the one-device result. */
fdb_status fdb_group_create_hessian(fdb_group **group, int n_devices, const int *devices, int64_t n, int64_t ldH,
                                    const fdb_plan_opts *opts);
fdb_status fdb_group_hessian(fdb_group *group, fdb_fn f, void *const *ctx, const double *d_x, double *d_H, double *d_fx,
                             double relstep, double absstep, void *stream);

/* ---- Derivatives with a scalar input per step size ----
 *   finite_difference_derivative!(df, f, x::StridedArray, cache::DerivativeCache; relstep, absstep, dir)
 *                                                                        src/derivatives.jl:197-233
 *   finite_difference_gradient!(df, f, x::Number, cache::GradientCache; relstep, absstep, dir)   src/gradients.jl:477-533
 * fdb_derivative_plan_create: the elementwise derivative of a scalar function over n components.  f is the batched
 *   fdb_fn with m = n, applied elementwise: d_fx[b*ldfx + i] = f(d_x[b*ldx + i]).  df, x: n doubles.
 * fdb_scalar_gradient_plan_create: the scalar -> vector "gradient" of an in-place f(fx, t) with m outputs: the fdb_fn
 *   with n = 1 (point b is the single double d_x[b*ldx]) and m outputs.  df: m doubles; x: ONE double (device memory,
 *   so that a solver writing t in place can replay a captured graph).
 * opts->fdtype: FDB_FORWARD, FDB_CENTRAL or FDB_COMPLEX (FDB_HCENTRAL => FDB_ERR_UNSUPPORTED); one device (world <= 1).
 * max_batch >= 2: a central call hands both points (rows 0: x+eps, 1: x-eps at the plan's ldx) to ONE f call.
 *
 * fdb_derivative evaluates, per component (derivative) or once (gradient), eps = max(relstep*|x|, absstep)*dir (forward;
 * central without dir) and, in the reference's order, f(x+eps) then f(x) (forward, unless d_fx is given: cache.fx, the
 * f values at x) or f(x+eps) then f(x-eps) (central), and writes
 *   forward  df = (f(x+eps) - f(x)) / eps
 *   central  df = (f(x+eps) - f(x-eps)) * (1 / (2eps))   derivative (the reciprocal is rounded first, derivatives.jl:220-222)
 *            df = (f(x+eps) - f(x-eps)) / (2eps)         scalar gradient (gradients.jl:520)
 * d_x is never modified; d_fx is ignored outside forward mode.  relstep / absstep: FDB_STEP_DEFAULT => default_relstep(fdtype)
 * and absstep = relstep.  fdb_derivative_complex (plans of fdtype FDB_COMPLEX): one complex128 evaluation at
 * (x + 0.0) + im*eps(Float64), df = imag(f) / eps(Float64).  Stream-ordered, no host synchronisation; use_graph as for
 * fdb_jacobian.  fdb_plan_info: n_entries = length(df), fcalls_per_jacobian = f evaluations of the last call (before
 * the first: 2 forward / central, 1 complex), alg_bytes / moved_bytes = the library's compulsory bytes per call.
 * The Jacobian, Hessian and JVP entry points reject these plans, and fdb_derivative rejects theirs (FDB_ERR_INVALID). ---- */
fdb_status fdb_derivative_plan_create(fdb_plan **plan, int64_t n, const fdb_plan_opts *opts);
fdb_status fdb_scalar_gradient_plan_create(fdb_plan **plan, int64_t m, const fdb_plan_opts *opts);
fdb_status fdb_derivative(fdb_plan *plan, fdb_fn f, void *ctx, double *d_df, const double *d_x, const double *d_fx,
                          double relstep, double absstep, double dir, void *stream);
fdb_status fdb_derivative_complex(fdb_plan *plan, fdb_fn_c f, void *ctx, double *d_df, const double *d_x, void *stream);

/* ---- Out-of-place Jacobian: J = finite_difference_jacobian(f, x, cache, f_in; relstep, absstep, colorvec, sparsity,
 *      jac_prototype, dir)  src/jacobians.jl:277-429 (cache-less form :240-259 = f(x) once, then the cached form).
 * Differences from the in-place colour loop, all reproduced:
 *   - every point starts from the caller's x: colour k gets x +- eps_k on its columns and x +- copysign(0, eps_k) on every
 *     other component (sparsity given, :341,381-382); the dense branch changes component i alone (:322,359-360);
 *   - central mode takes the forward step rule, dir included (:358,379-380);
 *   - the result is J + Ji summed over the colours, whose form depends on jac_prototype (result_kind):
 *       FDB_OOP_RAW     sparsity === nothing, no prototype: dense m x maximum(colorvec) holding the raw quotients (:329-331)
 *       FDB_OOP_DENSE   a dense result (prototype dense, or sparsity given without a sparse prototype): structural slots
 *                       hold 0.0 + q (-0.0 becomes +0.0), every other element +0.0
 *       FDB_OOP_SPARSE  a SparseMatrixCSC prototype: the structural entries whose quotient is not +-0.0 (NaN is kept), in
 *                       storage order (SparseArrays' zero-preserving `+`); sparsity === nothing: the nonzeros of every column
 *   f! call count and order: forward f(x) (unless d_f_in) then one call per colour; central f(x+) then f(x-) per colour;
 *   complex one call per colour.  d_x is never modified.
 * fdb_oop_plan_create_csc: sparsity is a CSC pattern (Int64, 1-based, host or device), result_kind FDB_OOP_DENSE (J dense
 *   m x n with leading dimension ldJ; a colouring in which two columns of one colour share a row is FDB_ERR_INVALID, as
 *   _make_Ji throws, :151-162) or FDB_OOP_SPARSE (ldJ ignored; any colouring).
 * fdb_oop_plan_create_dense: sparsity === nothing.  C = maximum(colorvec) (NULL => n) must be at most n.  FDB_OOP_RAW: J is
 *   m x C (ncols_out ignored; C < 1 is FDB_ERR_INVALID, as mapreduce over the empty colour range throws); FDB_OOP_DENSE: J
 *   is m x ncols_out with ncols_out >= C (a narrower prototype is not built: FDB_ERR_UNSUPPORTED); FDB_OOP_SPARSE:
 *   ncols_out >= C (else FDB_ERR_INVALID, as sparse() throws).  With the prototype kinds, C < 1 gives zero(jac_prototype):
 *   +0.0 everywhere, or colptr all 1 and nnz 0, after f(x) in forward mode without d_f_in and no other call.
 * fdb_oop_plan_create_banded: the sparsity is the in-matrix band (l, u) of an m x n matrix, E = {(r, c) : -u <= r - c <= l}
 *   (BandedMatrix(m, n, l, u); Diagonal (0, 0), Bidiagonal :U (0, 1) and :L (1, 0), SymTridiagonal and Tridiagonal (1, 1)),
 *   result_kind FDB_OOP_DENSE or FDB_OOP_SPARSE exactly as fdb_oop_plan_create_csc given the CSC of E: the same result,
 *   status and f! calls.  No entry list is built on the host or the device: the structure stays a closed form.  l < 0 or
 *   u < 0 is FDB_ERR_UNSUPPORTED; bandwidths beyond the matrix give the matrix's own band.  A dense result counts the
 *   colouring's conflicts on the device at plan time (skipped for a cyclic colouring with more than l + u colours, which has
 *   none).  A sparse result is compacted from the resident f! outputs in closed form, or, when they come in several groups
 *   or ranks, from candidates the band scatter wrote in band-data layout.
 * fdb_oop_plan_create_block_banded / fdb_oop_plan_create_block_dense: the sparsity is the entry set E of a square-block
 *   BandedBlockBandedMatrix (block bandwidths (l, u), sub-block bandwidths (lam, mu): rows max(0, j-mu) .. min(m_K-1, j+lam)
 *   of every block (K, J) with K in blockcolrange(J)) or BlockSkylineMatrix (every row of those blocks; BlockBandedMatrices'
 *   BlockBandedMatrix), `blocks` the nblocks block sizes as for fdb_plan_create_block_banded / _block_dense.  Only
 *   result_kind FDB_OOP_SPARSE is built (ldJ is ignored): the same result, status and f! calls as fdb_oop_plan_create_csc
 *   given the CSC of E, for any colorvec.  FDB_OOP_DENSE is FDB_ERR_UNSUPPORTED and FDB_OOP_RAW FDB_ERR_INVALID; sizes,
 *   bandwidths and the block list are refused as by the in-place block creators.  Host work is O(nblocks) plus reading the
 *   colorvec, and no entry, row or column-start list exists: the compaction finds each candidate's column and row from the
 *   block offsets and one table of nblocks + 1 block-column starts.  Candidate counts may pass 2^31.
 * fdb_oop_plan_create_csr: the sparsity is one CSR pattern (m x n, rowptr[m+1], colval[nnz]; Int64, 1-based, host or
 *   device), and the result a CSR.  Only result_kind FDB_OOP_SPARSE is built (ldJ is ignored); FDB_OOP_DENSE is
 *   FDB_ERR_UNSUPPORTED and FDB_OOP_RAW FDB_ERR_INVALID; sizes, the row pointer, the columns and nnz >= 2^31 are refused
 *   as by fdb_plan_create_csr.  The candidates are the stored entries, one per slot; a candidate is kept when its value is
 *   not +-0.0 (NaN is kept), and each kept value is bit-identical to what fdb_oop_plan_create_csc gives for the same
 *   (row, column) on the CSC of the same entry set.  Rows come in order and, within a row, the kept entries keep the
 *   pattern's own storage order (unsorted columns stay unsorted; a repeated (r, c) gives two entries of one value), so for
 *   rows of sorted, distinct columns the result is the CSC route's result converted to CSR.  f! calls and points are the
 *   CSC route's.  With more than 8 colours the step sizes come from per-colour column lists, as the CSC plan's do.
 * n = 0 is FDB_ERR_INVALID (maximum of an empty colorvec throws).  opts as for the in-place plans (rank plans below).
 * fdb_jacobian_oop / fdb_jacobian_oop_complex write the result to `out`:
 *   dense kinds: out->J (device, ldJ of the plan; the whole result, rank plans included);
 *   FDB_OOP_SPARSE: out->colptr [ncols + 1], out->rowval / out->nzval [out->cap >= the candidate count: nnz of the sparsity,
 *   or m*C], Int64 1-based; the kept count goes to the device scalar *out->nnz (stream-ordered, no host sync).
 *   A CSR plan writes the same fields in row-compressed form: out->colptr receives the m + 1 row starts and out->rowval
 *   the column of every kept entry (Int64, 1-based), with out->cap >= nnz.
 * fdb_plan_info(...).n_entries is the candidate count of the whole result (m*C on the dense branch, nnz with a CSC or CSR
 * sparsity, |E| with a band or a block structure); a CSR plan reports jkind FDB_J_CSR.
 *
 * Rank plans (opts.rank / opts.world, world in 2..64).  A rank evaluates only the colours it owns: the colour partition of
 * the in-place plans (opts.partition: round-robin or LPT, fdb_plan_color_owner) with a sparsity, the contiguous column
 * blocks of the dense plans over the C = maximum(colorvec) quotient columns (fdb_plan_dense_range) without one.  It uses
 * the same pristine points, step rule and dir, and writes exactly the slots it owns:
 *   FDB_OOP_RAW                 its column block of the m x C quotients;
 *   FDB_OOP_DENSE, no sparsity  0.0 + q on its own columns; rank 0 also writes +0.0 to the prototype's columns [C, ncols);
 *   FDB_OOP_DENSE, CSC          q, then + 0.0, on the structural slots of its own colours only; the owner of the buffer
 *                               zero-fills J before any rank starts (opts.shared_j = 1; without it a rank zero-fills J
 *                               itself, like an in-place rank plan);
 *   FDB_OOP_SPARSE, CSC         its colours' candidate quotients, in storage order, into the root's candidate buffer (rank 0
 *                               also writes the zeros of columns without a valid colour); the root then compacts all nnz
 *                               candidates into `out`;
 *   FDB_OOP_DENSE, band         as for a CSC sparsity, the + 0.0 in closed form over its own colours' band entries;
 *   FDB_OOP_SPARSE, band        its colours' columns of the band data into the root's buffer (rank 0 also writes the zeros
 *                               of columns without a valid colour); the root then compacts every band entry into `out`;
 *   FDB_OOP_SPARSE, block       its colours' columns into the root's buffer in the in-place layout (band data for
 *                               block-banded, slabs for block-dense; rank 0 also writes the zeros of columns without a valid
 *                               colour); the root then compacts every entry of E into `out`;
 *   FDB_OOP_SPARSE, CSR         its colours' candidate quotients, in slot order, into the root's candidate buffer (rank 0
 *                               also writes the zeros of columns without a valid colour); the root then compacts all nnz
 *                               candidates into `out`;
 *   FDB_OOP_SPARSE, no sparsity its column block of the m x C candidates at offset col_begin*m; the root then compacts all
 *                               m*C of them.
 * Per rank: forward mode without d_f_in evaluates f(x) first, then its own colours ascending; central f(x+) then f(x-) per
 * own colour; a rank > 0 that owns no colour (no column) calls nothing and launches nothing.  fdb_plan_info reports the
 * rank's share (fcalls_per_jacobian, n_local_colors, byte model); n_entries stays the whole result's candidate count.
 * A dense-kind rank plan may be driven on its own through fdb_jacobian_oop, every rank passing the same whole result: the
 * ranks are then ordered as in-place shared_j rank plans are (fdb_sync_barrier, fdb_jacobian_oop, fdb_sync_barrier, after
 * the owner's zero fill).  A sparse result needs every candidate on one device: fdb_jacobian_oop refuses a sparse rank
 * plan with world > 1 (FDB_ERR_INVALID); fdb_group_jacobian_oop runs it.  Every kind, mode, dir and step override gives
 * the one-device result bit for bit. */
enum { FDB_OOP_RAW = 0, FDB_OOP_DENSE = 1, FDB_OOP_SPARSE = 2 };

typedef struct {
  double *J;                 /* dense kinds */
  int64_t *colptr, *rowval;  /* FDB_OOP_SPARSE */
  double *nzval;
  int64_t cap;
  int64_t *nnz;              /* device scalar */
} fdb_oop_out;

fdb_status fdb_oop_plan_create_csc(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval,
                                   const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_oop_plan_create_dense(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colorvec, int64_t ncols_out,
                                     int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_oop_plan_create_banded(fdb_plan **plan, int64_t m, int64_t n, int64_t l, int64_t u, const int64_t *colorvec,
                                      int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_oop_plan_create_block_banded(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                            int64_t lam, int64_t mu, const int64_t *colorvec, int result_kind, int64_t ldJ,
                                            const fdb_plan_opts *opts);
fdb_status fdb_oop_plan_create_block_dense(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                           const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_oop_plan_create_csr(fdb_plan **plan, int64_t m, int64_t n, const int64_t *rowptr, const int64_t *colval,
                                   const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_jacobian_oop(fdb_plan *plan, fdb_fn f, void *ctx, const double *d_x, const fdb_oop_out *out, double *d_fx,
                            const double *d_f_in, double relstep, double absstep, double dir, void *stream);
fdb_status fdb_jacobian_oop_complex(fdb_plan *plan, fdb_fn_c f, void *ctx, const double *d_x, const fdb_oop_out *out,
                                    void *stream);

/* One process, n devices: the group form of the out-of-place rank plans (fdb_group_size / fdb_group_plan /
 * fdb_group_destroy as for Jacobians).  Member i runs rank i of n_devices on its own stream with ctx[i]; d_x, out, d_fx and
 * d_f_in live on devices[0] (the root), x (and d_f_in, forward mode) is replicated to members on other devices, every
 * member stores its slots straight into the root's result (sparse: the root's candidate buffer), and the members are
 * joined on `stream` (a stream of devices[0]) with events.  Before any member starts, the root zero-fills a dense result
 * of a CSC or band sparsity; after every member has finished, the root compacts a sparse result.  No host synchronisation: the
 * kept count lands in *out->nnz.  Only the root writes f(x) to d_fx.  Device ordinals may repeat.  The result is
 * bit-identical to fdb_jacobian_oop on one device.  Complex-step groups return FDB_ERR_UNSUPPORTED.
 * fdb_group_jacobian_oop on a Jacobian or Hessian group, and fdb_group_jacobian / fdb_group_hessian on an out-of-place
 * group, return FDB_ERR_INVALID before any launch. */
fdb_status fdb_group_create_oop_csc(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                    const int64_t *colptr, const int64_t *rowval, const int64_t *colorvec, int result_kind,
                                    int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_group_create_oop_csr(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                    const int64_t *rowptr, const int64_t *colval, const int64_t *colorvec, int result_kind,
                                    int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_group_create_oop_dense(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                      const int64_t *colorvec, int64_t ncols_out, int result_kind, int64_t ldJ,
                                      const fdb_plan_opts *opts);
fdb_status fdb_group_create_oop_banded(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n, int64_t l,
                                       int64_t u, const int64_t *colorvec, int result_kind, int64_t ldJ,
                                       const fdb_plan_opts *opts);
fdb_status fdb_group_create_oop_block_banded(fdb_group **group, int n_devices, const int *devices, int64_t nblocks,
                                            const int64_t *blocks, int64_t l, int64_t u, int64_t lam, int64_t mu,
                                            const int64_t *colorvec, int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_group_create_oop_block_dense(fdb_group **group, int n_devices, const int *devices, int64_t nblocks,
                                           const int64_t *blocks, int64_t l, int64_t u, const int64_t *colorvec,
                                           int result_kind, int64_t ldJ, const fdb_plan_opts *opts);
fdb_status fdb_group_jacobian_oop(fdb_group *group, fdb_fn f, void *const *ctx, const double *d_x, const fdb_oop_out *out,
                                  double *d_fx, const double *d_f_in, double relstep, double absstep, double dir,
                                  void *stream);

/* Out-of-place JVP: jvp = finite_difference_jvp(f, x, v, cache, f_in; relstep, absstep, dir)  src/jvp.jl:159-189.  Same
 * plan (fdb_jvp_plan_create) and arguments as fdb_jvp; central mode evaluates f(x + eps v) into d_jvp BEFORE f(x - eps v)
 * into d_fx1 (:180-183; the in-place form calls them the other way round). */
fdb_status fdb_jvp_oop(fdb_plan *plan, fdb_fn f, void *ctx, double *d_jvp, const double *d_x, const double *d_v, double *d_x1,
                       double *d_fx1, const double *d_f_in, double relstep, double absstep, double dir, void *stream);

/* ---- helpers for hosts without their own CUDA bindings ---- */
fdb_status fdb_host_alloc(void **p, size_t bytes);  /* pinned host memory */
fdb_status fdb_host_free(void *p);
fdb_status fdb_device_alloc(void **p, size_t bytes);
fdb_status fdb_device_free(void *p);
fdb_status fdb_memcpy_h2d(void *d, const void *h, size_t bytes, void *stream);
fdb_status fdb_memcpy_d2h(void *h, const void *d, size_t bytes, void *stream);
fdb_status fdb_stream_sync(void *stream);
/* CUDA IPC, for the one-process-per-GPU fused gather (handle is CUDA_IPC_HANDLE_SIZE = 64 bytes) */
fdb_status fdb_ipc_get_handle(void *d_ptr, unsigned char handle[64]);
fdb_status fdb_ipc_open(const unsigned char handle[64], void **d_ptr);
fdb_status fdb_ipc_close(void *d_ptr);

#ifdef __cplusplus
}
#endif
#endif /* FDJAC_B200_H */
