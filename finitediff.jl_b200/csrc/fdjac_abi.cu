// fdjac_abi.cu — libfdjac_b200.so: plan management + the C ABI declared in include/fdjac_b200.h.
// H100 / sm_90a only.  There is NO CPU fallback: without a CUDA device every compute entry point fails with
// FDB_ERR_NO_DEVICE.  Nothing here includes, links or calls anything under oracle/.
#include "../../include/fdjac_b200.h"

#include <algorithm>
#include <climits>
#include <cstdarg>
#include <cmath>
#include <cfloat>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <numeric>
#include <string>
#include <type_traits>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "kernels_eps.cuh"
#include "kernels_perturb.cuh"
#include "kernels_plan.cuh"
#include "kernels_scatter.cuh"
#include "kernels_staged.cuh"
#include "kernels_jvp.cuh"
#include "kernels_color.cuh"
#include "kernels_hessian.cuh"
#include "kernels_derivative.cuh"
#include "kernels_blockband.cuh"
#include "kernels_diagonals.cuh"
#include "kernels_csr.cuh"

using namespace fdb;

// ------------------------------------------------------------------------------------------------ errors
static thread_local std::string g_err;

static fdb_status fail(fdb_status st, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return st;
}

#define CU(expr)                                                                                       \
  do {                                                                                                 \
    cudaError_t e__ = (expr);                                                                          \
    if (e__ != cudaSuccess)                                                                            \
      return fail(FDB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

#define TRY(expr)                    \
  do {                               \
    fdb_status s__ = (expr);         \
    if (s__ != FDB_OK) return s__;   \
  } while (0)

enum { SP_NONE = 0, SP_CSC = 1, SP_COO = 3, SP_BANDED = 4, SP_JVP = 5, SP_EPS = 6, SP_HESS = 7, SP_DERIV = 8, SP_BLOCKBAND = 9, SP_CSR = 10 };

// Device memory that lives while a plan or a colouring is built: freed when it goes out of scope, unless release()
// hands it to a plan that keeps it (fdb_plan::adopt).  Declared after the builder's DeviceGuard, it is freed on the
// device it was allocated on.
template <typename T> struct DevBuf {
  T *p = nullptr;
  size_t bytes = 0;
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  fdb_status alloc(size_t count) {
    bytes = count * sizeof(T);
    if (bytes == 0) bytes = 16;
    const cudaError_t e = cudaMalloc((void **)&p, bytes);
    if (e != cudaSuccess) {
      p = nullptr;
      return fail(FDB_ERR_NOMEM, "cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
    }
    return FDB_OK;
  }
  T *get() const { return p; }
  T *release() { T *q = p; p = nullptr; return q; }
};

// copy `count` values back from the device; `what` names the value in the error text
template <typename T> static fdb_status read_back(T *h, const T *d, size_t count, const char *what) {
  const cudaError_t e = cudaMemcpy(h, d, count * sizeof(T), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return fail(FDB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return FDB_OK;
}

// a CUB device algorithm, called the two-phase way: `algo(nullptr, bytes)` sizes its scratch, `algo(tmp, bytes)` runs
template <typename F> static fdb_status cub_run(F &&algo) {
  size_t bytes = 0;
  CU(algo(nullptr, bytes));
  DevBuf<char> tmp;
  TRY(tmp.alloc(bytes));
  CU(algo((void *)tmp.get(), bytes));
  return FDB_OK;
}

struct DeviceGuard {
  int prev = -1;
  bool ok = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess) {
      if (prev == dev) ok = true;
      else ok = cudaSetDevice(dev) == cudaSuccess;
    }
  }
  ~DeviceGuard() {
    int cur = -1;
    if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
  }
};

// identity of a captured call: same function, buffers and scalar arguments => same launch sequence.  The scalars are
// compared by bit pattern: relstep = absstep = -0.0 gives the step -0.0, which keeps a -0.0 component of x negative where
// the step +0.0 does not, so a graph captured with one must not be replayed for the other.
static inline bool same_bits(double a, double b) { return std::memcmp(&a, &b, sizeof a) == 0; }

struct GraphKey {
  void *f = nullptr, *ctx = nullptr;
  const void *x = nullptr, *J = nullptr, *fx = nullptr, *f_in = nullptr;
  double relstep = 0, absstep = 0, dir = 0;
  int n_peers = 0;
  long long peer_generation = 0;
  const void *ext_eps = nullptr;
  bool operator==(const GraphKey &o) const {
    return f == o.f && ctx == o.ctx && x == o.x && J == o.J && fx == o.fx && f_in == o.f_in &&
           same_bits(relstep, o.relstep) && same_bits(absstep, o.absstep) && same_bits(dir, o.dir) &&
           n_peers == o.n_peers && peer_generation == o.peer_generation && ext_eps == o.ext_eps;
  }
};

// ------------------------------------------------------------------------------------------------ plan
// A plan's state: the fields every plan has, then one part per piece of work, each filled only by the plan kinds named
// on it (the other kinds leave it at its defaults).  SP_NONE is the dense-column plan.
struct fdb_plan {
  int device = 0, sm_count = 132;
  int64_t l2_bytes = 50 << 20;
  int fdtype = FDB_FORWARD, sp_kind = SP_CSC, jkind = FDB_J_CSC_NZVAL;
  int rank = 0, world = 1;
  int64_t m = 0, n = 0, j_len = 0, ldJ = 0;
  bool shared_J = false;            // member of an fdb_group: J is shared with the other members (root zero-fills it)
  int no_drift = 0;
  // A/B switches (environment, read ONCE when the plan is created — never on the hot path; DESIGN.md §4)
  struct Tunables {
    bool no_staged = false, no_eps_lists = false, no_eps_overlap = false, cm_prefetch = false, force_overlap = false;
    bool no_fx_cm = false, force_fx_cm = false, no_pack = false, no_band = false;
    int hi_stream = -1;                // -1: by pattern (random => evict-first slab gathers), 0 / 1: forced
    // walk direction: bit 0 the staged scatter
    // starts at the END of J's storage, bit 1 the perturbation pass at the end of x — each reads first what the kernel
    // before it streamed last (still in L2), and the first f! finds the heads of the points the perturbation wrote last
    int reverse = 3;
    int cm_slab_stream = 1;            // colour-major scatter, forward: slab gathers evict-first (CmArgs::slab_stream)
    int eps_depth = 2;                 // color_sumsq_reg: tiles of loads in flight per thread (same summation order, same bits)
    int cols_depth = 0, cols_gx = 64;  // diff_columns: loads in flight per thread (0 = by mode) / cap on the row blocks per column
    int stages = 2;
    char staged_variant[3] = {'6', 'n', 0};
  } tune;
  fdb_counters_t cnt{};
  int64_t alg_bytes = 0;
  std::vector<void *> allocs;
  size_t device_bytes = 0;

  // f! outputs and perturbed points: every kind but the step-size plan.  What batch, slabs and n_groups count:
  //   coloured (CSC, COO, banded, block-banded): points per f! call; colours whose f! outputs are resident at once;
  //     scatter groups per call
  //   dense: columns per f! call = slabs; column batches per call
  //   Hessian: points per f call = slabs; chunks of whole i-blocks
  //   derivative: 2 when the two central points go to f in one call, else 1 (no slabs, no groups)
  //   JVP: 1 (no slabs, no groups)
  struct Scratch {
    double *fx_own = nullptr, *Fp = nullptr, *Fm = nullptr, *xp = nullptr, *xm = nullptr;
    int64_t ldF = 0, ldx = 0;
    int64_t batch = 1, slabs = 0, n_groups = 0;
    int64_t pbatch = 1;   // coloured: perturbed points built per perturb pass (>= batch): x is read once for all of them
  } scratch;
  // colours: coloured plans and the step-size plan (C, the colour table and the column lists); coloured plans also fill
  // the ownership and local colours, and E
  struct Colors {
    int32_t C = 0;                    // maximum(colorvec)
    int bits = 8;                     // width of a colour in the tables: 8, 16 or 32
    bool has_invalid = false;
    bool cyclic = false;              // colorvec[j] == j mod C + 1 for every j: kernels use the closed form, jcolor is not read
    void *jcolor = nullptr;           // [n] CT
    int64_t E = 0;                    // structural entries of the coloured pattern (banded: in-band slots of valid colours)
    std::vector<int32_t> owner;       // [C] rank evaluating each colour
    std::vector<int32_t> local;       // this rank's colours, ascending
    int32_t *d_local = nullptr;       // [n_local] device copy of `local`
    int32_t *local_of = nullptr;      // [C] device: local index of each colour, -1 when another rank owns it
    // per-colour column lists (CSC plans, and plans with more than kEpsRegColors colours): bucket_start [C+2] offsets
    // into cols_by_color; bucket C = columns without a valid colour
    std::vector<int64_t> bucket_start;
    int32_t *cols_by_color = nullptr;
  } colors;
  // step sizes: coloured plans, the step-size plan (per colour) and the JVP plan (one)
  struct Steps {
    double *eps = nullptr, *sumsq = nullptr, *partial = nullptr;
    unsigned int *ticket = nullptr;   // last-block-done counter of color_sumsq_reg
    int blocks = 0;
    int64_t chunk = 0;
    int32_t group = 1;   // largest aligned lane group without a repeated colour (color_lane_conflicts)
    const double *ext = nullptr;   // step sizes supplied by the caller (fdb_plan_set_external_eps), device, >= C entries
    // eps from the per-colour column lists (more than kEpsRegColors colours)
    bool lists = false;
    int64_t *bucket_start_d = nullptr, *chunk_base_d = nullptr;
    double *list_partial = nullptr;
    int64_t list_max_chunks = 0;
  } steps;
  // compressed entry streams: CSC and COO plans.  strategy (CSC; internal, opts->strategy 0..3 is mapped onto it in
  // fdb_plan_create_csc): 0 = one fused pass over J's storage order, 1 = colour-major entry lists (per group of
  // resident colours)
  struct Entries {
    int32_t *row32 = nullptr;         // [E]
    void *ecolor = nullptr;           // [E] CT
    int64_t *dest = nullptr;          // [E] or null (identity)
    int32_t *colptr32 = nullptr;      // [n + 1] (CSC)
    int lanes = 1;
    double mean_row_jump = 0.0;
    int strategy = 0;
    bool strategy_auto = true;
    bool lists_resident = false;      // lists with every local colour's f! output resident: ONE launch over them
  } entries;
  // colour-major entry lists of this rank's colours: CSC plans with strategy 1 (built by build_cm_lists)
  struct ColorMajor {
    int32_t *row = nullptr;
    void *slot = nullptr;             // int32 (nzval slot) or int64 (explicit destination: entries.dest != nullptr)
    int64_t *start = nullptr;         // device [n_local + 1]
    double *fx = nullptr;             // forward: f(x) in colour-major order (rebuilt by every Jacobian)
    std::vector<int64_t> start_h;     // host copy; [n_local] .. invalid_end = entries of columns without a valid colour
    int64_t invalid_end = 0;
  } cm;
  // TMA-staged form of the fused pass: CSC plans with a row-local pattern (kernels_staged.cuh)
  struct Staged {
    bool on = false, packed = false;
    uint16_t *row16 = nullptr;
    int32_t *tile_w0 = nullptr;
    unsigned long long *claim = nullptr;   // walk-position counter of the staged pass (re-armed by every launch)
    int32_t W = 0;
    bool band = false;                // exact clipped band: the staged pass derives rows and columns, reads no index stream
    int32_t band_l = 0, band_col_a = 0, band_col_b = 0, band_e_a = 0, band_e_b = 0, band_w = 1;
  } staged;
  // bandwidths: banded and block-banded plans
  struct Band {
    int64_t l = 0, u = 0;
  } band;
  // block-banded and block-dense plans (kernels_blockband.cuh): block offsets on the device, sub-block bandwidths, slots
  // per column (block-banded), the slab starts (block-dense, jkind FDB_J_BLOCK_DENSE)
  struct BlockBand {
    int32_t *off = nullptr;           // [nblocks + 1]
    int32_t nblocks = 0, bs = 0;      // bs > 0: every block has bs columns
    int64_t lam = 0, mu = 0, w = 1;
    bool cyclic = false;              // colorvec is the block-cyclic closed form of matrix_colors
    int64_t *start = nullptr;         // block-dense: [nblocks + 1] first slot of every block column's slab
  } block_band;
  // CSR plans (kernels_csr.cuh): the row pointer and the columns, 0-based int32, on the device
  struct Csr {
    int32_t *rowptr = nullptr;        // [m + 1]
    int32_t *colval = nullptr;        // [nnz]
  } csr;
  // dense plans: this rank's column block [begin, end) and its steps
  struct Columns {
    int64_t begin = 0, end = 0;
    double *eps = nullptr;            // [end - begin]
  } columns;
  // Hessian plans (kernels_hessian.cuh): value buffer V (V[0] = f(x), then one chunk of whole i-blocks) and the chunk
  // boundaries [chunks[c], chunks[c+1]) in i
  struct Hessian {
    double *V = nullptr;
    std::vector<int64_t> chunks;
    // rank plans: local point q > 0 is global point q + off; points = the rank's f evaluations per call
    int64_t off = 0, points = 0;
    int64_t i_begin = 0, i_end = 0;   // this rank's i-blocks
    int64_t entries = 0;              // entries of H the rank's i-blocks write
    double *eps = nullptr;            // [n] per-component steps of all n components
  } hess;
  // derivative plans (kernels_derivative.cuh): elementwise derivative (m = n) or scalar -> vector gradient (n = 1)
  struct Derivative {
    bool elem = false;
    int64_t fcalls = 0;   // f evaluations of the most recent call (before any: the count without cache.fx)
  } deriv;
  // out-of-place Jacobian plans (fdjac_oop.cuh): the colour loop with pristine points and the forward step rule in
  // central mode, then the result form of the out-of-place finite_difference_jacobian
  struct OutOfPlace {
    bool on = false;                  // an out-of-place plan (fdb_jacobian rejects it)
    int kind = 0;                     // FDB_OOP_RAW / FDB_OOP_DENSE / FDB_OOP_SPARSE
    int64_t ncols = 0;                // columns of the result
    int64_t qcols = 0;                // dense branch: columns holding quotients, maximum(colorvec), over every rank
    const int64_t *dest = nullptr;    // dense result of a CSC sparsity: the slots of this rank's colours (entries.dest when world = 1)
    int64_t dest_n = 0;
    double *vals = nullptr;           // sparse result: the candidate values (nzval of the sparsity, or the m x C dense block)
    unsigned long long *state = nullptr;   // sparse result: look-back words of the compaction, then its tile counter
    int32_t *tile_col = nullptr;      // sparse result of a CSC sparsity: first column starting in each tile
    bool fused = false;               // sparse result, every colour's f! output resident: quotient + compaction fused
    int64_t band_nnz = 0;             // result of a band sparsity: |E|, every in-matrix band entry (colors.E counts coloured ones)
    int64_t *block_start = nullptr;   // result of a block-banded sparsity: [nblocks + 1] first entry of every block column of E
  } oop;
  // side stream and events: coloured plans.  Forward mode runs the eps pass beside f(x) on the side stream; with
  // double_buffer, two output buffers let a group's scatter overlap the next group's f!
  struct Overlap {
    bool double_buffer = false;
    cudaStream_t side = nullptr;
    cudaEvent_t ev_f[2] = {nullptr, nullptr}, ev_scat[2] = {nullptr, nullptr};
    cudaEvent_t ev_fork = nullptr, ev_eps = nullptr;
  } overlap;
  // peer J buffers (multi-GPU fused gather): CSC, COO, JVP and step-size plans (fdb_plan_set_peers)
  struct Peers {
    double **d = nullptr;
    int n = 0;
    long long generation = 0;
    bool aligned = true;
  } peers;
  // optional CUDA-graph replay of the whole call
  struct Graph {
    bool use = false;
    cudaStream_t stream = nullptr;
    cudaGraphExec_t exec = nullptr;
    GraphKey key;
    fdb_counters_t delta{};
  } graph;
  // optional device-side timing of the scatter launches
  struct Timing {
    bool on = false;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending, pool;
  } timing;
  // host-buffer path (fdb_jacobian_host): its stream and device staging buffers, made by the first call
  struct Host {
    cudaStream_t stream = nullptr;
    double *dx = nullptr, *dJ = nullptr, *dfx = nullptr, *dfin = nullptr;
  } host;

  // device memory the plan keeps until fdb_plan_destroy (build scratch is a DevBuf instead)
  void adopt(void *p, size_t bytes) {
    allocs.push_back(p);
    device_bytes += bytes;
  }
  fdb_status alloc(void **p, size_t bytes) {
    DevBuf<char> b;
    TRY(b.alloc(bytes));
    *p = b.get();
    adopt(b.release(), b.bytes);
    return FDB_OK;
  }
  template <typename T> fdb_status alloc_t(T **p, size_t count) { return alloc((void **)p, count * sizeof(T)); }
  int grid(int64_t items, int per_block = kThreads, int waves = 8) const {
    int64_t b = (items + per_block - 1) / per_block;
    const int64_t cap = (int64_t)sm_count * waves;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
  }
};

// A caller-supplied Int64 array that may live on the host or the device: make it readable by kernels.
struct I64View {
  const int64_t *d = nullptr;
  DevBuf<int64_t> copy;   // device copy of a host array
};

static fdb_status view_i64(const int64_t *p, int64_t count, I64View &v) {
  if (!p || count <= 0) { v.d = nullptr; return FDB_OK; }
  cudaPointerAttributes at{};
  cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
  if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) { v.d = p; return FDB_OK; }
  TRY(v.copy.alloc((size_t)count));
  CU(cudaMemcpy(v.copy.get(), p, (size_t)count * sizeof(int64_t), cudaMemcpyHostToDevice));
  v.d = v.copy.get();
  return FDB_OK;
}

static fdb_status check_device(const fdb_plan_opts *o, int *dev) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count <= 0) {
    cudaGetLastError();
    return fail(FDB_ERR_NO_DEVICE, "no CUDA device available (%s): libfdjac_b200 has no CPU fallback",
                e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
  }
  int d = 0;
  if (!o || o->use_current_device || o->device < 0) { CU(cudaGetDevice(&d)); }
  else d = o->device;
  if (d >= count) return fail(FDB_ERR_INVALID, "device %d out of range (%d devices)", d, count);
  *dev = d;
  return FDB_OK;
}

template <typename F> static fdb_status dispatch_ct(int bits, F &&fn) {
  if (bits == 8) return fn((uint8_t)0);
  if (bits == 16) return fn((uint16_t)0);
  return fn((int32_t)0);
}

// the per-column colour source of a plan whose table has type CT: the cyclic closed form when it holds, else the table
template <typename CT, typename F> static fdb_status dispatch_colors(const fdb_plan *P, F &&fn) {
  if (P->colors.cyclic) return fn(CyclicColors{make_fastdiv((uint32_t)P->colors.C)});
  return fn(TableColors<CT>{(const CT *)P->colors.jcolor});
}

// fn(tag) with the compile-time difference mode (kForward / kCentral / kComplex) of a plan's fdtype as decltype(tag)::value
template <typename F> static fdb_status dispatch_mode(int fdtype, F &&fn) {
  if (fdtype == FDB_CENTRAL) return fn(std::integral_constant<int, kCentral>{});
  if (fdtype == FDB_COMPLEX) return fn(std::integral_constant<int, kComplex>{});
  return fn(std::integral_constant<int, kForward>{});
}

// ------------------------------------------------------------------------------------------------ which calls a plan takes
// The compute and query calls whose acceptance depends on the plan.  fdb_jacobian_host is checked as fdb_jacobian,
// fdb_jvp_oop as fdb_jvp; a group call checks the group's member 0.
enum class Call {
  jacobian, jacobian_complex, jacobian_oop, jacobian_oop_complex, color_eps, set_external_eps, set_peers, color_owner,
  get_eps, jvp, hessian, derivative, derivative_complex, group_jacobian, group_jacobian_oop, group_hessian
};

// FDB_OK when plan P takes call c, else the refusal (its status and fdb_last_error() text): the one statement of the
// rule, listed per call in include/fdjac_b200.h.  The first refusal that applies is returned.  Every entry point checks
// before it allocates, launches or calls f.
static fdb_status check_call(const fdb_plan *P, Call c) {
  using K = Call;
  const int k = P->sp_kind;
  const bool cplx = P->fdtype == FDB_COMPLEX;
  const bool colored = k == SP_CSC || k == SP_COO || k == SP_BANDED || k == SP_BLOCKBAND || k == SP_CSR;   // coloured Jacobian plans
  const bool jac = c == K::jacobian || c == K::jacobian_complex, oop = c == K::jacobian_oop || c == K::jacobian_oop_complex;
  const bool group = c == K::group_jacobian || c == K::group_jacobian_oop;
  const fdb_status INV = FDB_ERR_INVALID;
  if (c == K::jacobian_complex && !cplx) return fail(INV, "fdb_jacobian_complex needs a plan created with fdtype = FDB_COMPLEX");
  if (jac && k == SP_JVP) return fail(INV, "this is a JVP plan: call fdb_jvp");
  if (jac && k == SP_EPS) return fail(INV, "this is a step-size plan: call fdb_color_eps");
  if (jac && k == SP_HESS) return fail(INV, "this is a Hessian plan: call fdb_hessian");
  if (jac && k == SP_DERIV) return fail(INV, "this is a derivative plan: call fdb_derivative");
  if (jac && P->oop.on) return fail(INV, "this is an out-of-place plan: call fdb_jacobian_oop");
  if (c == K::jacobian && cplx)
    return fail(INV, "this plan is a complex-step plan: call fdb_jacobian_complex with a complex128 callback");
  if (c == K::jacobian_oop && cplx)
    return fail(INV, "this plan is a complex-step plan: call fdb_jacobian_oop_complex with a complex128 callback");
  if (c == K::jacobian_oop_complex && !cplx)
    return fail(INV, "fdb_jacobian_oop_complex needs a plan created with fdtype = FDB_COMPLEX");
  if (oop && !P->oop.on) return fail(INV, "not an out-of-place plan (fdb_oop_plan_create_csc / _dense)");
  if (c == K::color_eps && !colored && k != SP_EPS) return fail(INV, "fdb_color_eps needs a coloured plan");
  if (c == K::set_external_eps && !colored) return fail(INV, "external step sizes apply to coloured Jacobian plans");
  if (c == K::set_peers && k != SP_CSC && k != SP_COO && k != SP_JVP && k != SP_EPS)
    return fail(FDB_ERR_UNSUPPORTED, "peer stores are implemented for the entry-driven (CSC / COO) scatters");
  if (c == K::color_owner && (k == SP_NONE || k == SP_HESS)) return fail(INV, "dense plans partition columns by range");
  if (c == K::color_owner && k == SP_DERIV) return fail(INV, "derivative plans have no colours");
  if (c == K::get_eps && k == SP_DERIV)
    return fail(INV, "derivative plans keep no step sizes (the quotient pass recomputes them)");
  if (c == K::jvp && k != SP_JVP) return fail(INV, "not a JVP plan (fdb_jvp_plan_create)");
  if (c == K::hessian && k != SP_HESS) return fail(INV, "not a Hessian plan (fdb_hessian_plan_create)");
  if (c == K::derivative && k != SP_DERIV)
    return fail(INV, "not a derivative plan (fdb_derivative_plan_create / fdb_scalar_gradient_plan_create)");
  if (c == K::derivative && cplx)
    return fail(INV, "this plan is a complex-step plan: call fdb_derivative_complex with a complex128 callback");
  if (c == K::derivative_complex && (k != SP_DERIV || !cplx))
    return fail(INV, "fdb_derivative_complex needs a derivative plan created with fdtype = FDB_COMPLEX");
  if (c == K::group_jacobian && k == SP_HESS) return fail(INV, "this is a Hessian group: call fdb_group_hessian");
  if (c == K::group_jacobian && P->oop.on) return fail(INV, "this is an out-of-place group: call fdb_group_jacobian_oop");
  if (c == K::group_jacobian_oop && !P->oop.on) return fail(INV, "not an out-of-place group (fdb_group_create_oop_csc / _dense)");
  if (group && cplx) return fail(FDB_ERR_UNSUPPORTED, "groups run forward / central plans");
  if (c == K::group_hessian && k != SP_HESS) return fail(INV, "not a Hessian group (fdb_group_create_hessian)");
  return FDB_OK;
}

static const char *plan_err_text(uint32_t e) {
  if (e & kErrColptr) return "colptr is not a valid CSC column pointer (must start at 1, be non-decreasing, end at nnz+1)";
  if (e & kErrRowRange) return "row index outside 1..m";
  if (e & kErrColRange) return "column index outside 1..n";
  if (e & kErrSlotRange) return "slot outside 1..j_len";
  if (e & kErrMissingInJ) return "a sparsity entry is absent from J's CSC pattern (the reference would insert a new stored entry; unsupported)";
  return "invalid pattern";
}

// maximum and minimum of a device colour vector of length n > 0 (order-free: the grid cannot change them)
static fdb_status color_range(const int64_t *d_colorvec, int64_t n, long long *mx, long long *mn) {
  DevBuf<long long> d_mm;
  TRY(d_mm.alloc(2));
  const long long init[2] = {LLONG_MIN, LLONG_MAX};
  CU(cudaMemcpy(d_mm.get(), init, sizeof init, cudaMemcpyHostToDevice));
  const int blocks = (int)std::min<int64_t>((n + kThreads - 1) / kThreads, 132 * 8);
  color_minmax<<<blocks, kThreads>>>(d_colorvec, n, d_mm.get(), d_mm.get() + 1);
  long long out[2];
  TRY(read_back(out, d_mm.get(), 2, "colour min/max failed"));
  *mx = out[0];
  *mn = out[1];
  return FDB_OK;
}

// colours: max/min, narrow type, per-column colour array
static fdb_status setup_colors(fdb_plan *P, const int64_t *colorvec /*host or device or null*/) {
  const int64_t n = P->n;
  I64View cv;
  TRY(view_i64(colorvec, n, cv));
  long long mx = n, mn = n > 0 ? 1 : 0;
  if (cv.d && n > 0) TRY(color_range(cv.d, n, &mx, &mn));
  if (n == 0) mx = 0;
  if (mx < 0) mx = 0;                       // maximum(colorvec) < 1: the colour loop 1:max is empty
  if (mx > 0x7FFFFFF0LL) return fail(FDB_ERR_UNSUPPORTED, "maximum(colorvec) = %lld exceeds 2^31", mx);
  P->colors.C = (int32_t)mx;
  P->colors.has_invalid = n > 0 && mn < 1;
  P->colors.bits = mx <= 255 ? 8 : (mx <= 65535 ? 16 : 32);
  TRY(P->alloc(&P->colors.jcolor, (size_t)std::max<int64_t>(n, 1) * (P->colors.bits / 8)));
  if (n > 0) {
    DevBuf<uint32_t> d_flags;   // [0] lane conflicts (window path), [1] not cyclic
    const bool window_path = P->colors.C > kEpsRegColors;
    TRY(d_flags.alloc(2));
    CU(cudaMemset(d_flags.get(), 0, 2 * sizeof(uint32_t)));
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      convert_colors<CT><<<P->grid(n), kThreads>>>(cv.d, n, (CT *)P->colors.jcolor);
      if (window_path) color_lane_conflicts<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, n, P->colors.C, d_flags.get());
      if (P->colors.C > 0) check_cyclic<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, n, P->colors.C, d_flags.get() + 1);
      CU(cudaGetLastError());
      return FDB_OK;
    }));
    uint32_t flags[2] = {0, 0};
    TRY(read_back(flags, d_flags.get(), 2, "colour flags"));
    P->colors.cyclic = P->colors.C > 0 && flags[1] == 0;
    if (window_path) {
      P->steps.group = 1;
      for (int lg = 1; lg <= 5 && !(flags[0] & (1u << lg)); ++lg) P->steps.group = 1 << lg;
    }
  }
  return FDB_OK;
}

// step-size buffers of a coloured plan: eps / sumsq per colour, block partials of the one-pass reduction
static fdb_status alloc_eps_buffers(fdb_plan *P) {
  const int32_t C = P->colors.C;
  TRY(P->alloc_t(&P->steps.eps, std::max<int32_t>(C, 1)));
  TRY(P->alloc_t(&P->steps.sumsq, std::max<int32_t>(C, 1)));
  {
    int64_t nb = (P->n + 2047) / 2048;
    // window path: 64 bytes of shared memory per window colour and block (<= 32 KB) -> one resident wave
    nb = std::max<int64_t>(1, std::min<int64_t>(nb, (int64_t)P->sm_count * (C <= 256 ? 8 : 6)));
    P->steps.blocks = (int)nb;
    int64_t chunk = (P->n + nb - 1) / nb;
    P->steps.chunk = (std::max<int64_t>(chunk, 1) + 31) & ~(int64_t)31;   // aligned 32-column steps on the window path
    const int64_t stride = C <= kEpsRegColors ? kEpsRegColors : std::min<int64_t>(C, kEpsWindow);
    TRY(P->alloc_t(&P->steps.partial, (size_t)nb * stride));
    TRY(P->alloc_t(&P->steps.ticket, 4));
    CU(cudaMemset(P->steps.ticket, 0, 16));
  }

  return FDB_OK;
}

// colour ownership (multi-GPU), local colour list, scratch sizing
static fdb_status finish_colored_plan(fdb_plan *P, const fdb_plan_opts *o, const std::vector<unsigned long long> &count) {
  const int32_t C = P->colors.C;
  P->colors.owner.assign(C, 0);
  const int world = P->world;
  if (world > 1) {
    if (o && o->partition == 1) {
      // LPT: heaviest colour first onto the least-loaded rank (ties -> lowest rank), deterministic on every rank
      std::vector<int32_t> order(C);
      std::iota(order.begin(), order.end(), 0);
      std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return count[a] > count[b]; });
      std::vector<unsigned long long> load(world, 0);
      for (int32_t k : order) {
        int best = 0;
        for (int r = 1; r < world; ++r) if (load[r] < load[best]) best = r;
        P->colors.owner[k] = best;
        load[best] += count[k] + 1;
      }
    } else {
      for (int32_t k = 0; k < C; ++k) P->colors.owner[k] = k % world;
    }
  }
  std::vector<int32_t> local_of(C, -1);
  P->colors.local.clear();
  for (int32_t k = 0; k < C; ++k)
    if (P->colors.owner[k] == P->rank) { local_of[k] = (int32_t)P->colors.local.size(); P->colors.local.push_back(k); }
  const int64_t n_local = (int64_t)P->colors.local.size();
  TRY(P->alloc_t(&P->colors.local_of, std::max<int32_t>(C, 1)));
  TRY(P->alloc_t(&P->colors.d_local, std::max<int64_t>(n_local, 1)));
  if (C > 0) CU(cudaMemcpy(P->colors.local_of, local_of.data(), (size_t)C * 4, cudaMemcpyHostToDevice));
  if (n_local > 0) CU(cudaMemcpy(P->colors.d_local, P->colors.local.data(), (size_t)n_local * 4, cudaMemcpyHostToDevice));

  TRY(alloc_eps_buffers(P));

  // scratch: stacked f! outputs (slabs) + perturbed points
  const bool central = P->fdtype == FDB_CENTRAL;
  const int64_t cw = P->fdtype == FDB_COMPLEX ? 2 : 1;     // doubles per element of the f! in/outputs
  P->scratch.ldF = (P->m + 1) & ~(int64_t)1;
  P->scratch.ldx = (P->n + 1) & ~(int64_t)1;
  if (P->scratch.ldF < 2) P->scratch.ldF = 2;
  if (P->scratch.ldx < 2) P->scratch.ldx = 2;
  int64_t budget = (o && o->scratch_bytes > 0) ? o->scratch_bytes : (int64_t)8 << 30;
  const int64_t per_slab = 8 * cw * P->scratch.ldF * (central ? 2 : 1);
  int64_t slabs = std::max<int64_t>(1, budget / per_slab);
  slabs = std::min<int64_t>(slabs, std::max<int64_t>(n_local, 1));
  if (P->sp_kind == SP_CSC && P->entries.strategy == 0 && P->entries.strategy_auto && slabs < n_local) P->entries.strategy = 1;
  if (P->entries.strategy == 1 && !P->entries.lists_resident) {
    // per-colour lists: keep only as many f! outputs in flight as stay L2-resident until their scatter (~40 % of the L2:
    // 20 MB of an H100's 50 MB, the rest is left to f(x) and the index streams)
    const int64_t l2_slabs = std::max<int64_t>(1, P->l2_bytes * 2 / 5 / per_slab);
    slabs = std::min<int64_t>(slabs, l2_slabs);
  }
  if (P->entries.strategy == 1) slabs = std::min<int64_t>(slabs, kCmMaxGroup);
  P->scratch.slabs = slabs;
  P->scratch.n_groups = n_local == 0 ? 0 : (n_local + slabs - 1) / slabs;
  int64_t batch = (o && o->max_batch > 1) ? o->max_batch : 1;
  batch = std::min<int64_t>(batch, slabs);
  P->scratch.batch = batch;
  // even when f! takes one point per call, build up to kPerturbMaxPoints points per pass over x (one read of x and
  // the colour stream instead of one per colour) when the point buffers fit in an eighth of the scratch budget
  int64_t pbatch = std::max<int64_t>(batch, std::min<int64_t>(kPerturbMaxPoints, std::max<int64_t>(n_local, 1)));
  while (pbatch > batch && pbatch * 8 * cw * P->scratch.ldx * (central ? 2 : 1) > budget / 8) --pbatch;
  P->scratch.pbatch = pbatch;
  // two output buffers + a side stream: a group's scatter (and its NVLink stores, when peers are set) overlaps the next
  // group's f! evaluations
  // Off by default: the scatter and the next f! compete for the same L2 / DRAM, and the NVLink stores of a 5 MB colour
  // need no hiding.  FDB_FORCE_OVERLAP=1 switches the double-buffered side-stream form back on.
  P->overlap.double_buffer = false;
  if (P->tune.force_overlap && P->sp_kind == SP_CSC && P->entries.strategy == 1 && (int64_t)P->colors.local.size() > slabs) P->overlap.double_buffer = true;
  const size_t nbuf = P->overlap.double_buffer ? 2 : 1;
  CU(cudaStreamCreateWithFlags(&P->overlap.side, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&P->overlap.ev_fork, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&P->overlap.ev_eps, cudaEventDisableTiming));
  if (P->overlap.double_buffer) {
    for (int b = 0; b < 2; ++b) {
      CU(cudaEventCreateWithFlags(&P->overlap.ev_f[b], cudaEventDisableTiming));
      CU(cudaEventCreateWithFlags(&P->overlap.ev_scat[b], cudaEventDisableTiming));
    }
  }
  TRY(P->alloc_t(&P->scratch.fx_own, (size_t)P->scratch.ldF));
  TRY(P->alloc_t(&P->scratch.Fp, nbuf * (size_t)slabs * P->scratch.ldF * cw));
  TRY(P->alloc_t(&P->scratch.xp, (size_t)pbatch * P->scratch.ldx * cw));
  if (central) {
    TRY(P->alloc_t(&P->scratch.Fm, nbuf * (size_t)slabs * P->scratch.ldF));
    TRY(P->alloc_t(&P->scratch.xm, (size_t)pbatch * P->scratch.ldx));
  }
  return FDB_OK;
}

// Per-colour column lists: bucket_start ([C+2] offsets into cols_by_color; bucket C = columns without a valid colour),
// cols_by_color (the column ids stable-sorted by colour: ascending inside a colour) and, for more colours than the
// register path takes, the chunk tables of the list-based eps pass.
static fdb_status build_color_lists(fdb_plan *P) {
  const int64_t n = P->n;
  const int32_t C = P->colors.C;
  TRY(P->alloc_t(&P->colors.cols_by_color, (size_t)std::max<int64_t>(n, 1)));
  std::vector<unsigned long long> bc((size_t)C + 1, 0);
  if (n > 0) {
    // a stable radix sort of the column ids by colour (deterministic: the list-based eps pass sums in list order, and
    // sharded and unsharded plans must produce the same bits)
    DevBuf<unsigned long long> d_bucket;
    DevBuf<uint32_t> k_in, k_out;
    DevBuf<int32_t> v_in;
    TRY(d_bucket.alloc((size_t)C + 1));
    CU(cudaMemset(d_bucket.get(), 0, ((size_t)C + 1) * 8));
    TRY(k_in.alloc((size_t)n));
    TRY(k_out.alloc((size_t)n));
    TRY(v_in.alloc((size_t)n));
    dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      count_color_buckets<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, n, C, d_bucket.get());
      color_sort_keys<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, n, C, k_in.get(), v_in.get());
      return FDB_OK;
    });
    int end_bit = 1;
    while (end_bit < 32 && ((uint64_t)1 << end_bit) <= (uint64_t)C) ++end_bit;
    TRY(cub_run([&](void *tmp, size_t &bytes) {
      return cub::DeviceRadixSort::SortPairs(tmp, bytes, k_in.get(), k_out.get(), v_in.get(), P->colors.cols_by_color, (int)n, 0, end_bit);
    }));
    TRY(read_back(bc.data(), d_bucket.get(), (size_t)C + 1, "column lists"));
  }
  P->colors.bucket_start.assign((size_t)C + 2, 0);
  for (int32_t k = 0; k <= C; ++k) P->colors.bucket_start[(size_t)k + 1] = P->colors.bucket_start[(size_t)k] + (int64_t)bc[(size_t)k];
  // step sizes from the column lists (more colours than the register path takes)
  if (C > kEpsRegColors && C <= (1 << 22) && n > 0) {
    std::vector<int64_t> cb((size_t)C + 1, 0);
    int64_t maxc = 1;
    for (int32_t k = 0; k < C; ++k) {
      const int64_t len = P->colors.bucket_start[(size_t)k + 1] - P->colors.bucket_start[(size_t)k];
      const int64_t nc = (len + kEpsListChunk - 1) / kEpsListChunk;
      cb[(size_t)k + 1] = cb[(size_t)k] + nc;
      maxc = std::max(maxc, nc);
    }
    TRY(P->alloc_t(&P->steps.bucket_start_d, (size_t)C + 2));
    TRY(P->alloc_t(&P->steps.chunk_base_d, (size_t)C + 1));
    TRY(P->alloc_t(&P->steps.list_partial, (size_t)std::max<int64_t>(cb[(size_t)C], 1)));
    CU(cudaMemcpy(P->steps.bucket_start_d, P->colors.bucket_start.data(), ((size_t)C + 2) * 8, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(P->steps.chunk_base_d, cb.data(), ((size_t)C + 1) * 8, cudaMemcpyHostToDevice));
    P->steps.list_max_chunks = maxc;
    P->steps.lists = true;
  }
  return FDB_OK;
}

// gather kernel for build_cm_lists: block b copies the column bucket of local colour (or of the invalid bucket) b
__global__ void __launch_bounds__(kThreads)
cm_gather_cols(const int32_t *__restrict__ cols_by_color, const int64_t *__restrict__ src_start /* [nseg] */,
               const int64_t *__restrict__ dst_start /* [nseg+1] */, int64_t nseg, int32_t *__restrict__ list_cols) {
  for (int64_t sgm = blockIdx.x; sgm < nseg; sgm += gridDim.x) {
    const int64_t s0 = src_start[sgm], d0 = dst_start[sgm], cnt = dst_start[sgm + 1] - d0;
    for (int64_t i = threadIdx.x; i < cnt; i += kThreads) list_cols[d0 + i] = cols_by_color[s0 + i];
  }
}

// Colour-major entry lists of the colours this rank evaluates (CSC plans, strategy 1): see kernels_scatter.cuh.
static fdb_status build_cm_lists(fdb_plan *P, const std::vector<unsigned long long> &count /* entries per colour */) {
  const int64_t n_local = (int64_t)P->colors.local.size();
  const int32_t C = P->colors.C;
  const bool zero_bucket = P->rank == 0 && P->colors.bucket_start[(size_t)C + 1] > P->colors.bucket_start[(size_t)C];
  const int64_t nseg = n_local + (zero_bucket ? 1 : 0);
  std::vector<int64_t> src(std::max<int64_t>(nseg, 1), 0), dst((size_t)nseg + 1, 0);
  P->cm.start_h.assign((size_t)n_local + 1, 0);
  unsigned long long valid_total = 0;
  for (int32_t k = 0; k < C; ++k) valid_total += count[(size_t)k];
  for (int64_t li = 0; li < n_local; ++li) {
    const int32_t k = P->colors.local[(size_t)li];
    src[(size_t)li] = P->colors.bucket_start[(size_t)k];
    dst[(size_t)li + 1] = dst[(size_t)li] + (P->colors.bucket_start[(size_t)k + 1] - P->colors.bucket_start[(size_t)k]);
    P->cm.start_h[(size_t)li + 1] = P->cm.start_h[(size_t)li] + (int64_t)count[(size_t)k];
  }
  int64_t e_local = P->cm.start_h[(size_t)n_local];
  P->cm.invalid_end = e_local;
  if (zero_bucket) {
    src[(size_t)n_local] = P->colors.bucket_start[(size_t)C];
    dst[(size_t)n_local + 1] = dst[(size_t)n_local] + (P->colors.bucket_start[(size_t)C + 1] - P->colors.bucket_start[(size_t)C]);
    e_local += P->colors.E - (int64_t)valid_total;
    P->cm.invalid_end = e_local;
  }
  const int64_t ncols = dst[(size_t)nseg];
  TRY(P->alloc_t(&P->cm.start, (size_t)n_local + 1));
  CU(cudaMemcpy(P->cm.start, P->cm.start_h.data(), ((size_t)n_local + 1) * 8, cudaMemcpyHostToDevice));
  TRY(P->alloc_t(&P->cm.row, (size_t)std::max<int64_t>(e_local, 1)));
  {
    // only where f(x) would otherwise be dragged through DRAM once per launch: several launches per Jacobian (colours
    // sharded over GPUs, or more colours than resident slabs).  One launch over all colours reads f(x) once anyway: not
    // used there (it would cost E_local * 8 bytes more for no gain).
    const bool want = P->scratch.n_groups > 1 || P->tune.force_fx_cm;
    if (P->fdtype == FDB_FORWARD && e_local > 0 && want && !P->tune.no_fx_cm) TRY(P->alloc_t(&P->cm.fx, (size_t)e_local));
  }
  const bool wide = P->entries.dest != nullptr;
  TRY(P->alloc(&P->cm.slot, (size_t)std::max<int64_t>(e_local, 1) * (wide ? 8 : 4)));
  if (ncols == 0 || e_local == 0) return FDB_OK;
  // temporaries: segment offsets, column list, counts, offsets
  DevBuf<int64_t> d_src, d_dst;
  DevBuf<int32_t> list_cols, list_cnt, list_off;
  TRY(d_src.alloc((size_t)nseg));
  TRY(d_dst.alloc((size_t)nseg + 1));
  TRY(list_cols.alloc((size_t)ncols));
  TRY(list_cnt.alloc((size_t)ncols));
  TRY(list_off.alloc((size_t)ncols));
  CU(cudaMemcpy(d_src.get(), src.data(), (size_t)nseg * 8, cudaMemcpyHostToDevice));
  CU(cudaMemcpy(d_dst.get(), dst.data(), ((size_t)nseg + 1) * 8, cudaMemcpyHostToDevice));
  cm_gather_cols<<<(int)std::min<int64_t>(nseg, (int64_t)P->sm_count * 16), kThreads>>>(P->colors.cols_by_color, d_src.get(), d_dst.get(), nseg, list_cols.get());
  cm_column_counts<<<P->grid(ncols), kThreads>>>(list_cols.get(), ncols, P->entries.colptr32, list_cnt.get());
  TRY(cub_run([&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, list_cnt.get(), list_off.get(), (int)ncols);
  }));
  {
    const int lanes = P->entries.lanes;
    const int64_t blocks = (ncols + (kThreads / lanes) - 1) / (kThreads / lanes);
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>(blocks, (int64_t)P->sm_count * 16));
    if (wide) cm_expand<int64_t><<<grid, kThreads>>>(list_cols.get(), list_off.get(), ncols, P->entries.colptr32, P->entries.row32, P->entries.dest, lanes, P->cm.row, (int64_t *)P->cm.slot);
    else cm_expand<int32_t><<<grid, kThreads>>>(list_cols.get(), list_off.get(), ncols, P->entries.colptr32, P->entries.row32, nullptr, lanes, P->cm.row, (int32_t *)P->cm.slot);
  }
  // consistency: the last column's end must be the entry total the per-colour counts promised
  int32_t last_off = 0, last_cnt = 0;
  TRY(read_back(&last_off, list_off.get() + (ncols - 1), 1, "colour-major list offsets"));
  TRY(read_back(&last_cnt, list_cnt.get() + (ncols - 1), 1, "colour-major list counts"));
  CU(cudaDeviceSynchronize());
  if ((int64_t)last_off + last_cnt != e_local)
    return fail(FDB_ERR_INVALID, "internal: colour-major list holds %lld entries, expected %lld", (long long)last_off + last_cnt,
                (long long)e_local);
  return FDB_OK;
}

// Band form of the staged pass: the pattern is exactly the clipped band of some (l, u) — column c holds the rows
// max(0, c-l) .. min(m-1, c+u), in order — so every entry's row and column follow from its position.
static fdb_status try_band_form(fdb_plan *P) {
  P->staged.band = false;
  const int64_t m = P->m, n = P->n;
  DevBuf<int> d_lu;
  DevBuf<uint32_t> d_flag;
  TRY(d_lu.alloc(2));
  TRY(d_flag.alloc(1));
  const int init[2] = {INT_MIN, INT_MIN};
  CU(cudaMemcpy(d_lu.get(), init, sizeof init, cudaMemcpyHostToDevice));
  CU(cudaMemset(d_flag.get(), 0, 4));
  band_extent<<<P->grid(n), kThreads>>>(P->entries.colptr32, P->entries.row32, n, d_lu.get());
  int lu[2];
  TRY(read_back(lu, d_lu.get(), 2, "band extent"));
  const int l = lu[0], u = lu[1];
  band_check<<<P->grid(n), kThreads>>>(P->entries.colptr32, P->entries.row32, m, n, l, u, d_flag.get());
  uint32_t bad = 1;
  TRY(read_back(&bad, d_flag.get(), 1, "band check"));
  if (bad) return FDB_OK;
  // interior columns [a, b): c - l >= 0 and c + u <= m - 1 — every one holds all w = l + u + 1 rows
  const int64_t a = std::min<int64_t>(std::max(l, 0), n), b = std::max<int64_t>(a, std::min<int64_t>(n, m - u));
  int32_t ea = 0, eb = 0;
  TRY(read_back(&ea, P->entries.colptr32 + a, 1, "band column pointer"));
  TRY(read_back(&eb, P->entries.colptr32 + b, 1, "band column pointer"));
  P->staged.band_l = l;
  P->staged.band_w = l + u + 1;
  P->staged.band_col_a = (int32_t)a;
  P->staged.band_col_b = (int32_t)b;
  P->staged.band_e_a = ea;
  P->staged.band_e_b = eb;
  P->staged.band = true;
  return FDB_OK;
}

// TMA-staged fused pass: eligible when the whole Jacobian is one resident group on one rank, the destination is the
// identity (CSC nzval) and every 1024-entry tile touches a short row window (row-local pattern).
static fdb_status try_stage_plan(fdb_plan *P) {
  P->staged.on = false;
  if (P->tune.no_staged) return FDB_OK;
  if (P->sp_kind != SP_CSC || P->entries.dest != nullptr || P->entries.strategy != 0 || P->world != 1 || P->scratch.n_groups != 1) return FDB_OK;
  if (P->fdtype == FDB_COMPLEX || P->colors.C < 1) return FDB_OK;
  const int nwin = P->fdtype == FDB_CENTRAL ? 2 * P->colors.C : P->colors.C + 1;
  const int64_t ntiles = P->colors.E / kTile;
  if (nwin > kStageMaxWin || ntiles < 1) return FDB_OK;
  // built here, kept by the plan only when the staged form is chosen
  DevBuf<unsigned int> d_span;
  DevBuf<int32_t> tile_w0;
  DevBuf<uint16_t> row16;
  TRY(d_span.alloc(1));
  CU(cudaMemset(d_span.get(), 0, 4));
  TRY(tile_w0.alloc((size_t)ntiles));
  TRY(row16.alloc((size_t)ntiles * kTile));
  const int pgrid = (int)std::min<int64_t>(ntiles, (int64_t)P->sm_count * 16);
  stage_prepare<uint8_t><<<pgrid, kThreads>>>(P->entries.row32, ntiles, tile_w0.get(), row16.get(), d_span.get(), nullptr, P->colors.C);
  unsigned int span = 0;
  TRY(read_back(&span, d_span.get(), 1, "staged row span"));
  const int64_t W = ((int64_t)span + 1) & ~(int64_t)1;
  // few colours, short windows: pack the entry's colour into the top 4 bits of its row offset (no colour stream at all)
  P->staged.packed = P->colors.C <= 14 && W <= 4096 && span > 0 && !P->tune.no_pack;
  if (P->staged.packed) {
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      stage_prepare<CT><<<pgrid, kThreads>>>(P->entries.row32, ntiles, tile_w0.get(), row16.get(), d_span.get(), (const CT *)P->entries.ecolor, P->colors.C);
      CU(cudaGetLastError());
      return FDB_OK;
    }));
    CU(cudaDeviceSynchronize());
  }
  const size_t smem = (size_t)2 * nwin * W * 8 + kStageCtlBytes + (size_t)P->colors.C * 8;
  if (span == 0 || span > 65535 || smem > (size_t)kStageMaxSmem) return FDB_OK;   // not row-local enough: keep the gather form
  P->adopt(P->staged.tile_w0 = tile_w0.release(), tile_w0.bytes);
  P->adopt(P->staged.row16 = row16.release(), row16.bytes);
  TRY(P->alloc_t(&P->staged.claim, 1));
  CU(cudaMemset(P->staged.claim, 0, sizeof(unsigned long long)));
  P->staged.W = (int32_t)W;
  P->staged.on = true;
  if (!P->tune.no_band) TRY(try_band_form(P));
  return FDB_OK;
}

static fdb_status read_plan_err(uint32_t *d_err, const char *what) {
  uint32_t h = 0;
  TRY(read_back(&h, d_err, 1, what));
  const uint32_t hard = h & ~(uint32_t)(kErrPatternDiff | kErrRowOrder);
  if (hard == kErrMissingInJ) return fail(FDB_ERR_UNSUPPORTED, "%s: %s", what, plan_err_text(hard));
  if (hard) return fail(FDB_ERR_INVALID, "%s: %s", what, plan_err_text(hard));
  return FDB_OK;
}

static bool env_is(const char *name, char c) {
  const char *v = getenv(name);
  return v && v[0] == c;
}

// Every default below is what an A/B on C2 / C4 chose; the switches exist to repeat such an A/B (DESIGN.md §4).
static void read_tunables(fdb_plan *P) {
  auto &t = P->tune;
  t.no_staged = env_is("FDB_NO_STAGED", '1');
  t.no_eps_lists = env_is("FDB_NO_EPS_LISTS", '1');
  t.no_eps_overlap = env_is("FDB_NO_EPS_OVERLAP", '1');
  t.cm_prefetch = env_is("FDB_CM_PREFETCH", '1');
  t.force_overlap = env_is("FDB_FORCE_OVERLAP", '1');
  t.no_fx_cm = env_is("FDB_NO_FX_CM", '1');
  t.force_fx_cm = env_is("FDB_FORCE_FX_CM", '1');
  t.no_pack = env_is("FDB_NO_PACK", '1');
  t.no_band = env_is("FDB_NO_BAND", '1');
  if (const char *hs = getenv("FDB_HI_STREAM")) t.hi_stream = hs[0] == '1' ? 1 : 0;
  if (const char *v = getenv("FDB_REVERSE")) { if (v[0] >= '0' && v[0] <= '3') t.reverse = v[0] - '0'; }
  if (env_is("FDB_CM_HINT", '0')) t.cm_slab_stream = 0;
  if (env_is("FDB_STAGES", '3')) t.stages = 3;
  if (env_is("FDB_EPS_DEPTH", '1')) t.eps_depth = 1;
  if (env_is("FDB_COLS_DEPTH", '4')) t.cols_depth = 4;
  if (env_is("FDB_COLS_DEPTH", '2')) t.cols_depth = 2;
  if (env_is("FDB_COLS_DEPTH", '1')) t.cols_depth = 1;
  if (const char *v = getenv("FDB_COLS_GX")) { const int g = atoi(v); if (g >= 1 && g <= 4096) t.cols_gx = g; }
  if (const char *v = getenv("FDB_STAGED_VARIANT")) {
    if (v[0]) { t.staged_variant[0] = v[0]; t.staged_variant[1] = v[1] ? v[1] : 'n'; }
  }
}

static void free_plan(fdb_plan *P) {
  if (!P) return;
  DeviceGuard g(P->device);
  for (void *p : P->allocs) cudaFree(p);   // the device buffers of every part
  for (auto &ev : P->timing.pending) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
  for (auto &ev : P->timing.pool) { cudaEventDestroy(ev.first); cudaEventDestroy(ev.second); }
  if (P->host.stream) cudaStreamDestroy(P->host.stream);
  const auto &o = P->overlap;
  if (o.side) cudaStreamDestroy(o.side);
  for (int b = 0; b < 2; ++b) { if (o.ev_f[b]) cudaEventDestroy(o.ev_f[b]); if (o.ev_scat[b]) cudaEventDestroy(o.ev_scat[b]); }
  if (o.ev_fork) cudaEventDestroy(o.ev_fork);
  if (o.ev_eps) cudaEventDestroy(o.ev_eps);
  if (P->graph.exec) cudaGraphExecDestroy(P->graph.exec);
  if (P->graph.stream) cudaStreamDestroy(P->graph.stream);
  delete P;
}

struct PlanFree { void operator()(fdb_plan *P) const { free_plan(P); } };
// a plan under construction: freed on every failure path, handed to the caller by release() once it is complete
using PlanPtr = std::unique_ptr<fdb_plan, PlanFree>;

static fdb_status new_plan(fdb_plan **out, PlanPtr &P, const fdb_plan_opts *o, int64_t m, int64_t n) {
  if (!out) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *out = nullptr;
  if (m < 0 || n < 0) return fail(FDB_ERR_INVALID, "negative dimensions m=%lld n=%lld", (long long)m, (long long)n);
  if (m > 0x7FFFFFF0LL || n > 0x7FFFFFF0LL) return fail(FDB_ERR_UNSUPPORTED, "m, n must be < 2^31");
  if (o && o->fdtype != FDB_FORWARD && o->fdtype != FDB_CENTRAL && o->fdtype != FDB_COMPLEX)
    return fail(FDB_ERR_UNSUPPORTED, "Unrecognized fdtype: valid values are forward (0), central (1) and complex (2)");
  int dev = 0;
  TRY(check_device(o, &dev));
  P.reset(new (std::nothrow) fdb_plan());
  if (!P) return fail(FDB_ERR_NOMEM, "out of host memory");
  P->device = dev;
  P->m = m;
  P->n = n;
  P->fdtype = o ? o->fdtype : FDB_FORWARD;
  P->no_drift = o ? o->no_drift : 0;
  P->graph.use = o && o->use_graph != 0;
  P->shared_J = o && o->shared_j != 0;
  read_tunables(P.get());
  P->world = (o && o->world > 1) ? o->world : 1;
  P->rank = (o && o->world > 1) ? o->rank : 0;
  if (P->rank < 0 || P->rank >= P->world) return fail(FDB_ERR_INVALID, "rank %d outside world %d", P->rank, P->world);
  cudaDeviceProp prop;
  cudaError_t e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) return fail(FDB_ERR_CUDA, "cudaGetDeviceProperties: %s", cudaGetErrorString(e));
  P->sm_count = prop.multiProcessorCount;
  // FDB_SM_COUNT=k (tests): size every grid as if the device had k SMs, so small problems already give each block several
  // tiles.  Launch geometry only: no plan decision reads sm_count.
  if (const char *v = getenv("FDB_SM_COUNT")) {
    const int k = atoi(v);
    if (k >= 1 && k < P->sm_count) P->sm_count = k;
  }
  P->l2_bytes = prop.l2CacheSize;
  return FDB_OK;
}

// the end of a creator that launched plan-build kernels: wait for them, then hand the plan to the caller
static fdb_status finish_plan(PlanPtr &P, fdb_plan **plan) {
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(FDB_ERR_CUDA, "plan build: %s", cudaGetErrorString(e));
  *plan = P.release();
  return FDB_OK;
}

// relstep / absstep keywords of jacobians.jl:508-510: `relstep = default_relstep(fdtype, eltype(x)), absstep = relstep`.
// FDB_STEP_DEFAULT (NaN) means "keyword not given"; every other value — 0 and negatives included — is used as passed
// (relstep = 0 is a pure absolute step, absstep = 0 a pure relative one, exactly as in the reference).
static inline void resolve_steps(int fdtype, double &relstep, double &absstep) {
  if (std::isnan(relstep)) relstep = fdb_default_relstep(fdtype);
  if (std::isnan(absstep)) absstep = relstep;
}

// The block sizes of a block-structured plan (host or device Int64), their 0-based offsets off[nblocks + 1] and their
// sum n: a negative size is FDB_ERR_INVALID, more than 2^31 columns FDB_ERR_UNSUPPORTED
static fdb_status read_block_sizes(int64_t nblocks, const int64_t *blocks, std::vector<int64_t> &hb,
                                   std::vector<int32_t> &off, int64_t &n) {
  hb.assign((size_t)nblocks, 0);
  if (nblocks > 0) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, blocks) != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
    if (at.type == cudaMemoryTypeDevice) CU(cudaMemcpy(hb.data(), blocks, (size_t)nblocks * 8, cudaMemcpyDeviceToHost));
    else std::memcpy(hb.data(), blocks, (size_t)nblocks * 8);
  }
  off.assign((size_t)nblocks + 1, 0);
  n = 0;
  for (int64_t K = 0; K < nblocks; ++K) {
    if (hb[(size_t)K] < 0) return fail(FDB_ERR_INVALID, "block %lld has negative size %lld", (long long)K, (long long)hb[(size_t)K]);
    n += hb[(size_t)K];
    if (n > 0x7FFFFFF0LL) return fail(FDB_ERR_UNSUPPORTED, "the block sizes sum to more than 2^31 columns");
    off[(size_t)K + 1] = (int32_t)n;
  }
  return FDB_OK;
}

// The rest of a block-structured plan once its colours are set up: pass(CT{}, cnt, not_cyclic) launches the kind's plan
// pass, which sums the structural entries per colour (the LPT weights; cnt[C]: columns without a valid colour) and
// clears nothing in *not_cyclic when the colouring is the kind's block-cyclic closed form.  Fills colors.E and
// block_band.cyclic, then the coloured plan's ownership and scratch.
template <typename Pass>
static fdb_status finish_block_plan(fdb_plan *P, const fdb_plan_opts *opts, Pass &&pass) {
  const int64_t n = P->n;
  DevBuf<unsigned long long> d_cnt;
  DevBuf<uint32_t> d_flag;
  TRY(d_cnt.alloc((size_t)P->colors.C + 1));
  TRY(d_flag.alloc(1));
  CU(cudaMemset(d_cnt.get(), 0, ((size_t)P->colors.C + 1) * 8));
  CU(cudaMemset(d_flag.get(), 0, 4));
  if (n > 0) {
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      pass(tag, d_cnt.get(), d_flag.get());
      CU(cudaGetLastError());
      return FDB_OK;
    }));
  }
  std::vector<unsigned long long> cnt((size_t)P->colors.C + 1, 0);
  TRY(read_back(cnt.data(), d_cnt.get(), (size_t)P->colors.C + 1, "block-banded entry counts"));
  uint32_t not_cyclic = 1;
  TRY(read_back(&not_cyclic, d_flag.get(), 1, "block-banded colouring form"));
  P->block_band.cyclic = n > 0 && P->colors.C > 0 && not_cyclic == 0;
  unsigned long long total = 0;
  for (auto c : cnt) total += c;
  P->colors.E = (int64_t)total;
  cnt.resize((size_t)std::max<int32_t>(P->colors.C, 1));
  return finish_colored_plan(P, opts, cnt);
}

// ------------------------------------------------------------------------------------------------ exported: misc
extern "C" {

int fdb_abi_version(void) { return FDB_ABI_VERSION; }
const char *fdb_last_error(void) { return g_err.c_str(); }
int fdb_device_count(void) {
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) { cudaGetLastError(); return 0; }
  return c;
}

// src/epsilons.jl:134-144
double fdb_default_relstep(int fdtype) {
  if (fdtype == FDB_FORWARD) return sqrt(DBL_EPSILON);
  if (fdtype == FDB_CENTRAL) return cbrt(DBL_EPSILON);
  if (fdtype == FDB_HCENTRAL) return ldexp(1.0, -13);   // eps(Float64)^(1/4) = (2^-52)^(1/4), exact
  return 1.0;
}
// src/epsilons.jl:26-29 / :50-53
double fdb_compute_epsilon(int fdtype, double x, double relstep, double absstep, double dir) {
  const double a = relstep * fabs(x);
  const double e = max_julia(a, absstep);
  return fdtype == FDB_FORWARD ? e * dir : e;
}

// ------------------------------------------------------------------------------------------------ plan creation
fdb_status fdb_plan_create_csc(fdb_plan **plan, int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval,
                               int jkind, const int64_t *j_colptr, const int64_t *j_rowval, int64_t ldJ,
                               const int64_t *colorvec, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (!colptr) return fail(FDB_ERR_INVALID, "colptr is NULL");
  if (jkind != FDB_J_CSC_NZVAL && jkind != FDB_J_DENSE)
    return fail(FDB_ERR_INVALID, "CSC sparsity supports J kinds CSC_NZVAL and DENSE");
  P->sp_kind = SP_CSC;
  P->jkind = jkind;
  // nnz = colptr[n]-1 : read the last element wherever it lives
  I64View cp, rv, jcp, jrv;
  TRY(view_i64(colptr, n + 1, cp));
  int64_t last = 1;
  TRY(read_back(&last, cp.d + n, 1, "reading colptr[n]"));
  const int64_t nnz = last - 1;
  if (nnz < 0 || nnz > 0x7FFFFFF0LL) return fail(FDB_ERR_UNSUPPORTED, "nnz=%lld unsupported (must be in [0, 2^31))", (long long)nnz);
  if (nnz > 0 && !rowval) return fail(FDB_ERR_INVALID, "rowval is NULL");
  P->colors.E = nnz;
  TRY(view_i64(rowval, nnz, rv));
  TRY(setup_colors(P, colorvec));

  DevBuf<uint32_t> d_err;
  DevBuf<unsigned long long> d_cnt;
  TRY(d_err.alloc(1));
  TRY(d_cnt.alloc(std::max<int32_t>(P->colors.C, 1)));
  CU(cudaMemset(d_err.get(), 0, 4));
  CU(cudaMemset(d_cnt.get(), 0, (size_t)std::max<int32_t>(P->colors.C, 1) * 8));
  TRY(P->alloc_t(&P->entries.row32, std::max<int64_t>(nnz, 4)));
  TRY(P->alloc(&P->entries.ecolor, (size_t)std::max<int64_t>(nnz, 4) * (P->colors.bits / 8) + 16));

  bool same_pattern = true;
  bool other_csc = false;
  if (jkind == FDB_J_CSC_NZVAL && j_colptr && j_rowval && (j_colptr != colptr || j_rowval != rowval)) {
    // ext/FiniteDiffSparseArraysExt.jl:51-52
    TRY(view_i64(j_colptr, n + 1, jcp));
    int64_t jlast = 1;
    TRY(read_back(&jlast, jcp.d + n, 1, "reading J.colptr[n]"));
    if (jlast < 1 || jlast - 1 > 0x7FFFFFF0LL) return fail(FDB_ERR_INVALID, "J.colptr[n+1]=%lld is not a valid CSC end pointer", (long long)jlast);
    const int64_t jnnz = jlast - 1;
    TRY(view_i64(j_rowval, jnnz, jrv));
    if (jnnz != nnz) same_pattern = false;
    else {
      compare_i64<<<P->grid(n + 1), kThreads>>>(cp.d, jcp.d, n + 1, d_err.get());
      if (nnz > 0) compare_i64<<<P->grid(nnz), kThreads>>>(rv.d, jrv.d, nnz, d_err.get());
      uint32_t h = 0;
      TRY(read_back(&h, d_err.get(), 1, "comparing J's pattern"));
      same_pattern = !(h & kErrPatternDiff);
      CU(cudaMemset(d_err.get(), 0, 4));
    }
    other_csc = !same_pattern;
    P->j_len = jnnz;
  } else if (jkind == FDB_J_CSC_NZVAL) {
    P->j_len = nnz;
  } else {
    if (ldJ < m) return fail(FDB_ERR_INVALID, "ldJ=%lld < m=%lld", (long long)ldJ, (long long)m);
    P->ldJ = ldJ;
    P->j_len = ldJ * n;
  }
  const bool need_dest = jkind == FDB_J_DENSE || other_csc;
  DevBuf<int32_t> col32;
  if (need_dest) {
    TRY(col32.alloc(std::max<int64_t>(nnz, 1)));
    TRY(P->alloc_t(&P->entries.dest, std::max<int64_t>(nnz, 1)));
  }
  validate_colptr<<<P->grid(n + 1), kThreads>>>(cp.d, n, nnz, d_err.get());
  TRY(read_plan_err(d_err.get(), "CSC sparsity"));
  if (other_csc) {   // J's own column pointer is searched by dest_other_csc: it must be a valid one too
    validate_colptr<<<P->grid(n + 1), kThreads>>>(jcp.d, n, P->j_len, d_err.get());
    TRY(read_plan_err(d_err.get(), "J's CSC pattern"));
  }
  if (nnz > 0) {
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      const size_t hsm = P->colors.C <= kPlanSmemColors ? (size_t)std::max<int32_t>(P->colors.C, 1) * sizeof(unsigned int) : 0;
      expand_csc<CT><<<P->grid(nnz), kThreads, hsm>>>(cp.d, rv.d, m, n, nnz, (const CT *)P->colors.jcolor, P->colors.C, P->entries.row32,
                                                 (CT *)P->entries.ecolor, col32.get(), d_cnt.get(), d_err.get());
      CU(cudaGetLastError());
      return FDB_OK;
    }));
    if (jkind == FDB_J_DENSE) dest_dense_from_rc<<<P->grid(nnz), kThreads>>>(P->entries.row32, col32.get(), nnz, ldJ, P->entries.dest);
    else if (other_csc) dest_other_csc<<<P->grid(nnz), kThreads>>>(P->entries.row32, col32.get(), nnz, jcp.d, jrv.d, P->entries.dest, d_err.get());
  }
  TRY(read_plan_err(d_err.get(), "CSC sparsity"));
  std::vector<unsigned long long> cnt(std::max<int32_t>(P->colors.C, 1), 0);
  if (P->colors.C > 0) TRY(read_back(cnt.data(), d_cnt.get(), (size_t)P->colors.C, "colour counts"));
  // ---- per-colour column lists + gather-locality metric -> scatter strategy
  {
    const int32_t C = P->colors.C;
    DevBuf<unsigned long long> d_jump;
    TRY(d_jump.alloc(1));
    CU(cudaMemset(d_jump.get(), 0, 8));
    TRY(P->alloc_t(&P->entries.colptr32, (size_t)n + 1));
    convert_colptr<<<P->grid(n + 1), kThreads>>>(cp.d, n, P->entries.colptr32);
    TRY(build_color_lists(P));
    if (nnz > 1) {
      row_jump_sum<<<P->grid(nnz), kThreads>>>(P->entries.row32, nnz, d_jump.get());
      unsigned long long js = 0;
      TRY(read_back(&js, d_jump.get(), 1, "row jump sum"));
      P->entries.mean_row_jump = (double)js / (double)(nnz - 1);
    }
    int lanes = 1;
    const double avg = n > 0 ? (double)nnz / (double)n : 1.0;
    while (lanes < 32 && lanes < avg) lanes *= 2;
    P->entries.lanes = lanes;
    // opts->strategy: 0 auto, 1 fused storage-order pass, 2 colour-major lists launched per group of resident colours,
    // 3 colour-major lists with every slab resident (one launch).  The lists are what a launch needs whenever it would
    // otherwise stream entries it does not own: several ranks sharing the colours, or more colours than resident slabs
    // (the latter is decided in finish_colored_plan).
    const int want = opts ? opts->strategy : 0;
    bool per_color = P->world > 1;
    if (want == 1) per_color = false;
    if (want == 2 || want == 3) per_color = true;
    P->entries.lists_resident = want == 3;       // colour-major lists, all slabs resident, one launch at the end
    // auto, one GPU, random pattern with many colours: colour-major lists with every slab resident (one launch) — the
    // colour-by-colour order keeps the gathers of a launch phase inside one 8m-byte slab + f(x) instead of spreading them
    // over C slabs at once.  That only pays while slab + f(x) stay in L2: on an H100 (50 MB) C4's 40 + 40 MB do not, and
    // the storage-order pass is the faster scatter there.  Row-local patterns stay fused / staged.
    if (want == 0 && P->world == 1 && P->entries.mean_row_jump > 4096.0 && C >= 16 && 16 * P->m <= P->l2_bytes) {
      per_color = true;
      P->entries.lists_resident = true;
    }
    P->entries.strategy = per_color ? 1 : 0;
    P->entries.strategy_auto = want == 0;
  }
  TRY(finish_colored_plan(P, opts, cnt));
  if (P->entries.strategy == 1) TRY(build_cm_lists(P, cnt));
  TRY(try_stage_plan(P));
  // SURVEY.md §8(d): B_alg = 32*nnz + 16*n + 8 (valid colouring; Int64 indices as at the ABI)
  P->alg_bytes = 32 * nnz + 16 * n + 8;
  return finish_plan(owner, plan);
}

fdb_status fdb_plan_create_coo(fdb_plan **plan, int64_t m, int64_t n, int64_t nnz, const int64_t *rows_index,
                               const int64_t *cols_index, int jkind, const int64_t *slots, int64_t ldJ_or_jlen,
                               const int64_t *colorvec, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (nnz < 0 || nnz > 0x7FFFFFF0LL) return fail(FDB_ERR_UNSUPPORTED, "nnz=%lld unsupported", (long long)nnz);
  if (nnz > 0 && (!rows_index || !cols_index)) return fail(FDB_ERR_INVALID, "rows_index/cols_index NULL");
  if (jkind != FDB_J_DENSE && jkind != FDB_J_SLOTS) return fail(FDB_ERR_INVALID, "COO sparsity supports J kinds DENSE and SLOTS");
  if (jkind == FDB_J_SLOTS && nnz > 0 && !slots) return fail(FDB_ERR_INVALID, "slots is NULL");
  if (jkind == FDB_J_DENSE && ldJ_or_jlen < m) return fail(FDB_ERR_INVALID, "ldJ < m");
  P->sp_kind = SP_COO;
  P->jkind = jkind;
  P->colors.E = nnz;
  if (jkind == FDB_J_DENSE) { P->ldJ = ldJ_or_jlen; P->j_len = ldJ_or_jlen * n; }
  else P->j_len = ldJ_or_jlen;
  I64View rv, cvw, sv;
  TRY(view_i64(rows_index, nnz, rv));
  TRY(view_i64(cols_index, nnz, cvw));
  if (jkind == FDB_J_SLOTS) TRY(view_i64(slots, nnz, sv));
  TRY(setup_colors(P, colorvec));
  DevBuf<uint32_t> d_err;
  DevBuf<unsigned long long> d_cnt;
  TRY(d_err.alloc(1));
  TRY(d_cnt.alloc(std::max<int32_t>(P->colors.C, 1)));
  CU(cudaMemset(d_err.get(), 0, 4));
  CU(cudaMemset(d_cnt.get(), 0, (size_t)std::max<int32_t>(P->colors.C, 1) * 8));
  TRY(P->alloc_t(&P->entries.row32, std::max<int64_t>(nnz, 4)));
  TRY(P->alloc(&P->entries.ecolor, (size_t)std::max<int64_t>(nnz, 4) * (P->colors.bits / 8) + 16));
  TRY(P->alloc_t(&P->entries.dest, std::max<int64_t>(nnz, 1)));
  if (nnz > 0) {
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      const size_t hsm = P->colors.C <= kPlanSmemColors ? (size_t)std::max<int32_t>(P->colors.C, 1) * sizeof(unsigned int) : 0;
      prepare_coo<CT><<<P->grid(nnz), kThreads, hsm>>>(rv.d, cvw.d, jkind == FDB_J_SLOTS ? sv.d : nullptr, nnz, m, n, P->ldJ,
                                                  P->j_len, (const CT *)P->colors.jcolor, P->colors.C, P->entries.row32, (CT *)P->entries.ecolor,
                                                  P->entries.dest, d_cnt.get(), d_err.get());
      CU(cudaGetLastError());
      return FDB_OK;
    }));
  }
  TRY(read_plan_err(d_err.get(), "COO sparsity"));
  std::vector<unsigned long long> cnt(std::max<int32_t>(P->colors.C, 1), 0);
  if (P->colors.C > 0) TRY(read_back(cnt.data(), d_cnt.get(), (size_t)P->colors.C, "colour counts"));
  TRY(finish_colored_plan(P, opts, cnt));
  P->alg_bytes = 32 * nnz + 16 * n + 8;
  return finish_plan(owner, plan);
}

fdb_status fdb_plan_create_banded(fdb_plan **plan, int64_t m, int64_t n, int64_t l, int64_t u, int jkind, int64_t ldJ,
                                  const int64_t *colorvec, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (jkind != FDB_J_BAND && jkind != FDB_J_DENSE && jkind != FDB_J_DIAGONALS)
    return fail(FDB_ERR_INVALID, "banded sparsity supports J kinds BAND and DENSE (and DIAGONALS for diagonal storage)");
  if (l + u + 1 < 1 || l < -n || u < -m) return fail(FDB_ERR_INVALID, "invalid bandwidths l=%lld u=%lld", (long long)l, (long long)u);
  if (jkind == FDB_J_DENSE && ldJ < m) return fail(FDB_ERR_INVALID, "ldJ < m");
  // diagonal storage (kernels_diagonals.cuh): the stored diagonals of a square matrix with l, u in {0, 1}, packed
  const int64_t diag_len = n > 0 ? (l + u + 1) * n - l - u : 0;
  if (jkind == FDB_J_DIAGONALS) {
    if (m != n) return fail(FDB_ERR_INVALID, "diagonal storage needs m == n (m=%lld n=%lld)", (long long)m, (long long)n);
    if (l < 0 || l > 1 || u < 0 || u > 1)
      return fail(FDB_ERR_INVALID, "diagonal storage needs l, u in {0, 1} (l=%lld u=%lld)", (long long)l, (long long)u);
    if (ldJ < diag_len) return fail(FDB_ERR_INVALID, "ldJ=%lld < (l+u+1)*n - l - u = %lld", (long long)ldJ, (long long)diag_len);
  }
  P->sp_kind = SP_BANDED;
  P->jkind = jkind;
  P->band.l = l;
  P->band.u = u;
  P->ldJ = ldJ;
  P->j_len = jkind == FDB_J_BAND ? (l + u + 1) * n : (jkind == FDB_J_DIAGONALS ? diag_len : ldJ * n);
  TRY(setup_colors(P, colorvec));
  DevBuf<unsigned long long> d_cnt;
  TRY(d_cnt.alloc(std::max<int32_t>(P->colors.C, 1)));
  CU(cudaMemset(d_cnt.get(), 0, (size_t)std::max<int32_t>(P->colors.C, 1) * 8));
  if (n > 0 && P->colors.C > 0) {
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      count_band_colors<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, m, n, l, u, P->colors.C, d_cnt.get());
      CU(cudaGetLastError());
      return FDB_OK;
    }));
  }
  std::vector<unsigned long long> cnt(std::max<int32_t>(P->colors.C, 1), 0);
  if (P->colors.C > 0) TRY(read_back(cnt.data(), d_cnt.get(), (size_t)P->colors.C, "colour counts"));
  unsigned long long total = 0;
  for (auto c : cnt) total += c;
  P->colors.E = (int64_t)total;
  TRY(finish_colored_plan(P, opts, cnt));
  // SURVEY.md §8(d) banded: 8*sum_c band_len(c) written + 16*m*C read (diagonal storage: every slot written once)
  P->alg_bytes = (jkind == FDB_J_DIAGONALS ? 8 * diag_len : 8 * (int64_t)total) + 16 * m * (int64_t)P->colors.C;
  return finish_plan(owner, plan);
}

// BandedBlockBandedMatrix with square blocks (ext/FiniteDiffBlockBandedMatricesExt.jl:16-42): host work O(nblocks), the
// structure stays a closed form (kernels_blockband.cuh)
fdb_status fdb_plan_create_block_banded(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                        int64_t lam, int64_t mu, int64_t ldata, const int64_t *colorvec,
                                        const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (nblocks < 0 || nblocks > 0x7FFFFFF0LL) return fail(FDB_ERR_INVALID, "nblocks=%lld outside [0, 2^31)", (long long)nblocks);
  if (nblocks > 0 && !blocks) return fail(FDB_ERR_INVALID, "blocks is NULL");
  if (l < 0 || u < 0 || lam < 0 || mu < 0)
    return fail(FDB_ERR_INVALID, "negative bandwidths (l, u) = (%lld, %lld), (lam, mu) = (%lld, %lld)", (long long)l,
                (long long)u, (long long)lam, (long long)mu);
  // slots per column: the kernels index a column with 32-bit offsets
  const int64_t kMaxW = 0x7FFFFFF0LL;
  if (l >= kMaxW || u >= kMaxW || lam >= kMaxW || mu >= kMaxW || (l + u + 1) > kMaxW / (lam + mu + 1))
    return fail(FDB_ERR_UNSUPPORTED, "(l+u+1)(lam+mu+1) slots per column must be below 2^31");
  const int64_t w = (l + u + 1) * (lam + mu + 1);
  std::vector<int64_t> hb;
  std::vector<int32_t> off;
  int64_t n = 0;
  TRY(read_block_sizes(nblocks, blocks, hb, off, n));
  if (ldata < w * n) return fail(FDB_ERR_INVALID, "ldata=%lld < (l+u+1)(lam+mu+1)*n = %lld", (long long)ldata, (long long)(w * n));
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, n, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->sp_kind = SP_BLOCKBAND;
  P->jkind = FDB_J_BLOCK_BAND;
  P->band.l = l;
  P->band.u = u;
  P->block_band.lam = lam;
  P->block_band.mu = mu;
  P->block_band.w = w;
  P->block_band.nblocks = (int32_t)nblocks;
  P->j_len = w * n;
  P->block_band.bs = nblocks > 0 && hb[0] > 0 && std::all_of(hb.begin(), hb.end(), [&](int64_t b) { return b == hb[0]; }) ? (int32_t)hb[0] : 0;
  TRY(P->alloc_t(&P->block_band.off, (size_t)nblocks + 1));
  CU(cudaMemcpy(P->block_band.off, off.data(), ((size_t)nblocks + 1) * 4, cudaMemcpyHostToDevice));
  TRY(setup_colors(P, colorvec));
  TRY(finish_block_plan(P, opts, [&](auto tag, unsigned long long *cnt, uint32_t *not_cyclic) {
    using CT = decltype(tag);
    block_band_plan_pass<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, P->block_band.off, (int32_t)nblocks, (int32_t)n, l, u,
                                                      lam, mu, P->colors.C, cnt, not_cyclic);
  }));
  // every slot written once + the f! outputs read (one slab and f(x) / the minus slab per colour)
  P->alg_bytes = 8 * w * n + 16 * n * (int64_t)P->colors.C;
  return finish_plan(owner, plan);
}

// BlockBandedMatrix with square blocks (ext/FiniteDiffBlockBandedMatricesExt.jl:44-68) in BlockBandedMatrices' own
// storage: one column-major slab per block column (kernels_blockband.cuh).  Host work O(nblocks); the plan keeps the
// block offsets and the slab starts on the device.
fdb_status fdb_plan_create_block_dense(fdb_plan **plan, int64_t nblocks, const int64_t *blocks, int64_t l, int64_t u,
                                       int64_t ldata, const int64_t *colorvec, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (nblocks < 0 || nblocks > 0x7FFFFFF0LL) return fail(FDB_ERR_INVALID, "nblocks=%lld outside [0, 2^31)", (long long)nblocks);
  if (nblocks > 0 && !blocks) return fail(FDB_ERR_INVALID, "blocks is NULL");
  if (l < 0 || u < 0) return fail(FDB_ERR_INVALID, "negative block bandwidths (l, u) = (%lld, %lld)", (long long)l, (long long)u);
  std::vector<int64_t> hb;
  std::vector<int32_t> off;
  int64_t n = 0;
  TRY(read_block_sizes(nblocks, blocks, hb, off, n));
  // bandwidths of nblocks or more describe the same structure (and the same closed-form colouring) as nblocks
  l = std::min(l, nblocks);
  u = std::min(u, nblocks);
  // slab J: the rows of block rows max(0, J-u) .. min(N-1, J+l), cb[J] columns; the kernel indexes a slab with 32 bits
  std::vector<int64_t> start((size_t)nblocks + 1, 0);
  for (int64_t J = 0; J < nblocks; ++J) {
    const int64_t K0 = std::max<int64_t>(0, J - u), K1 = std::min<int64_t>(nblocks - 1, J + l);
    const int64_t slab = (int64_t)(off[(size_t)K1 + 1] - off[(size_t)K0]) * hb[(size_t)J];
    if (slab > 0xFFFFFFFFLL)
      return fail(FDB_ERR_UNSUPPORTED, "block column %lld holds %lld slots; a block column is limited to 2^32", (long long)J,
                  (long long)slab);
    start[(size_t)J + 1] = start[(size_t)J] + slab;
  }
  const int64_t jlen = start[(size_t)nblocks];
  if (ldata < jlen) return fail(FDB_ERR_INVALID, "ldata=%lld < the %lld slots of the block columns", (long long)ldata, (long long)jlen);
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, n, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->sp_kind = SP_BLOCKBAND;
  P->jkind = FDB_J_BLOCK_DENSE;
  P->band.l = l;
  P->band.u = u;
  P->block_band.nblocks = (int32_t)nblocks;
  P->j_len = jlen;
  P->block_band.bs = nblocks > 0 && hb[0] > 0 && std::all_of(hb.begin(), hb.end(), [&](int64_t b) { return b == hb[0]; }) ? (int32_t)hb[0] : 0;
  TRY(P->alloc_t(&P->block_band.off, (size_t)nblocks + 1));
  CU(cudaMemcpy(P->block_band.off, off.data(), ((size_t)nblocks + 1) * 4, cudaMemcpyHostToDevice));
  TRY(P->alloc_t(&P->block_band.start, (size_t)nblocks + 1));
  CU(cudaMemcpy(P->block_band.start, start.data(), ((size_t)nblocks + 1) * 8, cudaMemcpyHostToDevice));
  TRY(setup_colors(P, colorvec));
  TRY(finish_block_plan(P, opts, [&](auto tag, unsigned long long *cnt, uint32_t *not_cyclic) {
    using CT = decltype(tag);
    block_dense_plan_pass<CT><<<P->grid(n), kThreads>>>((const CT *)P->colors.jcolor, P->block_band.off, (int32_t)nblocks, (int32_t)n, l, u,
                                                       P->block_band.bs, P->colors.C, cnt, not_cyclic);
  }));
  // the block-banded byte model: every slot written once + the f! outputs read
  P->alg_bytes = 8 * jlen + 16 * n * (int64_t)P->colors.C;
  return finish_plan(owner, plan);
}

// J a CSR matrix (rowptr, colval, nzval) with the sparsity's own pattern: the nzval scatter of kernels_csr.cuh.  The
// plan keeps the row pointer and the columns as 0-based int32; J is never zero-filled.
fdb_status fdb_plan_create_csr(fdb_plan **plan, int64_t m, int64_t n, const int64_t *rowptr, const int64_t *colval,
                               const int64_t *colorvec, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (!rowptr) return fail(FDB_ERR_INVALID, "rowptr is NULL");
  P->sp_kind = SP_CSR;
  P->jkind = FDB_J_CSR;
  // nnz = rowptr[m]-1: read the first and last elements wherever they live, then check the whole pointer on the device
  I64View rp, cv;
  TRY(view_i64(rowptr, m + 1, rp));
  int64_t first = 1, last = 1;
  TRY(read_back(&first, rp.d, 1, "reading rowptr[1]"));
  TRY(read_back(&last, rp.d + m, 1, "reading rowptr[m+1]"));
  if (first != 1) return fail(FDB_ERR_INVALID, "rowptr[1]=%lld: a CSR row pointer starts at 1", (long long)first);
  const int64_t nnz = last - 1;
  if (nnz < 0) return fail(FDB_ERR_INVALID, "rowptr is not a valid CSR row pointer (must start at 1, be non-decreasing, end at nnz+1)");
  {
    DevBuf<uint32_t> d_err;
    TRY(d_err.alloc(1));
    CU(cudaMemset(d_err.get(), 0, 4));
    validate_colptr<<<P->grid(m + 1), kThreads>>>(rp.d, m, nnz, d_err.get());
    uint32_t h = 0;
    TRY(read_back(&h, d_err.get(), 1, "CSR row pointer"));
    if (h) return fail(FDB_ERR_INVALID, "rowptr is not a valid CSR row pointer (must start at 1, be non-decreasing, end at nnz+1)");
  }
  if (nnz > 0x7FFFFFF0LL) return fail(FDB_ERR_UNSUPPORTED, "nnz=%lld unsupported (must be in [0, 2^31))", (long long)nnz);
  if (nnz > 0 && !colval) return fail(FDB_ERR_INVALID, "colval is NULL");
  TRY(view_i64(colval, nnz, cv));
  P->colors.E = nnz;
  P->j_len = nnz;
  TRY(setup_colors(P, colorvec));
  DevBuf<uint32_t> d_err;
  DevBuf<unsigned long long> d_cnt;
  TRY(d_err.alloc(1));
  TRY(d_cnt.alloc(std::max<int32_t>(P->colors.C, 1)));
  CU(cudaMemset(d_err.get(), 0, 4));
  CU(cudaMemset(d_cnt.get(), 0, (size_t)std::max<int32_t>(P->colors.C, 1) * 8));
  TRY(P->alloc_t(&P->csr.rowptr, (size_t)m + 1));
  TRY(P->alloc_t(&P->csr.colval, (size_t)std::max<int64_t>(nnz, 1)));
  csr_rowptr32<<<P->grid(m + 1), kThreads>>>(rp.d, m, P->csr.rowptr);
  if (nnz > 0) {
    TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      using CT = decltype(tag);
      const size_t hsm = P->colors.C <= kPlanSmemColors ? (size_t)std::max<int32_t>(P->colors.C, 1) * sizeof(unsigned int) : 0;
      csr_plan_pass<CT><<<P->grid(nnz), kThreads, hsm>>>(cv.d, n, nnz, (const CT *)P->colors.jcolor, P->colors.C, P->csr.colval,
                                                        d_cnt.get(), d_err.get());
      CU(cudaGetLastError());
      return FDB_OK;
    }));
  }
  TRY(read_plan_err(d_err.get(), "CSR sparsity"));
  std::vector<unsigned long long> cnt(std::max<int32_t>(P->colors.C, 1), 0);
  if (P->colors.C > 0) TRY(read_back(cnt.data(), d_cnt.get(), (size_t)P->colors.C, "colour counts"));
  TRY(finish_colored_plan(P, opts, cnt));
  // the CSC plan's SURVEY.md §8(d) model: B_alg = 32*nnz + 16*n + 8 (valid colouring; Int64 indices as at the ABI)
  P->alg_bytes = 32 * nnz + 16 * n + 8;
  return finish_plan(owner, plan);
}

// dense column branch over the leading `ncols` components (ncols == n for the default colorvec = 1:n)
static fdb_status create_dense(fdb_plan **plan, int64_t m, int64_t n, int64_t ldJ, int64_t ncols, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (ldJ < m) return fail(FDB_ERR_INVALID, "ldJ < m");
  P->sp_kind = SP_NONE;
  P->jkind = FDB_J_DENSE;
  P->ldJ = ldJ;
  // contiguous column blocks per rank (SURVEY.md §8e)
  const int64_t per = (ncols + P->world - 1) / P->world;
  P->columns.begin = std::min<int64_t>(ncols, per * P->rank);
  P->columns.end = std::min<int64_t>(ncols, P->columns.begin + per);
  const int64_t ncl = P->columns.end - P->columns.begin;
  P->j_len = ldJ * ncl;
  const bool central = P->fdtype == FDB_CENTRAL;
  P->scratch.ldF = std::max<int64_t>(2, (m + 1) & ~(int64_t)1);
  P->scratch.ldx = std::max<int64_t>(2, (n + 1) & ~(int64_t)1);
  int64_t batch = (opts && opts->max_batch > 1) ? opts->max_batch : 1;
  int64_t budget = (opts && opts->scratch_bytes > 0) ? opts->scratch_bytes : (int64_t)8 << 30;
  const int64_t cw = P->fdtype == FDB_COMPLEX ? 2 : 1;
  const int64_t per_point = 8 * cw * (P->scratch.ldx + P->scratch.ldF * (central ? 2 : 1));
  batch = std::max<int64_t>(1, std::min<int64_t>(batch, budget / per_point));
  batch = std::min<int64_t>(batch, std::max<int64_t>(ncl, 1));
  batch = std::min<int64_t>(batch, 65535);   // gridDim.y of diff_columns
  P->scratch.batch = batch;
  P->scratch.slabs = batch;
  P->scratch.n_groups = ncl == 0 ? 0 : (ncl + batch - 1) / batch;
  TRY(P->alloc_t(&P->scratch.fx_own, (size_t)P->scratch.ldF));
  TRY(P->alloc_t(&P->scratch.Fp, (size_t)batch * P->scratch.ldF * cw));
  if (central) TRY(P->alloc_t(&P->scratch.Fm, (size_t)batch * P->scratch.ldF));
  TRY(P->alloc_t(&P->scratch.xp, (size_t)batch * P->scratch.ldx * cw));
  TRY(P->alloc_t(&P->columns.eps, (size_t)std::max<int64_t>(ncl, 1)));
  // SURVEY.md §8(d) dense: 24*m per column
  P->alg_bytes = 24 * m * ncl;
  *plan = owner.release();
  return FDB_OK;
}

fdb_status fdb_plan_create_dense(fdb_plan **plan, int64_t m, int64_t n, int64_t ldJ, const fdb_plan_opts *opts) {
  return create_dense(plan, m, n, ldJ, n, opts);
}

// sparsity === nothing with a caller-supplied colorvec, exactly as jacobians.jl:547-557 / :589-598 / :625-631 are written:
// `for color_i in 1:maximum(colorvec)` perturbs COMPONENT color_i (the colour id is used as an index) and writes
// J[:, color_i]; J is not zero-filled (:530 only fills when sparsity !== nothing), so columns beyond maximum(colorvec)
// keep their contents.  maximum(colorvec) > n indexes x1 out of bounds in the reference (BoundsError) -> FDB_ERR_INVALID.
fdb_status fdb_plan_create_dense_colorvec(fdb_plan **plan, int64_t m, int64_t n, int64_t ldJ, const int64_t *colorvec,
                                          const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (!colorvec) return create_dense(plan, m, n, ldJ, n, opts);
  if (n < 0 || m < 0) return fail(FDB_ERR_INVALID, "negative dimensions");
  int dev = 0;
  TRY(check_device(opts, &dev));
  DeviceGuard g(dev);
  long long mx = 0, mn = 0;
  if (n > 0) {
    I64View cv;
    TRY(view_i64(colorvec, n, cv));
    TRY(color_range(cv.d, n, &mx, &mn));
  }
  if (mx > n) return fail(FDB_ERR_INVALID, "sparsity=nothing: maximum(colorvec)=%lld indexes x beyond length(x)=%lld "
                                           "(BoundsError in the reference, jacobians.jl:549)", mx, (long long)n);
  return create_dense(plan, m, n, ldJ, mx < 0 ? 0 : (int64_t)mx, opts);
}

fdb_status fdb_plan_destroy(fdb_plan *plan) {
  free_plan(plan);
  return FDB_OK;
}

// the part of the whole problem this rank evaluates, as the ABI reports it (fdb_plan_info, fdb_plan_dense_range): a dense
// plan's columns, a Hessian plan's i-blocks, and nothing for the other kinds
static std::pair<int64_t, int64_t> own_range(const fdb_plan *P) {
  if (P->sp_kind == SP_NONE) return {P->columns.begin, P->columns.end};
  if (P->sp_kind == SP_HESS) return {P->hess.i_begin, P->hess.i_end};
  return {0, 0};
}

// colours this rank evaluates (dense and Hessian plans: columns / i-blocks, counted as colours)
static int64_t local_units(const fdb_plan *P) {
  if (P->sp_kind != SP_NONE && P->sp_kind != SP_HESS) return (int64_t)P->colors.local.size();
  const auto r = own_range(P);
  return r.second - r.first;
}

// an out-of-place rank > 0 that owns no colour (dense branch: no column): it calls nothing and launches nothing
static bool oop_idle(const fdb_plan *P) {
  return P->oop.on && P->rank > 0 && local_units(P) == 0;
}

fdb_status fdb_plan_info(const fdb_plan *P, fdb_plan_info_t *info) {
  if (!P || !info) return fail(FDB_ERR_INVALID, "NULL argument");
  memset(info, 0, sizeof *info);
  info->m = P->m;
  info->n = P->n;
  info->j_len = P->j_len;
  const int64_t n_local = local_units(P);
  info->n_local_colors = n_local;
  switch (P->sp_kind) {   // maximum(colorvec) and the entries the scatter writes, by kind
    case SP_NONE:   // every column its own colour; out-of-place: the candidates of the whole result
      info->n_colors = P->n;
      info->n_entries = P->oop.on ? P->m * P->oop.qcols : P->m * n_local;
      break;
    case SP_HESS: info->n_colors = P->n; info->n_entries = P->hess.entries; break;
    case SP_JVP: info->n_colors = 1; break;
    case SP_DERIV: info->n_entries = P->m; break;
    default:   // coloured and step-size plans; out-of-place band: every in-matrix band entry
      info->n_colors = P->colors.C;
      info->n_entries = P->oop.on && P->sp_kind == SP_BANDED ? P->oop.band_nnz : P->colors.E;
  }
  info->n_groups = P->scratch.n_groups;
  info->slabs = P->scratch.slabs;
  info->fcalls_per_jacobian = P->fdtype == FDB_CENTRAL ? 2 * n_local : (P->fdtype == FDB_COMPLEX ? n_local : 1 + n_local);
  if (P->sp_kind == SP_HESS) info->fcalls_per_jacobian = P->hess.points;
  if (P->sp_kind == SP_DERIV) info->fcalls_per_jacobian = P->deriv.fcalls;
  if (oop_idle(P)) info->fcalls_per_jacobian = 0;
  info->device_bytes = (int64_t)P->device_bytes;
  info->fdtype = P->fdtype;
  info->jkind = P->jkind;
  info->sp_kind = P->sp_kind;
  info->color_bits = P->colors.bits;
  info->alg_bytes_scatter = P->alg_bytes;
  info->strategy = P->entries.strategy;
  info->lanes = P->entries.lanes;
  info->mean_row_jump = P->entries.mean_row_jump;
  info->staged = P->staged.on ? 1 : 0;
  info->lists_resident = P->entries.lists_resident ? 1 : 0;
  {
    // compulsory bytes of the formulation that runs (see the header); slabs read per entry: 1 (forward / complex), 2 (central)
    const int64_t ct = P->colors.bits / 8;
    const int64_t slabs_read = P->fdtype == FDB_CENTRAL ? 2 : 1;
    const int64_t fx_once = P->fdtype == FDB_FORWARD ? 8 * P->m : 0;
    if (P->sp_kind == SP_CSC || P->sp_kind == SP_COO) {
      if (P->sp_kind == SP_CSC && P->entries.strategy == 1) {
        const int64_t e_local = P->cm.start_h.empty() ? 0 : P->cm.start_h.back();
        info->moved_bytes_scatter = e_local * (4 + (P->entries.dest ? 8 : 4) + 8 * slabs_read + 8) + fx_once + (P->cm.fx ? e_local * (4 + 8 + 8) : 0);
      } else {
        const int64_t C = std::max<int32_t>(P->colors.C, 1);
        const int64_t owned = P->world > 1 ? P->colors.E * (int64_t)P->colors.local.size() / C : P->colors.E;   // approx. share
        info->moved_bytes_scatter = P->colors.E * (4 + ct) * std::max<int64_t>(P->scratch.n_groups, 1) + owned * (8 * slabs_read + 8 + (P->entries.dest ? 8 : 0)) + fx_once;
        const int64_t staged_rows = 8 * P->m * (int64_t)(P->fdtype == FDB_CENTRAL ? 2 * P->colors.C : P->colors.C + 1);
        if (P->staged.on && P->staged.band)   // no index stream; the column colour table unless the colouring is cyclic
          info->moved_bytes_scatter = 8 * P->colors.E + staged_rows + (P->colors.cyclic ? 0 : P->n * ct);
        else if (P->staged.on)   // 16-bit row offsets; every slab row and f(x) row staged once
          info->moved_bytes_scatter = P->colors.E * (2 + (P->staged.packed ? 0 : ct) + 8) + staged_rows;
      }
    } else if (P->sp_kind == SP_CSR) {
      // every launch streams the columns, the row pointer and (unless cyclic) the column colours; the entries it owns
      // gather their slab rows and store their slot once
      const int64_t launches = std::max<int64_t>(P->scratch.n_groups, 1);
      const int64_t C = std::max<int32_t>(P->colors.C, 1);
      const int64_t owned = P->world > 1 ? P->colors.E * (int64_t)P->colors.local.size() / C : P->colors.E;   // approx. share
      info->moved_bytes_scatter = launches * (4 * P->colors.E + 4 * (P->m + 1) + (P->colors.cyclic ? 0 : P->n * ct)) +
                                  owned * (8 * slabs_read + 8) + fx_once;
    } else {
      info->moved_bytes_scatter = P->alg_bytes;
    }
  }
  return FDB_OK;
}

fdb_status fdb_plan_counters(const fdb_plan *P, fdb_counters_t *out) {
  if (!P || !out) return fail(FDB_ERR_INVALID, "NULL argument");
  *out = P->cnt;
  return FDB_OK;
}

fdb_status fdb_plan_dense_range(const fdb_plan *P, int64_t *b, int64_t *e) {
  if (!P || !b || !e) return fail(FDB_ERR_INVALID, "NULL argument");
  const auto r = own_range(P);
  *b = r.first;
  *e = r.second;
  return FDB_OK;
}

fdb_status fdb_plan_color_owner(const fdb_plan *P, int32_t *owner_out, int64_t cap) {
  if (!P || !owner_out) return fail(FDB_ERR_INVALID, "NULL argument");
  TRY(check_call(P, Call::color_owner));
  if (cap < (int64_t)P->colors.owner.size()) return fail(FDB_ERR_INVALID, "owner_out too small");
  std::copy(P->colors.owner.begin(), P->colors.owner.end(), owner_out);
  return FDB_OK;
}

fdb_status fdb_plan_get_eps(fdb_plan *P, double *h_eps, int64_t cap, void *stream) {
  if (!P || !h_eps) return fail(FDB_ERR_INVALID, "NULL argument");
  TRY(check_call(P, Call::get_eps));
  DeviceGuard g(P->device);
  // dense plans: the steps of the rank's columns; Hessian plans: those of the rank's components (hess.eps holds all n);
  // JVP plans: the one step; coloured and step-size plans: one per colour
  const double *src = P->steps.eps;
  int64_t count = P->sp_kind == SP_JVP ? 1 : P->colors.C;
  if (P->sp_kind == SP_NONE) { src = P->columns.eps; count = local_units(P); }
  if (P->sp_kind == SP_HESS) { src = P->hess.eps + P->hess.i_begin; count = local_units(P); }
  if (cap < count) return fail(FDB_ERR_INVALID, "h_eps too small (%lld < %lld)", (long long)cap, (long long)count);
  if (count > 0) {
    CU(cudaMemcpyAsync(h_eps, src, (size_t)count * 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    CU(cudaStreamSynchronize((cudaStream_t)stream));
  }
  return FDB_OK;
}

fdb_status fdb_plan_enable_timing(fdb_plan *P, int enable) {
  if (!P) return fail(FDB_ERR_INVALID, "NULL plan");
  P->timing.on = enable != 0;
  return FDB_OK;
}

fdb_status fdb_plan_read_timing(fdb_plan *P, double *scatter_ms, int64_t *scatter_launches) {
  if (!P || !scatter_ms || !scatter_launches) return fail(FDB_ERR_INVALID, "NULL argument");
  DeviceGuard g(P->device);
  double total = 0.0;
  int64_t count = 0;
  for (auto &ev : P->timing.pending) {
    CU(cudaEventSynchronize(ev.second));
    float ms = 0.f;
    CU(cudaEventElapsedTime(&ms, ev.first, ev.second));
    total += ms;
    count += 1;
    P->timing.pool.push_back(ev);
  }
  P->timing.pending.clear();
  *scatter_ms = total;
  *scatter_launches = count;
  return FDB_OK;
}

fdb_status fdb_plan_set_peers(fdb_plan *P, int n_peers, double *const *peer_J) {
  if (!P) return fail(FDB_ERR_INVALID, "NULL plan");
  if (n_peers < 0 || n_peers > 64) return fail(FDB_ERR_INVALID, "n_peers out of range");
  TRY(check_call(P, Call::set_peers));
  DeviceGuard g(P->device);
  if (!P->peers.d) TRY(P->alloc_t(&P->peers.d, 64));
  if (n_peers > 0) CU(cudaMemcpy(P->peers.d, peer_J, (size_t)n_peers * sizeof(double *), cudaMemcpyHostToDevice));
  P->peers.n = n_peers;
  P->peers.generation += 1;
  P->peers.aligned = true;
  for (int i = 0; i < n_peers; ++i)
    if (reinterpret_cast<uintptr_t>(peer_J[i]) & 15) P->peers.aligned = false;
  return FDB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ the hot path
struct ScatterTimer {
  fdb_plan *P;
  cudaStream_t s;
  std::pair<cudaEvent_t, cudaEvent_t> ev{nullptr, nullptr};
  ScatterTimer(fdb_plan *p, cudaStream_t st) : P(p), s(st) {
    if (!P->timing.on) return;
    if (!P->timing.pool.empty()) { ev = P->timing.pool.back(); P->timing.pool.pop_back(); }
    else { cudaEventCreate(&ev.first); cudaEventCreate(&ev.second); }
    cudaEventRecord(ev.first, s);
  }
  ~ScatterTimer() {
    if (!P->timing.on || !ev.first) return;
    cudaEventRecord(ev.second, s);
    P->timing.pending.push_back(ev);
  }
};

// fill_matrix!(J, false) (jacobians.jl:530-532, :663).  A dense J may be a strided column-major view (ldJ > m): only
// rows [0, m) of every column belong to J — the padding rows between the columns are not touched.
static fdb_status zero_J(const fdb_plan *P, double *J, cudaStream_t s) {
  if (P->jkind == FDB_J_DENSE && P->ldJ > P->m) {
    const int64_t ncols = P->sp_kind == SP_NONE ? P->columns.end - P->columns.begin : P->n;
    if (P->m > 0 && ncols > 0)
      CU(cudaMemset2DAsync(J, (size_t)P->ldJ * 8, 0, (size_t)P->m * 8, (size_t)ncols, s));
    return FDB_OK;
  }
  CU(cudaMemsetAsync(J, 0, (size_t)P->j_len * 8, s));
  return FDB_OK;
}

// How a coloured plan turns a group's f! outputs into J: one launcher per family (scatter_lists ... scatter_entries), and
// none for an out-of-place sparse result whose compaction forms the quotients itself (fdjac_oop.cuh).  Fixed once the
// plan is built, but derived rather than stored: the out-of-place creators set oop.fused after the in-place creator.
enum class Scatter { none, lists, block_band, block_dense, diagonals, band, csr, entries };

static Scatter scatter_family(const fdb_plan *P) {
  if (P->oop.fused) return Scatter::none;
  if (P->sp_kind == SP_CSC && P->entries.strategy == 1) return Scatter::lists;
  if (P->sp_kind == SP_BLOCKBAND) return P->jkind == FDB_J_BLOCK_DENSE ? Scatter::block_dense : Scatter::block_band;
  if (P->sp_kind == SP_BANDED) return P->jkind == FDB_J_DIAGONALS ? Scatter::diagonals : Scatter::band;
  if (P->sp_kind == SP_CSR) return Scatter::csr;
  return Scatter::entries;
}

// fill_matrix!(J, false) (jacobians.jl:530-532) is needed unless the scatter launches over `colours` colours (one rank's
// or a whole group's) define every slot of J themselves, zeros for the columns without a valid colour included.  A fused
// out-of-place plan stores no candidate, and its candidate buffer is not J-sized: nothing to fill.
static bool scatter_defines_J(const fdb_plan *P, int64_t colours) {
  const Scatter f = scatter_family(P);
  if (f == Scatter::none || f == Scatter::block_band || f == Scatter::block_dense || f == Scatter::csr) return true;
  if (f == Scatter::band && P->jkind != FDB_J_BAND) return false;   // a dense J
  if ((f == Scatter::lists || f == Scatter::entries) && P->entries.dest != nullptr) return false;   // explicit destinations
  return colours > 0;
}

static fdb_status call_f(fdb_plan *P, fdb_fn f, void *ctx, double *fx, const double *x, int64_t batch, cudaStream_t s) {
  const int rc = f(ctx, fx, x, batch, P->scratch.ldF, P->scratch.ldx, (void *)s);
  P->cnt.f_invocations += 1;
  P->cnt.f_points += batch;
  if (rc != 0) return fail(FDB_ERR_CALLBACK, "user f! returned %d", rc);
  return FDB_OK;
}

// Persistent-grid sizing: exactly the number of blocks that are resident at once (SMs x blocks/SM from the occupancy
// calculator), capped by the work — a single full wave, no half-empty second wave.
template <typename K>
static int resident_grid(const fdb_plan *P, K kernel, size_t dyn_smem, int64_t work_blocks) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, dyn_smem) != cudaSuccess || per_sm < 1) {
    cudaGetLastError();
    per_sm = 4;
  }
  int64_t g = (int64_t)P->sm_count * per_sm;
  if (g > work_blocks) g = work_blocks;
  if (g < 1) g = 1;
  return (int)g;
}

// Store-heavy streams gain from an oversubscribed grid: `over` times the resident wave, capped by the work.
template <typename K>
static int oversubscribed_grid(const fdb_plan *P, K kernel, size_t dyn_smem, int64_t work_blocks, int over) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)resident_grid(P, kernel, dyn_smem, work_blocks) * over, work_blocks));
}

// launch `kern` on the resident grid that its occupancy gives for `work_blocks` blocks
template <typename... KArgs, typename... Args>
static void launch_resident(const fdb_plan *P, void (*kern)(KArgs...), int64_t work_blocks, size_t smem, cudaStream_t s,
                            Args... args) {
  kern<<<resident_grid(P, kern, smem, work_blocks), kThreads, smem, s>>>(args...);
}

// dynamic shared memory of a scatter that stages its per-colour (step size, slab) tables: none past kSmemTable colours
static size_t color_table_smem(const fdb_plan *P) {
  return P->colors.C <= kSmemTable ? (size_t)P->colors.C * (sizeof(double) + sizeof(int32_t)) : 0;
}

// Programmatic dependent launch: the kernel may be scheduled while the kernel before it on the stream drains, and runs
// its set-up (shared memory, barriers) meanwhile; it calls cudaGridDependencySynchronize() before it reads anything
// that kernel wrote.  A capture keeps the programmatic edge in the graph.
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kern)(KArgs...), int grid, size_t smem, cudaStream_t s, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, args...);
}

template <typename CT>
static fdb_status run_eps(fdb_plan *P, const double *x, double relstep, double absstep, double dir, cudaStream_t s) {
  const int32_t C = P->colors.C;
  if (C <= 0) return FDB_OK;
  if (P->fdtype == FDB_COMPLEX) {   // epsilon = eps(eltype(x))  jacobians.jl:624 — the same for every colour
    fill_value<<<(C + kThreads - 1) / kThreads, kThreads, 0, s>>>(P->steps.eps, C, DBL_EPSILON);
    P->cnt.kernel_launches += 1;
    CU(cudaGetLastError());
    return FDB_OK;
  }
  // out-of-place plans take the forward rule, dir included, in central mode too (jacobians.jl:379-380)
  EpsParams prm{P->fdtype == FDB_CENTRAL && !P->oop.on ? 1 : 0, relstep, absstep, dir};
  if (P->steps.lists) {
    if (!P->tune.no_eps_lists) {
      dim3 grid((unsigned)std::min<int64_t>(P->steps.list_max_chunks, 1024), (unsigned)std::min<int32_t>(C, 65535));
      color_sumsq_lists<<<grid, kThreads, 0, s>>>(x, P->colors.cols_by_color, P->steps.bucket_start_d, P->steps.chunk_base_d, C, P->steps.list_partial);
      finalize_eps_lists<<<(int)std::min<int64_t>(((int64_t)C * 32 + kThreads - 1) / kThreads, (int64_t)P->sm_count * 8), kThreads, 0, s>>>(
          P->steps.list_partial, P->steps.chunk_base_d, C, prm, P->steps.eps, P->steps.sumsq, x, P->colors.cols_by_color, P->steps.bucket_start_d, P->n);
      P->cnt.kernel_launches += 2;
      CU(cudaGetLastError());
      return FDB_OK;
    }
  }
  if (C <= kEpsRegColors) {
    const int64_t ntiles = (P->n + kTile - 1) / kTile;
    const int aligned = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    TRY(dispatch_colors<CT>(P, [&](auto cs) -> fdb_status {
      using CS = decltype(cs);
      auto go = [&](auto kern) {
        const int grid = std::min(resident_grid(P, kern, 0, ntiles), P->steps.blocks);  // partial capacity
        kern<<<grid, kThreads, 0, s>>>(x, cs, P->n, aligned, C, prm, P->steps.partial, P->steps.ticket, P->steps.eps, P->steps.sumsq);
      };
      if (C <= 4) { if (P->tune.eps_depth == 2) go(color_sumsq_reg<CS, 4, 2>); else go(color_sumsq_reg<CS, 4, 1>); }
      else { if (P->tune.eps_depth == 2) go(color_sumsq_reg<CS, 8, 2>); else go(color_sumsq_reg<CS, 8, 1>); }
      return FDB_OK;
    }));
    P->cnt.kernel_launches += 1;
  } else {
    for (int32_t k0 = 0; k0 < C; k0 += kEpsWindow) {
      const int32_t W = std::min<int32_t>(kEpsWindow, C - k0);
      color_sumsq_win<CT><<<P->steps.blocks, kThreads, (size_t)kEpsWarps * W * sizeof(double), s>>>(
          x, (const CT *)P->colors.jcolor, P->n, P->steps.chunk, k0, W, P->steps.group, P->steps.partial);
      // partial rows are W wide for this pass
      finalize_eps<CT><<<(W * 32 + kThreads - 1) / kThreads, kThreads, 0, s>>>(P->steps.partial, P->steps.blocks, W, k0, W, prm,
                                                                            P->steps.eps, P->steps.sumsq, x, (const CT *)P->colors.jcolor, P->n);
      P->cnt.kernel_launches += 2;
    }
  }
  CU(cudaGetLastError());
  return FDB_OK;
}

// ------------------------------------------------------------------------------------------------ the colour scatter
// What one colour group's scatter reads.  Every family takes its f! outputs and its stream from here, so the
// double-buffered overlap hands its buffer and side stream to whichever family it runs.
struct ScatterGroup {
  fdb_plan *P;
  double *J;
  const double *fx;        // f(x), forward mode
  double *Fp, *Fm;         // the group's f! outputs, one slab of ldF doubles per colour (Fm: central mode)
  int64_t ldF;
  cudaStream_t s;
  int64_t l0, G;           // local colours [l0, l0 + G); G = 0: a rank that owns no colour
  bool first;              // the first group of rank 0: it also writes the columns without a valid colour
};

// colour-major lists: the entries of the columns without a valid colour are 0
static void zero_uncoloured_slots(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  const int64_t z0 = P->cm.start_h[P->colors.local.size()], z1 = P->cm.invalid_end;
  if (z1 <= z0) return;
  const int grid = P->grid(z1 - z0);
  if (P->entries.dest != nullptr) zero_slots<int64_t><<<grid, kThreads, 0, g.s>>>(P->cm.slot, z0, z1, g.J, P->peers.d, P->peers.n);
  else zero_slots<int32_t><<<grid, kThreads, 0, g.s>>>(P->cm.slot, z0, z1, g.J, P->peers.d, P->peers.n);
  P->cnt.kernel_launches += 1;
}

// colour-major lists: the entry lists of the group's colours, <= kMaxSegs colours per launch
template <int MODE>
static fdb_status scatter_lists(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  const int64_t total = P->cm.start_h[(size_t)(g.l0 + g.G)] - P->cm.start_h[(size_t)g.l0];
  CmArgs a{};
  a.row = P->cm.row; a.slot = P->cm.slot; a.seg_start = P->cm.start; a.local_colors = P->colors.d_local;
  a.fx = g.fx; a.Fp = g.Fp; a.Fm = g.Fm; a.eps = P->steps.eps; a.J = g.J; a.peers = P->peers.d; a.n_peers = P->peers.n;
  a.fx_cm = MODE == kForward ? P->cm.fx : nullptr;
  a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G; a.ldF = g.ldF;
  a.m = MODE == kComplex ? 2 * P->m : P->m;
  // (software L2 prefetch of the next colour's slab: off unless FDB_CM_PREFETCH=1 — on C4 the 40 MB slab, the next one
  //  and f(x) do not fit the L2 together)
  a.prefetch_next = (g.G > 1 && P->tune.cm_prefetch) ? 1 : 0;
  a.slab_stream = P->tune.cm_slab_stream;
  const int64_t tiles = (total + kCmTile - 1) / kCmTile;
  ScatterTimer tm(P, g.s);
  if (P->entries.dest != nullptr) launch_resident(P, diff_scatter_cm<MODE, int64_t>, tiles, 0, g.s, a);
  else launch_resident(P, diff_scatter_cm<MODE, int32_t>, tiles, 0, g.s, a);
  return FDB_OK;
}

// block-banded: every slot of the columns of the group's colours, and (first group of rank 0) of the columns without a
// valid colour: storage order, closed-form structure
template <typename CT, int MODE>
static fdb_status scatter_block_band(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  BlockBandArgs a{};
  a.jcolor = P->colors.jcolor; a.boff = P->block_band.off; a.fx = g.fx; a.Fp = g.Fp; a.Fm = g.Fm; a.eps = P->steps.eps;
  a.local_of = P->colors.local_of; a.J = g.J; a.total = P->block_band.w * P->n; a.ldF = g.ldF;
  a.C = P->colors.C; a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G;
  a.write_other = g.first ? 1 : 0;
  a.nblocks = P->block_band.nblocks; a.u = (int32_t)P->band.u; a.mu = (int32_t)P->block_band.mu;
  a.uniform = P->block_band.bs > 0 ? 1 : 0;
  a.block_cyclic = P->block_band.cyclic ? 1 : 0;
  a.w = make_fastdiv((uint32_t)P->block_band.w);
  a.sw = make_fastdiv((uint32_t)(P->block_band.lam + P->block_band.mu + 1));
  a.bs = make_fastdiv((uint32_t)std::max<int32_t>(P->block_band.bs, 1));
  a.bw = make_fastdiv((uint32_t)(P->band.l + P->band.u + 1));
  const size_t sm = color_table_smem(P);
  const int64_t tiles = (a.total + kBbTile - 1) / kBbTile;
  // a store stream: an oversubscribed grid, as for the other band kernels
  const int grid = oversubscribed_grid(P, diff_scatter_block_band<CT, MODE>, sm, tiles, 16);
  ScatterTimer tm(P, g.s);
  diff_scatter_block_band<CT, MODE><<<grid, kThreads, sm, g.s>>>(a);
  return FDB_OK;
}

// block-dense: every slot of the columns of the group's colours, and (first group of rank 0) of the columns without a
// valid colour: storage order, block column from the slab starts
template <typename CT, int MODE>
static fdb_status scatter_block_dense(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  BlockDenseArgs a{};
  a.jcolor = P->colors.jcolor; a.boff = P->block_band.off; a.start = P->block_band.start; a.fx = g.fx; a.Fp = g.Fp;
  a.Fm = g.Fm; a.eps = P->steps.eps; a.local_of = P->colors.local_of; a.J = g.J; a.total = P->j_len; a.ldF = g.ldF;
  a.C = P->colors.C; a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G;
  a.write_other = g.first ? 1 : 0;
  a.nblocks = P->block_band.nblocks; a.l = (int32_t)P->band.l; a.u = (int32_t)P->band.u;
  a.bs = P->block_band.bs;
  a.block_cyclic = P->block_band.cyclic ? 1 : 0;
  a.bw = make_fastdiv((uint32_t)(P->band.l + P->band.u + 1));
  const size_t sm = color_table_smem(P);
  const int64_t tiles = (a.total + kBbTile - 1) / kBbTile;
  const int grid = oversubscribed_grid(P, diff_scatter_block_dense<CT, MODE>, sm, tiles, 16);
  ScatterTimer tm(P, g.s);
  diff_scatter_block_dense<CT, MODE><<<grid, kThreads, sm, g.s>>>(a);
  return FDB_OK;
}

// diagonal storage: every slot of the columns of the group's colours, and (first group of rank 0) of the columns without
// a valid colour: storage order, closed-form diagonal and (row, column)
template <typename CT, int MODE>
static fdb_status scatter_diagonals(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  DiagArgs a{};
  a.fx = g.fx; a.Fp = g.Fp; a.Fm = g.Fm; a.eps = P->steps.eps; a.local_of = P->colors.local_of; a.J = g.J;
  a.total = P->j_len; a.sub_end = P->band.l * (P->n - 1); a.main_end = a.sub_end + P->n; a.ldF = g.ldF;
  a.C = P->colors.C; a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G;
  a.write_other = g.first ? 1 : 0;
  const size_t sm = color_table_smem(P);
  const int64_t tiles = (a.total + kDgTile - 1) / kDgTile;
  ScatterTimer tm(P, g.s);
  return dispatch_colors<CT>(P, [&](auto cs) -> fdb_status {
    using CS = decltype(cs);
    // a store stream: an oversubscribed grid, as for the other band kernels
    const int grid = oversubscribed_grid(P, diff_scatter_diagonals<CS, MODE>, sm, tiles, 16);
    diff_scatter_diagonals<CS, MODE><<<grid, kThreads, sm, g.s>>>(a, cs);
    return FDB_OK;
  });
}

// CSR nzval: every entry of the columns of the group's colours, and (first group of rank 0) of the columns without a
// valid colour: storage order, row from the row pointer
template <typename CT, int MODE>
static fdb_status scatter_csr(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  CsrArgs a{};
  a.rowptr = P->csr.rowptr; a.colval = P->csr.colval; a.fx = g.fx; a.Fp = g.Fp; a.Fm = g.Fm; a.eps = P->steps.eps;
  a.local_of = P->colors.local_of; a.J = g.J; a.ldF = g.ldF;
  a.m = (int32_t)P->m; a.nnz = (int32_t)P->j_len;
  a.C = P->colors.C; a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G;
  // single group on a single rank: every valid colour is resident at its own slab (the first group of rank 0)
  a.full = P->scratch.n_groups == 1 && P->world == 1 ? 1 : 0;
  a.write_other = g.first ? 1 : 0;
  const size_t sm = color_table_smem(P);
  const int64_t tiles = (P->j_len + kCsrTile - 1) / kCsrTile;
  ScatterTimer tm(P, g.s);
  return dispatch_colors<CT>(P, [&](auto cs) -> fdb_status {
    using CS = decltype(cs);
    const int grid = oversubscribed_grid(P, diff_scatter_csr<CS, MODE>, sm, tiles, 16);
    diff_scatter_csr<CS, MODE><<<grid, kThreads, sm, g.s>>>(a, cs);
    return FDB_OK;
  });
}

// band data or a dense J of a banded sparsity: one timed region per group, the pre-division pass (when used) and the
// band kernel
template <typename CT, int MODE>
static fdb_status scatter_band(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  BandArgs a{};
  ScatterTimer tm(P, g.s);
  a.jcolor = P->colors.jcolor; a.fx = g.fx; a.Fp = g.Fp; a.Fm = g.Fm; a.eps = P->steps.eps; a.local_of = P->colors.local_of;
  a.J = g.J; a.C = P->colors.C; a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G;
  a.write_other = g.first ? 1 : 0;
  a.to_dense = P->jkind == FDB_J_DENSE ? 1 : 0;
  a.ldF = g.ldF; a.ldJ = P->ldJ; a.m = P->m; a.n = P->n; a.l = P->band.l; a.u = P->band.u;
  const int64_t w = P->band.l + P->band.u + 1;
  a.cols_per_tile = std::max<int64_t>(1, 4096 / w);
  // every (colour, row) quotient lands in about (l+u+1)/C columns of the whole-band fill: when that reuse is >= 2,
  // divide once per (colour, row) in place (the reference's own `vfx1 = (vfx1 - vfx)/eps` pass) and let the band
  // kernel copy; otherwise divide at gather time.
  // On C3 (16 GB band, 5 colours) the flat stream over pre-divided slabs with 4-deep batched loads was kept over
  // warp-per-column, dividing at gather time, row-stationary, colour-grouped columns and block-per-column forms.
  const bool prediv = MODE != kComplex && w >= 64 && w >= 2 * (int64_t)P->colors.C;
  if (prediv) {
    dim3 grid((unsigned)std::max(1, std::min(P->grid(P->m), std::max(1, P->sm_count * 8 / (int)g.G))), (unsigned)g.G);
    diff_slabs<MODE><<<grid, kThreads, 0, g.s>>>(g.Fp, MODE == kCentral ? g.Fm : g.fx, P->steps.eps, P->colors.d_local + g.l0, P->m, g.ldF);
    P->cnt.kernel_launches += 1;
  }
  if (w >= 64) {
    // wide band: one warp per column
    const size_t sm = color_table_smem(P);
    if (!a.to_dense && (reinterpret_cast<uintptr_t>(g.J) & 15) == 0) {
      // band-data target: aligned flat stream, 16-byte stores
      const int32_t CH = (int32_t)std::min<int64_t>(2048, w & ~(int64_t)1);
      const int64_t nchunks = (w * P->n + CH - 1) / CH;
      if (prediv) {
        // unlike the read-modify kernels (C2: no gain), this store-dominated stream gains from an oversubscribed grid
        // (64x the resident wave); a bare store-only stream (fdbs_store_probe) shows the same trend
        const int grid = oversubscribed_grid(P, diff_scatter_band_flat<CT, kCopy>, sm, (nchunks + 7) / 8, 64);
        diff_scatter_band_flat<CT, kCopy><<<grid, kThreads, sm, g.s>>>(a, CH);
      } else {
        launch_resident(P, diff_scatter_band_flat<CT, MODE>, (nchunks + 7) / 8, sm, g.s, a, CH);
      }
    } else if (prediv) launch_resident(P, diff_scatter_band_wide<CT, kCopy>, (P->n + 7) / 8, sm, g.s, a);
    else launch_resident(P, diff_scatter_band_wide<CT, MODE>, (P->n + 7) / 8, sm, g.s, a);
  } else {
    diff_scatter_band<CT, MODE><<<P->grid(P->n, (int)a.cols_per_tile, 16), kThreads, 0, g.s>>>(a);
  }
  return FDB_OK;
}

// CSC in storage order and COO: one pass over the entries.  Which kernel runs also depends on the call's pointers.
template <typename CT, int MODE>
static fdb_status scatter_entries(const ScatterGroup &g) {
  fdb_plan *P = g.P;
  ScatterArgs a{};
  a.row = P->entries.row32; a.ecolor = P->entries.ecolor; a.dest = P->entries.dest; a.fx = g.fx; a.Fp = g.Fp; a.Fm = g.Fm; a.eps = P->steps.eps;
  a.local_of = P->colors.local_of; a.J = g.J; a.peers = P->peers.d; a.n_peers = P->peers.n; a.C = P->colors.C;
  a.l0 = (int32_t)g.l0; a.G = (int32_t)g.G;
  a.write_invalid_zero = (g.first && P->colors.has_invalid) ? 1 : 0;
  a.ldF = g.ldF; a.E = P->colors.E;
  a.j_aligned = (reinterpret_cast<uintptr_t>(g.J) & 15) == 0 && P->peers.aligned;
  // random patterns (mean row jump beyond a few cache lines): slab gathers are read-once
  a.hi_stream = P->tune.hi_stream >= 0 ? P->tune.hi_stream : (P->entries.mean_row_jump > 4096.0 ? 1 : 0);
  const size_t sm = color_table_smem(P);
  ScatterTimer tm(P, g.s);
  const int64_t tiles = (P->colors.E + kTile - 1) / kTile;
  // single group on a single rank: every valid colour is resident -> the FULL variant (no ownership tests)
  const bool full = P->scratch.n_groups == 1 && P->world == 1 && P->peers.n == 0;
  // staged form (identity destination): needs 16-byte aligned sources and (forward) ldF readable doubles behind f(x)
  bool staged = P->entries.dest == nullptr && full && P->staged.on && MODE != kComplex;
  if (staged && MODE == kForward)
    staged = (reinterpret_cast<uintptr_t>(g.fx) & 15) == 0 && ((P->m & 1) == 0 || g.fx == P->scratch.fx_own);
  if (staged) {
    if constexpr (MODE != kComplex) {
      StagedArgs sa{};
      sa.row16 = P->staged.row16; sa.tile_w0 = P->staged.tile_w0; sa.row32 = P->entries.row32;
      sa.fx = g.fx; sa.Fp = g.Fp; sa.Fm = g.Fm; sa.eps = P->steps.eps; sa.J = g.J; sa.C = P->colors.C; sa.W = P->staged.W;
      sa.ldF = g.ldF; sa.src_len = P->scratch.ldF; sa.E = P->colors.E; sa.j_aligned = a.j_aligned; sa.claim = P->staged.claim;
      sa.reverse = P->tune.reverse & 1;
      sa.colptr32 = P->entries.colptr32; sa.l = P->staged.band_l; sa.n = (int32_t)P->n;
      sa.col_a = P->staged.band_col_a; sa.col_b = P->staged.band_col_b; sa.e_a = P->staged.band_e_a; sa.e_b = P->staged.band_e_b;
      sa.w = make_fastdiv((uint32_t)P->staged.band_w);
      const int nwin = MODE == kCentral ? 2 * P->colors.C : P->colors.C + 1;
      auto smem = [&](int stages) { return (size_t)stages * nwin * P->staged.W * 8 + kStageCtlBytes + (size_t)P->colors.C * 8; };
      sa.stages = smem(P->tune.stages) > (size_t)kStageMaxSmem ? 2 : P->tune.stages;
      const size_t ssm = smem(sa.stages);
      // variants (FDB_STAGED_VARIANT = 8n | 6p | 6n | 6e): resident blocks per SM x index prefetch / empty mbarrier
      const char v0 = P->tune.staged_variant[0], v1 = P->tune.staged_variant[1];
      auto go = [&](auto kern, auto cs) -> fdb_status {
        CU(launch_pdl(kern, resident_grid(P, kern, ssm, tiles), ssm, g.s, sa, cs));
        return FDB_OK;
      };
      if (P->staged.band) {
        return dispatch_colors<CT>(P, [&](auto cs) -> fdb_status {
          using CS = decltype(cs);
          if (v0 == '8') return go(diff_scatter_staged<CS, MODE, 8, false, false, false, true>, cs);
          if (v1 == 'e') return go(diff_scatter_staged<CS, MODE, 6, false, false, true, true>, cs);
          return go(diff_scatter_staged<CS, MODE, 6, false, false, false, true>, cs);
        });
      }
      using CS = TableColors<CT>;          // per-entry colours
      const CS ec{(const CT *)P->entries.ecolor};
      if (P->staged.packed && v1 == 'e') return go(diff_scatter_staged<CS, MODE, 6, false, true, true>, ec);
      if (P->staged.packed) return go(diff_scatter_staged<CS, MODE, 6, false, true>, ec);
      if (v0 == '8') return go(diff_scatter_staged<CS, MODE, 8, false, false>, ec);
      if (v1 == 'n') return go(diff_scatter_staged<CS, MODE, 6, false, false>, ec);
      return go(diff_scatter_staged<CS, MODE, 6, true, false>, ec);
    }
  }
  if (P->entries.dest != nullptr) launch_resident(P, diff_scatter_dest<CT, MODE>, (P->colors.E + kThreads - 1) / kThreads, sm, g.s, a);
  else if (full) launch_resident(P, diff_scatter_ident<CT, MODE, true, kScatterMinBlocks>, tiles, sm, g.s, a);
  else launch_resident(P, diff_scatter_ident<CT, MODE, false, kScatterMinBlocks>, tiles, sm, g.s, a);
  return FDB_OK;
}

// The scatter of one colour group (G = 0: once, on a rank that owns no colour).  Whether a family launches is decided
// here and counted here; what it launches, and which part of it is timed, is its launcher's.
template <typename CT, int MODE>
static fdb_status scatter(Scatter family, const ScatterGroup &g) {
  fdb_plan *P = g.P;
  // colour-major lists: rank 0 zeroes the entries of the columns without a valid colour with its first group; owning no
  // colour, it does so only where this call does not zero-fill J (peer stores, a shared J)
  if (family == Scatter::lists && g.first && (g.G > 0 || P->peers.n > 0 || P->shared_J)) zero_uncoloured_slots(g);
  // a rank that owns no colour launches the block-banded, block-dense or CSR scatter of rank 0 alone: the columns without
  // a valid colour
  const bool self_defining = family == Scatter::block_band || family == Scatter::block_dense || family == Scatter::csr;
  if (g.G == 0 && !(self_defining && g.first)) return FDB_OK;
  switch (family) {   // (a group has a colour: C > 0 and n > 0, so band and diagonal storage have slots)
    case Scatter::none: return FDB_OK;
    case Scatter::lists:
      if (P->cm.start_h[(size_t)(g.l0 + g.G)] == P->cm.start_h[(size_t)g.l0]) return FDB_OK;   // empty lists
      TRY(scatter_lists<MODE>(g)); break;
    case Scatter::block_band: if (P->block_band.w * P->n == 0) return FDB_OK; TRY((scatter_block_band<CT, MODE>(g))); break;
    case Scatter::block_dense: if (P->j_len == 0) return FDB_OK; TRY((scatter_block_dense<CT, MODE>(g))); break;
    case Scatter::diagonals: TRY((scatter_diagonals<CT, MODE>(g))); break;
    case Scatter::band: TRY((scatter_band<CT, MODE>(g))); break;
    case Scatter::csr: if (P->j_len == 0) return FDB_OK; TRY((scatter_csr<CT, MODE>(g))); break;
    case Scatter::entries: if (P->colors.E == 0) return FDB_OK; TRY((scatter_entries<CT, MODE>(g))); break;
  }
  P->cnt.kernel_launches += 1;
  P->cnt.scatter_launches += 1;
  return FDB_OK;
}

template <typename CT, int MODE>
static fdb_status run_colored(fdb_plan *P, fdb_fn f, void *ctx, const double *x, double *J, double *fx,
                              const double *f_in, double relstep, double absstep, double dir, cudaStream_t s) {
  constexpr bool CENTRAL = MODE == kCentral;
  constexpr bool COMPLEX = MODE == kComplex;
  // strides, in doubles, of one f! output slab / one perturbed point (complex128 in complex-step mode)
  const int64_t sF = COMPLEX ? 2 * P->scratch.ldF : P->scratch.ldF, sX = COMPLEX ? 2 * P->scratch.ldx : P->scratch.ldx;
  const int64_t n_local = (int64_t)P->colors.local.size();
  const Scatter family = scatter_family(P);
  // With peer buffers set the caller zero-fills J and synchronises the ranks BEFORE the call: a memset here would race
  // with the peers' stores.
  if (!scatter_defines_J(P, n_local) && P->peers.n == 0 && !P->shared_J && P->j_len > 0) TRY(zero_J(P, J, s));
  // build the perturbed points of local colours [li0, li0+kc) into the point buffers (one pass over x per 4 colours)
  auto perturb_window = [&](int64_t li0, int64_t kc, cudaStream_t ps) -> fdb_status {
      for (int64_t q0 = 0; q0 < kc; q0 += kPerturbMaxPoints) {
        PerturbArgs pa{};
        pa.x = x; pa.eps = P->steps.eps;
        pa.xp = P->scratch.xp + q0 * sX; pa.xm = CENTRAL ? P->scratch.xm + q0 * sX : nullptr;
        pa.n = P->n; pa.ldx = sX; pa.C = P->colors.C; pa.drift = (P->no_drift || P->oop.on) ? 0 : 1; pa.oop = P->oop.on;
        pa.reverse = (P->tune.reverse >> 1) & 1;
        pa.kcount = (int32_t)std::min<int64_t>(kPerturbMaxPoints, kc - q0);
        for (int32_t q = 0; q < pa.kcount; ++q) pa.k[q] = P->colors.local[(size_t)(li0 + q0 + q)];
        pa.aligned = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(P->scratch.xp) |
                       reinterpret_cast<uintptr_t>(P->scratch.xm)) & 15) == 0 && (P->scratch.ldx & 1) == 0;
        const size_t sm = P->colors.C <= kPerturbSmemColors ? (size_t)P->colors.C * sizeof(double) : 0;
        const int64_t tiles = (P->n + kTile - 1) / kTile;
        TRY(dispatch_colors<CT>(P, [&](auto cs) -> fdb_status {
          using CS = decltype(cs);
          if (COMPLEX) {
            if (pa.kcount == 1) perturb_complex<CS, 1><<<P->grid(P->n), kThreads, 0, ps>>>(pa, cs);
            else perturb_complex<CS, kPerturbMaxPoints><<<P->grid(P->n), kThreads, 0, ps>>>(pa, cs);
          } else {
            // store-heavy (NP points written per element read): an oversubscribed grid (16x the resident wave), like the
            // band and dense-column kernels
            auto go = [&](auto kern) { return launch_pdl(kern, oversubscribed_grid(P, kern, sm, tiles, 16), sm, ps, pa, cs); };
            if (pa.kcount == 1) CU(go(perturb_colors<CS, CENTRAL, 1>));
            else CU(go(perturb_colors<CS, CENTRAL, kPerturbMaxPoints>));
          }
          return FDB_OK;
        }));
        P->cnt.kernel_launches += 1;
      }
      return FDB_OK;
  };

  // forward mode without f_in: f(x) (jacobians.jl:541) and the step-size pass are independent — the eps kernels run on the
  // side stream beside the user's f(x) (a parallel branch of the CUDA graph)
  bool eps_beside_fx = MODE == kForward && !f_in && !P->steps.ext && P->overlap.side && P->overlap.ev_fork && P->colors.C > 0;
  if (P->tune.no_eps_overlap) eps_beside_fx = false;
  // ... and so is the first window of perturbed points, which reads x and the step sizes only: it is built on the side
  // stream behind the ε pass, and the call's stream waits for both before the first f!(xp).  f! is still called in the
  // reference's order, f(x) first.
  const bool perturb_beside_fx = eps_beside_fx && n_local > 0;
  if (P->steps.ext) {
    // sharded runs: the step sizes of the FULL x come from outside (fdb_color_eps on the full vector)
    if (P->colors.C > 0) CU(cudaMemcpyAsync(P->steps.eps, P->steps.ext, (size_t)P->colors.C * 8, cudaMemcpyDeviceToDevice, s));
  } else if (eps_beside_fx) {
    CU(cudaEventRecord(P->overlap.ev_fork, s));
    CU(cudaStreamWaitEvent(P->overlap.side, P->overlap.ev_fork, 0));
    TRY(run_eps<CT>(P, x, relstep, absstep, dir, P->overlap.side));
    if (perturb_beside_fx) TRY(perturb_window(0, std::min<int64_t>(P->scratch.pbatch, n_local), P->overlap.side));
    CU(cudaEventRecord(P->overlap.ev_eps, P->overlap.side));
  } else {
    TRY(run_eps<CT>(P, x, relstep, absstep, dir, s));
  }
  const double *vfx = nullptr;
  if (MODE == kForward) {
    if (f_in) vfx = f_in;                                  // jacobians.jl:543-544
    else { TRY(call_f(P, f, ctx, fx, x, 1, s)); vfx = fx; } // :541-542
  }
  if (eps_beside_fx) CU(cudaStreamWaitEvent(s, P->overlap.ev_eps, 0));
  // colour-major lists, forward: f(x) once into list order (read as a coalesced stream by every colour's launch)
  if (MODE == kForward && family == Scatter::lists && P->cm.fx && n_local > 0) {
    const int64_t cnt = P->cm.start_h[(size_t)n_local];
    if (cnt > 0) {
      ScatterTimer tm(P, s);            // part of the diff+scatter formulation: timed with it
      gather_fx_cm<<<P->grid(cnt, kThreads * 4, 16), kThreads, 0, s>>>(P->cm.row, vfx, cnt, P->cm.fx);
      P->cnt.kernel_launches += 1;
    }
  }
  // Double-buffered overlap (multi-GPU, column lists): group g's f! outputs live in buffer (g & 1); its scatter — the
  // kernel that also pushes the values to the peers over NVLink — runs on a side stream while the main stream already
  // evaluates group g+1 into the other buffer.  Events order buffer reuse; everything joins the caller's stream at the end.
  const bool overlap = P->overlap.double_buffer && P->overlap.side != nullptr;

  // colours ascending (jacobians.jl:547).  Points are built in windows of `pbatch` colours, f! is called once per point
  // (reference order f(fx1,x1) then f(fx,x) per colour, :563 / :605-606) or once per `batch` points for batch-capable
  // callbacks; a group's scatter is launched as soon as its `slabs` outputs are complete.
  int64_t li = 0;
  while (li < n_local) {
    const int64_t g = li / P->scratch.slabs, g0 = g * P->scratch.slabs, gend = std::min<int64_t>(g0 + P->scratch.slabs, n_local);
    if (li % P->scratch.pbatch == 0 && !(li == 0 && perturb_beside_fx)) TRY(perturb_window(li, std::min<int64_t>(P->scratch.pbatch, n_local - li), s));
    const int64_t wend = std::min<int64_t>((li / P->scratch.pbatch + 1) * P->scratch.pbatch, n_local);
    const int64_t fc = std::min<int64_t>(P->scratch.batch, std::min<int64_t>(wend - li, gend - li));
    const int64_t gb = overlap ? (g & 1) * P->scratch.slabs * sF : 0;           // this group's output buffer
    if (overlap && li == g0 && g >= 2) CU(cudaStreamWaitEvent(s, P->overlap.ev_scat[g & 1], 0));   // buffer free again?
    TRY(call_f(P, f, ctx, P->scratch.Fp + gb + (li - g0) * sF, P->scratch.xp + (li % P->scratch.pbatch) * sX, fc, s));
    if (CENTRAL) TRY(call_f(P, f, ctx, P->scratch.Fm + gb + (li - g0) * sF, P->scratch.xm + (li % P->scratch.pbatch) * sX, fc, s));
    li += fc;
    if (li == gend) {
      const ScatterGroup grp{P, J, vfx, P->scratch.Fp + gb, CENTRAL ? P->scratch.Fm + gb : nullptr, sF, overlap ? P->overlap.side : s,
                             g0, gend - g0, g == 0 && P->rank == 0};
      if (overlap) {
        CU(cudaEventRecord(P->overlap.ev_f[g & 1], s));
        CU(cudaStreamWaitEvent(P->overlap.side, P->overlap.ev_f[g & 1], 0));
      }
      TRY((scatter<CT, MODE>(family, grp)));
      if (overlap) CU(cudaEventRecord(P->overlap.ev_scat[g & 1], P->overlap.side));
    }
  }
  if (overlap) {   // join the side stream back into the caller's stream
    const int64_t ng = (n_local + P->scratch.slabs - 1) / P->scratch.slabs;
    for (int64_t b = 0; b < std::min<int64_t>(ng, 2); ++b) CU(cudaStreamWaitEvent(s, P->overlap.ev_scat[b], 0));
  }
  if (n_local == 0) TRY((scatter<CT, MODE>(family, {P, J, vfx, P->scratch.Fp, P->scratch.Fm, sF, s, 0, 0, P->rank == 0})));
  CU(cudaGetLastError());
  return FDB_OK;
}

template <int MODE>
static fdb_status run_dense(fdb_plan *P, fdb_fn f, void *ctx, const double *x, double *J, double *fx, const double *f_in,
                            double relstep, double absstep, double dir, cudaStream_t s) {
  constexpr bool CENTRAL = MODE == kCentral;
  constexpr bool COMPLEX = MODE == kComplex;
  const int64_t sF = COMPLEX ? 2 * P->scratch.ldF : P->scratch.ldF, sX = COMPLEX ? 2 * P->scratch.ldx : P->scratch.ldx;
  const int64_t ncl = P->columns.end - P->columns.begin;
  const double *vfx = nullptr;
  if (MODE == kForward) {
    if (f_in) vfx = f_in;
    else { TRY(call_f(P, f, ctx, fx, x, 1, s)); vfx = fx; }
  }
  if (ncl == 0) return FDB_OK;
  const int32_t B = (int32_t)P->scratch.batch;
  if (COMPLEX) {
    // epsilon = eps(eltype(x)) for every column (jacobians.jl:624); X[b] = complex(x)
    fill_value<<<(int)((ncl + kThreads - 1) / kThreads), kThreads, 0, s>>>(P->columns.eps, ncl, DBL_EPSILON);
    replicate_x_complex<<<P->grid(P->n), kThreads, 0, s>>>(x, P->n, sX, B, P->scratch.xp);
  } else {
    // out-of-place plans: the forward rule, dir included, in central mode too (jacobians.jl:358)
    component_eps<<<(int)((ncl + kThreads - 1) / kThreads), kThreads, 0, s>>>(x, P->columns.begin, ncl, CENTRAL && !P->oop.on ? 1 : 0,
                                                                            relstep, absstep, dir, P->columns.eps);
    replicate_x<<<P->grid(P->n), kThreads, 0, s>>>(x, P->n, P->scratch.ldx, B, P->scratch.xp);
  }
  P->cnt.kernel_launches += 2;
  int64_t prev_c0 = 0;
  int32_t prevB = 0;
  for (int64_t c0l = 0; c0l < ncl; c0l += B) {
    const int32_t kc = (int32_t)std::min<int64_t>(B, ncl - c0l);
    const int64_t c0 = P->columns.begin + c0l;
    const int sb = (std::max(kc, prevB) + kThreads - 1) / kThreads;
    if (COMPLEX) set_components_complex<<<sb, kThreads, 0, s>>>(x, P->columns.eps, c0l, c0, prev_c0, kc, prevB, sX, P->scratch.xp);
    else set_components<<<sb, kThreads, 0, s>>>(x, P->columns.eps, c0l, c0, prev_c0, kc, prevB, P->scratch.ldx, 1.0, P->scratch.xp);
    TRY(call_f(P, f, ctx, P->scratch.Fp, P->scratch.xp, kc, s));                         // f(fx1, x1)   jacobians.jl:553 / :594 / :629
    if (CENTRAL) {
      set_components<<<sb, kThreads, 0, s>>>(x, P->columns.eps, c0l, c0, 0, kc, 0, P->scratch.ldx, -1.0, P->scratch.xp);
      TRY(call_f(P, f, ctx, P->scratch.Fm, P->scratch.xp, kc, s));                       // f(fx, x1)    :596
      P->cnt.kernel_launches += 1;
    }
    // a store-heavy stream (24 bytes moved per 8 written): many small blocks rather than one resident wave — each thread
    // handles about four row pairs (see the band kernel's grid note)
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((P->m / 2 + kThreads * 4 - 1) / (kThreads * 4), P->tune.cols_gx));
    dim3 grid((unsigned)gx, (unsigned)kc);
    {
      const double *lo_ptr = CENTRAL ? P->scratch.Fm : vfx;
      const int pairs_ok = ((reinterpret_cast<uintptr_t>(J + c0l * P->ldJ) | reinterpret_cast<uintptr_t>(lo_ptr) |
                             reinterpret_cast<uintptr_t>(P->scratch.Fp)) & 15) == 0 && (P->ldJ & 1) == 0 && (sF & 1) == 0;
      ScatterTimer tm(P, s);
      auto go = [&](auto kern) { kern<<<grid, kThreads, 0, s>>>(P->scratch.Fp, lo_ptr, P->columns.eps, c0l, kc, P->m, sF, P->ldJ, J + c0l * P->ldJ, pairs_ok); };
      // independent 16-byte loads in flight per thread before the first quotient (C5 shape: 4 central, 2 forward)
      const int depth = P->tune.cols_depth ? P->tune.cols_depth : (CENTRAL ? 4 : 2);
      if (depth == 4) go(diff_columns<MODE, 4>);
      else if (depth == 2) go(diff_columns<MODE, 2>);
      else go(diff_columns<MODE, 1>);
    }
    P->cnt.kernel_launches += 2;
    P->cnt.scatter_launches += 1;
    prev_c0 = c0;
    prevB = kc;
  }
  CU(cudaGetLastError());
  return FDB_OK;
}

// The call as enqueued by `eager(stream)`, or — use_graph — a CUDA-graph replay of it: the launch sequence depends only on
// the plan and on the arguments in `key` (step sizes are computed on the device inside the graph), so it is captured once
// and re-launched while the key stays the same.
template <typename F>
static fdb_status run_maybe_graph(fdb_plan *P, const GraphKey &key, cudaStream_t s, const char *what, F &&eager) {
  if (!P->graph.use || P->timing.on) return eager(s);
  if (!P->graph.exec || !(key == P->graph.key)) {
    if (P->graph.exec) { cudaGraphExecDestroy(P->graph.exec); P->graph.exec = nullptr; }
    if (!P->graph.stream) CU(cudaStreamCreateWithFlags(&P->graph.stream, cudaStreamNonBlocking));
    const fdb_counters_t before = P->cnt;
    CU(cudaStreamBeginCapture(P->graph.stream, cudaStreamCaptureModeThreadLocal));
    const fdb_status st = eager(P->graph.stream);
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(P->graph.stream, &graph);
    if (st != FDB_OK) { if (graph) cudaGraphDestroy(graph); cudaGetLastError(); return st; }
    if (e != cudaSuccess || !graph) {
      cudaGetLastError();
      return fail(FDB_ERR_CUDA, "stream capture of the %s failed (%s): the f! callback must be capture-safe "
                                "(enqueue-only, no allocation) when use_graph is set", what, cudaGetErrorString(e));
    }
    e = cudaGraphInstantiate(&P->graph.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) { P->graph.exec = nullptr; return fail(FDB_ERR_CUDA, "cudaGraphInstantiate: %s", cudaGetErrorString(e)); }
    P->graph.key = key;
    // what one replay amounts to (the capture pass itself launched nothing)
    P->graph.delta.f_points = P->cnt.f_points - before.f_points;
    P->graph.delta.f_invocations = P->cnt.f_invocations - before.f_invocations;
    P->graph.delta.kernel_launches = P->cnt.kernel_launches - before.kernel_launches;
    P->graph.delta.scatter_launches = P->cnt.scatter_launches - before.scatter_launches;
    P->cnt = before;
  }
  CU(cudaGraphLaunch(P->graph.exec, s));
  P->cnt.f_points += P->graph.delta.f_points;
  P->cnt.f_invocations += P->graph.delta.f_invocations;
  P->cnt.kernel_launches += P->graph.delta.kernel_launches;
  P->cnt.scatter_launches += P->graph.delta.scatter_launches;
  return FDB_OK;
}

extern "C" {

static fdb_status jacobian_eager(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, double *d_J, double *fx,
                                 const double *d_f_in, double relstep, double absstep, double dir, cudaStream_t s) {
  return dispatch_mode(P->fdtype, [&](auto mode) -> fdb_status {
    constexpr int MODE = decltype(mode)::value;
    if (P->sp_kind == SP_NONE) return run_dense<MODE>(P, f, ctx, d_x, d_J, fx, d_f_in, relstep, absstep, dir, s);
    return dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
      return run_colored<decltype(tag), MODE>(P, f, ctx, d_x, d_J, fx, d_f_in, relstep, absstep, dir, s);
    });
  });
}

// A Jacobian call once check_call has accepted it (the complex, host-buffer, out-of-place and group entries included)
static fdb_status jacobian_run(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, double *d_J, double *d_fx,
                               const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  DeviceGuard g(P->device);
  if (!g.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", P->device);
  cudaStream_t s = (cudaStream_t)stream;
  // jacobians.jl:508-509 defaults
  resolve_steps(P->fdtype, relstep, absstep);
  double *fx = d_fx ? d_fx : P->scratch.fx_own;
  const GraphKey key{(void *)f, ctx, d_x, d_J, fx, d_f_in, relstep, absstep, dir, P->peers.n, P->peers.generation, P->steps.ext};
  const fdb_status st = run_maybe_graph(P, key, s, "Jacobian", [&](cudaStream_t cs) {
    return jacobian_eager(P, f, ctx, d_x, d_J, fx, d_f_in, relstep, absstep, dir, cs);
  });
  if (st == FDB_OK) P->cnt.jacobians += 1;
  return st;
}

fdb_status fdb_jacobian(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, double *d_J, double *d_fx,
                        const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  if ((P->n > 0 && !d_x) || (P->j_len > 0 && !d_J)) return fail(FDB_ERR_INVALID, "NULL x or J");
  TRY(check_call(P, Call::jacobian));
  return jacobian_run(P, f, ctx, d_x, d_J, d_fx, d_f_in, relstep, absstep, dir, stream);
}

fdb_status fdb_jacobian_complex(fdb_plan *P, fdb_fn_c f, void *ctx, const double *d_x, double *d_J, void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::jacobian_complex));
  if ((P->n > 0 && !d_x) || (P->j_len > 0 && !d_J)) return fail(FDB_ERR_INVALID, "NULL x or J");
  // same C signature up to the element type of the buffers: the complex128 slabs are handed over as raw pointers
  return jacobian_run(P, reinterpret_cast<fdb_fn>(f), ctx, d_x, d_J, nullptr, nullptr, FDB_STEP_DEFAULT, FDB_STEP_DEFAULT,
                      1.0, stream);
}

// ------------------------------------------------------------------------------------------------ step sizes on their own
// (column-block sharded runs: every shard perturbs with the step sizes of the FULL x — jacobians.jl:559-561 takes the
//  norm over all colour-k components)
fdb_status fdb_eps_plan_create(fdb_plan **plan, int64_t n, const int64_t *colorvec, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, 0, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->sp_kind = SP_EPS;
  TRY(setup_colors(P, colorvec));
  TRY(alloc_eps_buffers(P));
  // the same list-based eps pass as the Jacobian plans: a column block's external step sizes are then bit-identical to
  // the ones the unsharded plan computes for itself
  if (P->colors.C > kEpsRegColors && n > 0) TRY(build_color_lists(P));
  *plan = owner.release();
  return FDB_OK;
}

fdb_status fdb_color_eps(fdb_plan *P, const double *d_x, double relstep, double absstep, double dir, double *d_eps_out,
                         void *stream) {
  if (!P) return fail(FDB_ERR_INVALID, "NULL plan");
  TRY(check_call(P, Call::color_eps));
  if (P->n > 0 && !d_x) return fail(FDB_ERR_INVALID, "NULL x");
  DeviceGuard g(P->device);
  if (!g.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", P->device);
  cudaStream_t s = (cudaStream_t)stream;
  resolve_steps(P->fdtype, relstep, absstep);
  TRY(dispatch_ct(P->colors.bits, [&](auto tag) -> fdb_status {
    using CT = decltype(tag);
    return run_eps<CT>(P, d_x, relstep, absstep, dir, s);
  }));
  if (d_eps_out && P->colors.C > 0) CU(cudaMemcpyAsync(d_eps_out, P->steps.eps, (size_t)P->colors.C * 8, cudaMemcpyDeviceToDevice, s));
  return FDB_OK;
}

fdb_status fdb_plan_set_external_eps(fdb_plan *P, const double *d_eps) {
  if (!P) return fail(FDB_ERR_INVALID, "NULL plan");
  TRY(check_call(P, Call::set_external_eps));
  P->steps.ext = d_eps;
  return FDB_OK;
}

// ------------------------------------------------------------------------------------------------ JVP (src/jvp.jl:238-274)
fdb_status fdb_jvp_plan_create(fdb_plan **plan, int64_t m, int64_t n, const fdb_plan_opts *opts) {
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  if (P->fdtype == FDB_COMPLEX)
    return fail(FDB_ERR_UNSUPPORTED, "finite_difference_jvp doesn't support :complex-mode finite diff");   // jvp.jl:248-250
  P->sp_kind = SP_JVP;
  P->scratch.ldF = std::max<int64_t>(2, (m + 1) & ~(int64_t)1);
  P->scratch.ldx = std::max<int64_t>(2, (n + 1) & ~(int64_t)1);
  int64_t nb = std::max<int64_t>(1, std::min<int64_t>((n + kTile - 1) / kTile, (int64_t)P->sm_count * 8));
  P->steps.blocks = (int)nb;
  TRY(P->alloc_t(&P->steps.partial, (size_t)nb));
  TRY(P->alloc_t(&P->steps.ticket, 4));
  CU(cudaMemset(P->steps.ticket, 0, 16));
  TRY(P->alloc_t(&P->steps.eps, 2));
  TRY(P->alloc_t(&P->steps.sumsq, 2));
  TRY(P->alloc_t(&P->scratch.fx_own, (size_t)P->scratch.ldF));
  TRY(P->alloc_t(&P->scratch.xp, (size_t)P->scratch.ldx));
  P->alg_bytes = 24 * n + 24 * m;   // dot: 16n; point: 16n read + 8n write; quotient: 16m read + 8m write
  *plan = owner.release();
  return FDB_OK;
}

// plus_first: the out-of-place form's central order, f(x + eps v) then f(x - eps v) (jvp.jl:180-183); the in-place form
// evaluates the minus point first (:265-268)
static fdb_status jvp_run(fdb_plan *P, fdb_fn f, void *ctx, double *d_jvp, const double *d_x, const double *d_v, double *d_x1,
                          double *d_fx1, const double *d_f_in, double relstep, double absstep, double dir, void *stream,
                          bool plus_first) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::jvp));
  if ((P->n > 0 && (!d_x || !d_v)) || (P->m > 0 && !d_jvp)) return fail(FDB_ERR_INVALID, "NULL jvp, x or v");
  DeviceGuard g(P->device);
  if (!g.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", P->device);
  cudaStream_t s = (cudaStream_t)stream;
  resolve_steps(P->fdtype, relstep, absstep);                       // jvp.jl:245-246
  double *x1 = d_x1 ? d_x1 : P->scratch.xp;
  double *fx1 = d_fx1 ? d_fx1 : P->scratch.fx_own;
  const bool central = P->fdtype == FDB_CENTRAL;
  const int64_t n = P->n, m = P->m;
  const int al_xv = ((reinterpret_cast<uintptr_t>(d_x) | reinterpret_cast<uintptr_t>(d_v)) & 15) == 0;
  const int al_x1 = al_xv && (reinterpret_cast<uintptr_t>(x1) & 15) == 0;
  EpsParams prm{central ? 1 : 0, relstep, absstep, dir};
  const int64_t tiles = (n + kTile - 1) / kTile;
  const int grid_n = std::min(resident_grid(P, jvp_dot_eps, 0, tiles), P->steps.blocks);
  jvp_dot_eps<<<grid_n, kThreads, 0, s>>>(d_x, d_v, n, al_xv, prm, P->steps.partial, P->steps.ticket, P->steps.eps, P->steps.sumsq);   // :252-253
  P->cnt.kernel_launches += 1;
  const double *base = fx1;
  if (!central) {
    if (d_f_in) base = d_f_in;                                      // fx1 = f_in        :257-258
    else TRY(call_f(P, f, ctx, fx1, d_x, 1, s));                    // f(fx1, x)         :255
  } else if (plus_first) {
    jvp_point<<<resident_grid(P, jvp_point, 0, tiles), kThreads, 0, s>>>(d_x, d_v, P->steps.eps, 0, x1, n, al_x1);   // x + eps v :180
    TRY(call_f(P, f, ctx, d_jvp, x1, 1, s));                        // fx1 = f(x1)       :181
    jvp_point<<<resident_grid(P, jvp_point, 0, tiles), kThreads, 0, s>>>(d_x, d_v, P->steps.eps, 1, x1, n, al_x1);   // x - eps v :182
    TRY(call_f(P, f, ctx, fx1, x1, 1, s));                          // fx = f(x1)        :183
    jvp_quotient<<<P->grid(m), kThreads, 0, s>>>(d_jvp, fx1, P->steps.eps, 1, m);                                   // :184
    P->cnt.kernel_launches += 3;
    CU(cudaGetLastError());
    P->cnt.jacobians += 1;
    return FDB_OK;
  } else {
    jvp_point<<<resident_grid(P, jvp_point, 0, tiles), kThreads, 0, s>>>(d_x, d_v, P->steps.eps, 1, x1, n, al_x1);   // x1 = x - eps v :264
    P->cnt.kernel_launches += 1;
    TRY(call_f(P, f, ctx, fx1, x1, 1, s));                          // f(fx1, x1)        :265
  }
  jvp_point<<<resident_grid(P, jvp_point, 0, tiles), kThreads, 0, s>>>(d_x, d_v, P->steps.eps, 0, x1, n, al_x1);     // x1 = x + eps v :260/:266
  TRY(call_f(P, f, ctx, d_jvp, x1, 1, s));                          // f(jvp, x1)        :261/:267
  jvp_quotient<<<P->grid(m), kThreads, 0, s>>>(d_jvp, base, P->steps.eps, central ? 1 : 0, m);                        // :262/:268
  P->cnt.kernel_launches += 2;
  CU(cudaGetLastError());
  P->cnt.jacobians += 1;
  return FDB_OK;
}

fdb_status fdb_jvp(fdb_plan *P, fdb_fn f, void *ctx, double *d_jvp, const double *d_x, const double *d_v, double *d_x1,
                   double *d_fx1, const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  return jvp_run(P, f, ctx, d_jvp, d_x, d_v, d_x1, d_fx1, d_f_in, relstep, absstep, dir, stream, false);
}

// ------------------------------------------------------------------------------------------------ Hessian (src/hessians.jl:202-292)
// n above this would overflow the 64-bit sequence index 2n^2 + 1 long before any device could hold the work
static constexpr int64_t kHessMaxN = (int64_t)1 << 24;
// Cap on the points per f call.  scripts/hessian_bench.py's sweep at n = 1000 (fdbs_quartic; H100 80GB HBM3, 700 W; the
// run's output line is scripts/hessian_bench_h100.json): 64 -> 451 ms, 256 -> 119 ms, 1024 -> 30.4 ms, 4096 -> 10.8 ms per
// Hessian (requests above the cap are clamped to it).
static constexpr int64_t kHessBatchCap = 4096;

// First i-block of rank r of `world` (see fdb_hessian_plan_create in the header): i_0 = 0, i_world = n, and for
// 0 < r < world the i in [i_{r-1}, n] whose S(i) - 1 is nearest to r*T/world (T = 2n^2), ties to the smaller i.  The
// distance is compared exactly as |world*(S(i) - 1) - r*T| (below 2^56 for n <= 2^24, world <= 64).  S is increasing, so
// the nearest i is the first i whose S(i) - 1 reaches the target or the one before it.
static int64_t hess_rank_begin(int64_t n, int world, int r) {
  if (r >= world) return n;
  int64_t lo = 0;
  for (int k = 1; k <= r; ++k) {
    const int64_t target = (int64_t)k * 2 * n * n;
    int64_t a = lo, b = n;    // first i in [lo, n] with world*(S(i) - 1) >= target (n when none does)
    while (a < b) {
      const int64_t mid = (a + b) >> 1;
      if (world * (hess_block_start(mid, n) - 1) >= target) b = mid; else a = mid + 1;
    }
    if (a > lo && target - world * (hess_block_start(a - 1, n) - 1) <= world * (hess_block_start(a, n) - 1) - target) --a;
    lo = a;
  }
  return lo;
}

fdb_status fdb_hessian_plan_create(fdb_plan **plan, int64_t n, int64_t ldH, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (!opts || opts->fdtype != FDB_HCENTRAL)   // @assert fdtype == Val(:hcentral)   hessians.jl:206
    return fail(FDB_ERR_UNSUPPORTED, "finite_difference_hessian! supports fdtype = hcentral (%d) only", FDB_HCENTRAL);
  if (n < 0) return fail(FDB_ERR_INVALID, "negative dimension n=%lld", (long long)n);
  if (ldH < n) return fail(FDB_ERR_INVALID, "ldH < n");
  if (n > kHessMaxN) return fail(FDB_ERR_UNSUPPORTED, "Hessian plans need n <= %lld", (long long)kHessMaxN);
  if (opts->world > 64) return fail(FDB_ERR_INVALID, "Hessian plans take world <= 64");
  fdb_plan_opts o = *opts;
  o.fdtype = FDB_CENTRAL;   // new_plan validates the Jacobian fdtypes; the Hessian's is set below
  PlanPtr owner;
  TRY(new_plan(plan, owner, &o, 1, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->fdtype = FDB_HCENTRAL;
  P->sp_kind = SP_HESS;
  P->jkind = FDB_J_DENSE;
  P->ldJ = ldH;
  P->j_len = ldH * n;
  // this rank's i-blocks [i0, i1) (all of them on one device); it owns column i rows [i, n) and row i columns (i, n)
  const int64_t ib = hess_rank_begin(n, P->world, P->rank), ie = hess_rank_begin(n, P->world, P->rank + 1);
  const int64_t nb = ie - ib, own_points = hess_block_start(ie, n) - hess_block_start(ib, n);
  P->hess.i_begin = ib;
  P->hess.i_end = ie;
  P->hess.entries = nb * (2 * n - 1) - (ie * (ie - 1) - ib * (ib - 1));
  P->hess.off = hess_block_start(ib, n) - 1;
  // f(x) first (the diagonal needs it), then the rank's own points; rank 0 always evaluates f(x) (n = 0 included), a
  // rank > 0 without i-blocks evaluates nothing
  const bool idle = nb == 0 && P->rank > 0;
  P->hess.points = idle ? 0 : 1 + own_points;
  P->scratch.ldF = 1;
  P->scratch.ldx = std::max<int64_t>(2, (n + 1) & ~(int64_t)1);
  const int64_t budget = opts->scratch_bytes > 0 ? opts->scratch_bytes : (int64_t)8 << 30;
  // ONE budget for both buffers: the resident point rows X[0..B) take at most half of it, the value buffer V the rest
  int64_t batch = opts->max_batch > 1 ? opts->max_batch : 1;
  batch = std::max<int64_t>(1, std::min<int64_t>(batch, budget / 2 / (8 * P->scratch.ldx)));
  batch = std::min<int64_t>(std::min<int64_t>(batch, std::max<int64_t>(P->hess.points, 1)), kHessBatchCap);
  P->scratch.batch = batch;
  P->scratch.slabs = batch;
  // chunks of whole i-blocks whose values fit the budget (at least one i-block each), so that the <= 4 values of an
  // entry are always in the same chunk
  const int64_t cap = std::max<int64_t>((budget - batch * P->scratch.ldx * 8) / 8 - 1, 0);
  P->hess.chunks.assign(1, ib);
  int64_t max_vals = 0;
  for (int64_t i0 = ib; i0 < ie;) {
    int64_t i1 = i0 + 1;
    while (i1 < ie && hess_block_start(i1 + 1, n) - hess_block_start(i0, n) <= cap) ++i1;
    max_vals = std::max<int64_t>(max_vals, hess_block_start(i1, n) - hess_block_start(i0, n));
    P->hess.chunks.push_back(i1);
    i0 = i1;
  }
  if (nb == 0 && !idle) P->hess.chunks.push_back(ib);   // one chunk of no i-blocks: f(x) alone
  P->scratch.n_groups = (int64_t)P->hess.chunks.size() - 1;
  TRY(P->alloc_t(&P->hess.V, (size_t)(1 + max_vals)));
  TRY(P->alloc_t(&P->scratch.xp, (size_t)(batch * P->scratch.ldx)));
  TRY(P->alloc_t(&P->hess.eps, (size_t)std::max<int64_t>(n, 1)));
  // byte model per Hessian (this rank's share): values read back by the assembly, owned entries of H written, the
  // one-time replication of x into the B rows, and the patches (each changed component written once and restored once:
  // 2 per diagonal point, 4 per other point)
  const int64_t patched = 2 * own_points - 2 * nb;
  P->alg_bytes = idle ? 0 : 8 * P->hess.points + 8 * P->hess.entries + 8 * n * batch + 16 * patched;
  *plan = owner.release();
  return FDB_OK;
}

static fdb_status hessian_eager(fdb_plan *P, fdb_fn f, void *ctx, const double *x, double *H, double *fx_out,
                                double relstep, double absstep, cudaStream_t s) {
  const int64_t n = P->n, ldx = P->scratch.ldx;
  const int32_t B = (int32_t)P->scratch.batch;
  if (n > 0) {
    // eps_i = compute_epsilon(Val(:hcentral) / Val(:central), x_i, relstep, absstep) = max(relstep*|x_i|, absstep)  :223,234,252
    component_eps<<<(int)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>(x, 0, n, 1, relstep, absstep, 1.0, P->hess.eps);
    replicate_x<<<P->grid(n), kThreads, 0, s>>>(x, n, ldx, B, P->scratch.xp);
    P->cnt.kernel_launches += 2;
  }
  // p0 / p_end run over the rank's local sequence (point q > 0 is global point q + off, kernels_hessian.cuh); a chunk's
  // points sit at V[1 ..] whatever its rank
  const int64_t off = P->hess.off;
  int64_t prev_p0 = 0;
  int32_t prev_cnt = 0;
  for (size_t c = 0; c + 1 < P->hess.chunks.size(); ++c) {
    const int64_t i0 = P->hess.chunks[c], i1 = P->hess.chunks[c + 1];
    const int64_t cs = hess_block_start(i0, n) - off;
    const int64_t p_end = hess_block_start(i1, n) - off;
    for (int64_t p0 = c == 0 ? 0 : cs; p0 < p_end; p0 += B) {
      const int32_t cnt = (int32_t)std::min<int64_t>(B, p_end - p0);
      if (n > 0) {
        hess_patch<<<P->grid(std::max(cnt, prev_cnt)), kThreads, 0, s>>>(x, P->hess.eps, n, ldx, off, p0, cnt, prev_p0,
                                                                          prev_cnt, P->scratch.xp);
        P->cnt.kernel_launches += 1;
      }
      // f(x) (:209), f(_xpp), f(_xmm) (:233), f(_xpp), f(_xpm), f(_xmp), f(_xmm) (:268-269), in this order
      const int rc = f(ctx, P->hess.V + (p0 - cs + 1), P->scratch.xp, cnt, 1, ldx, (void *)s);
      P->cnt.f_invocations += 1;
      P->cnt.f_points += cnt;
      if (rc != 0) return fail(FDB_ERR_CALLBACK, "user f returned %d", rc);
      prev_p0 = p0;
      prev_cnt = cnt;
    }
    const int64_t tiles = hess_tiles(n, i0, i1);
    if (tiles > 0) {
      ScatterTimer tm(P, s);
      hess_assemble<<<P->grid(tiles, 1), kThreads, 0, s>>>(P->hess.V, P->hess.eps, n, i0, i1, tiles, H, P->ldJ);
      P->cnt.kernel_launches += 1;
      P->cnt.scatter_launches += 1;
    }
  }
  if (fx_out) CU(cudaMemcpyAsync(fx_out, P->hess.V, 8, cudaMemcpyDeviceToDevice, s));
  CU(cudaGetLastError());
  return FDB_OK;
}

fdb_status fdb_hessian(fdb_plan *P, fdb_fn f, void *ctx, const double *d_x, double *d_H, double *d_fx, double relstep,
                       double absstep, void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::hessian));
  if (P->n > 0 && (!d_x || !d_H)) return fail(FDB_ERR_INVALID, "NULL x or H");
  DeviceGuard g(P->device);
  if (!g.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", P->device);
  cudaStream_t s = (cudaStream_t)stream;
  if (P->hess.points == 0) {                 // a rank > 0 without i-blocks: no f call, no launch, d_fx untouched
    P->cnt.jacobians += 1;
    return FDB_OK;
  }
  resolve_steps(FDB_HCENTRAL, relstep, absstep);                    // hessians.jl:204-205
  const GraphKey key{(void *)f, ctx, d_x, d_H, d_fx, nullptr, relstep, absstep, 1.0, 0, 0, nullptr};
  const fdb_status st = run_maybe_graph(P, key, s, "Hessian", [&](cudaStream_t cs) {
    return hessian_eager(P, f, ctx, d_x, d_H, d_fx, relstep, absstep, cs);
  });
  if (st == FDB_OK) P->cnt.jacobians += 1;
  return st;
}

// ------------------------------------------------------------------------------------------------ derivatives with a
// scalar input per step size (src/derivatives.jl:197-233, src/gradients.jl:477-533; kernels_derivative.cuh)
// Scratch: the point rows xp (two rows of ldx doubles: x+eps and x-eps; complex: one complex128 row) and the f outputs
// F (two rows of ldF doubles: f(x+eps) and f(x) / f(x-eps); complex: one complex128 row).
static fdb_status create_derivative(fdb_plan **plan, int64_t m, int64_t n, bool elem, const fdb_plan_opts *opts) {
  if (!plan) return fail(FDB_ERR_INVALID, "plan output pointer is NULL");
  *plan = nullptr;
  if (opts && opts->fdtype == FDB_HCENTRAL)
    return fail(FDB_ERR_UNSUPPORTED, "derivative plans take fdtype forward, central or complex (hcentral is for Hessians)");
  if (opts && opts->world > 1) return fail(FDB_ERR_UNSUPPORTED, "derivative plans run on one device (world must be <= 1)");
  PlanPtr owner;
  TRY(new_plan(plan, owner, opts, m, n));
  fdb_plan *P = owner.get();
  DeviceGuard g(P->device);
  P->sp_kind = SP_DERIV;
  P->deriv.elem = elem;
  P->jkind = FDB_J_DENSE;
  P->j_len = m;
  P->ldJ = std::max<int64_t>(m, 1);
  P->scratch.batch = opts && opts->max_batch > 1 ? 2 : 1;
  P->scratch.ldx = std::max<int64_t>(2, (n + 1) & ~(int64_t)1);
  P->scratch.ldF = std::max<int64_t>(2, (m + 1) & ~(int64_t)1);
  TRY(P->alloc_t(&P->scratch.xp, (size_t)(2 * P->scratch.ldx)));
  TRY(P->alloc_t(&P->scratch.Fp, (size_t)(2 * P->scratch.ldF)));
  P->deriv.fcalls = P->fdtype == FDB_COMPLEX ? 1 : 2;
  // compulsory bytes per call: points pass (x read; one, two or one complex row written) + quotient pass (f rows and,
  // elementwise, x read; df written).  Complex reads the whole complex128 f row and no x.
  const int64_t pts = P->fdtype == FDB_FORWARD ? 16 : 24;
  const int64_t q = P->fdtype == FDB_COMPLEX || !elem ? 24 : 32;
  P->alg_bytes = pts * n + q * m;
  *plan = owner.release();
  return FDB_OK;
}

fdb_status fdb_derivative_plan_create(fdb_plan **plan, int64_t n, const fdb_plan_opts *opts) {
  return create_derivative(plan, n, n, true, opts);
}

fdb_status fdb_scalar_gradient_plan_create(fdb_plan **plan, int64_t m, const fdb_plan_opts *opts) {
  return create_derivative(plan, m, 1, false, opts);
}

}  // extern "C"

template <int MODE>
static fdb_status derivative_eager(fdb_plan *P, fdb_fn f, void *ctx, double *df, const double *x, const double *fx,
                                   const DerivSteps &st, cudaStream_t s) {
  const int64_t n = P->n, m = P->m;
  const int al_x = (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const int64_t tiles_n = (n + kTile - 1) / kTile, tiles_m = (m + kTile - 1) / kTile;
  if (n > 0) {
    deriv_points<MODE><<<resident_grid(P, deriv_points<MODE>, 0, tiles_n), kThreads, 0, s>>>(x, n, P->scratch.ldx, P->scratch.xp, st, al_x);
    P->cnt.kernel_launches += 1;
  }
  // f-call order of the reference: f(x+eps) first, then f(x) (forward without fx) or f(x-eps) (central)
  //   derivatives.jl:209-215,219-222 (per element) / gradients.jl:495-509,513-515
  // the two f rows of ldF doubles: f(x+eps), then f(x) / f(x-eps)
  double *const f_hi = P->scratch.Fp, *const f_lo = P->scratch.Fp + P->scratch.ldF;
  int64_t calls = 1;
  const double *fb = nullptr;
  if (MODE == kCentral && P->scratch.batch >= 2) {
    TRY(call_f(P, f, ctx, f_hi, P->scratch.xp, 2, s));                // both points in one call: rows 0 (+) and 1 (-)
    calls = 2;
    fb = f_lo;
  } else {
    TRY(call_f(P, f, ctx, f_hi, P->scratch.xp, 1, s));
    if (MODE == kCentral) {
      TRY(call_f(P, f, ctx, f_lo, P->scratch.xp + P->scratch.ldx, 1, s));
      calls = 2;
      fb = f_lo;
    } else if (MODE == kForward) {
      if (fx) fb = fx;
      else { TRY(call_f(P, f, ctx, f_lo, x, 1, s)); calls = 2; fb = f_lo; }
    }
  }
  P->deriv.fcalls = calls;
  if (m > 0) {
    const uintptr_t al = reinterpret_cast<uintptr_t>(df) | (fb ? reinterpret_cast<uintptr_t>(fb) : 0) |
                         (P->deriv.elem && MODE != kComplex ? reinterpret_cast<uintptr_t>(x) : 0);
    const int aligned = (al & 15) == 0;
    ScatterTimer tm(P, s);
    if (P->deriv.elem)
      deriv_quotient<MODE, true><<<resident_grid(P, deriv_quotient<MODE, true>, 0, tiles_m), kThreads, 0, s>>>(
          f_hi, fb, x, df, m, st, aligned);
    else
      deriv_quotient<MODE, false><<<resident_grid(P, deriv_quotient<MODE, false>, 0, tiles_m), kThreads, 0, s>>>(
          f_hi, fb, x, df, m, st, aligned);
    P->cnt.kernel_launches += 1;
    P->cnt.scatter_launches += 1;
  }
  CU(cudaGetLastError());
  return FDB_OK;
}

extern "C" {

// A derivative call once check_call has accepted it
static fdb_status derivative_run(fdb_plan *P, fdb_fn f, void *ctx, double *d_df, const double *d_x, const double *d_fx,
                                 double relstep, double absstep, double dir, void *stream) {
  if ((P->n > 0 && !d_x) || (P->m > 0 && !d_df)) return fail(FDB_ERR_INVALID, "NULL x or df");
  DeviceGuard g(P->device);
  if (!g.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", P->device);
  cudaStream_t s = (cudaStream_t)stream;
  resolve_steps(P->fdtype, relstep, absstep);                       // relstep = default_relstep(fdtype), absstep = relstep
  const double *fx = P->fdtype == FDB_FORWARD ? d_fx : nullptr;     // cache.fx is read in forward mode only
  const DerivSteps st{relstep, absstep, dir};
  const GraphKey key{(void *)f, ctx, d_x, d_df, fx, nullptr, relstep, absstep, dir, 0, 0, nullptr};
  const fdb_status rc = run_maybe_graph(P, key, s, "derivative", [&](cudaStream_t cs) {
    return dispatch_mode(P->fdtype, [&](auto mode) {
      return derivative_eager<decltype(mode)::value>(P, f, ctx, d_df, d_x, fx, st, cs);
    });
  });
  if (rc == FDB_OK) P->cnt.jacobians += 1;
  return rc;
}

fdb_status fdb_derivative(fdb_plan *P, fdb_fn f, void *ctx, double *d_df, const double *d_x, const double *d_fx,
                          double relstep, double absstep, double dir, void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::derivative));
  return derivative_run(P, f, ctx, d_df, d_x, d_fx, relstep, absstep, dir, stream);
}

fdb_status fdb_derivative_complex(fdb_plan *P, fdb_fn_c f, void *ctx, double *d_df, const double *d_x, void *stream) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::derivative_complex));
  return derivative_run(P, reinterpret_cast<fdb_fn>(f), ctx, d_df, d_x, nullptr, FDB_STEP_DEFAULT, FDB_STEP_DEFAULT, 1.0,
                        stream);
}

fdb_status fdb_jacobian_host(fdb_plan *P, fdb_fn f, void *ctx, const double *h_x, double *h_J, double *h_fx,
                             const double *h_f_in, double relstep, double absstep, double dir) {
  if (!P || !f) return fail(FDB_ERR_INVALID, "NULL plan or f");
  TRY(check_call(P, Call::jacobian));
  if ((P->n > 0 && !h_x) || (P->j_len > 0 && !h_J)) return fail(FDB_ERR_INVALID, "NULL x or J");
  DeviceGuard g(P->device);
  if (!g.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", P->device);
  if (!P->host.stream) {
    CU(cudaStreamCreateWithFlags(&P->host.stream, cudaStreamNonBlocking));
    TRY(P->alloc_t(&P->host.dx, (size_t)std::max<int64_t>(P->n, 1)));
    TRY(P->alloc_t(&P->host.dJ, (size_t)std::max<int64_t>(P->j_len, 1)));
    TRY(P->alloc_t(&P->host.dfx, (size_t)P->scratch.ldF));
    TRY(P->alloc_t(&P->host.dfin, (size_t)P->scratch.ldF));
  }
  cudaStream_t s = P->host.stream;
  if (P->n > 0) CU(cudaMemcpyAsync(P->host.dx, h_x, (size_t)P->n * 8, cudaMemcpyHostToDevice, s));
  const double *fin = nullptr;
  if (h_f_in && P->fdtype == FDB_FORWARD) {
    CU(cudaMemcpyAsync(P->host.dfin, h_f_in, (size_t)P->m * 8, cudaMemcpyHostToDevice, s));
    fin = P->host.dfin;
  }
  fdb_status st = jacobian_run(P, f, ctx, P->host.dx, P->host.dJ, P->host.dfx, fin, relstep, absstep, dir, (void *)s);
  if (st != FDB_OK) { cudaStreamSynchronize(s); return st; }
  if (P->j_len > 0) {
    if (P->jkind == FDB_J_DENSE && P->ldJ > P->m) {
      // strided dense view: only rows [0, m) of each column are J's (the host padding rows stay untouched)
      const int64_t ncols = P->sp_kind == SP_NONE ? P->columns.end - P->columns.begin : P->n;
      if (P->m > 0 && ncols > 0)
        CU(cudaMemcpy2DAsync(h_J, (size_t)P->ldJ * 8, P->host.dJ, (size_t)P->ldJ * 8, (size_t)P->m * 8, (size_t)ncols,
                             cudaMemcpyDeviceToHost, s));
    } else {
      CU(cudaMemcpyAsync(h_J, P->host.dJ, (size_t)P->j_len * 8, cudaMemcpyDeviceToHost, s));
    }
  }
  if (h_fx && P->fdtype == FDB_FORWARD && !fin && P->m > 0)
    CU(cudaMemcpyAsync(h_fx, P->host.dfx, (size_t)P->m * 8, cudaMemcpyDeviceToHost, s));
  CU(cudaStreamSynchronize(s));
  return FDB_OK;
}

// ------------------------------------------------------------------------------------------------ helpers
fdb_status fdb_host_alloc(void **p, size_t bytes) {
  if (!p) return fail(FDB_ERR_INVALID, "NULL argument");
  CU(cudaHostAlloc(p, bytes ? bytes : 16, cudaHostAllocDefault));
  return FDB_OK;
}
fdb_status fdb_host_free(void *p) { if (p) CU(cudaFreeHost(p)); return FDB_OK; }
fdb_status fdb_device_alloc(void **p, size_t bytes) {
  if (!p) return fail(FDB_ERR_INVALID, "NULL argument");
  CU(cudaMalloc(p, bytes ? bytes : 16));
  return FDB_OK;
}
fdb_status fdb_device_free(void *p) { if (p) CU(cudaFree(p)); return FDB_OK; }
fdb_status fdb_memcpy_h2d(void *d, const void *h, size_t bytes, void *stream) {
  CU(cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return FDB_OK;
}
fdb_status fdb_memcpy_d2h(void *h, const void *d, size_t bytes, void *stream) {
  CU(cudaMemcpyAsync(h, d, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return FDB_OK;
}
fdb_status fdb_stream_sync(void *stream) { CU(cudaStreamSynchronize((cudaStream_t)stream)); return FDB_OK; }

fdb_status fdb_ipc_get_handle(void *d_ptr, unsigned char handle[64]) {
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "CUDA IPC handle size");
  cudaIpcMemHandle_t h;
  CU(cudaIpcGetMemHandle(&h, d_ptr));
  memcpy(handle, &h, 64);
  return FDB_OK;
}
fdb_status fdb_ipc_open(const unsigned char handle[64], void **d_ptr) {
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, 64);
  CU(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return FDB_OK;
}
fdb_status fdb_ipc_close(void *d_ptr) { CU(cudaIpcCloseMemHandle(d_ptr)); return FDB_OK; }

}  // extern "C"

#include "fdjac_group.cuh"
#include "fdjac_oop.cuh"
