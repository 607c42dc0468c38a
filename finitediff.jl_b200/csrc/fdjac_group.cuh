// fdjac_group.cuh — multi-GPU behind the C ABI (included at the end of fdjac_abi.cu; same translation unit).
//
// Colours (dense plans: column blocks) are independent units given x, so N GPUs need no collective on the data path:
// every member evaluates its share and stores the entries it owns STRAIGHT INTO ONE Jacobian buffer (the root's) through
// peer-mapped memory over NVLink/NVSwitch — the "final gather of Jacobian columns" is the scatter kernel's own store.
// Two ways to drive it, both without NCCL:
//
//   fdb_group_*   ONE process drives n devices (what a Julia host calling finite_difference_jacobian! once needs):
//                 one plan per device (rank i of n, opts.shared_j = 1), cudaDeviceEnablePeerAccess to the root, x pushed
//                 to the members with cudaMemcpyPeerAsync, CUDA events order everything on the caller's stream.
//                 Device ordinals may repeat ({0,0}: two members on one GPU) — the same code path on a 1-GPU box.
//   fdb_sync_*    one process per GPU (torchrun-style launchers): every rank creates its plan with rank/world and
//                 opts.shared_j = 1, maps the root's J with CUDA IPC and passes that pointer as d_J; the ranks are
//                 ordered by a device-side flag barrier in peer memory (release/acquire at system scope) enqueued on
//                 the call's stream — no host synchronisation, CUDA-graph friendly (the epoch lives in device memory).
#pragma once

// ------------------------------------------------------------------------------------------------ device-side barrier
struct fdb_sync {
  int rank = 0, world = 1, device = 0;
  unsigned long long *flags = nullptr;        // [world] incoming slots + [world] = epoch counter (dedicated cudaMalloc)
  unsigned long long **d_peer_flags = nullptr;// device array [world]: every rank's flag block as mapped on this device
  bool peers_set = false;
};

// thread t: tell rank t that this rank reached epoch e, then wait until rank t has told us the same
__global__ void __launch_bounds__(64)
sync_barrier_kernel(unsigned long long *const *__restrict__ peer_flags, unsigned long long *my_flags, int rank, int world) {
  unsigned long long *epoch = my_flags + world;
  const unsigned long long e = *epoch + 1;
  __syncthreads();
  for (int t = threadIdx.x; t < world; t += blockDim.x) {
    __threadfence_system();   // everything this rank wrote before the barrier (peer stores included) is visible first
    unsigned long long *dst = peer_flags[t] + rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(e) : "memory");
    unsigned long long v;
    const unsigned long long *src = my_flags + t;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(src) : "memory");
    } while (v < e);
  }
  __syncthreads();
  if (threadIdx.x == 0) *epoch = e;
}

// ------------------------------------------------------------------------------------------------ single-process group
struct fdb_group {
  int n = 0;
  int kind = SP_CSC;
  std::vector<fdb_plan *> plans;
  std::vector<int> devices;
  std::vector<cudaStream_t> streams;     // members > 0 (index 0 unused: the root runs on the caller's stream)
  std::vector<cudaEvent_t> ev_done;
  cudaEvent_t ev_start = nullptr;
  std::vector<double *> x_rep, fin_rep;  // x / f_in replicas on members living on another device than the root
  int64_t nx = 0, m = 0;
};

static bool plan_self_defining(const fdb_plan *P) {
  // the scatter launches of all ranks together define every slot of J (identity CSC: nzval; band data: whole columns)
  const bool ident = P->dest == nullptr && P->sp_kind != SP_BANDED;
  const bool band_data = P->sp_kind == SP_BANDED && P->jkind == FDB_J_BAND;
  return (ident || band_data) && P->C > 0;
}

static void free_group(fdb_group *g) {
  if (!g) return;
  for (int i = 0; i < (int)g->plans.size(); ++i) {
    if (i < (int)g->devices.size()) {
      DeviceGuard dg(g->devices[i]);
      if (i < (int)g->streams.size() && g->streams[i]) cudaStreamDestroy(g->streams[i]);
      if (i < (int)g->ev_done.size() && g->ev_done[i]) cudaEventDestroy(g->ev_done[i]);
      if (i < (int)g->x_rep.size() && g->x_rep[i]) cudaFree(g->x_rep[i]);
      if (i < (int)g->fin_rep.size() && g->fin_rep[i]) cudaFree(g->fin_rep[i]);
    }
    free_plan(g->plans[i]);
  }
  if (g->ev_start) { DeviceGuard dg(g->devices.empty() ? 0 : g->devices[0]); cudaEventDestroy(g->ev_start); }
  delete g;
}

// common part of the fdb_group_create_* entry points: `make(i, opts_i, &plan)` creates member i's plan
template <typename Make>
static fdb_status group_create(fdb_group **out, int n_devices, const int *devices, const fdb_plan_opts *opts, Make &&make) {
  if (!out) return fail(FDB_ERR_INVALID, "group output pointer is NULL");
  *out = nullptr;
  if (n_devices < 1 || n_devices > 64 || !devices) return fail(FDB_ERR_INVALID, "n_devices must be in 1..64 and devices non-NULL");
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
    cudaGetLastError();
    return fail(FDB_ERR_NO_DEVICE, "no CUDA device available: libfdjac_b200 has no CPU fallback");
  }
  for (int i = 0; i < n_devices; ++i)
    if (devices[i] < 0 || devices[i] >= count) return fail(FDB_ERR_INVALID, "device %d out of range (%d devices)", devices[i], count);
  std::unique_ptr<fdb_group, void (*)(fdb_group *)> g(new (std::nothrow) fdb_group(), free_group);
  if (!g) return fail(FDB_ERR_NOMEM, "out of host memory");
  g->n = n_devices;
  g->devices.assign(devices, devices + n_devices);
  g->plans.assign(n_devices, nullptr);
  g->streams.assign(n_devices, nullptr);
  g->ev_done.assign(n_devices, nullptr);
  g->x_rep.assign(n_devices, nullptr);
  g->fin_rep.assign(n_devices, nullptr);
  const int root = devices[0];
  for (int i = 0; i < n_devices; ++i) {
    fdb_plan_opts o{};
    if (opts) o = *opts;
    o.device = devices[i];
    o.use_current_device = 0;
    o.rank = i;
    o.world = n_devices;
    o.shared_j = n_devices > 1 ? 1 : 0;
    // peer access to the root FIRST: the member's plan build may already read index arrays that live on the root device
    if (i > 0 && devices[i] != root) {
      DeviceGuard dgp(devices[i]);
      int can = 0;
      cudaDeviceCanAccessPeer(&can, devices[i], root);
      if (!can) return fail(FDB_ERR_UNSUPPORTED, "device %d cannot access device %d (no peer path)", devices[i], root);
      const cudaError_t e = cudaDeviceEnablePeerAccess(root, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled)
        return fail(FDB_ERR_CUDA, "cudaDeviceEnablePeerAccess(%d -> %d): %s", devices[i], root, cudaGetErrorString(e));
      cudaGetLastError();
    }
    TRY(make(i, &o, &g->plans[i]));
    if (i == 0) continue;
    DeviceGuard dg(devices[i]);
    cudaError_t e = cudaStreamCreateWithFlags(&g->streams[i], cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&g->ev_done[i], cudaEventDisableTiming);
    if (e != cudaSuccess) return fail(FDB_ERR_CUDA, "group stream/event: %s", cudaGetErrorString(e));
  }
  {
    DeviceGuard dg(root);
    const cudaError_t e = cudaEventCreateWithFlags(&g->ev_start, cudaEventDisableTiming);
    if (e != cudaSuccess) return fail(FDB_ERR_CUDA, "group event: %s", cudaGetErrorString(e));
  }
  g->nx = g->plans[0]->n;
  g->m = g->plans[0]->m;
  g->kind = g->plans[0]->sp_kind;
  *out = g.release();
  return FDB_OK;
}

extern "C" {

fdb_status fdb_group_create_csc(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n,
                                const int64_t *colptr, const int64_t *rowval, int jkind, const int64_t *j_colptr,
                                const int64_t *j_rowval, int64_t ldJ, const int64_t *colorvec, const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_plan_create_csc(p, m, n, colptr, rowval, jkind, j_colptr, j_rowval, ldJ, colorvec, o);
  });
}

fdb_status fdb_group_create_banded(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n, int64_t l,
                                   int64_t u, int jkind, int64_t ldJ, const int64_t *colorvec, const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_plan_create_banded(p, m, n, l, u, jkind, ldJ, colorvec, o);
  });
}

fdb_status fdb_group_create_dense(fdb_group **group, int n_devices, const int *devices, int64_t m, int64_t n, int64_t ldJ,
                                  const fdb_plan_opts *opts) {
  return group_create(group, n_devices, devices, opts, [&](int, const fdb_plan_opts *o, fdb_plan **p) {
    return fdb_plan_create_dense(p, m, n, ldJ, o);
  });
}

fdb_status fdb_group_destroy(fdb_group *group) {
  free_group(group);
  return FDB_OK;
}

fdb_status fdb_group_size(const fdb_group *group, int *n_members) {
  if (!group || !n_members) return fail(FDB_ERR_INVALID, "NULL argument");
  *n_members = group->n;
  return FDB_OK;
}

fdb_status fdb_group_plan(const fdb_group *group, int member, fdb_plan **plan) {
  if (!group || !plan) return fail(FDB_ERR_INVALID, "NULL argument");
  if (member < 0 || member >= group->n) return fail(FDB_ERR_INVALID, "member %d outside 0..%d", member, group->n - 1);
  *plan = group->plans[member];
  return FDB_OK;
}

fdb_status fdb_group_jacobian(fdb_group *g, fdb_fn f, void *const *ctx, const double *d_x, double *d_J, double *d_fx,
                              const double *d_f_in, double relstep, double absstep, double dir, void *stream) {
  if (!g || !f) return fail(FDB_ERR_INVALID, "NULL group or f");
  fdb_plan *P0 = g->plans[0];
  if (P0->fdtype == FDB_COMPLEX) return fail(FDB_ERR_UNSUPPORTED, "groups run forward / central plans");
  if ((P0->n > 0 && !d_x) || !d_J) return fail(FDB_ERR_INVALID, "NULL x or J");
  const int root = g->devices[0];
  cudaStream_t s0 = (cudaStream_t)stream;
  {
    DeviceGuard dg(root);
    if (!dg.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", root);
    // fill_matrix!(J, false) once, by the owner of the buffer, before any member may store into it
    if (g->n > 1 && P0->sp_kind != SP_NONE && !plan_self_defining(P0) && P0->j_len > 0) TRY(zero_J(P0, d_J, s0));
    CU(cudaEventRecord(g->ev_start, s0));
  }
  for (int i = 1; i < g->n; ++i) {
    fdb_plan *P = g->plans[i];
    const int dev = g->devices[i];
    DeviceGuard dg(dev);
    if (!dg.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", dev);
    cudaStream_t s = g->streams[i];
    CU(cudaStreamWaitEvent(s, g->ev_start, 0));
    const double *xi = d_x, *fin_i = d_f_in;
    if (dev != root) {
      if (!g->x_rep[i]) CU(cudaMalloc((void **)&g->x_rep[i], (size_t)std::max<int64_t>(g->nx, 2) * 8));
      if (g->nx > 0) CU(cudaMemcpyPeerAsync(g->x_rep[i], dev, d_x, root, (size_t)g->nx * 8, s));
      xi = g->x_rep[i];
      if (d_f_in && P->fdtype == FDB_FORWARD) {
        if (!g->fin_rep[i]) CU(cudaMalloc((void **)&g->fin_rep[i], (size_t)std::max<int64_t>(g->m, 2) * 8));
        if (g->m > 0) CU(cudaMemcpyPeerAsync(g->fin_rep[i], dev, d_f_in, root, (size_t)g->m * 8, s));
        fin_i = g->fin_rep[i];
      }
    }
    double *Ji = P->sp_kind == SP_NONE ? d_J + P->col_begin * P->ldJ : d_J;
    TRY(fdb_jacobian(P, f, ctx ? ctx[i] : nullptr, xi, Ji, nullptr, fin_i, relstep, absstep, dir, (void *)s));
    CU(cudaEventRecord(g->ev_done[i], s));
  }
  {
    DeviceGuard dg(root);
    double *J0 = P0->sp_kind == SP_NONE ? d_J + P0->col_begin * P0->ldJ : d_J;
    TRY(fdb_jacobian(P0, f, ctx ? ctx[0] : nullptr, d_x, J0, d_fx, d_f_in, relstep, absstep, dir, (void *)s0));
    for (int i = 1; i < g->n; ++i) CU(cudaStreamWaitEvent(s0, g->ev_done[i], 0));
  }
  return FDB_OK;
}

// ------------------------------------------------------------------------------------------------ fdb_sync (one process per GPU)
fdb_status fdb_sync_create(fdb_sync **out, int rank, int world, int device) {
  if (!out) return fail(FDB_ERR_INVALID, "NULL argument");
  *out = nullptr;
  if (world < 1 || world > 64 || rank < 0 || rank >= world) return fail(FDB_ERR_INVALID, "rank %d / world %d invalid (world <= 64)", rank, world);
  fdb_plan_opts o{};
  o.device = device;
  o.use_current_device = device < 0 ? 1 : 0;
  int dev = 0;
  TRY(check_device(&o, &dev));
  DeviceGuard dg(dev);
  std::unique_ptr<fdb_sync, fdb_status (*)(fdb_sync *)> s(new (std::nothrow) fdb_sync(), fdb_sync_destroy);
  if (!s) return fail(FDB_ERR_NOMEM, "out of host memory");
  s->rank = rank; s->world = world; s->device = dev;
  cudaError_t e = cudaMalloc((void **)&s->flags, ((size_t)world + 1) * 8);
  if (e == cudaSuccess) e = cudaMemset(s->flags, 0, ((size_t)world + 1) * 8);
  if (e == cudaSuccess) e = cudaMalloc((void **)&s->d_peer_flags, (size_t)world * sizeof(void *));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(FDB_ERR_CUDA, "fdb_sync_create: %s", cudaGetErrorString(e));
  *out = s.release();
  return FDB_OK;
}

fdb_status fdb_sync_flags(fdb_sync *s, void **d_flags) {
  if (!s || !d_flags) return fail(FDB_ERR_INVALID, "NULL argument");
  *d_flags = s->flags;
  return FDB_OK;
}

fdb_status fdb_sync_set_peers(fdb_sync *s, void *const *d_flags_by_rank) {
  if (!s || !d_flags_by_rank) return fail(FDB_ERR_INVALID, "NULL argument");
  DeviceGuard dg(s->device);
  std::vector<unsigned long long *> p((size_t)s->world);
  for (int r = 0; r < s->world; ++r) {
    p[(size_t)r] = r == s->rank ? s->flags : (unsigned long long *)d_flags_by_rank[r];
    if (!p[(size_t)r]) return fail(FDB_ERR_INVALID, "flag block of rank %d is NULL", r);
  }
  CU(cudaMemcpy(s->d_peer_flags, p.data(), (size_t)s->world * sizeof(void *), cudaMemcpyHostToDevice));
  s->peers_set = true;
  return FDB_OK;
}

fdb_status fdb_sync_barrier(fdb_sync *s, void *stream) {
  if (!s) return fail(FDB_ERR_INVALID, "NULL argument");
  if (!s->peers_set) return fail(FDB_ERR_INVALID, "fdb_sync_set_peers has not been called");
  DeviceGuard dg(s->device);
  if (!dg.ok) return fail(FDB_ERR_CUDA, "cannot select device %d", s->device);
  sync_barrier_kernel<<<1, 64, 0, (cudaStream_t)stream>>>(s->d_peer_flags, s->flags, s->rank, s->world);
  CU(cudaGetLastError());
  return FDB_OK;
}

fdb_status fdb_sync_destroy(fdb_sync *s) {
  if (!s) return FDB_OK;
  DeviceGuard dg(s->device);
  cudaFree(s->flags);
  cudaFree(s->d_peer_flags);
  delete s;
  return FDB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------ on-device colouring
// ArrayInterface.matrix_colors analogues (kernels_color.cuh).  Plan-time operations: they synchronise.
struct CsrPattern {
  DevBuf<int32_t> rowptr, rcols;
  I64View cp, rv;
  int64_t nnz = 0;
};

static fdb_status build_csr_pattern(int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval, CsrPattern &P) {
  if (m < 0 || n < 0 || m > 0x7FFFFFF0LL || n > 0x7FFFFFF0LL) return fail(FDB_ERR_INVALID, "m, n must be in [0, 2^31)");
  if (!colptr) return fail(FDB_ERR_INVALID, "colptr is NULL");
  TRY(view_i64(colptr, n + 1, P.cp));
  int64_t last = 1;
  TRY(read_back(&last, P.cp.d + n, 1, "reading colptr[n]"));
  P.nnz = last - 1;
  if (P.nnz < 0 || P.nnz > 0x7FFFFFF0LL) return fail(FDB_ERR_INVALID, "nnz=%lld unsupported", (long long)P.nnz);
  if (P.nnz > 0 && !rowval) return fail(FDB_ERR_INVALID, "rowval is NULL");
  TRY(view_i64(rowval, P.nnz, P.rv));
  DevBuf<uint32_t> d_err;
  DevBuf<int32_t> cnt, cursor;
  TRY(d_err.alloc(1));
  CU(cudaMemset(d_err.get(), 0, 4));
  TRY(cnt.alloc((size_t)m + 1));
  CU(cudaMemset(cnt.get(), 0, ((size_t)m + 1) * 4));
  TRY(cursor.alloc((size_t)m + 1));
  CU(cudaMemset(cursor.get(), 0, ((size_t)m + 1) * 4));
  TRY(P.rowptr.alloc((size_t)m + 1));
  TRY(P.rcols.alloc((size_t)std::max<int64_t>(P.nnz, 1)));
  const int gb = (int)std::max<int64_t>(1, std::min<int64_t>((std::max<int64_t>(P.nnz, n + 1) + kThreads - 1) / kThreads, 132 * 16));
  validate_colptr<<<gb, kThreads>>>(P.cp.d, n, P.nnz, d_err.get());
  if (P.nnz > 0) csr_count_rows<<<gb, kThreads>>>(P.rv.d, P.nnz, m, cnt.get(), d_err.get());
  uint32_t herr = 0;
  TRY(read_back(&herr, d_err.get(), 1, "CSC pattern check"));
  if (herr) return fail(FDB_ERR_INVALID, "invalid CSC pattern (%s)", (herr & 1u) ? "colptr" : "row index outside 1..m");
  TRY(cub_run([&](void *tmp, size_t &bytes) {
    return cub::DeviceScan::ExclusiveSum(tmp, bytes, cnt.get(), P.rowptr.get(), (int)(m + 1));
  }));
  if (n > 0 && P.nnz > 0) csr_fill<<<gb, kThreads>>>(P.cp.d, P.rv.d, n, m, P.rowptr.get(), cursor.get(), P.rcols.get());
  CU(cudaDeviceSynchronize());
  return FDB_OK;
}

extern "C" {

fdb_status fdb_matrix_colors_banded(int64_t n, int64_t l, int64_t u, int64_t *d_colorvec, void *stream) {
  if (n < 0 || l + u + 1 < 1) return fail(FDB_ERR_INVALID, "invalid n / bandwidths");
  if (n > 0 && !d_colorvec) return fail(FDB_ERR_INVALID, "colorvec is NULL");
  if (n == 0) return FDB_OK;
  const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, 132 * 8));
  cyclic_colors<<<blocks, kThreads, 0, (cudaStream_t)stream>>>(n, l + u + 1, d_colorvec);
  CU(cudaGetLastError());
  return FDB_OK;
}

fdb_status fdb_matrix_colors_csc(int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval, int64_t *d_colorvec,
                                 int64_t *n_colors, int64_t *n_rounds) {
  if (n > 0 && !d_colorvec) return fail(FDB_ERR_INVALID, "colorvec is NULL");
  int dev = 0;
  TRY(check_device(nullptr, &dev));
  if (n_colors) *n_colors = 0;
  if (n_rounds) *n_rounds = 0;
  if (n == 0) return FDB_OK;
  CsrPattern P;
  TRY(build_csr_pattern(m, n, colptr, rowval, P));
  DevBuf<int32_t> buf_a, buf_b;
  DevBuf<unsigned long long> d_pending;
  DevBuf<int> d_max;
  TRY(buf_a.alloc((size_t)n));
  TRY(buf_b.alloc((size_t)n));
  TRY(d_pending.alloc(1));
  TRY(d_max.alloc(1));
  CU(cudaMemset(buf_a.get(), 0, (size_t)n * 4));
  CU(cudaMemset(d_max.get(), 0, 4));
  int32_t *col_a = buf_a.get(), *col_b = buf_b.get();
  const int gb = (int)std::max<int64_t>(1, std::min<int64_t>((n + kThreads - 1) / kThreads, 132 * 16));
  int64_t rounds = 0;
  unsigned long long pending = (unsigned long long)n;
  while (pending > 0) {
    CU(cudaMemset(d_pending.get(), 0, 8));
    jp_color_round<<<gb, kThreads>>>(P.cp.d, P.rv.d, P.rowptr.get(), P.rcols.get(), n, m, col_a, col_b, d_pending.get());
    TRY(read_back(&pending, d_pending.get(), 1, "colouring round"));
    std::swap(col_a, col_b);
    if (++rounds > 100000) return fail(FDB_ERR_INVALID, "colouring did not converge");
  }
  colors_to_i64<<<gb, kThreads>>>(col_a, n, d_colorvec, d_max.get());
  int mx = 0;
  TRY(read_back(&mx, d_max.get(), 1, "colour count"));
  if (n_colors) *n_colors = mx;
  if (n_rounds) *n_rounds = rounds;
  return FDB_OK;
}

fdb_status fdb_check_coloring_csc(int64_t m, int64_t n, const int64_t *colptr, const int64_t *rowval, const int64_t *colorvec,
                                  int64_t *n_conflicts) {
  if (!n_conflicts) return fail(FDB_ERR_INVALID, "NULL argument");
  *n_conflicts = 0;
  int dev = 0;
  TRY(check_device(nullptr, &dev));
  if (n == 0 || m == 0) return FDB_OK;
  if (!colorvec) return FDB_OK;                     // 1:n: every column its own colour
  CsrPattern P;
  TRY(build_csr_pattern(m, n, colptr, rowval, P));
  I64View cv;
  TRY(view_i64(colorvec, n, cv));
  DevBuf<unsigned long long> d_c;
  TRY(d_c.alloc(1));
  CU(cudaMemset(d_c.get(), 0, 8));
  const int gb = (int)std::max<int64_t>(1, std::min<int64_t>((m + kThreads - 1) / kThreads, 132 * 16));
  count_color_conflicts<<<gb, kThreads>>>(P.rowptr.get(), P.rcols.get(), m, cv.d, d_c.get());
  unsigned long long h = 0;
  TRY(read_back(&h, d_c.get(), 1, "conflict count"));
  *n_conflicts = (int64_t)h;
  return FDB_OK;
}

}  // extern "C"
