// kernels_plan.cuh — plan-time device kernels: validate the caller's Int64 1-based index arrays and build the
// compressed per-entry streams the hot kernels read (0-based int32 rows, narrow colour ids, destination offsets).
// This replaces the per-call index work of the reference's prologue (jacobians.jl:515-535: reshape of colorvec,
// findstructralnz / _findstructralnz, the O(n+nnz) same-pattern comparison of ext/FiniteDiffSparseArraysExt.jl:51-52)
// — done once per (pattern, colorvec), on the device, instead of on every Jacobian.
#pragma once
#include "common.cuh"

namespace fdb {

enum PlanErr : uint32_t {
  kErrColptr = 1u,        // colptr not monotone / wrong ends
  kErrRowRange = 2u,      // row index outside 1..m
  kErrColRange = 4u,      // column index outside 1..n
  kErrSlotRange = 8u,     // slot outside 1..j_len
  kErrPatternDiff = 16u,  // J pattern != sparsity pattern (informational)
  kErrMissingInJ = 32u,   // sparsity entry absent from J's pattern (setindex! would have to insert)
  kErrRowOrder = 64u      // rows within a column not strictly increasing (binary search needs it)
};

// max / min of colorvec
__global__ void __launch_bounds__(kThreads)
color_minmax(const int64_t *__restrict__ colorvec, int64_t n, long long *__restrict__ out_max,
             long long *__restrict__ out_min) {
  long long mx = LLONG_MIN, mn = LLONG_MAX;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride) {
    const long long c = colorvec[j];
    mx = c > mx ? c : mx;
    mn = c < mn ? c : mn;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const long long a = __shfl_xor_sync(0xffffffffu, mx, o), b = __shfl_xor_sync(0xffffffffu, mn, o);
    mx = a > mx ? a : mx;
    mn = b < mn ? b : mn;
  }
  if ((threadIdx.x & 31) == 0) {
    atomicMax(out_max, mx);
    atomicMin(out_min, mn);
  }
}

// jcolor[j] = colorvec[j]-1 (or j for the default 1:n), invalid marker for colorvec[j] < 1
template <typename CT>
__global__ void __launch_bounds__(kThreads)
convert_colors(const int64_t *__restrict__ colorvec /* null => 1:n */, int64_t n, CT *__restrict__ jcolor) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride) {
    const int64_t c = colorvec ? colorvec[j] : j + 1;
    jcolor[j] = c >= 1 ? (CT)(c - 1) : (CT)ColorTraits<CT>::invalid;
  }
}

// cyclic colouring test: flag = 1 unless jcolor[j] == j mod C for every j (a column without a valid colour never matches)
template <typename CT>
__global__ void __launch_bounds__(kThreads)
check_cyclic(const CT *__restrict__ jcolor, int64_t n, int32_t C, uint32_t *__restrict__ flag) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t j = blockIdx.x * (int64_t)kThreads + threadIdx.x; j < n; j += stride)
    if ((uint32_t)jcolor[j] != (uint32_t)(j % C)) { *flag = 1u; return; }
}

// exact-band test, pass 1: l = max(c - r), u = max(r - c) over all entries (0-based rows, CSC column pointer)
__global__ void __launch_bounds__(kThreads)
band_extent(const int32_t *__restrict__ colptr32, const int32_t *__restrict__ row32, int64_t n, int *__restrict__ lu) {
  int l = INT_MIN, u = INT_MIN;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c < n; c += stride) {
    const int32_t p0 = colptr32[c], p1 = colptr32[c + 1];
    if (p1 > p0) {                                       // rows may be unsorted here: look at every one
      for (int32_t p = p0; p < p1; ++p) {
        const int r = row32[p];
        l = max(l, (int)c - r);
        u = max(u, r - (int)c);
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    l = max(l, __shfl_xor_sync(0xffffffffu, l, o));
    u = max(u, __shfl_xor_sync(0xffffffffu, u, o));
  }
  if ((threadIdx.x & 31) == 0) { atomicMax(lu, l); atomicMax(lu + 1, u); }
}

// pass 2: every column c holds exactly the rows max(0, c-l) .. min(m-1, c+u), in order; flag = 1 on the first mismatch
__global__ void __launch_bounds__(kThreads)
band_check(const int32_t *__restrict__ colptr32, const int32_t *__restrict__ row32, int64_t m, int64_t n, int l, int u,
           uint32_t *__restrict__ flag) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c < n; c += stride) {
    const int64_t lo = c - l > 0 ? c - l : 0, hi = c + u < m - 1 ? c + u : m - 1;
    const int64_t len = hi >= lo ? hi - lo + 1 : 0;
    const int32_t p0 = colptr32[c];
    bool bad = colptr32[c + 1] - p0 != len;
    for (int64_t i = 0; !bad && i < len; ++i) bad = row32[p0 + i] != lo + i;
    if (bad) { *flag = 1u; return; }
  }
}

__global__ void __launch_bounds__(kThreads)
validate_colptr(const int64_t *__restrict__ colptr, int64_t n, int64_t nnz, uint32_t *__restrict__ err) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c <= n; c += stride) {
    bool bad = false;
    if (c == 0 && colptr[0] != 1) bad = true;
    if (c == n && colptr[n] != nnz + 1) bad = true;
    if (c < n && colptr[c + 1] < colptr[c]) bad = true;
    if (bad) atomicOr(err, kErrColptr);
  }
}

// column (0-based) of CSC slot p (0-based): largest c with colptr[c]-1 <= p
__device__ __forceinline__ int64_t csc_col_of(const int64_t *__restrict__ colptr, int64_t n, int64_t p) {
  int64_t lo = 0, hi = n;  // invariant: colptr[lo]-1 <= p < colptr[hi]-1
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (colptr[mid] - 1 <= p) lo = mid; else hi = mid;
  }
  return lo;
}

// Per-colour counting shared by the plan kernels: lanes of a warp holding the same colour are combined (match.any),
// the group's leader adds the population to the block's shared-memory histogram (C <= kPlanSmemColors) or straight
// to the global counters.  Must be reached by all 32 lanes of the warp (`k` >= C for lanes with nothing to count).
constexpr int kPlanSmemColors = 4096;
__device__ __forceinline__ void count_color(uint32_t k, int32_t C, unsigned int *s_cnt /* null => global */,
                                            unsigned long long *__restrict__ color_count) {
  const bool valid = k < (uint32_t)C;
  const unsigned act = __ballot_sync(0xffffffffu, valid);
  if (!valid) return;
  const unsigned peers = __match_any_sync(act, k);
  if ((int)(threadIdx.x & 31) != __ffs(peers) - 1) return;
  if (s_cnt) atomicAdd(s_cnt + k, (unsigned int)__popc(peers));
  else atomicAdd(color_count + k, (unsigned long long)__popc(peers));
}
__device__ __forceinline__ unsigned int *count_begin(unsigned int *smem, int32_t C, const unsigned long long *color_count) {
  if (color_count == nullptr || C > kPlanSmemColors) return nullptr;
  for (int i = threadIdx.x; i < C; i += kThreads) smem[i] = 0u;
  __syncthreads();
  return smem;
}
__device__ __forceinline__ void count_end(unsigned int *s_cnt, int32_t C, unsigned long long *__restrict__ color_count) {
  if (!s_cnt) return;
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += kThreads)
    if (s_cnt[i]) atomicAdd(color_count + i, (unsigned long long)s_cnt[i]);
}

// For every CSC slot p: row32[p], ecolor[p] (colour of its column), optional col32[p]; per-colour entry counts
// (one global atomic per entry would serialise 3*10^7 atomics on 3 addresses for C2).
template <typename CT>
__global__ void __launch_bounds__(kThreads)
expand_csc(const int64_t *__restrict__ colptr, const int64_t *__restrict__ rowval, int64_t m, int64_t n, int64_t nnz,
           const CT *__restrict__ jcolor, int32_t C, int32_t *__restrict__ row32, CT *__restrict__ ecolor,
           int32_t *__restrict__ col32 /* nullable */, unsigned long long *__restrict__ color_count /* [C] nullable */,
           uint32_t *__restrict__ err) {
  extern __shared__ unsigned int s_hist[];   // [C] when C <= kPlanSmemColors and counts are wanted
  unsigned int *s_cnt = count_begin(s_hist, C, color_count);
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int lane = threadIdx.x & 31;
  // warp-uniform trip count: count_color uses full-warp collectives
  for (int64_t p0 = blockIdx.x * (int64_t)kThreads + threadIdx.x - lane; p0 < nnz; p0 += stride) {
    const int64_t p = p0 + lane;
    uint32_t k = 0xffffffffu;
    if (p < nnz) {
      const int64_t c = csc_col_of(colptr, n, p);
      const int64_t r = rowval[p];
      if (r < 1 || r > m) { atomicOr(err, kErrRowRange); row32[p] = 0; }
      else row32[p] = (int32_t)(r - 1);
      if (p > colptr[c] - 1 && rowval[p - 1] >= r) atomicOr(err, kErrRowOrder);
      const CT kc = jcolor[c];
      ecolor[p] = kc;
      if (col32) col32[p] = (int32_t)c;
      k = (uint32_t)kc;
    }
    if (color_count) count_color(k, C, s_cnt, color_count);
  }
  count_end(s_cnt, C, color_count);
}

// same-pattern test of ext/FiniteDiffSparseArraysExt.jl:51-52:  J.colptr == sp.colptr && J.rowval == sp.rowval
__global__ void __launch_bounds__(kThreads)
compare_i64(const int64_t *__restrict__ a, const int64_t *__restrict__ b, int64_t count, uint32_t *__restrict__ err) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  bool diff = false;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < count; i += stride) diff |= a[i] != b[i];
  if (diff) atomicOr(err, kErrPatternDiff);
}

// dest[p] = col*ldJ + row  (dense column-major J)
__global__ void __launch_bounds__(kThreads)
dest_dense_from_rc(const int32_t *__restrict__ row32, const int32_t *__restrict__ col32, int64_t E, int64_t ldJ,
                   int64_t *__restrict__ dest) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < E; e += stride)
    dest[e] = (int64_t)col32[e] * ldJ + row32[e];
}

// dest[p] = slot of (row,col) in another CSC pattern (J[r,c] = v on a SparseMatrixCSC: binary search in the column)
__global__ void __launch_bounds__(kThreads)
dest_other_csc(const int32_t *__restrict__ row32, const int32_t *__restrict__ col32, int64_t E,
               const int64_t *__restrict__ j_colptr, const int64_t *__restrict__ j_rowval, int64_t *__restrict__ dest,
               uint32_t *__restrict__ err) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e < E; e += stride) {
    const int64_t c = col32[e], r = (int64_t)row32[e] + 1;
    int64_t lo = j_colptr[c] - 1, hi = j_colptr[c + 1] - 1;  // [lo,hi)
    int64_t found = -1;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      const int64_t rv = j_rowval[mid];
      if (rv == r) { found = mid; break; }
      if (rv < r) lo = mid + 1; else hi = mid;
    }
    if (found < 0) { atomicOr(err, kErrMissingInJ); found = 0; }
    dest[e] = found;
  }
}

// COO entries (rows_index/cols_index, 1-based): row32, ecolor, dest (dense or explicit slots), validation, counts
template <typename CT>
__global__ void __launch_bounds__(kThreads)
prepare_coo(const int64_t *__restrict__ rows, const int64_t *__restrict__ cols, const int64_t *__restrict__ slots,
            int64_t nnz, int64_t m, int64_t n, int64_t ldJ, int64_t j_len, const CT *__restrict__ jcolor, int32_t C,
            int32_t *__restrict__ row32, CT *__restrict__ ecolor, int64_t *__restrict__ dest,
            unsigned long long *__restrict__ color_count, uint32_t *__restrict__ err) {
  extern __shared__ unsigned int s_hist[];
  unsigned int *s_cnt = count_begin(s_hist, C, color_count);
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int lane = threadIdx.x & 31;
  for (int64_t e0 = blockIdx.x * (int64_t)kThreads + threadIdx.x - lane; e0 < nnz; e0 += stride) {
    const int64_t e = e0 + lane;
    uint32_t kk = 0xffffffffu;
    if (e < nnz) {
      int64_t r = rows[e], c = cols[e];
      if (r < 1 || r > m) { atomicOr(err, kErrRowRange); r = 1; }
      if (c < 1 || c > n) { atomicOr(err, kErrColRange); c = 1; }
      row32[e] = (int32_t)(r - 1);
      const CT k = jcolor[c - 1];
      ecolor[e] = k;
      int64_t d;
      if (slots) {
        d = slots[e] - 1;
        if (d < 0 || d >= j_len) { atomicOr(err, kErrSlotRange); d = 0; }
      } else {
        d = (c - 1) * ldJ + (r - 1);
      }
      dest[e] = d;
      kk = (uint32_t)k;
    }
    if (color_count) count_color(kk, C, s_cnt, color_count);
  }
  count_end(s_cnt, C, color_count);
}

// ---- per-colour column lists (the reference's "for col in 1:ncols; if colorvec[col]==color_i" test, done ONCE) ----
// colptr32[c] = colptr[c]-1 (0-based int32), column counts per colour bucket (bucket C = columns without a valid colour)
template <typename CT>
__global__ void __launch_bounds__(kThreads)
colptr32_and_count(const int64_t *__restrict__ colptr, int64_t n, const CT *__restrict__ jcolor, int32_t C,
                   int32_t *__restrict__ colptr32, unsigned long long *__restrict__ bucket_count /* [C+1] */) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c <= n; c += stride) {
    colptr32[c] = (int32_t)(colptr[c] - 1);
    if (c < n) {
      uint32_t k = (uint32_t)jcolor[c];
      if (k >= (uint32_t)C) k = (uint32_t)C;
      // warp-aggregated histogram: lanes holding the same colour elect a leader that adds the group's population
      const unsigned act = __activemask();
      const unsigned peers = __match_any_sync(act, k);
      if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(bucket_count + k, (unsigned long long)__popc(peers));
    }
  }
}

// column counts per colour bucket (bucket C = columns without a valid colour) — plans without a CSC colptr
template <typename CT>
__global__ void __launch_bounds__(kThreads)
count_color_buckets(const CT *__restrict__ jcolor, int64_t n, int32_t C, unsigned long long *__restrict__ bucket_count /* [C+1] */) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c < n; c += stride) {
    uint32_t k = (uint32_t)jcolor[c];
    if (k >= (uint32_t)C) k = (uint32_t)C;
    const unsigned act = __activemask();
    const unsigned peers = __match_any_sync(act, k);
    if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(bucket_count + k, (unsigned long long)__popc(peers));
  }
}

// sort keys of the per-colour column lists: colour id, C for columns without a valid colour; values = the column ids
template <typename CT>
__global__ void __launch_bounds__(kThreads)
color_sort_keys(const CT *__restrict__ jcolor, int64_t n, int32_t C, uint32_t *__restrict__ keys, int32_t *__restrict__ vals) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c < n; c += stride) {
    uint32_t k = (uint32_t)jcolor[c];
    if (k >= (uint32_t)C) k = (uint32_t)C;
    keys[c] = k;
    vals[c] = (int32_t)c;
  }
}

// ---- colour-major entry lists (diff_scatter_cm) ----
// list_cols[i] = i-th column of this rank's colour-major order (its local colours one after the other, then — rank 0
// only — the columns without a valid colour); list_cnt[i] = stored entries of that column.
__global__ void __launch_bounds__(kThreads)
cm_column_counts(const int32_t *__restrict__ list_cols, int64_t ncols, const int32_t *__restrict__ colptr32,
                 int32_t *__restrict__ list_cnt) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t i = blockIdx.x * (int64_t)kThreads + threadIdx.x; i < ncols; i += stride) {
    const int32_t c = list_cols[i];
    list_cnt[i] = colptr32[c + 1] - colptr32[c];
  }
}

// cm_row / cm_slot from the exclusive scan of list_cnt: column i's entries land at [off[i], off[i] + cnt)
template <typename ST>
__global__ void __launch_bounds__(kThreads)
cm_expand(const int32_t *__restrict__ list_cols, const int32_t *__restrict__ list_off, int64_t ncols,
          const int32_t *__restrict__ colptr32, const int32_t *__restrict__ row32, const int64_t *__restrict__ dest,
          int lanes, int32_t *__restrict__ cm_row, ST *__restrict__ cm_slot) {
  const int cols_per_block = kThreads / lanes;
  const int sub = threadIdx.x % lanes;
  for (int64_t i = blockIdx.x * (int64_t)cols_per_block + threadIdx.x / lanes; i < ncols; i += (int64_t)gridDim.x * cols_per_block) {
    const int32_t c = list_cols[i];
    const int32_t p0 = colptr32[c], p1 = colptr32[c + 1];
    const int64_t q0 = list_off[i];
    for (int32_t p = p0 + sub; p < p1; p += lanes) {
      cm_row[q0 + (p - p0)] = row32[p];
      cm_slot[q0 + (p - p0)] = dest ? (ST)dest[p] : (ST)p;
    }
  }
}

// Step-size plan aid: in which aligned lane groups of g = 2,4,8,16,32 consecutive columns does a colour repeat?
// bit log2(g) of *flags is set when some aligned g-group holds two columns of the same valid colour.  The window
// sum-of-squares kernel lets the lanes of a conflict-free group update their shared-memory accumulators without any
// matching (cyclic / banded colourings with C >= 32 are conflict-free at g = 32).
template <typename CT>
__global__ void __launch_bounds__(kThreads)
color_lane_conflicts(const CT *__restrict__ jcolor, int64_t n, int32_t C, uint32_t *__restrict__ flags) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int lane = threadIdx.x & 31;
  uint32_t bad = 0;
  for (int64_t c0 = blockIdx.x * (int64_t)kThreads + threadIdx.x - lane; c0 < n; c0 += stride) {
    const int64_t c = c0 + lane;
    const uint32_t k = c < n ? (uint32_t)jcolor[c] : 0xffffffffu;
    const bool valid = k < (uint32_t)C;
    const unsigned act = __ballot_sync(0xffffffffu, valid);
    if (!valid) continue;
    const unsigned others = __match_any_sync(act, k) & ~(1u << lane);
#pragma unroll
    for (int lg = 1; lg <= 5; ++lg) {
      const int g = 1 << lg;
      const unsigned group = (g == 32 ? 0xffffffffu : ((1u << g) - 1u)) << (lane & ~(g - 1));
      if (others & group) bad |= 1u << lg;
    }
  }
  if (bad) atomicOr(flags, bad);
}

// gather-locality metric: sum over entries of min(|row[e+1]-row[e]|, 2^20) (decides fused single pass vs per-colour passes)
__global__ void __launch_bounds__(kThreads)
row_jump_sum(const int32_t *__restrict__ row32, int64_t E, unsigned long long *__restrict__ out) {
  unsigned long long acc = 0;
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t e = blockIdx.x * (int64_t)kThreads + threadIdx.x; e + 1 < E; e += stride) {
    long long d = (long long)row32[e + 1] - row32[e];
    if (d < 0) d = -d;
    acc += (unsigned long long)(d > (1 << 20) ? (1 << 20) : d);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

// per-colour column counts (banded plans: entries per colour = sum of band lengths of its columns)
template <typename CT>
__global__ void __launch_bounds__(kThreads)
count_band_colors(const CT *__restrict__ jcolor, int64_t m, int64_t n, int64_t l, int64_t u, int32_t C,
                  unsigned long long *__restrict__ color_count) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  for (int64_t c = blockIdx.x * (int64_t)kThreads + threadIdx.x; c < n; c += stride) {
    const uint32_t k = (uint32_t)jcolor[c];
    if (k >= (uint32_t)C) continue;
    int64_t r_lo = c - u; if (r_lo < 0) r_lo = 0;
    int64_t r_hi = c + l; if (r_hi > m - 1) r_hi = m - 1;
    if (r_hi >= r_lo) atomicAdd(color_count + k, (unsigned long long)(r_hi - r_lo + 1));
  }
}

}  // namespace fdb
