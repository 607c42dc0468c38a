// common.cuh — shared device helpers for libfdjac_b200 (sm_90a only; no other arch is built).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fdb {

// Colour ids are stored 0-based and compressed to the narrowest type that holds maximum(colorvec):
// uint8 (C <= 255), uint16 (C <= 65535) or int32.  The all-ones pattern marks "no valid colour"
// (colorvec[j] < 1 in the caller's array: such a column is never perturbed and its entries stay 0,
// exactly what the reference's `colorvec[col] == color_i` test yields).
template <typename CT> struct ColorTraits;
template <> struct ColorTraits<uint8_t>  { static constexpr uint32_t invalid = 0xFFu; };
template <> struct ColorTraits<uint16_t> { static constexpr uint32_t invalid = 0xFFFFu; };
template <> struct ColorTraits<int32_t>  { static constexpr uint32_t invalid = 0x7FFFFFFFu; };

constexpr int kThreads = 256;

// Streaming kernels walk their data in tiles of kTile consecutive elements per block step.  Lane t of the block owns
// the element PAIRS (tile + 2t, tile + 2t + 1) and (tile + kTile/2 + 2t, ...): every warp-level access is one
// contiguous run (512 B for a double2, 64..256 B for the index/colour pairs) — full sectors in both directions — and
// each thread has two independent pairs in flight.
constexpr int kPairsPerThread = 2;
constexpr int kTile = kThreads * 2 * kPairsPerThread;   // 1024 elements per block step

// streaming (read-once) loads / stores: keep L1/L2 for the gathered vectors
__device__ __forceinline__ double ld_stream(const double *p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(double *p, double v) { __stcs(p, v); }
__device__ __forceinline__ double2 ld_stream2(const double *p) { return __ldcs(reinterpret_cast<const double2 *>(p)); }
__device__ __forceinline__ void st_stream2(double *p, double a, double b) {
  __stcs(reinterpret_cast<double2 *>(p), make_double2(a, b));
}

// two consecutive colour ids with ONE load (16 / 32 / 64 bit)
template <typename CT> __device__ __forceinline__ void ld_color_pair(const CT *p, uint32_t &a, uint32_t &b);
template <> __device__ __forceinline__ void ld_color_pair<uint8_t>(const uint8_t *p, uint32_t &a, uint32_t &b) {
  const uint16_t v = __ldcs(reinterpret_cast<const unsigned short *>(p));
  a = v & 0xFFu; b = v >> 8;
}
template <> __device__ __forceinline__ void ld_color_pair<uint16_t>(const uint16_t *p, uint32_t &a, uint32_t &b) {
  const uint32_t v = __ldcs(reinterpret_cast<const unsigned int *>(p));
  a = v & 0xFFFFu; b = v >> 16;
}
template <> __device__ __forceinline__ void ld_color_pair<int32_t>(const int32_t *p, uint32_t &a, uint32_t &b) {
  const int2 v = __ldcs(reinterpret_cast<const int2 *>(p));
  a = (uint32_t)v.x; b = (uint32_t)v.y;
}

// j / d and j mod d for a divisor fixed at plan time, j < 2^32: one multiply-high, two shifts and a multiply-add instead
// of a division loop (Granlund & Montgomery, "Division by invariant integers using multiplication", PLDI 1994, fig. 4.1)
struct FastDiv {
  uint32_t d, magic, s1, s2;
  __device__ __forceinline__ uint32_t div(uint32_t j) const {
    const uint32_t t = __umulhi(j, magic);
    return (t + ((j - t) >> s1)) >> s2;
  }
  __device__ __forceinline__ uint32_t mod(uint32_t j) const { return j - div(j) * d; }
};
inline FastDiv make_fastdiv(uint32_t d) {   // d >= 1
  uint32_t l = 0;
  while ((1ull << l) < d) ++l;
  FastDiv f;
  f.d = d;
  f.magic = (uint32_t)(((1ull << 32) * ((1ull << l) - d)) / d + 1);
  f.s1 = l > 0 ? 1 : 0;
  f.s2 = l > 0 ? l - 1 : 0;
  return f;
}

// Colour sources: where a kernel finds the 0-based colour of element j (a column, or a structural entry).
//   TableColors<CT>  the plan's array, one CT per element (all-ones = no valid colour);
//   CyclicColors     colorvec[j] == j mod P + 1 (what matrix_colors gives banded / tridiagonal matrices): the closed form,
//                    no array is read.
// tile(base, tid2, ...) yields the colours of the two element pairs a lane owns in the tile at `base` (common tile shape).
template <typename CT> struct TableColors {
  const CT *p;
  __device__ __forceinline__ uint32_t at(int64_t j) const { return (uint32_t)__ldg(p + j); }
  __device__ __forceinline__ void tile(int64_t base, int tid2, uint32_t &a0, uint32_t &a1, uint32_t &b0, uint32_t &b1) const {
    ld_color_pair<CT>(p + base + tid2, a0, a1);
    ld_color_pair<CT>(p + base + kTile / 2 + tid2, b0, b1);
  }
};
struct CyclicColors {
  FastDiv P;                                          // P = maximum(colorvec); element indices are < 2^31
  __device__ __forceinline__ uint32_t at(int64_t j) const { return P.mod((uint32_t)j); }
  __device__ __forceinline__ uint32_t plus(uint32_t a, uint32_t b) const {   // (a + b) mod P for a < P, b <= P
    const uint32_t s = a + b;
    return s >= P.d ? s - P.d : s;
  }
  // one modulo per tile; the lane offsets mod P do not depend on the tile (hoisted out of the tile loops)
  __device__ __forceinline__ void tile(int64_t base, int tid2, uint32_t &a0, uint32_t &a1, uint32_t &b0, uint32_t &b1) const {
    const uint32_t b = P.mod((uint32_t)base);
    a0 = plus(b, P.mod((uint32_t)tid2));
    a1 = plus(a0, 1u);
    b0 = plus(b, P.mod((uint32_t)(kTile / 2 + tid2)));
    b1 = plus(b0, 1u);
  }
};

// Julia Base max(a, b) on Float64: NaN when either argument is NaN (it returns a - b then), otherwise the larger one,
// with +0.0 counted larger than -0.0.  The step-size formula max(relstep*|x|, absstep) uses it, so a NaN in x gives a
// NaN step (a plain `a > b ? a : b` would return absstep).
__host__ __device__ __forceinline__ double max_julia(double a, double b) {
  if (isnan(a) || isnan(b)) return a - b;
  return signbit(a - b) ? b : a;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace fdb
