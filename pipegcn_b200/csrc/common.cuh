// Shared device/host helpers of libpipegcn_b200 (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/pipegcn_b200.h"

namespace pg {

void set_error(const char* fmt, ...);

// SMs of the current device (132 on an H100 SXM, also the answer without a device): persistent grids and the caps of
// the grid-stride kernels are multiples of it
int sm_count();

#define PG_CHECK_CUDA(expr)                                                              \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      pg::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PG_ERR_CUDA;                                                                \
    }                                                                                    \
  } while (0)

#define PG_REQUIRE(cond, ...)          \
  do {                                 \
    if (!(cond)) {                     \
      pg::set_error(__VA_ARGS__);      \
      return PG_ERR_INVALID;           \
    }                                  \
  } while (0)

#define PG_LAUNCH_CHECK()                                                               \
  do {                                                                                  \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess) {                                                            \
      pg::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return PG_ERR_CUDA;                                                               \
    }                                                                                   \
  } while (0)

// ---- raw vectors of VB bytes -------------------------------------------------------------
template <int VB> struct RawVec;
template <> struct RawVec<16> { using type = uint4; };
template <> struct RawVec<8>  { using type = uint2; };
template <> struct RawVec<4>  { using type = uint32_t; };
template <> struct RawVec<2>  { using type = uint16_t; };

// read-only gather path; rows are re-read by other CTAs, so keep them cacheable in L2/L1
template <int VB>
__device__ __forceinline__ typename RawVec<VB>::type ld_vec(const void* p) {
  return __ldg(reinterpret_cast<const typename RawVec<VB>::type*>(p));
}
template <int VB>
__device__ __forceinline__ void st_vec(void* p, typename RawVec<VB>::type v) {
  *reinterpret_cast<typename RawVec<VB>::type*>(p) = v;
}

// ---- fp32 pairs: two round-to-nearest scalar operations (never contracted into a different rounding) ------
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// ---- unpack VB bytes of T into floats / pack back / accumulate -------------------------------
// Accumulators are float2 pairs: one bf16x2 word unpacks into one pair.
template <typename T, int VB> struct Pack;

template <int VB> struct Pack<float, VB> {
  static constexpr int V = VB / 4;
  static constexpr int NA = (V + 1) / 2;      // float2 accumulators per vector
  using Raw = typename RawVec<VB>::type;
  __device__ __forceinline__ static void unpack(const Raw& r, float* f) {
    const float* p = reinterpret_cast<const float*>(&r);
#pragma unroll
    for (int i = 0; i < V; ++i) f[i] = p[i];
  }
  __device__ __forceinline__ static Raw pack(const float* f) {
    Raw r;
    float* p = reinterpret_cast<float*>(&r);
#pragma unroll
    for (int i = 0; i < V; ++i) p[i] = f[i];
    return r;
  }
  __device__ __forceinline__ static void add(float2* acc, const Raw& r) {
    const float* p = reinterpret_cast<const float*>(&r);
    if constexpr (V == 1) {
      acc[0].x += p[0];
    } else {
#pragma unroll
      for (int i = 0; i < NA; ++i) acc[i] = add2(acc[i], make_float2(p[2 * i], p[2 * i + 1]));
    }
  }
};

template <int VB> struct Pack<__nv_bfloat16, VB> {
  static constexpr int V = VB / 2;
  static constexpr int NA = (V + 1) / 2;
  using Raw = typename RawVec<VB>::type;
  __device__ __forceinline__ static void unpack(const Raw& r, float* f) {
    if constexpr (V == 1) {
      f[0] = __uint_as_float(static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&r)) << 16);
    } else {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&r);
#pragma unroll
      for (int i = 0; i < V / 2; ++i) {           // one word = two bf16: low half, high half
        f[2 * i] = __uint_as_float(w[i] << 16);
        f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
      }
    }
  }
  __device__ __forceinline__ static Raw pack(const float* f) {
    Raw r;
    __nv_bfloat16* p = reinterpret_cast<__nv_bfloat16*>(&r);
#pragma unroll
    for (int i = 0; i < V; ++i) p[i] = __float2bfloat16_rn(f[i]);
    return r;
  }
  __device__ __forceinline__ static void add(float2* acc, const Raw& r) {
    if constexpr (V == 1) {
      acc[0].x += __uint_as_float(static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&r)) << 16);
    } else {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&r);
#pragma unroll
      for (int i = 0; i < NA; ++i)
        acc[i] = add2(acc[i], make_float2(__uint_as_float(w[i] << 16), __uint_as_float(w[i] & 0xffff0000u)));
    }
  }
};

// ---- dropout with a counter-based generator -------------------------------------------------------------------------
// keep(i, k) is a pure function of (seed, step, element): i = row * nvec + (16-byte vector index inside the row), k =
// element inside the vector; 16 random bits per element, two elements per hash.  Every kernel that produces or consumes
// a dropped tensor (pg_dropout, the LayerNorm epilogue, the halo push, the aggregate / fix-up store) evaluates the SAME
// function, so a mask is never stored: out = keep ? x / (1 - p) : 0.
struct DropArg {
  uint32_t thresh16;           // p * 65536 (0: no dropout)
  float scale;                 // 1 / (1 - p)
  uint32_t seed_lo, seed_hi;
  const uint32_t* step_dev;    // device-side epoch counter (may be null: no step mixing)
  int32_t step_off;
};
__device__ __forceinline__ uint32_t mix32(uint32_t x) {       // lowbias32 finaliser
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}
// per-kernel key: the seed's high word mixed with the device-side epoch counter, hashed ONCE per thread
__device__ __forceinline__ uint32_t drop_seed_hi(const DropArg& a) {
  return mix32(a.step_dev != nullptr ? a.seed_hi + 0x632be5abU * (*a.step_dev + static_cast<uint32_t>(a.step_off) + 1u)
                                     : a.seed_hi);
}
// One full-avalanche hash per 16-byte vector (the key enters BEFORE the mix: masks of different epochs are
// uncorrelated), then one odd multiply + xor-shift per pair of elements: 23 integer instructions per 8 elements
// instead of 54 for a full mix per pair.  tools/dropout_hash_quality.py checks keep rate, in-vector, neighbour and
// cross-epoch correlations of exactly this function.
__device__ __forceinline__ uint32_t drop_base(uint64_t i, uint32_t seed_lo, uint32_t key) {
  const uint32_t lo = static_cast<uint32_t>(i), hi = static_cast<uint32_t>(i >> 32);
  return mix32((lo ^ seed_lo) + (key + hi * 0x9e3779b9U));
}
// 2 x 16 random bits for elements (2 * pair, 2 * pair + 1) of the vector
__device__ __forceinline__ uint32_t drop_bits(uint32_t base, int pair) {
  constexpr uint32_t kMul[4] = {0x9e3779b1U, 0x85ebca6bU, 0xc2b2ae35U, 0x27d4eb2fU};
  const uint32_t h = base * kMul[pair & 3];
  return h ^ (h >> 16);
}
template <int V>
__device__ __forceinline__ void drop_apply(float (&f)[V], uint64_t i, uint32_t thresh16, float scale, uint32_t seed_lo,
                                           uint32_t key) {
  const uint32_t base = drop_base(i, seed_lo, key);
#pragma unroll
  for (int k = 0; k < V; k += 2) {
    const uint32_t h = drop_bits(base, k / 2);
    f[k] = ((h & 0xffffU) >= thresh16) ? f[k] * scale : 0.f;
    if (k + 1 < V) f[k + 1] = ((h >> 16) >= thresh16) ? f[k + 1] * scale : 0.f;
  }
}
// one pair of a vector: elements (2 * pair, 2 * pair + 1) of 16-byte vector i, for a kernel whose threads hold pairs
__device__ __forceinline__ void drop_pair(float& a, float& b, uint64_t i, int pair, uint32_t thresh16, float scale,
                                          uint32_t seed_lo, uint32_t key) {
  const uint32_t h = drop_bits(drop_base(i, seed_lo, key), pair);
  a = ((h & 0xffffU) >= thresh16) ? a * scale : 0.f;
  b = ((h >> 16) >= thresh16) ? b * scale : 0.f;
}
// the same function on float2 pairs
template <int H>
__device__ __forceinline__ void drop_apply2(float2 (&f)[H], uint64_t i, uint32_t thresh16, float scale, uint32_t seed_lo,
                                            uint32_t key) {
  const uint32_t base = drop_base(i, seed_lo, key);
  const float2 sc = make_float2(scale, scale);
#pragma unroll
  for (int k = 0; k < H; ++k) {
    const uint32_t h = drop_bits(base, k);
    const float2 m = mul2(f[k], sc);
    f[k].x = ((h & 0xffffU) >= thresh16) ? m.x : 0.f;
    f[k].y = ((h >> 16) >= thresh16) ? m.y : 0.f;
  }
}
// ---- boundary-node sampling (pg_bns) ---------------------------------------------------------------------------------
// Rank r keeps halo row h (its row in r's `_U` space) in epoch t iff mix32(mix32(h ^ k) + k) < thresh, with the key
// k = bns_key(seed, t, r).  A pure function of (seed, t, r, h): the receiver, the sender and the boundary add draw
// the same sample without exchanging it.  tests/test_boundary_sampling_cpu.py ports it to the host.
__device__ __forceinline__ uint32_t bns_epoch(const pg_bns& s) {
  return s.epoch + (s.epoch_dev != nullptr ? *s.epoch_dev : 0u);
}
__device__ __forceinline__ uint32_t bns_key(uint64_t seed, uint32_t t, uint32_t r) {
  const uint32_t k = mix32(static_cast<uint32_t>(seed >> 32) + 0x632be5abU * (t + 1u));
  return mix32((static_cast<uint32_t>(seed) ^ k) + 0x85ebca6bU * (r + 1u));
}
__device__ __forceinline__ bool bns_keep(uint32_t key, uint32_t h, uint32_t thresh) {
  return mix32(mix32(h ^ key) + key) < thresh;
}

inline DropArg make_drop(const pg_drop* d) {
  DropArg a{0u, 1.f, 0u, 0u, nullptr, 0};
  if (d != nullptr && d->p > 0.f) {
    a.thresh16 = static_cast<uint32_t>(d->p * 65536.0f + 0.5f);
    a.scale = 1.0f / (1.0f - d->p);
    a.seed_lo = static_cast<uint32_t>(d->seed);
    a.seed_hi = static_cast<uint32_t>(d->seed >> 32);
    a.step_dev = d->step_dev;
    a.step_off = d->step_off;
  }
  return a;
}

__host__ __device__ inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// largest power-of-two vector width (bytes, <= 16) that divides both the byte stride of a row
// and the base address
inline int vec_bytes(const void* base, int64_t ld_elems, int elem_bytes) {
  uintptr_t a = reinterpret_cast<uintptr_t>(base);
  int64_t stride = ld_elems * elem_bytes;
  int vb = 16;
  while (vb > elem_bytes && ((a % vb) != 0 || (stride % vb) != 0)) vb >>= 1;
  return vb;
}

inline int elem_size(int dtype) { return dtype == PG_BF16 ? 2 : 4; }

}  // namespace pg
