// The chunk walk shared by the plan-walking kernels (pool.cu, pna.cu, genconv.cu): one warp owns one chunk of a
// pg_csr plan (include/pipegcn_b200.h: pg_csr::chunks) and visits its rows, or its one long-row segment, through
// walk_chunk.
#pragma once
#include "common.cuh"

namespace pg {
namespace {

constexpr int32_t kColMask = 0x7fffffff;  // pidx bit 31 is the "hot row" hint

// the plan's chunk table (include/pipegcn_b200.h: pg_csr::chunks)
struct Walk {
  const int4* chunks;
  int32_t n_chunks;
  const int32_t* pidx;
  const int32_t* prow;
  const int32_t* long_row;
  const int32_t* long_seg_ptr;
  const int32_t* seg_long;
  int32_t n_long;
};

Walk make_walk(const pg_csr* g) {
  return Walk{reinterpret_cast<const int4*>(g->chunks), g->n_chunks, g->pidx, g->prow, g->long_row, g->long_seg_ptr,
              g->seg_long, g->n_long};
}

// Calls f(row, first entry, entries, slot) for every row (slot -1) or long-row segment (slot = its scratch slot) of
// chunk c.
template <typename F>
__device__ __forceinline__ void walk_chunk(const Walk& w, int c, F&& f) {
  const int4 ch = w.chunks[c];
  const int kind = ch.w & 3, nr = ch.w >> 2;
  if (kind == 2) {
    f(w.long_row[w.seg_long[ch.z]], ch.x, ch.y, ch.z);
  } else if (kind == 1) {
    f(w.prow[ch.z], ch.x, ch.y, -1);
  } else {
    for (int j = 0; j < nr; ++j) f(w.prow[ch.z + j], ch.x + j * ch.y, ch.y, -1);
  }
}

// (m, a) <- (x, u) when the row has no candidate yet, x is larger, or x is the first NaN
__device__ __forceinline__ void take_max(float& m, int32_t& a, float x, int32_t u) {
  if (a < 0 || x > m || (x != x && m == m)) { m = x; a = u; }
}

// 16-byte vectors of T
template <typename T> struct Vec {
  static constexpr int V = 16 / static_cast<int>(sizeof(T));
  using P = Pack<T, 16>;
};

template <typename T> __device__ __forceinline__ T to_t(float x);
template <> __device__ __forceinline__ float to_t<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 to_t<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

// V consecutive fp32 values at p (16-byte aligned when all V are valid and V is a multiple of 4): the side outputs and
// operands of pna.cu and genconv.cu
template <int V>
__device__ __forceinline__ void st_f32(float* p, const float (&f)[V], int valid) {
  if (valid >= V && V % 4 == 0) {
#pragma unroll
    for (int k = 0; k < V; k += 4) *reinterpret_cast<float4*>(p + k) = make_float4(f[k], f[k + 1], f[k + 2], f[k + 3]);
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) if (k < valid) p[k] = f[k];
  }
}
template <int V>
__device__ __forceinline__ void ld_f32(const float* p, float (&f)[V], int valid) {
  if (valid >= V && V % 4 == 0) {
#pragma unroll
    for (int k = 0; k < V; k += 4) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(p + k));
      f[k] = x.x; f[k + 1] = x.y; f[k + 2] = x.z; f[k + 3] = x.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) f[k] = k < valid ? __ldg(p + k) : 0.f;
  }
}
// one 16-byte vector of T from V floats (one rounding each), or its first `valid` elements
template <typename T, int V>
__device__ __forceinline__ void st_t(T* p, const float (&f)[V], int valid) {
  if (valid >= V) {
    st_vec<16>(p, Pack<T, 16>::pack(f));
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) if (k < valid) p[k] = to_t<T>(f[k]);
  }
}

int check_plan(const pg_csr* g, const char* who) {
  PG_REQUIRE(g != nullptr, "%s: null plan", who);
  PG_REQUIRE(g->n_rows == 0 || (g->chunks != nullptr && g->pidx != nullptr && g->prow != nullptr),
             "%s: the plan has no chunk table (build it with sorted rows and chunks enabled)", who);
  PG_REQUIRE(g->n_seg == 0 || (g->long_row && g->long_seg_ptr && g->seg_long), "%s: the plan has no long-row split", who);
  return PG_OK;
}

// 16-byte vectors of whole rows: the base is 16-byte aligned and the stride a multiple of 16 bytes
bool vec_ok(const void* p, int64_t ld, int es) {
  return (reinterpret_cast<uintptr_t>(p) % 16) == 0 && (ld * es) % 16 == 0;
}

}  // namespace
}  // namespace pg
