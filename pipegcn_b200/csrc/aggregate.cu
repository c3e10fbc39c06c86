// CSR neighbour aggregate (SURVEY.md K6/K7 forward, K11 backward) for sm_90a.
//
//   out[r,:] = ( sum_{e in row r} x[indices[e],:] ) / row_div[r]  (+ out[r,:] if r < acc_rows)
//
// HBM/L2-bound gather: no tensor cores.  A group of G lanes owns one row (or one segment of a
// long row) and walks its edge list; every lane keeps VPL vectors of VB bytes of the feature
// row in fp32 accumulators, so a neighbour row is fetched with coalesced 16-byte loads
// (one 512 B row of 256 bf16 = one load instruction of a full warp).  U neighbour rows are
// in flight per group before they are accumulated.  Rows longer than seg_len are cut into
// segments reduced by different groups into fp32 partials and summed in segment order by a
// fix-up kernel: deterministic, no atomics.
//
// Every kernel has a compile-time switch SC (pg_aggregate_scaled, GraphConv's symmetric norm):
//   out[r,:] = dst_scale[r] * ( sum_{e in row r} src_scale[indices[e]] * x[indices[e],:] )  (+ bias)
// The lane that loads a column id also loads its source scale; the scale travels with the id (one more shuffle per
// edge) and is applied as a multiply-add per element.  dst_scale arrives in the row_div slot and is a multiplier.
// SC = 0 instantiations are the plain aggregate, instruction for instruction.  The SC kernels hold the scales of
// the rows in flight as well: they are compiled for one resident CTA per SM fewer (agg_occ does not apply), which
// keeps every one of them free of local-memory spills.
//
// SC = 2 (pg_aggregate_scaled_res, GCNII's initial residual) is SC = 1 plus, wherever a finished row is stored,
//   out[r,:] = dst_scale[r] * ( ... ) + alpha * res[r,:]  (+ bias)
// one fp32 multiply-add per element after the row scale, before the single rounding to the output type.  A long row
// gets it in the fix-up only: its segment partials carry the bare sums.  SC = 0 and 1 compile to the code they had.
#include <algorithm>
#include <mutex>
#include <type_traits>
#include <string.h>
#include "common.cuh"

namespace pg {

// the operands of the SC instantiations that have no slot in the plain aggregate's arguments
struct ScaleCore {
  const float* src;    // [source rows] multiplier of every gathered row
  const float* bias;   // [d] added after the row scale, or NULL
  int d;               // columns of the bias and the residual (the pad columns of a vector get none)
};
struct ScaleArg : ScaleCore {
  const void* res;     // SC = 2: [n_rows, ldr] rows of the output type, added times alpha
  int64_t ldr;
  float alpha;
};

// the factor every output row is multiplied by: dst_scale[row] (SC), else the IEEE reciprocal of row_div[row]
template <int SC>
__device__ __forceinline__ float row_scale(const float* __restrict__ row_div, int row) {
  if constexpr (SC != 0) return __ldg(row_div + row);
  return row_div != nullptr ? 1.f / __ldg(row_div + row) : 1.f;
}
// the scale operands a walker holds: none in the plain instantiations, so their code is that of pg_aggregate, and no
// residual operands in the SC = 1 ones, so theirs is that of pg_aggregate_scaled
struct NoScale {};
template <int SC> using ScaleOf = std::conditional_t<SC == 0, NoScale, std::conditional_t<SC == 1, ScaleCore, ScaleArg>>;

// r[0:V] holds columns o .. o+V of the scaled output row `row`: SC = 2 adds alpha * res[row, o:o+V] (one multiply-add),
// then SC with a bias adds bias[o:o+V]; columns past d add nothing
template <int SC, typename P, typename S>
__device__ __forceinline__ void row_epilogue(float* r, const S& sc, int row, int64_t o) {
  constexpr int V = P::V;
  if constexpr (SC == 2) {
    float rv[V];
    P::unpack(*reinterpret_cast<const typename P::Raw*>(static_cast<const typename P::Elem*>(sc.res) + static_cast<int64_t>(row) * sc.ldr + o), rv);
#pragma unroll
    for (int i = 0; i < V; ++i)
      if (o + i < sc.d) r[i] = __fmaf_rn(sc.alpha, rv[i], r[i]);
  }
  if constexpr (SC != 0) {
    if (sc.bias != nullptr) {
#pragma unroll
      for (int i = 0; i < V; ++i)
        if (o + i < sc.d) r[i] += __ldg(sc.bias + o + i);
    }
  }
}

template <typename T, int VB, int G, int VPL, int U, int SC>
__global__ void __launch_bounds__(256)
agg_kernel(pg_csr g, const T* __restrict__ x, uint32_t ldx_bytes, T* __restrict__ out, int64_t ldo, int nvec,
           const float* __restrict__ row_div, int acc_rows, float* __restrict__ scratch, int64_t lds, DropArg drop,
           ScaleArg sc) {
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  constexpr int V = P::V;
  constexpr int NA = P::NA;
  constexpr int GROUPS = 256 / G;
  const int lane_g = threadIdx.x % G;
  const int64_t item = static_cast<int64_t>(blockIdx.x) * GROUPS + threadIdx.x / G;
  const int64_t n_items = static_cast<int64_t>(g.n_rows) + g.n_seg;
  if (item >= n_items) return;   // whole group leaves together

  int row, beg, end, seg = -1;
  if (item < g.n_rows) {
    row = g.row_order ? __ldg(g.row_order + item) : static_cast<int>(item);
    beg = __ldg(g.indptr + row);
    end = __ldg(g.indptr + row + 1);
    if (end - beg > g.seg_len) return;   // long row: its segments do the work
  } else {
    seg = static_cast<int>(item - g.n_rows);
    const int li = __ldg(g.seg_long + seg);
    row = __ldg(g.long_row + li);
    const int k = seg - __ldg(g.long_seg_ptr + li);
    const int rb = __ldg(g.indptr + row), re = __ldg(g.indptr + row + 1);
    beg = rb + k * g.seg_len;
    end = min(re, beg + g.seg_len);
  }

  for (int c0 = 0; c0 < nvec; c0 += G * VPL) {
    float2 acc[VPL][NA];
#pragma unroll
    for (int j = 0; j < VPL; ++j)
#pragma unroll
      for (int i = 0; i < NA; ++i) acc[j][i] = make_float2(0.f, 0.f);
    bool act[VPL];
    const char* xc[VPL];                   // this lane's column(s) of row 0
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      const int vi = c0 + lane_g + j * G;
      act[j] = vi < nvec;
      xc[j] = reinterpret_cast<const char*>(x + static_cast<int64_t>(vi) * V);
    }

    // main loop: U neighbour rows per batch, no tail predicates: U index loads (one broadcast
    // transaction each), then U*VPL 16-byte row loads in flight before the first add.
    // row address = base + src * ldx: one 32x32+64 multiply-add (IMAD.WIDE.U32) per row.
    int e = beg;
    for (; e + U <= end; e += U) {
      uint32_t src[U];
#pragma unroll
      for (int u = 0; u < U; ++u) src[u] = static_cast<uint32_t>(__ldg(g.indices + e + u));
      Raw v[U][VPL];
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < VPL; ++j)
          if (act[j]) v[u][j] = ld_vec<VB>(xc[j] + static_cast<uint64_t>(src[u]) * ldx_bytes);
      float ss[U];
      if constexpr (SC != 0) {
#pragma unroll
        for (int u = 0; u < U; ++u) ss[u] = __ldg(sc.src + src[u]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < VPL; ++j) {
          if constexpr (SC != 0) {
            if (act[j]) P::fma(acc[j], v[u][j], ss[u]);
          } else {
            if (act[j]) P::add(acc[j], v[u][j]);
          }
        }
    }
    for (; e < end; ++e) {
      const uint32_t s = static_cast<uint32_t>(__ldg(g.indices + e));
      if constexpr (SC != 0) {
        const float s1 = __ldg(sc.src + s);
#pragma unroll
        for (int j = 0; j < VPL; ++j)
          if (act[j]) P::fma(acc[j], ld_vec<VB>(xc[j] + static_cast<uint64_t>(s) * ldx_bytes), s1);
      } else {
#pragma unroll
        for (int j = 0; j < VPL; ++j)
          if (act[j]) P::add(acc[j], ld_vec<VB>(xc[j] + static_cast<uint64_t>(s) * ldx_bytes));
      }
    }

    if (seg >= 0) {
      float* sp = scratch + static_cast<int64_t>(seg) * lds;
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        if (!act[j]) continue;
        const int64_t o = static_cast<int64_t>(c0 + lane_g + j * G) * V;
#pragma unroll
        for (int i = 0; i < V; ++i) sp[o + i] = (i & 1) ? acc[j][i / 2].y : acc[j][i / 2].x;
      }
    } else {
      // `/ degs` (layer.py:50) as one IEEE reciprocal per row and a multiply per element (<= 1 ulp from the
      // division): the per-element IEEE division took its slow path on every exact zero (dropout) and was
      // a third of the kernel's instructions in the ncu source view
      const float inv = row_scale<SC>(row_div, row);
      T* op = out + static_cast<int64_t>(row) * ldo;
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        if (!act[j]) continue;
        const int64_t o = static_cast<int64_t>(c0 + lane_g + j * G) * V;
        float r[V];
#pragma unroll
        for (int i = 0; i < V; ++i) {
          const float a = (i & 1) ? acc[j][i / 2].y : acc[j][i / 2].x;
          r[i] = a * inv;
        }
        row_epilogue<SC, P>(r, sc, row, o);
        if (row < acc_rows) {
          float ov[V];
          P::unpack(*reinterpret_cast<const Raw*>(op + o), ov);
#pragma unroll
          for (int i = 0; i < V; ++i) r[i] += ov[i];
        }
        if (drop.thresh16 != 0u)
          drop_apply<V>(r, static_cast<uint64_t>(row) * nvec + (c0 + lane_g + j * G), drop.thresh16, drop.scale, drop.seed_lo, drop_seed_hi(drop));
        st_vec<VB>(op + o, P::pack(r));
      }
    }
  }
}

// sums the fp32 partials of every long row and writes the row: one CTA per long row, warp w adds the segments
// s0 + w, s0 + w + 8, ... (four in flight), then the eight warp sums are added in warp order -- a fixed order, so the
// result does not depend on scheduling
template <typename T, int VB, int SC>
__global__ void __launch_bounds__(256)
agg_fixup_kernel(pg_csr g, T* __restrict__ out, int64_t ldo, int nvec, const float* __restrict__ row_div,
                 int acc_rows, const float* __restrict__ scratch, int64_t lds, DropArg drop, ScaleArg sc) {
  using P = Pack<T, VB>;
  constexpr int V = P::V;
  __shared__ float part[8][32 * V];
  const int li = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int row = __ldg(g.long_row + li);
  const int s0 = __ldg(g.long_seg_ptr + li), s1 = __ldg(g.long_seg_ptr + li + 1);
  const float inv = row_scale<SC>(row_div, row);
  T* op = out + static_cast<int64_t>(row) * ldo;
  for (int v0 = 0; v0 < nvec; v0 += 32) {
    const int vi = v0 + lane;
    float r[V];
#pragma unroll
    for (int i = 0; i < V; ++i) r[i] = 0.f;
    if (vi < nvec) {
      const float* sp = scratch + static_cast<int64_t>(vi) * V;
      int s = s0 + warp;
      for (; s + 24 < s1; s += 32) {
        float t[4][V];
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int i = 0; i < V; ++i) t[u][i] = __ldcs(sp + static_cast<int64_t>(s + 8 * u) * lds + i);
#pragma unroll
        for (int u = 0; u < 4; ++u)
#pragma unroll
          for (int i = 0; i < V; ++i) r[i] += t[u][i];
      }
      for (; s < s1; s += 8)
#pragma unroll
        for (int i = 0; i < V; ++i) r[i] += __ldcs(sp + static_cast<int64_t>(s) * lds + i);
    }
#pragma unroll
    for (int i = 0; i < V; ++i) part[warp][lane * V + i] = r[i];
    __syncthreads();
    if (warp == 0 && vi < nvec) {
#pragma unroll
      for (int i = 0; i < V; ++i) {
        float a = part[0][lane * V + i];
#pragma unroll
        for (int w = 1; w < 8; ++w) a += part[w][lane * V + i];
        r[i] = a * inv;
      }
      row_epilogue<SC, P>(r, sc, row, static_cast<int64_t>(vi) * V);
      if (row < acc_rows) {
        float o[V];
        P::unpack(*reinterpret_cast<const typename P::Raw*>(op + static_cast<int64_t>(vi) * V), o);
#pragma unroll
        for (int i = 0; i < V; ++i) r[i] += o[i];
      }
      if (drop.thresh16 != 0u)
        drop_apply<V>(r, static_cast<uint64_t>(row) * nvec + vi, drop.thresh16, drop.scale, drop.seed_lo, drop_seed_hi(drop));
      st_vec<VB>(op + static_cast<int64_t>(vi) * V, P::pack(r));
    }
    __syncthreads();
  }
}

extern int g_ln_stage, g_ce_subwarp;   // rowops.cu
extern int g_gemm_epi_slabs;   // linear_wgmma.cu
int g_agg_narrow = 1;  // pg_set_option("agg_narrow", 0|1): chunked sub-warp kernels for rows of at most 16 vectors
int g_agg_overlap = 1; // pg_set_option("agg_overlap", 0|1): short-row kernel on a side stream next to the long-row kernel
int g_agg_impl = 2;     // pg_set_option("agg_impl", 1|2|3): 1 = row-per-group kernel, 2 = chunked kernels (need pg_csr::chunks),
                        // 3 = chunked, long rows staged through shared memory with cp.async
int g_agg_unroll = 8;   // pg_set_option("agg_unroll", 4|8): neighbour rows in flight per group (VPL == 1, agg_impl 1)
int g_agg_occ = 4;      // pg_set_option("agg_occ", 4|5): resident CTAs per SM the long-row kernel is compiled for (64 / 48 registers)
int g_agg_l2_hint = 0; // pg_set_option("agg_l2_hint", 0|1): L2 eviction policies by source hotness in the chunked kernels.
                       // OFF by default: the policy select costs 5 of 23 instructions per edge; not measured on H100

// ---------------------------------------------------------------------------------------------------------
// v2: chunked walk over the degree-sorted, permuted CSR (pg_csr::chunks / pidx / prow).
//
// v1 walks a chain of DEPENDENT loads per row --
// row_order -> indptr -> index -> feature row, then one index + one row load per edge in the scalar tail -- while
// 77 % of the rows of an RMAT graph have fewer than 8 entries.  Here a warp takes one CHUNK: either up to 32
// edges' worth of whole rows of equal length (the rows are sorted by length, so a chunk is `n_rows` x `len`), or
// one longer row, or one segment of a long row.  One 16-byte descriptor load, then ONE coalesced load fetches the
// chunk's (next 32) column indices, which are broadcast by shuffles; neighbour rows are fetched U at a time with
// warp-uniform predicates on the ragged end: the dependent chain per chunk is descriptor -> indices -> rows.
// L2 residency by source hotness: bit 31 of a permuted column id marks a source row that is referenced often enough
// to be worth keeping in the 50 MB L2 (the plan marks the most-referenced rows up to a byte budget).  Hot rows are
// loaded with an evict_last policy, everything that is touched once or rarely (cold rows, the index stream, the
// output) with evict_first / streaming hints, so that the long tail does not flush the hubs.
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
template <int VB> __device__ __forceinline__ typename RawVec<VB>::type ld_vec_policy(const void* p, uint64_t pol);
template <> __device__ __forceinline__ uint4 ld_vec_policy<16>(const void* p, uint64_t pol) {
  uint4 v;
  asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0, %1, %2, %3}, [%4], %5;"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol));
  return v;
}
template <> __device__ __forceinline__ uint2 ld_vec_policy<8>(const void* p, uint64_t pol) {
  uint2 v;
  asm volatile("ld.global.nc.L2::cache_hint.v2.u32 {%0, %1}, [%2], %3;" : "=r"(v.x), "=r"(v.y) : "l"(p), "l"(pol));
  return v;
}
template <> __device__ __forceinline__ uint32_t ld_vec_policy<4>(const void* p, uint64_t pol) {
  uint32_t v;
  asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
template <int VB> __device__ __forceinline__ void st_vec_cs(void* p, typename RawVec<VB>::type v);
template <> __device__ __forceinline__ void st_vec_cs<16>(void* p, uint4 v) { __stcs(reinterpret_cast<uint4*>(p), v); }
template <> __device__ __forceinline__ void st_vec_cs<8>(void* p, uint2 v) { __stcs(reinterpret_cast<uint2*>(p), v); }
template <> __device__ __forceinline__ void st_vec_cs<4>(void* p, uint32_t v) { __stcs(reinterpret_cast<uint32_t*>(p), v); }

struct Chunk { int e_beg, n, item, kind_rows; };   // kind = kind_rows & 3 (0: n_rows rows of n edges, 1: one row, 2: segment)

template <typename T, int VB, int VPL, int U, bool HINT, int SC>
struct Agg2 {
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  static constexpr int V = P::V;
  static constexpr int NA = P::NA;
  static constexpr int kVPL = VPL;
  static constexpr bool kSC = SC != 0;
  static constexpr unsigned kFull = 0xffffffffu;

  const char* xc[VPL];      // this lane's column(s) of source row 0
  bool act[VPL];
  uint32_t ldx_bytes;
  uint64_t pol_hot, pol_cold;
  T* out;
  int64_t ldo;
  int col0;                 // first vector column of this lane (c0 + lane)
  int acc_rows;
  int nvec;
  DropArg drop;             // dropout applied to every row as it is written (thresh16 == 0: none)
  uint32_t drop_hi;
  ScaleOf<SC> sc;
  float2 acc[VPL][NA];

  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int j = 0; j < VPL; ++j)
#pragma unroll
      for (int i = 0; i < NA; ++i) acc[j][i] = make_float2(0.f, 0.f);
  }
  // one neighbour-row vector; `s` = column id with the hot flag in bit 31
  __device__ __forceinline__ Raw ld_row(int j, uint32_t s) const {
    const char* p = xc[j] + static_cast<uint64_t>(s & 0x7fffffffu) * ldx_bytes;
    if (HINT) return ld_vec_policy<VB>(p, (s >> 31) ? pol_hot : pol_cold);
    return ld_vec<VB>(p);
  }
  // lanes past the row width (act[j] false) read column 0 like lane 0 does (same address: no extra traffic) and
  // are only masked at the store: the loads and adds of the inner loops carry no predicates
  __device__ __forceinline__ void add(const Raw (&v)[VPL], float s) {
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      if constexpr (SC != 0) P::fma(acc[j], v[j], s);
      else P::add(acc[j], v[j]);
    }
  }
  // source scale of column id `id` (hot flag in bit 31)
  __device__ __forceinline__ float scale_of(uint32_t id) const {
    if constexpr (SC != 0) return __ldg(sc.src + (id & 0x7fffffffu));
    else return 1.f;
  }
  // the ragged end of a batch: every load is issued (positions past the end fetch a valid row: lanes past the
  // chunk hold column 0) and the fetched bits are ANDed with 0 / ~0 -- no predicated loads, no divergent code
  __device__ __forceinline__ void add_masked(const Raw (&v)[VPL], bool keep) {
    const uint32_t m = keep ? 0xffffffffu : 0u;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      Raw t = v[j];
      uint32_t* w = reinterpret_cast<uint32_t*>(&t);
#pragma unroll
      for (int i = 0; i < VB / 4; ++i) w[i] &= m;
      P::add(acc[j], t);
    }
  }
  __device__ __forceinline__ void ld_rows(Raw (&v)[VPL], uint32_t s) const {
#pragma unroll
    for (int j = 0; j < VPL; ++j) v[j] = ld_row(j, s);
  }
  // out[row] = acc * inv (+ out[row] when row < acc_rows); acc = 0
  __device__ __forceinline__ void flush(int row, float inv) {
    T* op = out + static_cast<int64_t>(row) * ldo;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      if (act[j]) {
        const int64_t o = static_cast<int64_t>(col0 + j * 32) * V;
        float r[V];
#pragma unroll
        for (int i = 0; i < V; ++i) r[i] = ((i & 1) ? acc[j][i / 2].y : acc[j][i / 2].x) * inv;
        row_epilogue<SC, P>(r, sc, row, o);
        if (row < acc_rows) {
          float ov[V];
          P::unpack(*reinterpret_cast<const Raw*>(op + o), ov);
#pragma unroll
          for (int i = 0; i < V; ++i) r[i] += ov[i];
        }
        if (drop.thresh16 != 0u)
          drop_apply<V>(r, static_cast<uint64_t>(row) * nvec + (col0 + j * 32), drop.thresh16, drop.scale, drop.seed_lo, drop_hi);
        if (HINT) st_vec_cs<VB>(op + o, P::pack(r));
        else st_vec<VB>(op + o, P::pack(r));
      }
    }
    zero();
  }

  // a chunk of n_rows whole rows of `len` (<= 32) entries each, n_rows * len <= 32: U neighbour rows in flight
  // across row boundaries; a row is flushed as soon as its last entry has been added (warp-uniform branch)
  __device__ __forceinline__ void small_chunk(uint32_t my_idx, float my_sc, int my_row, float my_inv, int n_rows,
                                              int len) {
    const int n_e = n_rows * len;
    int r = 0, cnt = 0;
#pragma unroll 1
    for (int u0 = 0; u0 < n_e; u0 += U) {
      Raw v[U][VPL];
      float s[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        ld_rows(v[u], __shfl_sync(kFull, my_idx, (u0 + u) & 31));   // lanes >= n_e hold 0
        s[u] = SC ? __shfl_sync(kFull, my_sc, (u0 + u) & 31) : 1.f;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (u0 + u < n_e) {
          add(v[u], s[u]);
          if (++cnt == len) {
            flush(__shfl_sync(kFull, my_row, r), __shfl_sync(kFull, my_inv, r));
            ++r;
            cnt = 0;
          }
        }
      }
    }
    if (len == 0)                                          // rows without entries: the empty sum
      for (r = 0; r < n_rows; ++r) flush(__shfl_sync(kFull, my_row, r), 1.f);
  }

  // B neighbour rows (columns my_idx[u0 .. u0+B) of the current 32 indices) fetched, then added in order
  template <int B>
  __device__ __forceinline__ void batch(uint32_t my_idx, float my_sc, int u0) {
    Raw v[B][VPL];
    float s[B];
#pragma unroll
    for (int u = 0; u < B; ++u) {
      ld_rows(v[u], __shfl_sync(kFull, my_idx, u0 + u));
      s[u] = SC ? __shfl_sync(kFull, my_sc, u0 + u) : 1.f;
    }
#pragma unroll
    for (int u = 0; u < B; ++u) add(v[u], s[u]);
  }

  // one row / one segment of n_e entries: 32 indices per coalesced load (the next 32 prefetched), U rows in flight
  __device__ __forceinline__ void long_row(const uint32_t* __restrict__ pidx, int n_e, int lane) {
    uint32_t nxt = lane < n_e ? __ldcs(pidx + lane) : 0u;
    float nxt_sc = (SC && lane < n_e) ? scale_of(nxt) : 1.f;
#pragma unroll 1
    for (int base = 0; base < n_e; base += 32) {
      const uint32_t my_idx = nxt;
      const float my_sc = nxt_sc;
      if (base + 32 + lane < n_e) {
        nxt = __ldcs(pidx + base + 32 + lane);
        if constexpr (SC != 0) nxt_sc = scale_of(nxt);
      }
      const int n = min(32, n_e - base);
      int u0 = 0;
#pragma unroll 1
      for (; u0 + U <= n; u0 += U) batch<U>(my_idx, my_sc, u0);
      // ragged end of the row: 4 + 2 + 1 neighbour rows, no predicated loads
      if (n - u0 >= 4) { batch<4>(my_idx, my_sc, u0); u0 += 4; }
      if (n - u0 >= 2) { batch<2>(my_idx, my_sc, u0); u0 += 2; }
      if (n - u0 >= 1) { batch<1>(my_idx, my_sc, u0); }
    }
  }
};

template <typename A, typename T>
__device__ __forceinline__ void agg2_setup(A& a, const T* x, uint32_t ldx_bytes, T* out, int64_t ldo, int acc_rows, int nvec,
                                           const DropArg& drop, const ScaleArg& sc) {
  if constexpr (A::kSC) a.sc = sc;
  a.ldx_bytes = ldx_bytes;
  a.out = out;
  a.ldo = ldo;
  a.acc_rows = acc_rows;
  a.nvec = nvec;
  a.drop = drop;
  a.drop_hi = drop_seed_hi(drop);
  a.pol_hot = a.pol_cold = 0;
}
template <typename A, typename T>
__device__ __forceinline__ void agg2_columns(A& a, const T* x, int c0, int lane, int nvec) {
  a.col0 = c0 + lane;
#pragma unroll
  for (int j = 0; j < A::kVPL; ++j) {
    const int vi = c0 + lane + j * 32;
    a.act[j] = vi < nvec;
    a.xc[j] = reinterpret_cast<const char*>(x + static_cast<int64_t>(a.act[j] ? vi : 0) * A::V);
  }
  a.zero();
}

// chunks [0, n_chunks_long): one row (kind 1) or one segment of a long row (kind 2) per warp
template <typename T, int VB, int VPL, int U, bool HINT, int OCC, int SC>
__global__ void __launch_bounds__(256, (VPL == 1 ? (SC ? (HINT ? 2 : 3) : OCC) : (VPL == 2 ? 2 : 1)))
agg2_long_kernel(pg_csr g, const T* __restrict__ x, uint32_t ldx_bytes, T* __restrict__ out, int64_t ldo, int nvec,
                 const float* __restrict__ row_div, int acc_rows, float* __restrict__ scratch, int64_t lds, DropArg drop,
                 ScaleArg sc) {
  using A = Agg2<T, VB, VPL, U, HINT, SC>;
  constexpr int V = A::V;
  const int lane = threadIdx.x & 31;
  const int cid = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (cid >= g.n_chunks_long) return;
  const int4 c = __ldcs(reinterpret_cast<const int4*>(g.chunks) + cid);
  const uint32_t* __restrict__ pidx = reinterpret_cast<const uint32_t*>(g.pidx) + c.x;
  A a;
  agg2_setup(a, x, ldx_bytes, out, ldo, acc_rows, nvec, drop, sc);
  if (HINT) {
    a.pol_hot = l2_policy_evict_last();
    a.pol_cold = l2_policy_evict_first();
  }
  for (int c0 = 0; c0 < nvec; c0 += 32 * VPL) {
    agg2_columns(a, x, c0, lane, nvec);
    a.long_row(pidx, c.y, lane);
    if ((c.w & 3) == 2) {
      float* sp = scratch + static_cast<int64_t>(c.z) * lds;
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        if (!a.act[j]) continue;
        const int64_t o = static_cast<int64_t>(c0 + lane + j * 32) * V;
#pragma unroll
        for (int i = 0; i < V; ++i) sp[o + i] = (i & 1) ? a.acc[j][i / 2].y : a.acc[j][i / 2].x;
      }
    } else {
      const int row = __ldg(g.prow + c.z);
      a.flush(row, row_scale<SC>(row_div, row));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// v3 of the long-row kernel: neighbour rows are STAGED THROUGH SHARED MEMORY with asynchronous copies.
// The register-landing kernels are bound by latency x bytes in flight -- a load in flight owns its
// destination registers (32 warps x 8 rows x 512 B = 131 KB per SM).  Here every warp owns a ring of D row slots in shared
// memory; `cp.async` (LDGSTS) moves 16 bytes per lane straight from global memory into the ring, one commit group
// per row, D - 1 rows ahead of the row being added.  A lane reads back exactly the 16 bytes it copied itself, so the
// ring needs no barrier at all: `cp.async.wait_group` is the only synchronisation.
__device__ __forceinline__ void cp_async16(uint32_t smem, const void* gmem) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async16_policy(uint32_t smem, const void* gmem, uint64_t pol) {
  asm volatile("cp.async.ca.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem), "l"(gmem), "l"(pol) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <typename T, int VPL, int D, bool HINT, int SC>
__global__ void __launch_bounds__(256, (VPL == 1 ? (SC ? 4 : 6) : (SC ? 2 : 3)))
agg3_long_kernel(pg_csr g, const T* __restrict__ x, uint32_t ldx_bytes, T* __restrict__ out, int64_t ldo, int nvec,
                 const float* __restrict__ row_div, int acc_rows, float* __restrict__ scratch, int64_t lds, DropArg drop,
                 ScaleArg sc) {
  using A = Agg2<T, 16, VPL, 1, HINT, SC>;
  using Raw = typename A::Raw;
  constexpr int V = A::V;
  constexpr unsigned kFull = 0xffffffffu;
  constexpr int kSlotBytes = VPL * 512;
  extern __shared__ __align__(16) uint8_t agg3_ring[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cid = blockIdx.x * 8 + warp;
  if (cid >= g.n_chunks_long) return;
  const int4 c = __ldcs(reinterpret_cast<const int4*>(g.chunks) + cid);
  const uint32_t* __restrict__ pidx = reinterpret_cast<const uint32_t*>(g.pidx) + c.x;
  const int n_e = c.y;
  // this lane's 16 bytes of slot 0 (piece j at + j * 512)
  const uint32_t ring = static_cast<uint32_t>(__cvta_generic_to_shared(agg3_ring)) + warp * (D * kSlotBytes) + lane * 16;
  A a;
  agg2_setup(a, x, ldx_bytes, out, ldo, acc_rows, nvec, drop, sc);
  if (HINT) {
    a.pol_hot = l2_policy_evict_last();
    a.pol_cold = l2_policy_evict_first();
  }
  auto issue = [&](int e, uint32_t s) {
    const uint32_t dst = ring + static_cast<uint32_t>(e & (D - 1)) * kSlotBytes;
    const uint64_t off = static_cast<uint64_t>(s & 0x7fffffffu) * ldx_bytes;
#pragma unroll
    for (int j = 0; j < VPL; ++j) {
      if (HINT) cp_async16_policy(dst + j * 512, a.xc[j] + off, (s >> 31) ? a.pol_hot : a.pol_cold);
      else cp_async16(dst + j * 512, a.xc[j] + off);
    }
  };
  for (int c0 = 0; c0 < nvec; c0 += 32 * VPL) {
    agg2_columns(a, x, c0, lane, nvec);
    uint32_t idx_a = lane < n_e ? __ldcs(pidx + lane) : 0u;
    uint32_t idx_b = 32 + lane < n_e ? __ldcs(pidx + 32 + lane) : 0u;
    float sc_a = (SC && lane < n_e) ? a.scale_of(idx_a) : 1.f;
#pragma unroll
    for (int k = 0; k < D - 1; ++k) {                       // prologue: rows 0 .. D-2 (all inside the first 32 indices)
      const uint32_t s = __shfl_sync(kFull, idx_a, k);
      if (k < n_e) issue(k, s);
      cp_async_commit();
    }
#pragma unroll 1
    for (int base = 0; base < n_e; base += 32) {
      const int n = min(32, n_e - base);
#pragma unroll 4
      for (int u = 0; u < n; ++u) {
        const int ui = u + D - 1;                            // position of the row to fetch now, relative to `base`
        const uint32_t sa = __shfl_sync(kFull, idx_a, ui & 31), sb = __shfl_sync(kFull, idx_b, ui & 31);
        if (base + ui < n_e) issue(base + ui, ui < 32 ? sa : sb);
        cp_async_commit();
        cp_async_wait<D - 1>();                              // row base + u has landed
        const uint32_t src = ring + static_cast<uint32_t>((base + u) & (D - 1)) * kSlotBytes;
        Raw v[VPL];
#pragma unroll
        for (int j = 0; j < VPL; ++j)
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                       : "=r"(v[j].x), "=r"(v[j].y), "=r"(v[j].z), "=r"(v[j].w) : "r"(src + j * 512));
        a.add(v, SC ? __shfl_sync(kFull, sc_a, u) : 1.f);
      }
      idx_a = idx_b;
      if constexpr (SC != 0) sc_a = base + 32 + lane < n_e ? a.scale_of(idx_a) : 1.f;
      idx_b = base + 64 + lane < n_e ? __ldcs(pidx + base + 64 + lane) : 0u;
    }
    if ((c.w & 3) == 2) {
      float* sp = scratch + static_cast<int64_t>(c.z) * lds;
#pragma unroll
      for (int j = 0; j < VPL; ++j) {
        if (!a.act[j]) continue;
        const int64_t o = static_cast<int64_t>(c0 + lane + j * 32) * V;
#pragma unroll
        for (int i = 0; i < V; ++i) sp[o + i] = (i & 1) ? a.acc[j][i / 2].y : a.acc[j][i / 2].x;
      }
    } else {
      const int row = __ldg(g.prow + c.z);
      a.flush(row, row_scale<SC>(row_div, row));
    }
  }
}

// chunks [n_chunks_long, n_chunks): n_rows whole rows of equal length (<= 32 entries together) per warp
template <typename T, int VB, int VPL, int U, bool HINT, int SC>
__global__ void __launch_bounds__(256, (VPL == 1 ? (SC ? (HINT ? 2 : 3) : 4) : (VPL == 2 ? 2 : 1)))
agg2_small_kernel(pg_csr g, const T* __restrict__ x, uint32_t ldx_bytes, T* __restrict__ out, int64_t ldo, int nvec,
                  const float* __restrict__ row_div, int acc_rows, DropArg drop, ScaleArg sc) {
  using A = Agg2<T, VB, VPL, U, HINT, SC>;
  const int lane = threadIdx.x & 31;
  const int cid = g.n_chunks_long + blockIdx.x * 8 + (threadIdx.x >> 5);
  if (cid >= g.n_chunks) return;
  const int4 c = __ldcs(reinterpret_cast<const int4*>(g.chunks) + cid);
  const int n_rows = c.w >> 2, len = c.y, n_e = len * n_rows;
  const uint32_t my_idx = lane < n_e ? __ldcs(reinterpret_cast<const uint32_t*>(g.pidx) + c.x + lane) : 0u;
  const float my_sc = (SC && lane < n_e) ? __ldg(sc.src + (my_idx & 0x7fffffffu)) : 1.f;
  int my_row = 0;
  float my_inv = 1.f;
  if (lane < n_rows) {
    my_row = __ldg(g.prow + c.z + lane);
    if constexpr (SC != 0) my_inv = __ldg(row_div + my_row);
    else if (row_div != nullptr) my_inv = 1.f / __ldg(row_div + my_row);
  }
  A a;
  agg2_setup(a, x, ldx_bytes, out, ldo, acc_rows, nvec, drop, sc);
  if (HINT) {
    a.pol_hot = l2_policy_evict_last();
    a.pol_cold = l2_policy_evict_first();
  }
  for (int c0 = 0; c0 < nvec; c0 += 32 * VPL) {
    agg2_columns(a, x, c0, lane, nvec);
    a.small_chunk(my_idx, my_sc, my_row, my_inv, n_rows, len);
  }
}

// ---------------------------------------------------------------------------------------------------------
// Narrow rows (at most 16 vectors of 16 bytes: the d_out-wide aggregates of transform-first layers, class-wide
// rows).  G = 4 / 8 / 16 lanes cover one row, so a warp fetches R = 32 / G neighbour rows per load instruction:
//   long rows / segments : lane group q takes the entries q, q + R, q + 2R, ... of the row; the R partial sums are
//                          added with xor-shuffles at the end (fixed order)
//   chunks of short rows : lane group q takes the rows q, q + R, ... of the chunk; all groups walk rows of the same
//                          length, so the flush points are warp-uniform and only the stores are predicated
// Same chunk plan, same coalesced index loads + shuffles as the full-width kernels.
template <typename T, int VB, int G, int SC>
struct AggN {
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  static constexpr int V = P::V;
  static constexpr int NA = P::NA;
  static constexpr int R = 32 / G;
  static constexpr int U = 8;
  static constexpr bool kSC = SC != 0;
  static constexpr unsigned kFull = 0xffffffffu;
  const char* xc;           // this lane's column of source row 0
  bool act;                 // lane's column exists
  uint32_t ldx_bytes;
  T* out;
  int64_t ldo;
  int col, q, acc_rows, nvec;
  DropArg drop;
  uint32_t drop_hi;
  ScaleOf<SC> sc;
  float2 acc[NA];

  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int i = 0; i < NA; ++i) acc[i] = make_float2(0.f, 0.f);
  }
  __device__ __forceinline__ Raw ld_row(uint32_t s) const {
    return ld_vec<VB>(xc + static_cast<uint64_t>(s & 0x7fffffffu) * ldx_bytes);
  }
  __device__ __forceinline__ void add(const Raw& t, float s) {
    if constexpr (SC != 0) P::fma(acc, t, s);
    else P::add(acc, t);
  }
  __device__ __forceinline__ void add_masked(Raw t, bool keep, float s) {
    const uint32_t m = keep ? 0xffffffffu : 0u;
    uint32_t* w = reinterpret_cast<uint32_t*>(&t);
#pragma unroll
    for (int i = 0; i < VB / 4; ++i) w[i] &= m;
    add(t, s);
  }
  __device__ __forceinline__ float scale_of(uint32_t id) const {
    if constexpr (SC != 0) return __ldg(sc.src + (id & 0x7fffffffu));
    else return 1.f;
  }
  __device__ __forceinline__ void store(int row, float inv, bool valid) {
    if (valid && act) {
      T* op = out + static_cast<int64_t>(row) * ldo + static_cast<int64_t>(col) * V;
      float r[V];
#pragma unroll
      for (int i = 0; i < V; ++i) r[i] = ((i & 1) ? acc[i / 2].y : acc[i / 2].x) * inv;
      row_epilogue<SC, P>(r, sc, row, static_cast<int64_t>(col) * V);
      if (row < acc_rows) {
        float ov[V];
        P::unpack(*reinterpret_cast<const Raw*>(op), ov);
#pragma unroll
        for (int i = 0; i < V; ++i) r[i] += ov[i];
      }
      if (drop.thresh16 != 0u)
        drop_apply<V>(r, static_cast<uint64_t>(row) * nvec + col, drop.thresh16, drop.scale, drop.seed_lo, drop_hi);
      st_vec<VB>(op, P::pack(r));
    }
    zero();
  }
  // sum of the R group partials into every lane (xor butterflies: the same order on every lane)
  __device__ __forceinline__ void reduce_groups() {
#pragma unroll
    for (int off = G; off < 32; off <<= 1)
#pragma unroll
      for (int i = 0; i < NA; ++i) {
        acc[i].x += __shfl_xor_sync(kFull, acc[i].x, off);
        acc[i].y += __shfl_xor_sync(kFull, acc[i].y, off);
      }
  }
};

template <typename A, typename T>
__device__ __forceinline__ void aggn_setup(A& a, const T* x, uint32_t ldx_bytes, T* out, int64_t ldo, int acc_rows, int nvec,
                                           const DropArg& drop, const ScaleArg& sc, int lane) {
  if constexpr (A::kSC) a.sc = sc;
  constexpr int G = 32 / A::R;
  a.col = lane % G;
  a.q = lane / G;
  a.act = a.col < nvec;
  a.xc = reinterpret_cast<const char*>(x + static_cast<int64_t>(a.act ? a.col : 0) * A::V);
  a.ldx_bytes = ldx_bytes;
  a.out = out;
  a.ldo = ldo;
  a.acc_rows = acc_rows;
  a.nvec = nvec;
  a.drop = drop;
  a.drop_hi = drop_seed_hi(drop);
  a.zero();
}

template <typename T, int VB, int G, int SC>
__global__ void __launch_bounds__(256, SC ? (G == 16 ? 2 : 3) : 4)
aggn_long_kernel(pg_csr g, const T* __restrict__ x, uint32_t ldx_bytes, T* __restrict__ out, int64_t ldo, int nvec,
                 const float* __restrict__ row_div, int acc_rows, float* __restrict__ scratch, int64_t lds, DropArg drop,
                 ScaleArg sc) {
  using A = AggN<T, VB, G, SC>;
  using Raw = typename A::Raw;
  constexpr int V = A::V, R = A::R, U = A::U;
  constexpr unsigned kFull = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int cid = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (cid >= g.n_chunks_long) return;
  const int4 c = __ldcs(reinterpret_cast<const int4*>(g.chunks) + cid);
  const uint32_t* __restrict__ pidx = reinterpret_cast<const uint32_t*>(g.pidx) + c.x;
  const int n_e = c.y;
  A a;
  aggn_setup(a, x, ldx_bytes, out, ldo, acc_rows, nvec, drop, sc, lane);
  uint32_t nxt = lane < n_e ? __ldcs(pidx + lane) : 0u;
  float nxt_sc = (SC && lane < n_e) ? a.scale_of(nxt) : 1.f;
#pragma unroll 1
  for (int base = 0; base < n_e; base += 32) {
    const uint32_t my_idx = nxt;                          // lanes past the end hold column 0: a valid row
    const float my_sc = nxt_sc;
    if (base + 32 + lane < n_e) {
      nxt = __ldcs(pidx + base + 32 + lane);
      if constexpr (SC != 0) nxt_sc = a.scale_of(nxt);
    }
    const int n = min(32, n_e - base);
    // step u of this block: group q fetches entry u * R + q
#pragma unroll 1
    for (int u0 = 0; u0 * R < n; u0 += U) {
      Raw v[U];
      float s[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        v[u] = a.ld_row(__shfl_sync(kFull, my_idx, ((u0 + u) * R + a.q) & 31));
        s[u] = SC ? __shfl_sync(kFull, my_sc, ((u0 + u) * R + a.q) & 31) : 1.f;
      }
      if (n == 32 && (u0 + U) * R <= 32) {
#pragma unroll
        for (int u = 0; u < U; ++u) a.add(v[u], s[u]);
      } else {
#pragma unroll
        for (int u = 0; u < U; ++u) a.add_masked(v[u], (u0 + u) * R + a.q < n, s[u]);
      }
    }
  }
  a.reduce_groups();
  if ((c.w & 3) == 2) {
    if (a.q == 0 && a.act) {
      float* sp = scratch + static_cast<int64_t>(c.z) * lds + static_cast<int64_t>(a.col) * V;
#pragma unroll
      for (int i = 0; i < V; ++i) sp[i] = (i & 1) ? a.acc[i / 2].y : a.acc[i / 2].x;
    }
  } else {
    const int row = __ldg(g.prow + c.z);
    a.store(row, row_scale<SC>(row_div, row), a.q == 0);
  }
}

template <typename T, int VB, int G, int SC>
__global__ void __launch_bounds__(256, SC ? (G == 16 ? 2 : 3) : 4)
aggn_small_kernel(pg_csr g, const T* __restrict__ x, uint32_t ldx_bytes, T* __restrict__ out, int64_t ldo, int nvec,
                  const float* __restrict__ row_div, int acc_rows, DropArg drop, ScaleArg sc) {
  using A = AggN<T, VB, G, SC>;
  using Raw = typename A::Raw;
  constexpr int R = A::R, U = A::U;
  constexpr unsigned kFull = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int cid = g.n_chunks_long + blockIdx.x * 8 + (threadIdx.x >> 5);
  if (cid >= g.n_chunks) return;
  const int4 c = __ldcs(reinterpret_cast<const int4*>(g.chunks) + cid);
  const int n_rows = c.w >> 2, len = c.y, n_e = len * n_rows;
  const uint32_t my_idx = lane < n_e ? __ldcs(reinterpret_cast<const uint32_t*>(g.pidx) + c.x + lane) : 0u;
  const float my_sc = (SC && lane < n_e) ? __ldg(sc.src + (my_idx & 0x7fffffffu)) : 1.f;
  int my_row = 0;
  float my_inv = 1.f;
  if (lane < n_rows) {
    my_row = __ldg(g.prow + c.z + lane);
    if constexpr (SC != 0) my_inv = __ldg(row_div + my_row);
    else if (row_div != nullptr) my_inv = 1.f / __ldg(row_div + my_row);
  }
  A a;
  aggn_setup(a, x, ldx_bytes, out, ldo, acc_rows, nvec, drop, sc, lane);
  // group q walks the rows q, q + R, ...: T rows of `len` entries each, the same positions in every group
  const int t_rows = (n_rows + R - 1) / R;
  if (len == 0) {
    for (int t = 0; t < t_rows; ++t) {
      const int rq = t * R + a.q;
      a.store(__shfl_sync(kFull, my_row, rq & 31), 1.f, rq < n_rows);
    }
    return;
  }
  const int n_pos = t_rows * len;
  int t_ld = 0, k_ld = 0;                                 // (row-in-group, entry) of the next position to fetch
  int t_add = 0, k_add = 0;
#pragma unroll 1
  for (int p0 = 0; p0 < n_pos; p0 += U) {
    Raw v[U];
    float s[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int rq = t_ld * R + a.q;
      v[u] = a.ld_row(__shfl_sync(kFull, my_idx, (rq * len + k_ld) & 31));      // lanes >= n_e hold column 0
      s[u] = SC ? __shfl_sync(kFull, my_sc, (rq * len + k_ld) & 31) : 1.f;
      if (++k_ld == len) { k_ld = 0; ++t_ld; }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (p0 + u < n_pos) {                                 // warp-uniform
        const int rq = t_add * R + a.q;
        a.add_masked(v[u], rq < n_rows, s[u]);
        if (++k_add == len) {
          a.store(__shfl_sync(kFull, my_row, rq & 31), __shfl_sync(kFull, my_inv, rq & 31), rq < n_rows);
          k_add = 0;
          ++t_add;
        }
      }
    }
  }
}

template <typename T, int VB, int G, int SC>
static int launch_aggn(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec, const float* row_div,
                       int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st);

// The long-row kernel is bound by instruction issue and L2 bandwidth, the short-row kernel by DRAM latency (it
// touches the cold sources and writes most of the output): they run side by side, the short rows on a side stream
// forked from and joined to the caller's stream with events (legal inside a CUDA-graph capture).
struct AggSide { cudaStream_t main; cudaStream_t side; cudaEvent_t fork, join; };
static AggSide g_agg_side[32];
static int g_agg_n_side = 0;
static AggSide* agg_side_for(cudaStream_t st) {
  for (int i = 0; i < g_agg_n_side; ++i)
    if (g_agg_side[i].main == st) return &g_agg_side[i];
  if (g_agg_n_side == 32) return nullptr;
  AggSide& e = g_agg_side[g_agg_n_side];
  e.main = st;
  if (cudaStreamCreateWithFlags(&e.side, cudaStreamNonBlocking) != cudaSuccess ||
      cudaEventCreateWithFlags(&e.fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&e.join, cudaEventDisableTiming) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  ++g_agg_n_side;
  return &e;
}

template <typename T, int VB, int VPL, bool HINT, int SC>
static int launch_agg2h(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec,
                        const float* row_div, int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
  constexpr int U = (VPL >= 4) ? 2 : (VPL == 2 ? 4 : 8);
  const uint32_t ldxb = static_cast<uint32_t>(ldx * sizeof(T));
  AggSide* side = nullptr;
  if (g.n_chunks > g.n_chunks_long) {                     // the short rows first, on the side stream if there is other work
    const unsigned blocks = static_cast<unsigned>((g.n_chunks - g.n_chunks_long + 7) / 8);
    cudaStream_t ss = st;
    if (g_agg_overlap && g.n_chunks_long > 0 && (side = agg_side_for(st)) != nullptr) {
      PG_CHECK_CUDA(cudaEventRecord(side->fork, st));
      PG_CHECK_CUDA(cudaStreamWaitEvent(side->side, side->fork, 0));
      ss = side->side;
    }
    agg2_small_kernel<T, VB, VPL, U, HINT, SC><<<blocks, 256, 0, ss>>>(g, x, ldxb, out, ldo, nvec, row_div, acc_rows, da, sc);
    PG_LAUNCH_CHECK();
    if (side != nullptr) PG_CHECK_CUDA(cudaEventRecord(side->join, ss));
  }
  if (g.n_chunks_long > 0 && g_agg_impl == 3 && VB == 16) {
    constexpr int D = (VPL >= 4) ? 4 : 8;
    const unsigned blocks = static_cast<unsigned>((g.n_chunks_long + 7) / 8);
    const size_t smem = static_cast<size_t>(8) * D * VPL * 512;
    static bool attr_done = false;
    if (!attr_done) {
      PG_CHECK_CUDA(cudaFuncSetAttribute(agg3_long_kernel<T, VPL, D, HINT, SC>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
      PG_CHECK_CUDA(cudaFuncSetAttribute(agg3_long_kernel<T, VPL, D, HINT, SC>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
      attr_done = true;
    }
    agg3_long_kernel<T, VPL, D, HINT, SC><<<blocks, 256, smem, st>>>(g, x, ldxb, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  } else if (g.n_chunks_long > 0) {
    const unsigned blocks = static_cast<unsigned>((g.n_chunks_long + 7) / 8);
    if (VPL == 1 && g_agg_occ == 5)
      agg2_long_kernel<T, VB, VPL, U, HINT, (VPL == 1 && !SC ? 5 : 4), SC><<<blocks, 256, 0, st>>>(g, x, ldxb, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    else
      agg2_long_kernel<T, VB, VPL, U, HINT, 4, SC><<<blocks, 256, 0, st>>>(g, x, ldxb, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  }
  if (g.n_long > 0) {
    agg_fixup_kernel<T, VB, SC><<<g.n_long, 256, 0, st>>>(g, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  }
  if (side != nullptr) PG_CHECK_CUDA(cudaStreamWaitEvent(st, side->join, 0));
  return PG_OK;
}

template <typename T, int VB, int G, int SC>
static int launch_aggn(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec, const float* row_div,
                       int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
  const uint32_t ldxb = static_cast<uint32_t>(ldx * sizeof(T));
  AggSide* side = nullptr;
  if (g.n_chunks > g.n_chunks_long) {
    const unsigned blocks = static_cast<unsigned>((g.n_chunks - g.n_chunks_long + 7) / 8);
    cudaStream_t ss = st;
    if (g_agg_overlap && g.n_chunks_long > 0 && (side = agg_side_for(st)) != nullptr) {
      PG_CHECK_CUDA(cudaEventRecord(side->fork, st));
      PG_CHECK_CUDA(cudaStreamWaitEvent(side->side, side->fork, 0));
      ss = side->side;
    }
    aggn_small_kernel<T, VB, G, SC><<<blocks, 256, 0, ss>>>(g, x, ldxb, out, ldo, nvec, row_div, acc_rows, da, sc);
    PG_LAUNCH_CHECK();
    if (side != nullptr) PG_CHECK_CUDA(cudaEventRecord(side->join, ss));
  }
  if (g.n_chunks_long > 0) {
    const unsigned blocks = static_cast<unsigned>((g.n_chunks_long + 7) / 8);
    aggn_long_kernel<T, VB, G, SC><<<blocks, 256, 0, st>>>(g, x, ldxb, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  }
  if (g.n_long > 0) {
    agg_fixup_kernel<T, VB, SC><<<g.n_long, 256, 0, st>>>(g, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  }
  if (side != nullptr) PG_CHECK_CUDA(cudaStreamWaitEvent(st, side->join, 0));
  return PG_OK;
}

template <typename T, int VB, int VPL, int SC>
static int launch_agg2(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec,
                       const float* row_div, int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
  if (g_agg_l2_hint) return launch_agg2h<T, VB, VPL, true, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
  return launch_agg2h<T, VB, VPL, false, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
}

int g_agg_pack_short = 0;   // pg_set_option("agg_pack_short", 0|1): 16 lanes x 2 vectors per row when rows are short.
                            // OFF by default; not measured on H100

template <typename T, int VB, int G, int VPL, int U, int SC>
static int launch_agg_u(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec,
                        const float* row_div, int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st);

template <typename T, int VB, int G, int VPL, int SC>
static int launch_agg(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec,
                      const float* row_div, int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
  if (VPL == 1 && g_agg_unroll == 4)
    return launch_agg_u<T, VB, G, VPL, 4, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
  constexpr int U = (VPL >= 4) ? 2 : (VPL == 2 ? 4 : 8);
  return launch_agg_u<T, VB, G, VPL, U, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
}

template <typename T, int VB, int G, int VPL, int U, int SC>
static int launch_agg_u(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec,
                        const float* row_div, int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
  constexpr int GROUPS = 256 / G;
  const int64_t n_items = static_cast<int64_t>(g.n_rows) + g.n_seg;
  if (n_items > 0) {
    const int64_t blocks = (n_items + GROUPS - 1) / GROUPS;
    agg_kernel<T, VB, G, VPL, U, SC><<<static_cast<unsigned>(blocks), 256, 0, st>>>(g, x, static_cast<uint32_t>(ldx * sizeof(T)), out, ldo, nvec, row_div,
                                                                                acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  }
  if (g.n_long > 0) {
    agg_fixup_kernel<T, VB, SC><<<g.n_long, 256, 0, st>>>(g, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

template <typename T, int VB, int SC>
static int dispatch_agg(const pg_csr& g, const T* x, int64_t ldx, T* out, int64_t ldo, int nvec,
                        const float* row_div, int acc_rows, float* scratch, int64_t lds, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
#define PG_AGG(G_, VPL_) return launch_agg<T, VB, G_, VPL_, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st)
  if (g_agg_impl >= 2 && g.chunks != nullptr && nvec > 16) {
    if (nvec <= 32) return launch_agg2<T, VB, 1, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    if (nvec <= 64) return launch_agg2<T, VB, 2, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    return launch_agg2<T, VB, 4, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
  }
  if (g_agg_impl >= 2 && g.chunks != nullptr && g_agg_narrow) {
    if (nvec <= 4) return launch_aggn<T, VB, 4, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    if (nvec <= 8) return launch_aggn<T, VB, 8, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    return launch_aggn<T, VB, 16, SC>(g, x, ldx, out, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
  }
  if (nvec <= 4) PG_AGG(4, 1);
  if (nvec <= 8) PG_AGG(8, 1);
  if (nvec <= 16) PG_AGG(16, 1);
  // short rows (mean length < 12, e.g. the backward over a partition's halo rows): two rows per warp, each lane
  // owning two 16-byte vectors, doubles the rows in flight for the same bytes per load instruction
  if (nvec <= 32 && g_agg_pack_short && g.n_rows > 0 && g.nnz < 12 * static_cast<int64_t>(g.n_rows)) PG_AGG(16, 2);
  if (nvec <= 32) PG_AGG(32, 1);
  if (nvec <= 64) PG_AGG(32, 2);
  PG_AGG(32, 4);
#undef PG_AGG
}

template <typename T, int SC>
static int aggregate_t(const pg_csr& g, const void* x, int64_t ldx, void* out, int64_t ldo, int d,
                       const float* row_div, int acc_rows, float* scratch, const DropArg& da, const ScaleArg& sc, cudaStream_t st) {
  const int es = sizeof(T);
  int vb = min(vec_bytes(x, ldx, es), vec_bytes(out, ldo, es));
  if constexpr (SC == 2) vb = min(vb, vec_bytes(sc.res, sc.ldr, es));
  // a vector must not straddle two rows: either d is a multiple of the vector or every stride leaves room
  while (vb > es) {
    const int v = vb / es;
    const int64_t dp = round_up(d, v);
    if (d % v == 0 || (dp <= ldx && dp <= ldo && (SC != 2 || dp <= sc.ldr))) break;
    vb >>= 1;
  }
  const int v = vb / es;
  const int nvec = static_cast<int>(round_up(d, v) / v);
  const int64_t lds = round_up(d, 8);
  PG_REQUIRE(g.n_seg == 0 || scratch != nullptr, "pg_aggregate: scratch is NULL but the graph has %d long-row segments", g.n_seg);
  PG_REQUIRE(da.thresh16 == 0u || vb == 16, "pg_aggregate_drop: the dropout mask is defined on 16-byte vectors (rows must be 16-byte aligned and padded)");
  const T* xp = static_cast<const T*>(x);
  T* op = static_cast<T*>(out);
  switch (vb) {
    case 16: return dispatch_agg<T, 16, SC>(g, xp, ldx, op, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    case 8: return dispatch_agg<T, 8, SC>(g, xp, ldx, op, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    case 4: return dispatch_agg<T, 4, SC>(g, xp, ldx, op, ldo, nvec, row_div, acc_rows, scratch, lds, da, sc, st);
    default:
      set_error("pg_aggregate: rows must be at least 4-byte aligned (vector width %d)", vb);
      return PG_ERR_INVALID;
  }
}

template <typename T, int VB>
__global__ void __launch_bounds__(256)
row_div_kernel(const T* __restrict__ x, int64_t ldx, T* __restrict__ out, int64_t ldo, int n_rows, int nvec,
               const float* __restrict__ row_div) {
  using P = Pack<T, VB>;
  constexpr int V = P::V;
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / nvec), vi = static_cast<int>(i % nvec);
    float f[V];
    P::unpack(ld_vec<VB>(x + static_cast<int64_t>(r) * ldx + static_cast<int64_t>(vi) * V), f);
    const float inv = 1.f / __ldg(row_div + r);
#pragma unroll
    for (int k = 0; k < V; ++k) f[k] *= inv;
    st_vec<VB>(out + static_cast<int64_t>(r) * ldo + static_cast<int64_t>(vi) * V, P::pack(f));
  }
}

template <typename T>
static int row_div_t(const void* x, int64_t ldx, void* out, int64_t ldo, int n_rows, int d, const float* row_div,
                     cudaStream_t st) {
  const int es = sizeof(T);
  int vb = min(vec_bytes(x, ldx, es), vec_bytes(out, ldo, es));
  while (vb > es) {
    const int v = vb / es;
    const int64_t dp = round_up(d, v);
    if (d % v == 0 || (dp <= ldx && dp <= ldo)) break;
    vb >>= 1;
  }
  const int v = vb / es;
  const int nvec = static_cast<int>(round_up(d, v) / v);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  if (total == 0) return PG_OK;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, sm_count() * 16));
  const T* xp = static_cast<const T*>(x);
  T* op = static_cast<T*>(out);
  switch (vb) {
    case 16: row_div_kernel<T, 16><<<blocks, 256, 0, st>>>(xp, ldx, op, ldo, n_rows, nvec, row_div); break;
    case 8: row_div_kernel<T, 8><<<blocks, 256, 0, st>>>(xp, ldx, op, ldo, n_rows, nvec, row_div); break;
    case 4: row_div_kernel<T, 4><<<blocks, 256, 0, st>>>(xp, ldx, op, ldo, n_rows, nvec, row_div); break;
    default:
      set_error("pg_row_div: rows must be at least 4-byte aligned");
      return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

// CUDA loads kernels lazily, and loading one may wait for the device: every SC instantiation is loaded at the first
// pg_aggregate_scaled call (or pg_aggregate_scaled_preload), before a halo wait of a simulated rank can spin; the SC = 2
// ones likewise at the first pg_aggregate_scaled_res call (or pg_aggregate_scaled_res_preload)
template <typename T, int VB, int VPL, bool HINT, int SC>
static void preload_agg2(cudaFuncAttributes* a) {
  constexpr int U = (VPL >= 4) ? 2 : (VPL == 2 ? 4 : 8);
  constexpr int D = (VPL >= 4) ? 4 : 8;
  cudaFuncGetAttributes(a, agg2_small_kernel<T, VB, VPL, U, HINT, SC>);
  cudaFuncGetAttributes(a, agg2_long_kernel<T, VB, VPL, U, HINT, 4, SC>);
  cudaFuncGetAttributes(a, agg3_long_kernel<T, VPL, D, HINT, SC>);
}
template <typename T, int VB, int SC>
static void preload_vb(cudaFuncAttributes* a) {
  preload_agg2<T, VB, 1, false, SC>(a); preload_agg2<T, VB, 2, false, SC>(a); preload_agg2<T, VB, 4, false, SC>(a);
  preload_agg2<T, VB, 1, true, SC>(a); preload_agg2<T, VB, 2, true, SC>(a); preload_agg2<T, VB, 4, true, SC>(a);
  cudaFuncGetAttributes(a, aggn_small_kernel<T, VB, 4, SC>);
  cudaFuncGetAttributes(a, aggn_small_kernel<T, VB, 8, SC>);
  cudaFuncGetAttributes(a, aggn_small_kernel<T, VB, 16, SC>);
  cudaFuncGetAttributes(a, aggn_long_kernel<T, VB, 4, SC>);
  cudaFuncGetAttributes(a, aggn_long_kernel<T, VB, 8, SC>);
  cudaFuncGetAttributes(a, aggn_long_kernel<T, VB, 16, SC>);
  cudaFuncGetAttributes(a, agg_fixup_kernel<T, VB, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 4, 1, 8, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 4, 1, 4, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 8, 1, 8, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 8, 1, 4, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 16, 1, 8, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 16, 1, 4, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 16, 2, 4, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 32, 1, 8, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 32, 1, 4, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 32, 2, 4, SC>);
  cudaFuncGetAttributes(a, agg_kernel<T, VB, 32, 4, 2, SC>);
}
template <int SC>
static void aggregate_scaled_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncAttributes a;
    preload_vb<float, 16, SC>(&a); preload_vb<float, 8, SC>(&a); preload_vb<float, 4, SC>(&a);
    preload_vb<__nv_bfloat16, 16, SC>(&a); preload_vb<__nv_bfloat16, 8, SC>(&a); preload_vb<__nv_bfloat16, 4, SC>(&a);
    cudaGetLastError();
  });
}

}  // namespace pg

extern "C" int pg_set_option(const char* name, int value) {
  PG_REQUIRE(name != nullptr, "pg_set_option: null name");
  if (strcmp(name, "agg_unroll") == 0) {
    PG_REQUIRE(value == 4 || value == 8, "agg_unroll must be 4 or 8");
    pg::g_agg_unroll = value;
    return PG_OK;
  }
  if (strcmp(name, "agg_narrow") == 0) {
    pg::g_agg_narrow = value ? 1 : 0;
    return PG_OK;
  }
  if (strcmp(name, "agg_overlap") == 0) {
    pg::g_agg_overlap = value ? 1 : 0;
    return PG_OK;
  }
  if (strcmp(name, "agg_occ") == 0) {
    PG_REQUIRE(value == 4 || value == 5, "agg_occ must be 4 or 5");
    pg::g_agg_occ = value;
    return PG_OK;
  }
  if (strcmp(name, "agg_l2_hint") == 0) {
    pg::g_agg_l2_hint = value ? 1 : 0;
    return PG_OK;
  }
  if (strcmp(name, "agg_impl") == 0) {
    PG_REQUIRE(value >= 1 && value <= 3, "agg_impl must be 1, 2 or 3");
    pg::g_agg_impl = value;
    return PG_OK;
  }
  if (strcmp(name, "agg_pack_short") == 0) {
    pg::g_agg_pack_short = value ? 1 : 0;
    return PG_OK;
  }
  if (strcmp(name, "ln_stage") == 0) {
    PG_REQUIRE(value >= 0 && value <= 2, "ln_stage must be 0, 1 or 2");
    pg::g_ln_stage = value;
    return PG_OK;
  }
  if (strcmp(name, "gemm_epi_slabs") == 0) {
    PG_REQUIRE(value == 1 || value == 2, "gemm_epi_slabs must be 1 or 2");
    pg::g_gemm_epi_slabs = value;
    return PG_OK;
  }
  if (strcmp(name, "ce_subwarp") == 0) {
    pg::g_ce_subwarp = value ? 1 : 0;
    return PG_OK;
  }
  pg::set_error("pg_set_option: unknown option '%s'", name);
  return PG_ERR_INVALID;
}

extern "C" int pg_aggregate(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d, int dtype,
                            const float* row_div, int32_t acc_rows, float* scratch, void* stream) {
  return pg_aggregate_drop(g, x, ldx, out, ldo, d, dtype, row_div, acc_rows, scratch, nullptr, stream);
}

extern "C" int pg_aggregate_drop(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d, int dtype,
                                 const float* row_div, int32_t acc_rows, float* scratch, const pg_drop* drop, void* stream) {
  const pg::DropArg da = pg::make_drop(drop);
  PG_REQUIRE(g && x && out, "pg_aggregate: null argument");
  PG_REQUIRE(g->n_rows >= 0 && g->seg_len > 0 && d > 0, "pg_aggregate: bad sizes (n_rows=%d seg_len=%d d=%d)", g->n_rows, g->seg_len, d);
  PG_REQUIRE(ldx >= d && ldo >= d && ldx < (1ll << 29), "pg_aggregate: row stride smaller than d (or >= 2^29 elements)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const pg::ScaleArg sc{{nullptr, nullptr, 0}, nullptr, 0, 0.f};
  if (dtype == PG_F32) return pg::aggregate_t<float, 0>(*g, x, ldx, out, ldo, d, row_div, acc_rows, scratch, da, sc, st);
  if (dtype == PG_BF16)
    return pg::aggregate_t<__nv_bfloat16, 0>(*g, x, ldx, out, ldo, d, row_div, acc_rows, scratch, da, sc, st);
  pg::set_error("pg_aggregate: unknown dtype %d", dtype);
  return PG_ERR_INVALID;
}

extern "C" int pg_aggregate_scaled(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d,
                                   int dtype, const float* src_scale, const float* dst_scale, const float* bias,
                                   float* scratch, const pg_drop* drop, void* stream) {
  const pg::DropArg da = pg::make_drop(drop);
  PG_REQUIRE(g && x && out && src_scale && dst_scale, "pg_aggregate_scaled: null argument");
  PG_REQUIRE(g->n_rows >= 0 && g->seg_len > 0 && d > 0, "pg_aggregate_scaled: bad sizes (n_rows=%d seg_len=%d d=%d)",
             g->n_rows, g->seg_len, d);
  PG_REQUIRE(ldx >= d && ldo >= d && ldx < (1ll << 29), "pg_aggregate_scaled: row stride smaller than d (or >= 2^29 elements)");
  pg::aggregate_scaled_preload<1>();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const pg::ScaleArg sc{{src_scale, bias, d}, nullptr, 0, 0.f};
  if (dtype == PG_F32) return pg::aggregate_t<float, 1>(*g, x, ldx, out, ldo, d, dst_scale, 0, scratch, da, sc, st);
  if (dtype == PG_BF16)
    return pg::aggregate_t<__nv_bfloat16, 1>(*g, x, ldx, out, ldo, d, dst_scale, 0, scratch, da, sc, st);
  pg::set_error("pg_aggregate_scaled: unknown dtype %d", dtype);
  return PG_ERR_INVALID;
}

extern "C" int pg_aggregate_scaled_preload(void) {
  pg::aggregate_scaled_preload<1>();
  return PG_OK;
}

extern "C" int pg_aggregate_scaled_res(const pg_csr* g, const void* x, int64_t ldx, void* out, int64_t ldo, int32_t d,
                                       int dtype, const float* src_scale, const float* dst_scale, const void* res,
                                       int64_t ldr, float alpha, const float* bias, float* scratch, const pg_drop* drop,
                                       void* stream) {
  if (res == nullptr)      // no residual: pg_aggregate_scaled, the same kernels and bits
    return pg_aggregate_scaled(g, x, ldx, out, ldo, d, dtype, src_scale, dst_scale, bias, scratch, drop, stream);
  const pg::DropArg da = pg::make_drop(drop);
  PG_REQUIRE(g && x && out && src_scale && dst_scale, "pg_aggregate_scaled_res: null argument");
  PG_REQUIRE(g->n_rows >= 0 && g->seg_len > 0 && d > 0, "pg_aggregate_scaled_res: bad sizes (n_rows=%d seg_len=%d d=%d)",
             g->n_rows, g->seg_len, d);
  PG_REQUIRE(ldx >= d && ldo >= d && ldr >= d && ldx < (1ll << 29),
             "pg_aggregate_scaled_res: row stride smaller than d (or >= 2^29 elements)");
  pg::aggregate_scaled_preload<2>();
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const pg::ScaleArg sc{{src_scale, bias, d}, res, ldr, alpha};
  if (dtype == PG_F32) return pg::aggregate_t<float, 2>(*g, x, ldx, out, ldo, d, dst_scale, 0, scratch, da, sc, st);
  if (dtype == PG_BF16)
    return pg::aggregate_t<__nv_bfloat16, 2>(*g, x, ldx, out, ldo, d, dst_scale, 0, scratch, da, sc, st);
  pg::set_error("pg_aggregate_scaled_res: unknown dtype %d", dtype);
  return PG_ERR_INVALID;
}

extern "C" int pg_aggregate_scaled_res_preload(void) {
  pg::aggregate_scaled_preload<2>();
  return PG_OK;
}

extern "C" int pg_row_div(const void* x, int64_t ldx, void* out, int64_t ldo, int32_t n_rows, int32_t d, int dtype,
                          const float* row_div, void* stream) {
  PG_REQUIRE(x && out && row_div, "pg_row_div: null argument");
  PG_REQUIRE(n_rows >= 0 && d > 0 && ldx >= d && ldo >= d, "pg_row_div: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) return pg::row_div_t<float>(x, ldx, out, ldo, n_rows, d, row_div, st);
  if (dtype == PG_BF16) return pg::row_div_t<__nv_bfloat16>(x, ldx, out, ldo, n_rows, d, row_div, st);
  pg::set_error("pg_row_div: unknown dtype %d", dtype);
  return PG_ERR_INVALID;
}
