// Max-pool GraphSAGE (Hamilton et al.'s pool aggregator, DGL SAGEConv(aggregator_type='pool')) on sm_90a: the
// element-wise neighbour maximum with its argmax, and the argmax backward.
//
// One warp owns one chunk of the pg_csr plan (the chunked aggregate's table) and one tile of columns: lane l holds
// 16-byte vectors l, l + 32, ... of the tile, so every gather is a 16-byte load per lane, and the warp keeps four
// neighbour rows in flight before it folds them in CSR order.  Long rows come as segments that write their partials to
// `scratch`; a fix-up merges each long row's partials in segment order.  The forward compares with a strict `>`, so the
// first source in CSR order wins a tie, and a NaN, once taken, is never replaced.  The backward walks the CSC: source u
// collects the gradients of the destinations whose argmax is u, in CSC order, in fp32.  No atomics anywhere: the results
// are the same bits from run to run.
#include <math.h>
#include <mutex>

#include "chunk_walk.cuh"

namespace pg {
namespace {

constexpr int kPoolWarps = 4;             // warps per CTA
constexpr int kInFlight = 4;              // neighbour rows loaded before they are folded in

// ---------------------------------------------------------------------------------------------------- forward
struct FwdArgs {
  Walk w;
  const void* q; int64_t ldq;
  void* hn; int64_t ldh;             // ReLU(max) in the activation dtype
  int32_t* arg; int64_t lda;         // argmax (`_U` row ids, -1 for a row without in-edges)
  float* scratch; int64_t lds;       // [n_seg][lds]: max values at [0, d), argmax bits at [d, 2d)
  int32_t d, nvec;
};

template <typename T, int NJ>
__device__ __forceinline__ void fwd_store(const FwdArgs& a, int v, int vbase, const float (&m)[NJ][Vec<T>::V],
                                          const int32_t (&am)[NJ][Vec<T>::V]) {
  constexpr int V = Vec<T>::V;
  T* ho = static_cast<T*>(a.hn) + static_cast<int64_t>(v) * a.ldh;
  int32_t* ao = a.arg + static_cast<int64_t>(v) * a.lda;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int vi = vbase + 32 * j;
    if (vi >= a.nvec) continue;
    float r[V];
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const float x = m[j][k];
      r[k] = am[j][k] < 0 ? 0.f : (x > 0.f || x != x) ? x : 0.f;      // ReLU(max), NaN kept
    }
    const int c0 = vi * V;
    if (c0 + V <= a.d) {
      st_vec<16>(ho + c0, Vec<T>::P::pack(r));
      int4* ap = reinterpret_cast<int4*>(ao + c0);
#pragma unroll
      for (int k = 0; k < V; k += 4) ap[k / 4] = make_int4(am[j][k], am[j][k + 1], am[j][k + 2], am[j][k + 3]);
    } else {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        if (c0 + k < a.d) {
          ho[c0 + k] = to_t<T>(r[k]);
          ao[c0 + k] = am[j][k];
        }
      }
    }
  }
}

template <typename T, int NJ>
__device__ __forceinline__ void fwd_row(const FwdArgs& a, int v, int e0, int n, int slot, int vbase, int lane) {
  constexpr int V = Vec<T>::V;
  const T* q = static_cast<const T*>(a.q);
  float m[NJ][V];
  int32_t am[NJ][V];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int k = 0; k < V; ++k) { m[j][k] = 0.f; am[j][k] = -1; }
  for (int b = 0; b < n; b += 32) {
    const int32_t ul = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const int cnt = min(32, n - b);
    for (int t = 0; t < cnt; t += kInFlight) {
      int32_t us[kInFlight];
      uint4 raw[kInFlight][NJ];
#pragma unroll
      for (int i = 0; i < kInFlight; ++i) {
        us[i] = __shfl_sync(0xffffffffu, ul, min(t + i, cnt - 1));
        const T* row = q + static_cast<int64_t>(us[i]) * a.ldq;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int vi = vbase + 32 * j;
          if (t + i < cnt && vi < a.nvec) raw[i][j] = ld_vec<16>(row + vi * V);
        }
      }
#pragma unroll
      for (int i = 0; i < kInFlight; ++i) {
        if (t + i >= cnt) break;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          if (vbase + 32 * j >= a.nvec) continue;
          float f[V];
          Vec<T>::P::unpack(raw[i][j], f);
#pragma unroll
          for (int k = 0; k < V; ++k) take_max(m[j][k], am[j][k], f[k], us[i]);
        }
      }
    }
  }
  if (slot < 0) {
    fwd_store<T, NJ>(a, v, vbase, m, am);
    return;
  }
  float* p = a.scratch + static_cast<int64_t>(slot) * a.lds;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c0 = (vbase + 32 * j) * V;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      if (c0 + k < a.d) {
        p[c0 + k] = m[j][k];
        p[a.d + c0 + k] = __int_as_float(am[j][k]);
      }
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kPoolWarps * 32) pool_fwd_kernel(FwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kPoolWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vbase = blockIdx.y * 32 * NJ + lane;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { fwd_row<T, NJ>(a, v, e0, n, slot, vbase, lane); });
}

// merge the (max, argmax) partials of every long row in segment order (an earlier segment keeps a tie)
template <typename T, int NJ>
__global__ void __launch_bounds__(kPoolWarps * 32) pool_fwd_fixup_kernel(FwdArgs a) {
  constexpr int V = Vec<T>::V;
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kPoolWarps + (threadIdx.x >> 5);
  if (li >= a.w.n_long) return;
  const int vbase = blockIdx.y * 32 * NJ + lane;
  float m[NJ][V];
  int32_t am[NJ][V];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int k = 0; k < V; ++k) { m[j][k] = 0.f; am[j][k] = -1; }
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.lds;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c0 = (vbase + 32 * j) * V;
#pragma unroll
      for (int k = 0; k < V; ++k)
        if (c0 + k < a.d) take_max(m[j][k], am[j][k], p[c0 + k], __float_as_int(p[a.d + c0 + k]));
    }
  }
  fwd_store<T, NJ>(a, a.w.long_row[li], vbase, m, am);
}

// ---------------------------------------------------------------------------------------------------- backward
struct BwdArgs {
  Walk w;
  const void* q; int64_t ldq;        // the pre-activation Q: its sign gates the gradient
  const int32_t* arg; int64_t lda;   // forward argmax [N_in]
  const void* g; int64_t ldg;        // g_neigh = dL/d ReLU(max) [N_in]
  void* gq; int64_t ldgq;            // dL/dQ [num_all]
  float* scratch; int64_t lds;       // [n_seg][lds] fp32 partial sums
  int32_t d, nvec;
};

template <typename T, int NJ>
__device__ __forceinline__ void bwd_store(const BwdArgs& a, int u, int vbase, const float (&acc)[NJ][Vec<T>::V]) {
  constexpr int V = Vec<T>::V;
  const T* qr = static_cast<const T*>(a.q) + static_cast<int64_t>(u) * a.ldq;
  T* o = static_cast<T*>(a.gq) + static_cast<int64_t>(u) * a.ldgq;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int vi = vbase + 32 * j;
    if (vi >= a.nvec) continue;
    float qf[V], r[V];
    Vec<T>::P::unpack(ld_vec<16>(qr + vi * V), qf);
#pragma unroll
    for (int k = 0; k < V; ++k) r[k] = qf[k] > 0.f ? acc[j][k] : 0.f;
    const int c0 = vi * V;
    if (c0 + V <= a.d) {
      st_vec<16>(o + c0, Vec<T>::P::pack(r));
    } else {
#pragma unroll
      for (int k = 0; k < V; ++k)
        if (c0 + k < a.d) o[c0 + k] = to_t<T>(r[k]);
    }
  }
}

template <typename T, int NJ>
__device__ __forceinline__ void bwd_row(const BwdArgs& a, int u, int e0, int n, int slot, int vbase, int lane) {
  constexpr int V = Vec<T>::V;
  const T* g = static_cast<const T*>(a.g);
  float acc[NJ][V];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int k = 0; k < V; ++k) acc[j][k] = 0.f;
  // a vector whose Q is <= 0 everywhere gets no gradient: its lane skips the loads (the gate of a long row's fix-up
  // zeroes such a vector too, so its segments may skip them as well)
  bool live[NJ];
  {
    const T* qr = static_cast<const T*>(a.q) + static_cast<int64_t>(u) * a.ldq;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int vi = vbase + 32 * j;
      live[j] = false;
      if (vi < a.nvec) {
        float qf[V];
        Vec<T>::P::unpack(ld_vec<16>(qr + vi * V), qf);
#pragma unroll
        for (int k = 0; k < V; ++k) live[j] |= qf[k] > 0.f;
      }
    }
  }
  for (int b = 0; b < n; b += 32) {
    const int32_t vl = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const int cnt = min(32, n - b);
    for (int t = 0; t < cnt; t += kInFlight) {
      int32_t vs[kInFlight];
      uint4 graw[kInFlight][NJ];
      uint32_t hit[kInFlight][NJ];         // bit k: A[v, c] == u for element k of the vector
#pragma unroll
      for (int i = 0; i < kInFlight; ++i) {
        vs[i] = __shfl_sync(0xffffffffu, vl, min(t + i, cnt - 1));
        const T* gr = g + static_cast<int64_t>(vs[i]) * a.ldg;
        const int4* ar = reinterpret_cast<const int4*>(a.arg + static_cast<int64_t>(vs[i]) * a.lda);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int vi = vbase + 32 * j;
          if (t + i < cnt && live[j]) {
            graw[i][j] = ld_vec<16>(gr + vi * V);
            uint32_t h = 0;
#pragma unroll
            for (int k4 = 0; k4 < V / 4; ++k4) {
              const int4 av = __ldg(ar + vi * (V / 4) + k4);
              h |= (av.x == u ? 1u : 0u) << (4 * k4) | (av.y == u ? 2u : 0u) << (4 * k4) |
                   (av.z == u ? 4u : 0u) << (4 * k4) | (av.w == u ? 8u : 0u) << (4 * k4);
            }
            hit[i][j] = h;
          }
        }
      }
#pragma unroll
      for (int i = 0; i < kInFlight; ++i) {
        if (t + i >= cnt) break;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          if (!live[j]) continue;
          float f[V];
          Vec<T>::P::unpack(graw[i][j], f);
#pragma unroll
          for (int k = 0; k < V; ++k)
            if (hit[i][j] >> k & 1u) acc[j][k] = __fadd_rn(acc[j][k], f[k]);
        }
      }
    }
  }
  if (slot < 0) {
    bwd_store<T, NJ>(a, u, vbase, acc);
    return;
  }
  float* p = a.scratch + static_cast<int64_t>(slot) * a.lds;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c0 = (vbase + 32 * j) * V;
#pragma unroll
    for (int k = 0; k < V; ++k)
      if (c0 + k < a.d) p[c0 + k] = acc[j][k];
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kPoolWarps * 32) pool_bwd_kernel(BwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kPoolWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vbase = blockIdx.y * 32 * NJ + lane;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { bwd_row<T, NJ>(a, u, e0, n, slot, vbase, lane); });
}

// sum the partials of every long CSC row in segment order, then gate by Q > 0
template <typename T, int NJ>
__global__ void __launch_bounds__(kPoolWarps * 32) pool_bwd_fixup_kernel(BwdArgs a) {
  constexpr int V = Vec<T>::V;
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kPoolWarps + (threadIdx.x >> 5);
  if (li >= a.w.n_long) return;
  const int vbase = blockIdx.y * 32 * NJ + lane;
  float acc[NJ][V];
#pragma unroll
  for (int j = 0; j < NJ; ++j)
#pragma unroll
    for (int k = 0; k < V; ++k) acc[j][k] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.lds;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c0 = (vbase + 32 * j) * V;
#pragma unroll
      for (int k = 0; k < V; ++k)
        if (c0 + k < a.d) acc[j][k] = __fadd_rn(acc[j][k], p[c0 + k]);
    }
  }
  bwd_store<T, NJ>(a, a.w.long_row[li], vbase, acc);
}

// ---------------------------------------------------------------------------------------------------- dispatch
// vectors per lane: one for rows of up to 32 vectors, else two (a tile of 64 vectors; wider rows take more tiles)
int nj_of(int32_t nvec) { return nvec <= 32 ? 1 : 2; }
int tiles_of(int32_t nvec, int nj) { return (nvec + 32 * nj - 1) / (32 * nj); }

template <typename T>
void preload_t() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, pool_fwd_kernel<T, 1>);
  cudaFuncGetAttributes(&a, pool_fwd_kernel<T, 2>);
  cudaFuncGetAttributes(&a, pool_fwd_fixup_kernel<T, 1>);
  cudaFuncGetAttributes(&a, pool_fwd_fixup_kernel<T, 2>);
  cudaFuncGetAttributes(&a, pool_bwd_kernel<T, 1>);
  cudaFuncGetAttributes(&a, pool_bwd_kernel<T, 2>);
  cudaFuncGetAttributes(&a, pool_bwd_fixup_kernel<T, 1>);
  cudaFuncGetAttributes(&a, pool_bwd_fixup_kernel<T, 2>);
}

template <typename T, typename K, typename A>
void launch(const pg_csr* g, A& a, cudaStream_t st, bool fixup) {
  const int nj = nj_of(a.nvec);
  const dim3 grid((g->n_chunks + kPoolWarps - 1) / kPoolWarps, tiles_of(a.nvec, nj));
  const dim3 grid_fix((g->n_long + kPoolWarps - 1) / kPoolWarps, tiles_of(a.nvec, nj));
  K::template run<T>(nj, grid, grid_fix, st, a, g->n_chunks > 0, fixup && g->n_long > 0);
}

struct FwdLaunch {
  template <typename T>
  static void run(int nj, dim3 grid, dim3 grid_fix, cudaStream_t st, FwdArgs& a, bool main, bool fix) {
    if (nj == 1) {
      if (main) pool_fwd_kernel<T, 1><<<grid, kPoolWarps * 32, 0, st>>>(a);
      if (fix) pool_fwd_fixup_kernel<T, 1><<<grid_fix, kPoolWarps * 32, 0, st>>>(a);
    } else {
      if (main) pool_fwd_kernel<T, 2><<<grid, kPoolWarps * 32, 0, st>>>(a);
      if (fix) pool_fwd_fixup_kernel<T, 2><<<grid_fix, kPoolWarps * 32, 0, st>>>(a);
    }
  }
};

struct BwdLaunch {
  template <typename T>
  static void run(int nj, dim3 grid, dim3 grid_fix, cudaStream_t st, BwdArgs& a, bool main, bool fix) {
    if (nj == 1) {
      if (main) pool_bwd_kernel<T, 1><<<grid, kPoolWarps * 32, 0, st>>>(a);
      if (fix) pool_bwd_fixup_kernel<T, 1><<<grid_fix, kPoolWarps * 32, 0, st>>>(a);
    } else {
      if (main) pool_bwd_kernel<T, 2><<<grid, kPoolWarps * 32, 0, st>>>(a);
      if (fix) pool_bwd_fixup_kernel<T, 2><<<grid_fix, kPoolWarps * 32, 0, st>>>(a);
    }
  }
};

}  // namespace

// CUDA loads kernels lazily, and loading one may wait for the device: see exchange.cu's bns_preload.
static void pool_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_t<float>();
    preload_t<__nv_bfloat16>();
    cudaGetLastError();
  });
}

}  // namespace pg

extern "C" int pg_pool_preload(void) {
  pg::pool_preload();
  return PG_OK;
}

extern "C" int pg_max_aggregate(const pg_csr* g, const void* q, int64_t ldq, int32_t d, int dtype, void* hn,
                                int64_t ldh, int32_t* arg, int64_t lda, float* scratch, int64_t ld_scratch,
                                void* stream) {
  pg::pool_preload();
  if (int rc = pg::check_plan(g, "pg_max_aggregate")) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_max_aggregate: unknown dtype %d", dtype);
  const int es = pg::elem_size(dtype);
  PG_REQUIRE(d > 0 && ldq >= d && ldh >= d && lda >= d, "pg_max_aggregate: bad sizes (d %d)", d);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(q && hn && arg && (g->n_seg == 0 || scratch), "pg_max_aggregate: null argument");
  PG_REQUIRE(g->n_seg == 0 || ld_scratch >= 2 * static_cast<int64_t>(d), "pg_max_aggregate: scratch rows < 2d");
  PG_REQUIRE(pg::vec_ok(q, ldq, es) && pg::vec_ok(hn, ldh, es) && pg::vec_ok(arg, lda, 4),
             "pg_max_aggregate: rows must start on 16-byte boundaries with a 16-byte multiple stride");
  const int V = 16 / es;
  const int32_t nvec = (d + V - 1) / V;
  PG_REQUIRE(ldq >= static_cast<int64_t>(nvec) * V && lda >= static_cast<int64_t>(nvec) * V,
             "pg_max_aggregate: row stride shorter than the last 16-byte vector");
  pg::FwdArgs a{pg::make_walk(g), q, ldq, hn, ldh, arg, lda, scratch, ld_scratch, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) pg::launch<float, pg::FwdLaunch>(g, a, st, true);
  else pg::launch<__nv_bfloat16, pg::FwdLaunch>(g, a, st, true);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_max_aggregate_bwd(const pg_csr* gt, const void* q, int64_t ldq, const int32_t* arg, int64_t lda,
                                    const void* grad, int64_t ldg, int32_t d, int dtype, void* gq, int64_t ldgq,
                                    float* scratch, int64_t ld_scratch, void* stream) {
  pg::pool_preload();
  if (int rc = pg::check_plan(gt, "pg_max_aggregate_bwd")) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_max_aggregate_bwd: unknown dtype %d", dtype);
  const int es = pg::elem_size(dtype);
  PG_REQUIRE(d > 0 && ldq >= d && lda >= d && ldg >= d && ldgq >= d, "pg_max_aggregate_bwd: bad sizes (d %d)", d);
  if (gt->n_rows == 0) return PG_OK;
  PG_REQUIRE(q && gq && (gt->nnz == 0 || (arg && grad)) && (gt->n_seg == 0 || scratch),
             "pg_max_aggregate_bwd: null argument");
  PG_REQUIRE(gt->n_seg == 0 || ld_scratch >= d, "pg_max_aggregate_bwd: scratch rows < d");
  PG_REQUIRE(pg::vec_ok(q, ldq, es) && pg::vec_ok(gq, ldgq, es) &&
                 (gt->nnz == 0 || (pg::vec_ok(arg, lda, 4) && pg::vec_ok(grad, ldg, es))),
             "pg_max_aggregate_bwd: rows must start on 16-byte boundaries with a 16-byte multiple stride");
  const int V = 16 / es;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  PG_REQUIRE(ldq >= full && (gt->nnz == 0 || (lda >= full && ldg >= full)),
             "pg_max_aggregate_bwd: row stride shorter than the last 16-byte vector");
  pg::BwdArgs a{pg::make_walk(gt), q, ldq, arg, lda, grad, ldg, gq, ldgq, scratch, ld_scratch, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) pg::launch<float, pg::BwdLaunch>(gt, a, st, true);
  else pg::launch<__nv_bfloat16, pg::BwdLaunch>(gt, a, st, true);
  PG_LAUNCH_CHECK();
  return PG_OK;
}
