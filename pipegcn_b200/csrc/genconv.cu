// Softmax-aggregation graph convolution (Li et al., "DeeperGCN", 2020; PyG GENConv, aggr='softmax') on sm_90a: the
// per-channel online-softmax aggregate of the messages m_u = ReLU(x_src[u]) + 1e-7 and its backward.
//
// The aggregate walks the forward chunk plan as pna.cu does: one warp per (chunk, column tile), lane l holding 16-byte
// vector l of the tile, four neighbour rows in flight.  Per element it keeps an online softmax state in fp32: the running
// maximum M of s = t m, W = sum exp(s - M), A = sum exp(s - M) m and, for the temperature's gradient, B = sum
// exp(s - M) m^2.  Every edge costs one expf: exp(-|s - M|) is the new edge's weight when s <= M and the old state's
// rescale when s > M.  Long rows come as segments whose partial states a fix-up merges in segment order.  The backward's
// source pass walks the CSC the same way and sums in CSC order.  No atomics anywhere: the results are the same bits from
// run to run.
#include <math.h>

#include <algorithm>
#include <mutex>

#include "chunk_walk.cuh"

namespace pg {
namespace {

constexpr int kGenWarps = 4;        // warps per CTA of the plan walks
constexpr int kAggInFlight = 4;     // neighbour rows of the aggregate loaded before they are folded in
constexpr int kSrcInFlight = 2;     // destination rows of the source pass (each brings three fp32 operands)
constexpr int kRowThreads = 256;    // threads per CTA of the element kernels
constexpr float kMsgEps = 1e-7f;    // GENConv's eps: m = ReLU(x) + eps

__device__ __forceinline__ bool gen_kept(const uint8_t* keep, int32_t num_in, int32_t u) {
  return keep == nullptr || u < num_in || keep[u - num_in] != 0;
}

// m = ReLU(x) + eps; a NaN stays NaN (torch's relu keeps it)
__device__ __forceinline__ float gen_msg(float x) { return __fadd_rn(x < 0.f ? 0.f : x, kMsgEps); }

// the online softmax state of V elements
template <int V, bool MOM> struct Soft {
  float mx[V], w[V], a[V], b[MOM ? V : 1];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < V; ++k) {
      mx[k] = -INFINITY;
      w[k] = a[k] = 0.f;
      if (MOM) b[k] = 0.f;
    }
  }
  // fold in a state (s_max, sw, sa, sb) of element k: one expf, exp(-|s_max - M|), scales whichever side has the
  // smaller maximum.  A single edge is (t m, 1, m, m^2).  A NaN poisons W, A and B and never becomes the maximum.
  __device__ __forceinline__ void fold(int k, float s, float sw, float sa, float sb) {
    const bool up = s > mx[k];
    const float e = expf(-fabsf(__fsub_rn(s, mx[k])));
    const float ca = up ? e : 1.f, cb = up ? 1.f : e;
    w[k] = __fmaf_rn(w[k], ca, __fmul_rn(cb, sw));
    a[k] = __fmaf_rn(a[k], ca, __fmul_rn(cb, sa));
    if (MOM) b[k] = __fmaf_rn(b[k], ca, __fmul_rn(cb, sb));
    mx[k] = up ? s : mx[k];
  }
};

// ---------------------------------------------------------------------------------------------------- aggregate
struct AggArgs {
  Walk w;
  const int32_t* indptr;             // forward CSR: D_v = indptr[v + 1] - indptr[v]
  int32_t seg_len;
  const void* xs; int64_t ldxs;      // [num_all, d] activation dtype
  const void* xd; int64_t ldxd;      // [N_in, d] activation dtype
  const float* t;                    // device scalar
  const uint8_t* keep; int32_t num_in;          // keep mask of the halo rows, or NULL
  void* s; int64_t lds;              // [N_in, d] activation dtype: agg + x_dst
  float* agg; int64_t ldagg;         // [N_in, d] fp32, or NULL (then lse and var are NULL too)
  float* lse; int64_t ldlse;         // [N_in, d] fp32
  float* var; int64_t ldvar;         // [N_in, d] fp32, or NULL
  float* scratch; int64_t ldsc;      // [n_seg][ldsc]: M, W, A (, B) at [k d, (k + 1) d)
  int32_t d, nvec;
};

template <typename T, bool MOM>
__device__ __forceinline__ void agg_store(const AggArgs& a, int v, int vi, const Soft<Vec<T>::V, MOM>& s) {
  constexpr int V = Vec<T>::V;
  if (vi >= a.nvec) return;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float xd[V], ag[V], l[V], vr[V], o[V];
  Vec<T>::P::unpack(ld_vec<16>(static_cast<const T*>(a.xd) + static_cast<int64_t>(v) * a.ldxd + c0), xd);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if (s.w[k] == 0.f) {             // no (kept) in-edge: agg = 0, log-sum-exp -inf
      ag[k] = 0.f;
      l[k] = -INFINITY;
      vr[k] = 0.f;
    } else {
      ag[k] = __fdiv_rn(s.a[k], s.w[k]);
      l[k] = __fadd_rn(s.mx[k], logf(s.w[k]));
      if (MOM) {
        const float x = __fsub_rn(__fdiv_rn(s.b[k], s.w[k]), __fmul_rn(ag[k], ag[k]));
        vr[k] = x < 0.f ? 0.f : x;
      }
    }
    o[k] = __fadd_rn(ag[k], xd[k]);
  }
  st_t<T, V>(static_cast<T*>(a.s) + static_cast<int64_t>(v) * a.lds + c0, o, valid);
  if (a.agg != nullptr) {
    st_f32<V>(a.agg + static_cast<int64_t>(v) * a.ldagg + c0, ag, valid);
    st_f32<V>(a.lse + static_cast<int64_t>(v) * a.ldlse + c0, l, valid);
    if (MOM) st_f32<V>(a.var + static_cast<int64_t>(v) * a.ldvar + c0, vr, valid);
  }
}

template <typename T, bool MOM>
__device__ __forceinline__ void agg_row(const AggArgs& a, int v, int e0, int n, int slot, int vi, int lane, float t) {
  constexpr int V = Vec<T>::V;
  const T* xs = static_cast<const T*>(a.xs);
  const bool live = vi < a.nvec;
  Soft<V, MOM> s;
  s.init();
  for (int b = 0; b < n; b += 32) {
    int32_t ul = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    if (!gen_kept(a.keep, a.num_in, ul)) ul = -1;
    const int cnt = min(32, n - b);
    for (int j = 0; j < cnt; j += kAggInFlight) {
      int32_t us[kAggInFlight];
      uint4 raw[kAggInFlight];
#pragma unroll
      for (int i = 0; i < kAggInFlight; ++i) {
        us[i] = __shfl_sync(0xffffffffu, ul, min(j + i, cnt - 1));
        if (j + i < cnt && us[i] >= 0 && live) raw[i] = ld_vec<16>(xs + static_cast<int64_t>(us[i]) * a.ldxs + vi * V);
      }
#pragma unroll
      for (int i = 0; i < kAggInFlight; ++i) {
        if (j + i >= cnt) break;
        if (!live || us[i] < 0) continue;
        float f[V];
        Vec<T>::P::unpack(raw[i], f);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float m = gen_msg(f[k]);
          s.fold(k, __fmul_rn(t, m), 1.f, m, MOM ? __fmul_rn(m, m) : 0.f);
        }
      }
    }
  }
  if (slot < 0) {
    agg_store<T, MOM>(a, v, vi, s);
    return;
  }
  if (!live) return;
  float* p = a.scratch + static_cast<int64_t>(slot) * a.ldsc;
  const int c0 = vi * V;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if (c0 + k < a.d) {
      p[c0 + k] = s.mx[k];
      p[a.d + c0 + k] = s.w[k];
      p[2 * a.d + c0 + k] = s.a[k];
      if (MOM) p[3 * a.d + c0 + k] = s.b[k];
    }
  }
}

template <typename T, bool MOM>
__global__ void __launch_bounds__(kGenWarps * 32) genconv_agg_kernel(AggArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGenWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  const float t = *a.t;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { agg_row<T, MOM>(a, v, e0, n, slot, vi, lane, t); });
}

// merge the partial states of every long row in segment order; a segment without a kept source (W = 0) is skipped
template <typename T, bool MOM>
__global__ void __launch_bounds__(kGenWarps * 32) genconv_agg_fixup_kernel(AggArgs a) {
  constexpr int V = Vec<T>::V;
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGenWarps + (threadIdx.x >> 5);
  if (li >= a.w.n_long) return;
  const int vi = blockIdx.y * 32 + lane;
  if (vi >= a.nvec) return;
  const int v = a.w.long_row[li];
  const int c0 = vi * V;
  Soft<V, MOM> s;
  s.init();
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.ldsc;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      const int c = c0 + k;
      if (c >= a.d) continue;
      const float sw = p[a.d + c];
      if (sw == 0.f) continue;
      s.fold(k, p[c], sw, p[2 * a.d + c], MOM ? p[3 * a.d + c] : 0.f);
    }
  }
  agg_store<T, MOM>(a, v, vi, s);
}

// ---------------------------------------------------------------------------------------------------- backward
// Q = t (g_S agg) per destination element (fp32, one rounding per product), g_S rounded to T when gst is given, and
// with var the block partials of dt = sum g_S var (fp64, each thread in grid-stride order, then a fixed tree)
template <typename T>
__global__ void __launch_bounds__(kRowThreads) genconv_bwd_dst_kernel(const float* g, int64_t ldg, const float* agg,
                                                                     int64_t ldagg, const float* var, int64_t ldvar,
                                                                     const float* tp, int32_t n, int32_t d, float* q,
                                                                     int64_t ldq, T* gst, int64_t ldgst,
                                                                     double* partial) {
  __shared__ double red[kRowThreads];
  const float t = *tp;
  const int64_t total = static_cast<int64_t>(n) * d;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * kRowThreads;
  double acc = 0.0;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x; i < total; i += stride) {
    const int v = static_cast<int>(i / d), c = static_cast<int>(i % d);
    const float gs = g[static_cast<int64_t>(v) * ldg + c];
    q[static_cast<int64_t>(v) * ldq + c] = __fmul_rn(t, __fmul_rn(gs, agg[static_cast<int64_t>(v) * ldagg + c]));
    if (gst != nullptr) gst[static_cast<int64_t>(v) * ldgst + c] = to_t<T>(gs);
    if (var != nullptr) acc += static_cast<double>(gs) * static_cast<double>(var[static_cast<int64_t>(v) * ldvar + c]);
  }
  if (var == nullptr) return;
  red[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int h = kRowThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = red[0];
}

// dt = the partials summed in a fixed order (one CTA), rounded once to fp32
__global__ void __launch_bounds__(kRowThreads) genconv_dt_sum_kernel(const double* partial, int32_t n, float* dt) {
  __shared__ double red[kRowThreads];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kRowThreads) acc += partial[i];
  red[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int h = kRowThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) *dt = static_cast<float>(red[0]);
}

struct SrcArgs {
  Walk w;
  const void* xs; int64_t ldxs;      // [num_all, d] activation dtype
  const float* t;
  const uint8_t* keep; int32_t num_in;
  const float* lse; int64_t ldlse;   // [N_in, d] fp32
  const float* g; int64_t ldg;       // [N_in, d] fp32
  const float* q; int64_t ldq;       // [N_in, d] fp32
  const float* add; int64_t ldadd; int32_t n_add;   // fp32 [n_add, d] added to rows < n_add, or NULL
  DropArg drop;
  void* dx; int64_t lddx;            // [num_all, d] activation dtype
  float* scratch; int64_t ldsc;      // [n_seg][ldsc]: the partial sums at [0, d)
  int32_t d, nvec;
};

// dx[u] = dropout([x_src[u] > 0] acc + add[u]) rounded once to T; acc is 0 for a row without (kept) out-edges
template <typename T>
__device__ __forceinline__ void src_store(const SrcArgs& a, int u, int vi, const float (&acc)[Vec<T>::V]) {
  constexpr int V = Vec<T>::V;
  if (vi >= a.nvec) return;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float x[V], r[V];
  Vec<T>::P::unpack(ld_vec<16>(static_cast<const T*>(a.xs) + static_cast<int64_t>(u) * a.ldxs + c0), x);
#pragma unroll
  for (int k = 0; k < V; ++k) r[k] = x[k] > 0.f ? acc[k] : 0.f;
  if (u < a.n_add) {
    float ad[V];
    ld_f32<V>(a.add + static_cast<int64_t>(u) * a.ldadd + c0, ad, valid);
#pragma unroll
    for (int k = 0; k < V; ++k) r[k] = __fadd_rn(r[k], ad[k]);
  }
  if (a.drop.thresh16 != 0u)
    drop_apply<V>(r, static_cast<uint64_t>(u) * a.nvec + vi, a.drop.thresh16, a.drop.scale, a.drop.seed_lo,
                  drop_seed_hi(a.drop));
  st_t<T, V>(static_cast<T*>(a.dx) + static_cast<int64_t>(u) * a.lddx + c0, r, valid);
}

// acc = sum over the destinations v of u (CSC order) of exp(t m - L_v) (G_v (1 + t m) - Q_v), one multiply-add per term
template <typename T>
__device__ __forceinline__ void src_row(const SrcArgs& a, int u, int e0, int n, int slot, int vi, int lane, float t) {
  constexpr int V = Vec<T>::V;
  const bool live = vi < a.nvec;
  const int c0 = vi * V;
  const int valid = live ? min(V, a.d - c0) : 0;
  float acc[V], tm[V], p1[V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.f;
  if (!gen_kept(a.keep, a.num_in, u)) n = 0;
  if (n > 0 && live) {
    float x[V];
    Vec<T>::P::unpack(ld_vec<16>(static_cast<const T*>(a.xs) + static_cast<int64_t>(u) * a.ldxs + c0), x);
#pragma unroll
    for (int k = 0; k < V; ++k) {
      tm[k] = __fmul_rn(t, gen_msg(x[k]));
      p1[k] = __fadd_rn(1.f, tm[k]);
    }
  }
  for (int b = 0; b < n; b += 32) {
    const int32_t vl = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const int cnt = min(32, n - b);
    for (int j = 0; j < cnt; j += kSrcInFlight) {
      float l[kSrcInFlight][V], g[kSrcInFlight][V], q[kSrcInFlight][V];
#pragma unroll
      for (int i = 0; i < kSrcInFlight; ++i) {
        const int v = __shfl_sync(0xffffffffu, vl, min(j + i, cnt - 1));
        if (j + i < cnt && live) {
          ld_f32<V>(a.lse + static_cast<int64_t>(v) * a.ldlse + c0, l[i], valid);
          ld_f32<V>(a.g + static_cast<int64_t>(v) * a.ldg + c0, g[i], valid);
          ld_f32<V>(a.q + static_cast<int64_t>(v) * a.ldq + c0, q[i], valid);
        }
      }
#pragma unroll
      for (int i = 0; i < kSrcInFlight; ++i) {
        if (j + i >= cnt) break;
        if (!live) continue;
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float e = expf(__fsub_rn(tm[k], l[i][k]));
          acc[k] = __fmaf_rn(e, __fsub_rn(__fmul_rn(g[i][k], p1[k]), q[i][k]), acc[k]);
        }
      }
    }
  }
  if (slot < 0) {
    src_store<T>(a, u, vi, acc);
    return;
  }
  if (!live) return;
  float* p = a.scratch + static_cast<int64_t>(slot) * a.ldsc;
#pragma unroll
  for (int k = 0; k < V; ++k)
    if (c0 + k < a.d) p[c0 + k] = acc[k];
}

template <typename T>
__global__ void __launch_bounds__(kGenWarps * 32) genconv_src_kernel(SrcArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGenWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  const float t = *a.t;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { src_row<T>(a, u, e0, n, slot, vi, lane, t); });
}

// sum the partials of every long CSC row in segment order (an unkept row's segments hold zeros)
template <typename T>
__global__ void __launch_bounds__(kGenWarps * 32) genconv_src_fixup_kernel(SrcArgs a) {
  constexpr int V = Vec<T>::V;
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGenWarps + (threadIdx.x >> 5);
  if (li >= a.w.n_long) return;
  const int vi = blockIdx.y * 32 + lane;
  if (vi >= a.nvec) return;
  const int c0 = vi * V;
  float acc[V];
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.ldsc;
#pragma unroll
    for (int k = 0; k < V; ++k)
      if (c0 + k < a.d) acc[k] = __fadd_rn(acc[k], p[c0 + k]);
  }
  src_store<T>(a, a.w.long_row[li], vi, acc);
}

// ---------------------------------------------------------------------------------------------------- dispatch
template <typename T>
void preload_t() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, genconv_agg_kernel<T, false>);
  cudaFuncGetAttributes(&a, genconv_agg_kernel<T, true>);
  cudaFuncGetAttributes(&a, genconv_agg_fixup_kernel<T, false>);
  cudaFuncGetAttributes(&a, genconv_agg_fixup_kernel<T, true>);
  cudaFuncGetAttributes(&a, genconv_bwd_dst_kernel<T>);
  cudaFuncGetAttributes(&a, genconv_src_kernel<T>);
  cudaFuncGetAttributes(&a, genconv_src_fixup_kernel<T>);
}

template <typename T, bool MOM>
void launch_agg(const AggArgs& a, const pg_csr* g, cudaStream_t st) {
  const int tiles = (a.nvec + 31) / 32;
  if (g->n_chunks > 0)
    genconv_agg_kernel<T, MOM><<<dim3((g->n_chunks + kGenWarps - 1) / kGenWarps, tiles), kGenWarps * 32, 0, st>>>(a);
  if (g->n_long > 0)
    genconv_agg_fixup_kernel<T, MOM><<<dim3((g->n_long + kGenWarps - 1) / kGenWarps, tiles), kGenWarps * 32, 0, st>>>(a);
}

template <typename T>
void launch_src(const SrcArgs& a, const pg_csr* g, cudaStream_t st) {
  const int tiles = (a.nvec + 31) / 32;
  if (g->n_chunks > 0)
    genconv_src_kernel<T><<<dim3((g->n_chunks + kGenWarps - 1) / kGenWarps, tiles), kGenWarps * 32, 0, st>>>(a);
  if (g->n_long > 0)
    genconv_src_fixup_kernel<T><<<dim3((g->n_long + kGenWarps - 1) / kGenWarps, tiles), kGenWarps * 32, 0, st>>>(a);
}

bool f32_rows_ok(const void* p, int64_t ld) { return vec_ok(p, ld, 4); }

}  // namespace

// CUDA loads kernels lazily, and loading one may wait for the device: see exchange.cu's bns_preload.
static void genconv_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_t<float>();
    preload_t<__nv_bfloat16>();
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, genconv_dt_sum_kernel);
    cudaGetLastError();
  });
}

}  // namespace pg

extern "C" int pg_genconv_preload(void) {
  pg::genconv_preload();
  return PG_OK;
}

extern "C" int pg_genconv_aggregate(const pg_csr* g, const void* xs, int64_t ldxs, const void* xd, int64_t ldxd,
                                    int32_t d, int dtype, const float* t, const uint8_t* keep, int32_t num_in,
                                    void* s, int64_t lds, float* agg, int64_t ldagg, float* lse, int64_t ldlse,
                                    float* var, int64_t ldvar, float* scratch, int64_t ld_scratch, void* stream) {
  pg::genconv_preload();
  if (int rc = pg::check_plan(g, "pg_genconv_aggregate")) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_genconv_aggregate: unknown dtype %d", dtype);
  const int es = pg::elem_size(dtype);
  const int V = 16 / es;
  PG_REQUIRE(d > 0 && ldxs >= d && ldxd >= d && lds >= d, "pg_genconv_aggregate: bad sizes (d %d)", d);
  if (g->n_rows == 0) return PG_OK;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  PG_REQUIRE(xs && xd && s && t && (g->n_seg == 0 || scratch) && ((agg == nullptr) == (lse == nullptr)) &&
                 (var == nullptr || agg != nullptr),
             "pg_genconv_aggregate: null argument");
  PG_REQUIRE(ldxs >= full && ldxd >= full && lds >= full &&
                 (agg == nullptr || (ldagg >= full && ldlse >= full)) && (var == nullptr || ldvar >= full),
             "pg_genconv_aggregate: row stride shorter than the last 16-byte vector");
  const int parts = var != nullptr ? 4 : 3;
  PG_REQUIRE(g->n_seg == 0 || ld_scratch >= parts * static_cast<int64_t>(d),
             "pg_genconv_aggregate: scratch rows < %d d", parts);
  PG_REQUIRE(pg::vec_ok(xs, ldxs, es) && pg::vec_ok(xd, ldxd, es) && pg::vec_ok(s, lds, es) &&
                 (agg == nullptr || (pg::f32_rows_ok(agg, ldagg) && pg::f32_rows_ok(lse, ldlse))) &&
                 (var == nullptr || pg::f32_rows_ok(var, ldvar)),
             "pg_genconv_aggregate: rows must start on 16-byte boundaries with a 16-byte multiple stride");
  pg::AggArgs a{pg::make_walk(g), g->indptr, g->seg_len, xs, ldxs, xd, ldxd, t, keep, num_in, s, lds,
                agg, ldagg, lse, ldlse, var, ldvar, scratch, ld_scratch, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) {
    if (var != nullptr) pg::launch_agg<float, true>(a, g, st);
    else pg::launch_agg<float, false>(a, g, st);
  } else {
    if (var != nullptr) pg::launch_agg<__nv_bfloat16, true>(a, g, st);
    else pg::launch_agg<__nv_bfloat16, false>(a, g, st);
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_genconv_bwd_dst(const float* gs, int64_t ldg, const float* agg, int64_t ldagg, const float* var,
                                  int64_t ldvar, const float* t, int32_t n_rows, int32_t d, int dtype, float* q,
                                  int64_t ldq, void* gst, int64_t ldgst, double* partial, float* dt, void* stream) {
  pg::genconv_preload();
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_genconv_bwd_dst: unknown dtype %d", dtype);
  PG_REQUIRE(n_rows >= 0 && d > 0 && ldg >= d && ldagg >= d && ldq >= d && (var == nullptr || ldvar >= d) &&
                 (gst == nullptr || ldgst >= d),
             "pg_genconv_bwd_dst: bad sizes (d %d)", d);
  PG_REQUIRE(t && ((var == nullptr) == (dt == nullptr)) && (var == nullptr || partial),
             "pg_genconv_bwd_dst: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t total = static_cast<int64_t>(n_rows) * d;
  const int nb = static_cast<int>(std::min<int64_t>(PG_GENCONV_DT_PARTIALS,
                                                    std::max<int64_t>(1, (total + pg::kRowThreads - 1) / pg::kRowThreads)));
  if (total > 0) PG_REQUIRE(gs && agg && q, "pg_genconv_bwd_dst: null argument");
  if (dtype == PG_F32)
    pg::genconv_bwd_dst_kernel<float><<<nb, pg::kRowThreads, 0, st>>>(gs, ldg, agg, ldagg, var, ldvar, t, n_rows, d, q,
                                                                       ldq, static_cast<float*>(gst), ldgst, partial);
  else
    pg::genconv_bwd_dst_kernel<__nv_bfloat16><<<nb, pg::kRowThreads, 0, st>>>(
        gs, ldg, agg, ldagg, var, ldvar, t, n_rows, d, q, ldq, static_cast<__nv_bfloat16*>(gst), ldgst, partial);
  if (var != nullptr) pg::genconv_dt_sum_kernel<<<1, pg::kRowThreads, 0, st>>>(partial, nb, dt);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_genconv_bwd_src(const pg_csr* gt, const void* xs, int64_t ldxs, const float* t, const uint8_t* keep,
                                  int32_t num_in, const float* lse, int64_t ldlse, const float* gs, int64_t ldg,
                                  const float* q, int64_t ldq, const float* add, int64_t ldadd, int32_t n_add,
                                  const pg_drop* drop, int32_t d, int dtype, void* dx, int64_t lddx, float* scratch,
                                  int64_t ld_scratch, void* stream) {
  pg::genconv_preload();
  if (int rc = pg::check_plan(gt, "pg_genconv_bwd_src")) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_genconv_bwd_src: unknown dtype %d", dtype);
  const int es = pg::elem_size(dtype);
  const int V = 16 / es;
  PG_REQUIRE(d > 0 && ldxs >= d && lddx >= d && n_add >= 0 && n_add <= gt->n_rows,
             "pg_genconv_bwd_src: bad sizes (d %d)", d);
  if (gt->n_rows == 0) return PG_OK;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  PG_REQUIRE(xs && dx && t && (gt->nnz == 0 || (lse && gs && q)) && (n_add == 0 || add) &&
                 (gt->n_seg == 0 || scratch),
             "pg_genconv_bwd_src: null argument");
  PG_REQUIRE(ldxs >= full && lddx >= full && (gt->nnz == 0 || (ldlse >= full && ldg >= full && ldq >= full)) &&
                 (n_add == 0 || ldadd >= full),
             "pg_genconv_bwd_src: row stride shorter than the last 16-byte vector");
  PG_REQUIRE(gt->n_seg == 0 || ld_scratch >= d, "pg_genconv_bwd_src: scratch rows < d");
  PG_REQUIRE(pg::vec_ok(xs, ldxs, es) && pg::vec_ok(dx, lddx, es) &&
                 (gt->nnz == 0 || (pg::f32_rows_ok(lse, ldlse) && pg::f32_rows_ok(gs, ldg) && pg::f32_rows_ok(q, ldq))) &&
                 (n_add == 0 || pg::f32_rows_ok(add, ldadd)),
             "pg_genconv_bwd_src: rows must start on 16-byte boundaries with a 16-byte multiple stride");
  pg::SrcArgs a{pg::make_walk(gt), xs, ldxs, t, keep, num_in, lse, ldlse, gs, ldg, q, ldq, add, ldadd, n_add,
                pg::make_drop(drop), dx, lddx, scratch, ld_scratch, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) pg::launch_src<float>(a, gt, st);
  else pg::launch_src<__nv_bfloat16>(a, gt, st);
  PG_LAUNCH_CHECK();
  return PG_OK;
}
