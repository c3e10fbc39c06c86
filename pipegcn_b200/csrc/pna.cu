// Principal neighbourhood aggregation (Corso et al., NeurIPS 2020; DGL PNAConv) on sm_90a: one gather that keeps the
// mean, variance, maximum and minimum of the neighbour rows, the degree-scaler combine, and the backward.
//
// The aggregate walks the forward chunk plan as pool.cu does: one warp per (chunk, column tile), lane l holding 16-byte
// vector l of the tile, four neighbour rows in flight.  Per element it keeps Welford's (mean, M2) and the extremes with
// their sources; long rows come as segments whose partials a fix-up merges in segment order (Chan's merge for the
// moments, pool.cu's rule for the extremes: an earlier source keeps a tie, the first NaN stays).  The backward's source
// pass walks the CSC the same way and sums in CSC order.  No atomics anywhere: the results are the same bits from run
// to run.
#include <math.h>
#include <mutex>

#include "chunk_walk.cuh"

namespace pg {
namespace {

constexpr int kPnaWarps = 4;      // warps per CTA of the plan walks
constexpr int kAggInFlight = 4;   // neighbour rows of the aggregate loaded before they are folded in
constexpr int kSrcInFlight = 2;   // destination rows of the source pass (each brings six operands)
constexpr int kRowThreads = 256;  // threads per CTA of the element kernels

// (m, a) <- (x, u) when the row has no candidate yet, x is smaller, or x is the first NaN
__device__ __forceinline__ void take_min(float& m, int32_t& a, float x, int32_t u) {
  if (a < 0 || x < m || (x != x && m == m)) { m = x; a = u; }
}

// V consecutive int32 values at p (16-byte aligned when all V are valid and V is a multiple of 4)
template <int V>
__device__ __forceinline__ void st_i32(int32_t* p, const int32_t (&f)[V], int valid) {
  if (valid >= V && V % 4 == 0) {
#pragma unroll
    for (int k = 0; k < V; k += 4) *reinterpret_cast<int4*>(p + k) = make_int4(f[k], f[k + 1], f[k + 2], f[k + 3]);
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) if (k < valid) p[k] = f[k];
  }
}
// std of a row from its variance: sqrt(max(var, 0) + 1e-30), a NaN variance kept
__device__ __forceinline__ float pna_sigma(float var) { return sqrtf(__fadd_rn(var < 0.f ? 0.f : var, 1e-30f)); }

// ---------------------------------------------------------------------------------------------------- aggregate
struct AggArgs {
  Walk w;
  const int32_t* indptr;             // forward CSR: D_v = indptr[v + 1] - indptr[v]
  int32_t seg_len;
  const void* zs; int64_t ldz;       // [num_all, d] activation dtype
  const float* zd; int64_t ldzd;     // [N_in, d] fp32
  void* agg; int64_t ldagg, seg;     // [N_in, 4 seg]: [mu + zd | max + zd | min + zd | sigma], segment stride seg
  float* mu; float* var; int64_t ldst;          // [N_in, d] fp32 each, or NULL
  int32_t* amax; int32_t* amin; int64_t lda;    // [N_in, d] int32 each, or NULL
  float* scratch; int64_t lds;       // [n_seg][lds]: mean, M2, max, argmax bits, min, argmin bits at [k d, (k + 1) d)
  int32_t d, nvec;
};

template <int V> struct Stats {
  float mean[V], m2[V], mx[V], mn[V];
  int32_t ax[V], an[V];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < V; ++k) { mean[k] = m2[k] = mx[k] = mn[k] = 0.f; ax[k] = an[k] = -1; }
  }
};

template <typename T>
__device__ __forceinline__ void agg_store(const AggArgs& a, int v, int vi, int n, const Stats<Vec<T>::V>& s) {
  constexpr int V = Vec<T>::V;
  if (vi >= a.nvec) return;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float zd[V], mu[V], var[V], o[4][V];
  ld_f32<V>(a.zd + static_cast<int64_t>(v) * a.ldzd + c0, zd, valid);
  const float nf = static_cast<float>(n);
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if (n == 0) {
      mu[k] = var[k] = 0.f;
      o[0][k] = o[1][k] = o[2][k] = o[3][k] = 0.f;
    } else {
      mu[k] = s.mean[k];
      var[k] = __fdiv_rn(s.m2[k], nf);
      o[0][k] = __fadd_rn(s.mean[k], zd[k]);
      o[1][k] = __fadd_rn(s.mx[k], zd[k]);
      o[2][k] = __fadd_rn(s.mn[k], zd[k]);
      o[3][k] = pna_sigma(var[k]);
    }
  }
  T* out = static_cast<T*>(a.agg) + static_cast<int64_t>(v) * a.ldagg + c0;
#pragma unroll
  for (int j = 0; j < 4; ++j) st_t<T, V>(out + j * a.seg, o[j], valid);
  if (a.mu != nullptr) {
    st_f32<V>(a.mu + static_cast<int64_t>(v) * a.ldst + c0, mu, valid);
    st_f32<V>(a.var + static_cast<int64_t>(v) * a.ldst + c0, var, valid);
  }
  if (a.amax != nullptr) {
    st_i32<V>(a.amax + static_cast<int64_t>(v) * a.lda + c0, s.ax, valid);
    st_i32<V>(a.amin + static_cast<int64_t>(v) * a.lda + c0, s.an, valid);
  }
}

template <typename T>
__device__ __forceinline__ void agg_row(const AggArgs& a, int v, int e0, int n, int slot, int vi, int lane) {
  constexpr int V = Vec<T>::V;
  const T* zs = static_cast<const T*>(a.zs);
  const bool live = vi < a.nvec;
  Stats<V> s;
  s.init();
  int seen = 0;
  for (int b = 0; b < n; b += 32) {
    const int32_t ul = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const int cnt = min(32, n - b);
    for (int t = 0; t < cnt; t += kAggInFlight) {
      int32_t us[kAggInFlight];
      uint4 raw[kAggInFlight];
#pragma unroll
      for (int i = 0; i < kAggInFlight; ++i) {
        us[i] = __shfl_sync(0xffffffffu, ul, min(t + i, cnt - 1));
        if (t + i < cnt && live) raw[i] = ld_vec<16>(zs + static_cast<int64_t>(us[i]) * a.ldz + vi * V);
      }
#pragma unroll
      for (int i = 0; i < kAggInFlight; ++i) {
        if (t + i >= cnt) break;
        ++seen;
        if (!live) continue;
        const float r = __frcp_rn(static_cast<float>(seen));
        float f[V];
        Vec<T>::P::unpack(raw[i], f);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          take_max(s.mx[k], s.ax[k], f[k], us[i]);
          take_min(s.mn[k], s.an[k], f[k], us[i]);
          // Welford: an all-equal row keeps delta = 0, so its M2 stays exactly 0
          const float delta = __fsub_rn(f[k], s.mean[k]);
          s.mean[k] = __fadd_rn(s.mean[k], __fmul_rn(delta, r));
          s.m2[k] = __fadd_rn(s.m2[k], __fmul_rn(delta, __fsub_rn(f[k], s.mean[k])));
        }
      }
    }
  }
  if (slot < 0) {
    agg_store<T>(a, v, vi, n, s);
    return;
  }
  if (!live) return;
  float* p = a.scratch + static_cast<int64_t>(slot) * a.lds;
  const int c0 = vi * V;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if (c0 + k < a.d) {
      p[c0 + k] = s.mean[k];
      p[a.d + c0 + k] = s.m2[k];
      p[2 * a.d + c0 + k] = s.mx[k];
      p[3 * a.d + c0 + k] = __int_as_float(s.ax[k]);
      p[4 * a.d + c0 + k] = s.mn[k];
      p[5 * a.d + c0 + k] = __int_as_float(s.an[k]);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kPnaWarps * 32) pna_agg_kernel(AggArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kPnaWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { agg_row<T>(a, v, e0, n, slot, vi, lane); });
}

// merge the partials of every long row in segment order: Chan's pairwise update for (n, mean, M2), the earlier segment
// keeping a tie of the extremes
template <typename T>
__global__ void __launch_bounds__(kPnaWarps * 32) pna_agg_fixup_kernel(AggArgs a) {
  constexpr int V = Vec<T>::V;
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kPnaWarps + (threadIdx.x >> 5);
  if (li >= a.w.n_long) return;
  const int vi = blockIdx.y * 32 + lane;
  if (vi >= a.nvec) return;
  const int v = a.w.long_row[li];
  const int deg = a.indptr[v + 1] - a.indptr[v];
  const int c0 = vi * V;
  Stats<V> s;
  s.init();
  int na = 0;
  for (int sg = a.w.long_seg_ptr[li], k = 0; sg < a.w.long_seg_ptr[li + 1]; ++sg, ++k) {
    const int nb = min(a.seg_len, deg - k * a.seg_len);
    const int nn = na + nb;
    const float wb = __fdiv_rn(static_cast<float>(nb), static_cast<float>(nn));
    const float wab = __fdiv_rn(__fmul_rn(static_cast<float>(na), static_cast<float>(nb)), static_cast<float>(nn));
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.lds;
#pragma unroll
    for (int e = 0; e < V; ++e) {
      const int c = c0 + e;
      if (c >= a.d) continue;
      const float mb = p[c], m2b = p[a.d + c];
      if (na == 0) {
        s.mean[e] = mb;
        s.m2[e] = m2b;
      } else {
        const float delta = __fsub_rn(mb, s.mean[e]);
        s.mean[e] = __fadd_rn(s.mean[e], __fmul_rn(delta, wb));
        s.m2[e] = __fadd_rn(__fadd_rn(s.m2[e], m2b), __fmul_rn(__fmul_rn(delta, delta), wab));
      }
      take_max(s.mx[e], s.ax[e], p[2 * a.d + c], __float_as_int(p[3 * a.d + c]));
      take_min(s.mn[e], s.an[e], p[4 * a.d + c], __float_as_int(p[5 * a.d + c]));
    }
    na = nn;
  }
  agg_store<T>(a, v, vi, deg, s);
}

// ---------------------------------------------------------------------------------------------------- combine
// out = y + a Z2 + t Z3, each product and sum rounded once in fp32, then one rounding to T
template <typename T>
__global__ void __launch_bounds__(kRowThreads) pna_combine_kernel(const float* y, int64_t ldy, const float* z,
                                                                 int64_t ldz, const float* sa, const float* st,
                                                                 int32_t n, int32_t d, T* out, int64_t ldo) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  if (i >= static_cast<int64_t>(n) * d) return;
  const int v = static_cast<int>(i / d), c = static_cast<int>(i % d);
  const float* zr = z + static_cast<int64_t>(v) * ldz;
  const float r = __fadd_rn(__fadd_rn(y[static_cast<int64_t>(v) * ldy + c], __fmul_rn(sa[v], zr[c])),
                            __fmul_rn(st[v], zr[d + c]));
  out[static_cast<int64_t>(v) * ldo + c] = to_t<T>(r);
}

// G3 = [g | a g | t g] with segment stride seg
template <typename T>
__global__ void __launch_bounds__(kRowThreads) pna_grad_scale_kernel(const T* g, int64_t ldg, const float* sa,
                                                                    const float* st, int32_t n, int32_t d, T* out,
                                                                    int64_t ldo, int64_t seg) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  if (i >= static_cast<int64_t>(n) * d) return;
  const int v = static_cast<int>(i / d), c = static_cast<int>(i % d);
  const float x = static_cast<float>(g[static_cast<int64_t>(v) * ldg + c]);
  T* o = out + static_cast<int64_t>(v) * ldo + c;
  o[0] = g[static_cast<int64_t>(v) * ldg + c];
  o[seg] = to_t<T>(__fmul_rn(sa[v], x));
  o[2 * seg] = to_t<T>(__fmul_rn(st[v], x));
}

// ---------------------------------------------------------------------------------------------------- backward
// per destination element: g_zd = g_mu + g_mx + g_mn, beta = [var > 0] g_sigma / (D sigma), alpha = g_mu / D - beta mu,
// g_mx and g_mn copied to T for the source pass; everything 0 on a row without in-edges
template <typename T>
__global__ void __launch_bounds__(kRowThreads) pna_bwd_dst_kernel(const int32_t* indptr, const float* gagg,
                                                                 int64_t ldga, int64_t seg, const float* mu,
                                                                 const float* var, int64_t ldst, int32_t n, int32_t d,
                                                                 T* gzd, int64_t ldgzd, float* alpha, float* beta,
                                                                 int64_t ldab, T* gmx, T* gmn, int64_t ldgm) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * kRowThreads + threadIdx.x;
  if (i >= static_cast<int64_t>(n) * d) return;
  const int v = static_cast<int>(i / d), c = static_cast<int>(i % d);
  const int deg = indptr[v + 1] - indptr[v];
  const float* gr = gagg + static_cast<int64_t>(v) * ldga + c;
  float zd = 0.f, al = 0.f, be = 0.f, gx = 0.f, gn = 0.f;
  if (deg > 0) {
    const float df = static_cast<float>(deg);
    const float gm = gr[0], gs = gr[3 * seg];
    gx = gr[seg];
    gn = gr[2 * seg];
    zd = __fadd_rn(__fadd_rn(gm, gx), gn);
    const float vv = var[static_cast<int64_t>(v) * ldst + c];
    be = vv > 0.f ? __fdiv_rn(gs, __fmul_rn(df, pna_sigma(vv))) : 0.f;
    al = __fsub_rn(__fdiv_rn(gm, df), __fmul_rn(be, mu[static_cast<int64_t>(v) * ldst + c]));
  }
  gzd[static_cast<int64_t>(v) * ldgzd + c] = to_t<T>(zd);
  alpha[static_cast<int64_t>(v) * ldab + c] = al;
  beta[static_cast<int64_t>(v) * ldab + c] = be;
  gmx[static_cast<int64_t>(v) * ldgm + c] = to_t<T>(gx);
  gmn[static_cast<int64_t>(v) * ldgm + c] = to_t<T>(gn);
}

struct SrcArgs {
  Walk w;
  const void* zs; int64_t ldz;                    // [num_all, d]
  const float* alpha; const float* beta; int64_t ldab;   // [N_in, d]
  const int32_t* amax; const int32_t* amin; int64_t lda; // [N_in, d]
  const void* gmx; const void* gmn; int64_t ldgm;       // [N_in, d] activation dtype
  void* gzs; int64_t ldgzs;                       // [num_all, d]
  float* scratch; int64_t lds;                    // [n_seg][lds]: sum alpha + routed at [0, d), sum beta at [d, 2d)
  int32_t d, nvec;
};

template <typename T>
__device__ __forceinline__ void src_store(const SrcArgs& a, int u, int vi, bool any, const float (&s1)[Vec<T>::V],
                                          const float (&s2)[Vec<T>::V]) {
  constexpr int V = Vec<T>::V;
  if (vi >= a.nvec) return;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float r[V];
  if (any) {
    float zf[V];
    Vec<T>::P::unpack(ld_vec<16>(static_cast<const T*>(a.zs) + static_cast<int64_t>(u) * a.ldz + c0), zf);
#pragma unroll
    for (int k = 0; k < V; ++k) r[k] = __fadd_rn(s1[k], __fmul_rn(zf[k], s2[k]));
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) r[k] = 0.f;
  }
  st_t<T, V>(static_cast<T*>(a.gzs) + static_cast<int64_t>(u) * a.ldgzs + c0, r, valid);
}

template <typename T>
__device__ __forceinline__ void src_row(const SrcArgs& a, int u, int e0, int n, int slot, int vi, int lane) {
  constexpr int V = Vec<T>::V;
  const bool live = vi < a.nvec;
  const int c0 = vi * V;
  const int valid = live ? min(V, a.d - c0) : 0;
  float s1[V], s2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) s1[k] = s2[k] = 0.f;
  for (int b = 0; b < n; b += 32) {
    const int32_t vl = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const int cnt = min(32, n - b);
    for (int t = 0; t < cnt; t += kSrcInFlight) {
      float al[kSrcInFlight][V], be[kSrcInFlight][V];
      uint32_t hx[kSrcInFlight], hn[kSrcInFlight];       // bit k: A+ / A- of element k is u
      uint4 rx[kSrcInFlight], rn[kSrcInFlight];
#pragma unroll
      for (int i = 0; i < kSrcInFlight; ++i) {
        const int v = __shfl_sync(0xffffffffu, vl, min(t + i, cnt - 1));
        hx[i] = hn[i] = 0u;
        if (t + i < cnt && live) {
          const int64_t ro = static_cast<int64_t>(v) * a.ldab + c0;
          ld_f32<V>(a.alpha + ro, al[i], valid);
          ld_f32<V>(a.beta + ro, be[i], valid);
          const int32_t* px = a.amax + static_cast<int64_t>(v) * a.lda + c0;
          const int32_t* pn = a.amin + static_cast<int64_t>(v) * a.lda + c0;
#pragma unroll
          for (int k4 = 0; k4 < V; k4 += 4) {
            const int4 x = __ldg(reinterpret_cast<const int4*>(px + k4));
            const int4 m = __ldg(reinterpret_cast<const int4*>(pn + k4));
            hx[i] |= ((x.x == u ? 1u : 0u) | (x.y == u ? 2u : 0u) | (x.z == u ? 4u : 0u) | (x.w == u ? 8u : 0u)) << k4;
            hn[i] |= ((m.x == u ? 1u : 0u) | (m.y == u ? 2u : 0u) | (m.z == u ? 4u : 0u) | (m.w == u ? 8u : 0u)) << k4;
          }
          const int64_t go = static_cast<int64_t>(v) * a.ldgm + c0;
          if (hx[i]) rx[i] = ld_vec<16>(static_cast<const T*>(a.gmx) + go);
          if (hn[i]) rn[i] = ld_vec<16>(static_cast<const T*>(a.gmn) + go);
        }
      }
#pragma unroll
      for (int i = 0; i < kSrcInFlight; ++i) {
        if (t + i >= cnt) break;
        if (!live) continue;
        float fx[V], fn[V];
        if (hx[i]) Vec<T>::P::unpack(rx[i], fx);
        if (hn[i]) Vec<T>::P::unpack(rn[i], fn);
#pragma unroll
        for (int k = 0; k < V; ++k) {
          s1[k] = __fadd_rn(s1[k], al[i][k]);
          if (hx[i] >> k & 1u) s1[k] = __fadd_rn(s1[k], fx[k]);
          if (hn[i] >> k & 1u) s1[k] = __fadd_rn(s1[k], fn[k]);
          s2[k] = __fadd_rn(s2[k], be[i][k]);
        }
      }
    }
  }
  if (slot < 0) {
    src_store<T>(a, u, vi, n > 0, s1, s2);
    return;
  }
  if (!live) return;
  float* p = a.scratch + static_cast<int64_t>(slot) * a.lds;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    if (c0 + k < a.d) {
      p[c0 + k] = s1[k];
      p[a.d + c0 + k] = s2[k];
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kPnaWarps * 32) pna_src_kernel(SrcArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kPnaWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { src_row<T>(a, u, e0, n, slot, vi, lane); });
}

// sum the partials of every long CSC row in segment order, then apply zs * sum beta
template <typename T>
__global__ void __launch_bounds__(kPnaWarps * 32) pna_src_fixup_kernel(SrcArgs a) {
  constexpr int V = Vec<T>::V;
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kPnaWarps + (threadIdx.x >> 5);
  if (li >= a.w.n_long) return;
  const int vi = blockIdx.y * 32 + lane;
  if (vi >= a.nvec) return;
  const int c0 = vi * V;
  float s1[V], s2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) s1[k] = s2[k] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.lds;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      if (c0 + k < a.d) {
        s1[k] = __fadd_rn(s1[k], p[c0 + k]);
        s2[k] = __fadd_rn(s2[k], p[a.d + c0 + k]);
      }
    }
  }
  src_store<T>(a, a.w.long_row[li], vi, true, s1, s2);
}

// ---------------------------------------------------------------------------------------------------- dispatch
template <typename T>
void preload_t() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, pna_agg_kernel<T>);
  cudaFuncGetAttributes(&a, pna_agg_fixup_kernel<T>);
  cudaFuncGetAttributes(&a, pna_combine_kernel<T>);
  cudaFuncGetAttributes(&a, pna_grad_scale_kernel<T>);
  cudaFuncGetAttributes(&a, pna_bwd_dst_kernel<T>);
  cudaFuncGetAttributes(&a, pna_src_kernel<T>);
  cudaFuncGetAttributes(&a, pna_src_fixup_kernel<T>);
}

// a tile is 32 vectors of 16 bytes; wider rows take more tiles
int tiles_of(int32_t nvec) { return (nvec + 31) / 32; }

int row_blocks(int32_t n, int32_t d) {
  return static_cast<int>((static_cast<int64_t>(n) * d + kRowThreads - 1) / kRowThreads);
}

bool f32_ok(const void* p, int64_t ld) { return vec_ok(p, ld, 4); }

}  // namespace

// CUDA loads kernels lazily, and loading one may wait for the device: see exchange.cu's bns_preload.
static void pna_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_t<float>();
    preload_t<__nv_bfloat16>();
    cudaGetLastError();
  });
}

}  // namespace pg

extern "C" int pg_pna_preload(void) {
  pg::pna_preload();
  return PG_OK;
}

extern "C" int pg_pna_aggregate(const pg_csr* g, const void* zs, int64_t ldz, const float* zd, int64_t ldzd,
                                int32_t d, int dtype, void* agg, int64_t ldagg, int64_t seg, float* mu, float* var,
                                int64_t ldst, int32_t* amax, int32_t* amin, int64_t lda, float* scratch,
                                int64_t ld_scratch, void* stream) {
  pg::pna_preload();
  if (int rc = pg::check_plan(g, "pg_pna_aggregate")) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_pna_aggregate: unknown dtype %d", dtype);
  const int es = pg::elem_size(dtype);
  const int V = 16 / es;
  PG_REQUIRE(d > 0 && ldz >= d && ldzd >= d, "pg_pna_aggregate: bad sizes (d %d)", d);
  if (g->n_rows == 0) return PG_OK;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  PG_REQUIRE(zs && zd && agg && (g->n_seg == 0 || scratch) && ((mu == nullptr) == (var == nullptr)) &&
                 ((amax == nullptr) == (amin == nullptr)),
             "pg_pna_aggregate: null argument");
  PG_REQUIRE(seg >= full && seg % V == 0 && ldagg >= 4 * seg && ldz >= full && ldzd >= full &&
                 (mu == nullptr || ldst >= full) && (amax == nullptr || lda >= full),
             "pg_pna_aggregate: segment or row stride shorter than the last 16-byte vector");
  PG_REQUIRE(g->n_seg == 0 || ld_scratch >= 6 * static_cast<int64_t>(d), "pg_pna_aggregate: scratch rows < 6d");
  PG_REQUIRE(pg::vec_ok(zs, ldz, es) && pg::vec_ok(agg, ldagg, es) && pg::f32_ok(zd, ldzd) &&
                 (mu == nullptr || (pg::f32_ok(mu, ldst) && pg::f32_ok(var, ldst))) &&
                 (amax == nullptr || (pg::vec_ok(amax, lda, 4) && pg::vec_ok(amin, lda, 4))),
             "pg_pna_aggregate: rows must start on 16-byte boundaries with a 16-byte multiple stride");
  pg::AggArgs a{pg::make_walk(g), g->indptr, g->seg_len, zs, ldz, zd, ldzd, agg, ldagg, seg, mu, var, ldst,
                amax, amin, lda, scratch, ld_scratch, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + pg::kPnaWarps - 1) / pg::kPnaWarps, pg::tiles_of(nvec));
  const dim3 grid_fix((g->n_long + pg::kPnaWarps - 1) / pg::kPnaWarps, pg::tiles_of(nvec));
  if (dtype == PG_F32) {
    if (g->n_chunks > 0) pg::pna_agg_kernel<float><<<grid, pg::kPnaWarps * 32, 0, st>>>(a);
    if (g->n_long > 0) pg::pna_agg_fixup_kernel<float><<<grid_fix, pg::kPnaWarps * 32, 0, st>>>(a);
  } else {
    if (g->n_chunks > 0) pg::pna_agg_kernel<__nv_bfloat16><<<grid, pg::kPnaWarps * 32, 0, st>>>(a);
    if (g->n_long > 0) pg::pna_agg_fixup_kernel<__nv_bfloat16><<<grid_fix, pg::kPnaWarps * 32, 0, st>>>(a);
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_pna_combine(const float* y, int64_t ldy, const float* z, int64_t ldz, const float* a,
                              const float* t, int32_t n_rows, int32_t d_out, int dtype, void* out, int64_t ldo,
                              void* stream) {
  pg::pna_preload();
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_pna_combine: unknown dtype %d", dtype);
  PG_REQUIRE(n_rows >= 0 && d_out > 0 && ldy >= d_out && ldz >= 2 * static_cast<int64_t>(d_out) && ldo >= d_out,
             "pg_pna_combine: bad sizes (d_out %d)", d_out);
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(y && z && a && t && out, "pg_pna_combine: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nb = pg::row_blocks(n_rows, d_out);
  if (dtype == PG_F32)
    pg::pna_combine_kernel<float><<<nb, pg::kRowThreads, 0, st>>>(y, ldy, z, ldz, a, t, n_rows, d_out,
                                                                   static_cast<float*>(out), ldo);
  else
    pg::pna_combine_kernel<__nv_bfloat16><<<nb, pg::kRowThreads, 0, st>>>(y, ldy, z, ldz, a, t, n_rows, d_out,
                                                                           static_cast<__nv_bfloat16*>(out), ldo);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_pna_grad_scale(const void* g, int64_t ldg, const float* a, const float* t, int32_t n_rows,
                                 int32_t d_out, int dtype, void* out, int64_t ldo, int64_t seg, void* stream) {
  pg::pna_preload();
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_pna_grad_scale: unknown dtype %d", dtype);
  PG_REQUIRE(n_rows >= 0 && d_out > 0 && ldg >= d_out && seg >= d_out && ldo >= 3 * seg,
             "pg_pna_grad_scale: bad sizes (d_out %d)", d_out);
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(g && a && t && out, "pg_pna_grad_scale: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nb = pg::row_blocks(n_rows, d_out);
  if (dtype == PG_F32)
    pg::pna_grad_scale_kernel<float><<<nb, pg::kRowThreads, 0, st>>>(static_cast<const float*>(g), ldg, a, t, n_rows,
                                                                      d_out, static_cast<float*>(out), ldo, seg);
  else
    pg::pna_grad_scale_kernel<__nv_bfloat16><<<nb, pg::kRowThreads, 0, st>>>(
        static_cast<const __nv_bfloat16*>(g), ldg, a, t, n_rows, d_out, static_cast<__nv_bfloat16*>(out), ldo, seg);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_pna_bwd_dst(const int32_t* indptr, const float* gagg, int64_t ldga, int64_t seg, const float* mu,
                              const float* var, int64_t ldst, int32_t n_rows, int32_t d, int dtype, void* gzd,
                              int64_t ldgzd, float* alpha, float* beta, int64_t ldab, void* gmx, void* gmn,
                              int64_t ldgm, void* stream) {
  pg::pna_preload();
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_pna_bwd_dst: unknown dtype %d", dtype);
  PG_REQUIRE(n_rows >= 0 && d > 0 && seg >= d && ldga >= 4 * seg && ldst >= d && ldgzd >= d && ldab >= d && ldgm >= d,
             "pg_pna_bwd_dst: bad sizes (d %d)", d);
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(indptr && gagg && mu && var && gzd && alpha && beta && gmx && gmn, "pg_pna_bwd_dst: null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int nb = pg::row_blocks(n_rows, d);
  if (dtype == PG_F32)
    pg::pna_bwd_dst_kernel<float><<<nb, pg::kRowThreads, 0, st>>>(
        indptr, gagg, ldga, seg, mu, var, ldst, n_rows, d, static_cast<float*>(gzd), ldgzd, alpha, beta, ldab,
        static_cast<float*>(gmx), static_cast<float*>(gmn), ldgm);
  else
    pg::pna_bwd_dst_kernel<__nv_bfloat16><<<nb, pg::kRowThreads, 0, st>>>(
        indptr, gagg, ldga, seg, mu, var, ldst, n_rows, d, static_cast<__nv_bfloat16*>(gzd), ldgzd, alpha, beta,
        ldab, static_cast<__nv_bfloat16*>(gmx), static_cast<__nv_bfloat16*>(gmn), ldgm);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_pna_bwd_src(const pg_csr* gt, const void* zs, int64_t ldz, const float* alpha, const float* beta,
                              int64_t ldab, const int32_t* amax, const int32_t* amin, int64_t lda, const void* gmx,
                              const void* gmn, int64_t ldgm, int32_t d, int dtype, void* gzs, int64_t ldgzs,
                              float* scratch, int64_t ld_scratch, void* stream) {
  pg::pna_preload();
  if (int rc = pg::check_plan(gt, "pg_pna_bwd_src")) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_pna_bwd_src: unknown dtype %d", dtype);
  const int es = pg::elem_size(dtype);
  const int V = 16 / es;
  PG_REQUIRE(d > 0 && ldz >= d && ldgzs >= d, "pg_pna_bwd_src: bad sizes (d %d)", d);
  if (gt->n_rows == 0) return PG_OK;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  PG_REQUIRE(zs && gzs && (gt->nnz == 0 || (alpha && beta && amax && amin && gmx && gmn)) &&
                 (gt->n_seg == 0 || scratch),
             "pg_pna_bwd_src: null argument");
  PG_REQUIRE(ldz >= full && (gt->nnz == 0 || (ldab >= full && lda >= full && ldgm >= full)),
             "pg_pna_bwd_src: row stride shorter than the last 16-byte vector");
  PG_REQUIRE(gt->n_seg == 0 || ld_scratch >= 2 * static_cast<int64_t>(d), "pg_pna_bwd_src: scratch rows < 2d");
  PG_REQUIRE(pg::vec_ok(zs, ldz, es) && pg::vec_ok(gzs, ldgzs, es) &&
                 (gt->nnz == 0 || (pg::f32_ok(alpha, ldab) && pg::f32_ok(beta, ldab) && pg::vec_ok(amax, lda, 4) &&
                                   pg::vec_ok(amin, lda, 4) && pg::vec_ok(gmx, ldgm, es) && pg::vec_ok(gmn, ldgm, es))),
             "pg_pna_bwd_src: rows must start on 16-byte boundaries with a 16-byte multiple stride");
  pg::SrcArgs a{pg::make_walk(gt), zs, ldz, alpha, beta, ldab, amax, amin, lda, gmx, gmn, ldgm, gzs, ldgzs,
                scratch, ld_scratch, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((gt->n_chunks + pg::kPnaWarps - 1) / pg::kPnaWarps, pg::tiles_of(nvec));
  const dim3 grid_fix((gt->n_long + pg::kPnaWarps - 1) / pg::kPnaWarps, pg::tiles_of(nvec));
  if (dtype == PG_F32) {
    if (gt->n_chunks > 0) pg::pna_src_kernel<float><<<grid, pg::kPnaWarps * 32, 0, st>>>(a);
    if (gt->n_long > 0) pg::pna_src_fixup_kernel<float><<<grid_fix, pg::kPnaWarps * 32, 0, st>>>(a);
  } else {
    if (gt->n_chunks > 0) pg::pna_src_kernel<__nv_bfloat16><<<grid, pg::kPnaWarps * 32, 0, st>>>(a);
    if (gt->n_long > 0) pg::pna_src_fixup_kernel<__nv_bfloat16><<<grid_fix, pg::kPnaWarps * 32, 0, st>>>(a);
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}
