// Residual gated graph convolution (Bresson & Laurent, "Residual Gated Graph ConvNets", 2017; PyG ResGatedGraphConv)
// on sm_90a: the per-channel edge-gate aggregate and its two backward passes.
//
//   out[v] = skip[v] + sum_{u -> v} sigmoid(k[v] + q[u]) val[u]      (per column; skip carries the output bias)
//
// The plan walks are genconv.cu's: one warp per (chunk, tile of 32 column vectors of VB bytes), lane l holding vector l
// of the tile, several neighbour rows in flight.  Sums are fp32, in CSR order (aggregate, destination pass) or CSC
// order (source pass); long rows come as segments whose fp32 partials a fix-up adds in segment order.  There is no
// normalisation across the in-edges, so no softmax state, and no per-edge array: both backward passes recompute every
// gate.  No atomics: the results are the same bits from run to run.  A gate and its derivative take one expf:
//   e = exp(-|x|),  r = 1 / (1 + e),  sigmoid(x) = x >= 0 ? r : e r,  sigmoid'(x) = e r r
// which is finite for every finite x and has no 1 - sigmoid cancellation.  Every output vector is written whole: the
// columns between d and the end of the row's last vector are written as 0.
#include <math.h>

#include <algorithm>
#include <mutex>

#include "chunk_walk.cuh"

namespace pg {
namespace {

constexpr int kRgWarps = 4;         // warps per CTA
// neighbour rows loaded before they are folded in (two vectors each): the most every instance compiles with without
// local-memory spills
template <int V, bool SRC> __host__ __device__ constexpr int rg_in_flight() { return V == 1 ? 2 : SRC && V >= 8 ? 2 : 4; }

__device__ __forceinline__ bool rg_kept(const uint8_t* keep, int32_t num_in, int32_t u) {
  return keep == nullptr || u < num_in || keep[u - num_in] != 0;
}

// sigmoid(x) and sigmoid'(x) from one expf (a NaN x gives NaN for both)
__device__ __forceinline__ void rg_gate(float x, float& s, float& ds) {
  const float e = expf(-fabsf(x));
  const float r = __frcp_rn(__fadd_rn(1.f, e));
  const float er = __fmul_rn(e, r);
  s = x >= 0.f ? r : er;
  ds = __fmul_rn(er, r);
}

struct RgArgs {
  Walk w;
  const void* qv; int64_t ldqv;      // [num_all rows]: q at columns [0, d), val at [half, half + d)
  const void* ks; int64_t ldks;      // [N_in rows]: k at [0, d), skip at [half, half + d)
  const void* g; int64_t ldg;        // backward: the gradient G of out [N_in, d]
  const uint8_t* keep; int32_t num_in;
  void* out; int64_t ldo;            // aggregate: out [N_in, d]; destination pass: [dk | G]; source pass: [dq | dval]
  float* scratch; int64_t ldsc;      // [n_seg][ldsc] fp32 partials: [0, d) (and [d, 2 d) in the source pass)
  int32_t half, d, nvec;
};

template <typename T, int VB>
__device__ __forceinline__ void ld_row(const void* base, int64_t ld, int r, int64_t c, float (&f)[Pack<T, VB>::V]) {
  Pack<T, VB>::unpack(ld_vec<VB>(static_cast<const T*>(base) + static_cast<int64_t>(r) * ld + c), f);
}

// one whole vector of T at column c of row r: the first `valid` values (one rounding each), zeros after them
template <typename T, int VB>
__device__ __forceinline__ void st_row(void* base, int64_t ld, int r, int64_t c, const float (&f)[Pack<T, VB>::V],
                                       int valid) {
  constexpr int V = Pack<T, VB>::V;
  float o[V];
#pragma unroll
  for (int k = 0; k < V; ++k) o[k] = k < valid ? f[k] : 0.f;
  st_vec<VB>(static_cast<T*>(base) + static_cast<int64_t>(r) * ld + c, Pack<T, VB>::pack(o));
}

// Sums over the kept in-edges u -> v of CSR row v (entries e0 .. e0 + n) of the forward plan, per element of vector
// vi: DER = false: acc = sum sigmoid(k_v + q_u) val_u (the aggregate); DER = true: acc = sum sigmoid'(k_v + q_u) val_u
// (the destination pass).  kv: the k row of v.
template <typename T, int VB, bool DER>
__device__ __forceinline__ void dst_sum(const RgArgs& a, int e0, int n, int vi, int lane, bool live,
                                        const float (&kv)[Pack<T, VB>::V], float (&acc)[Pack<T, VB>::V]) {
  using P = Pack<T, VB>;
  constexpr int V = P::V;
  constexpr int kRgInFlight = rg_in_flight<V, false>();
  const T* qv = static_cast<const T*>(a.qv);
  const int c0 = vi * V;
#pragma unroll
  for (int k = 0; k < V; ++k) acc[k] = 0.f;
  for (int b = 0; b < n; b += 32) {
    int32_t ul = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    if (!rg_kept(a.keep, a.num_in, ul)) ul = -1;
    const int cnt = min(32, n - b);
    for (int j = 0; j < cnt; j += kRgInFlight) {
      int32_t us[kRgInFlight];
      typename P::Raw rq[kRgInFlight], rv[kRgInFlight];
#pragma unroll
      for (int i = 0; i < kRgInFlight; ++i) {
        us[i] = __shfl_sync(0xffffffffu, ul, min(j + i, cnt - 1));
        if (j + i < cnt && us[i] >= 0 && live) {
          const T* row = qv + static_cast<int64_t>(us[i]) * a.ldqv + c0;
          rq[i] = ld_vec<VB>(row);
          rv[i] = ld_vec<VB>(row + a.half);
        }
      }
#pragma unroll
      for (int i = 0; i < kRgInFlight; ++i) {
        if (j + i < cnt && us[i] >= 0 && live) {
          float fq[V], fv[V];
          P::unpack(rq[i], fq);
          P::unpack(rv[i], fv);
#pragma unroll
          for (int k = 0; k < V; ++k) {
            float s, ds;
            rg_gate(__fadd_rn(kv[k], fq[k]), s, ds);
            acc[k] = __fmaf_rn(DER ? ds : s, fv[k], acc[k]);
          }
        }
      }
    }
  }
}

template <typename T, int VB>
__device__ __forceinline__ void save_partial(const RgArgs& a, int slot, int c0, int off, const float* f) {
  constexpr int V = Pack<T, VB>::V;
  float* p = a.scratch + static_cast<int64_t>(slot) * a.ldsc + off;
#pragma unroll
  for (int k = 0; k < V; ++k)
    if (c0 + k < a.d) p[c0 + k] = f[k];
}

template <typename T, int VB>
__device__ __forceinline__ void add_partials(const RgArgs& a, int li, int c0, int off, float* f) {
  constexpr int V = Pack<T, VB>::V;
#pragma unroll
  for (int k = 0; k < V; ++k) f[k] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.ldsc + off;
#pragma unroll
    for (int k = 0; k < V; ++k)
      if (c0 + k < a.d) f[k] = __fadd_rn(f[k], p[c0 + k]);
  }
}

// ---------------------------------------------------------------------------------------------------- aggregate
// out[v] = skip[v] + acc, rounded once to T
template <typename T, int VB>
__device__ __forceinline__ void fwd_store(const RgArgs& a, int v, int vi, const float (&acc)[Pack<T, VB>::V]) {
  constexpr int V = Pack<T, VB>::V;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float sk[V], o[V];
  ld_row<T, VB>(a.ks, a.ldks, v, a.half + c0, sk);
#pragma unroll
  for (int k = 0; k < V; ++k) o[k] = __fadd_rn(sk[k], acc[k]);
  st_row<T, VB>(a.out, a.ldo, v, c0, o, valid);
}

template <typename T, int VB>
__device__ __forceinline__ void fwd_row(const RgArgs& a, int v, int e0, int n, int slot, int vi, int lane) {
  constexpr int V = Pack<T, VB>::V;
  const bool live = vi < a.nvec;
  float kv[V], acc[V];
  if (live) ld_row<T, VB>(a.ks, a.ldks, v, vi * V, kv);
  dst_sum<T, VB, false>(a, e0, n, vi, lane, live, kv, acc);
  if (!live) return;
  if (slot < 0) fwd_store<T, VB>(a, v, vi, acc);
  else save_partial<T, VB>(a, slot, vi * V, 0, acc);
}

template <typename T, int VB>
__global__ void __launch_bounds__(kRgWarps * 32) resgated_fwd_kernel(RgArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kRgWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { fwd_row<T, VB>(a, v, e0, n, slot, vi, lane); });
}

template <typename T, int VB>
__global__ void __launch_bounds__(kRgWarps * 32) resgated_fwd_fixup_kernel(RgArgs a) {
  constexpr int V = Pack<T, VB>::V;
  const int li = blockIdx.x * kRgWarps + (threadIdx.x >> 5);
  const int vi = blockIdx.y * 32 + (threadIdx.x & 31);
  if (li >= a.w.n_long || vi >= a.nvec) return;
  float acc[V];
  add_partials<T, VB>(a, li, vi * V, 0, acc);
  fwd_store<T, VB>(a, a.w.long_row[li], vi, acc);
}

// ---------------------------------------------------------------------------------------------------- destination pass
// dk[v] = G[v] s1 (one rounding to T) at [0, d), G[v] at [half, half + d) of the output row
template <typename T, int VB>
__device__ __forceinline__ void dst_store(const RgArgs& a, int v, int vi, const float (&s1)[Pack<T, VB>::V]) {
  constexpr int V = Pack<T, VB>::V;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float gv[V], dk[V];
  ld_row<T, VB>(a.g, a.ldg, v, c0, gv);
#pragma unroll
  for (int k = 0; k < V; ++k) dk[k] = __fmul_rn(gv[k], s1[k]);
  st_row<T, VB>(a.out, a.ldo, v, c0, dk, valid);
  st_row<T, VB>(a.out, a.ldo, v, a.half + c0, gv, valid);
}

template <typename T, int VB>
__device__ __forceinline__ void dst_row(const RgArgs& a, int v, int e0, int n, int slot, int vi, int lane) {
  constexpr int V = Pack<T, VB>::V;
  const bool live = vi < a.nvec;
  float kv[V], s1[V];
  if (live) ld_row<T, VB>(a.ks, a.ldks, v, vi * V, kv);
  dst_sum<T, VB, true>(a, e0, n, vi, lane, live, kv, s1);
  if (!live) return;
  if (slot < 0) dst_store<T, VB>(a, v, vi, s1);
  else save_partial<T, VB>(a, slot, vi * V, 0, s1);
}

template <typename T, int VB>
__global__ void __launch_bounds__(kRgWarps * 32) resgated_dst_kernel(RgArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kRgWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { dst_row<T, VB>(a, v, e0, n, slot, vi, lane); });
}

template <typename T, int VB>
__global__ void __launch_bounds__(kRgWarps * 32) resgated_dst_fixup_kernel(RgArgs a) {
  constexpr int V = Pack<T, VB>::V;
  const int li = blockIdx.x * kRgWarps + (threadIdx.x >> 5);
  const int vi = blockIdx.y * 32 + (threadIdx.x & 31);
  if (li >= a.w.n_long || vi >= a.nvec) return;
  float s1[V];
  add_partials<T, VB>(a, li, vi * V, 0, s1);
  dst_store<T, VB>(a, a.w.long_row[li], vi, s1);
}

// ---------------------------------------------------------------------------------------------------- source pass
// dq[u] = val[u] B at [0, d), dval[u] = A at [half, half + d), both rounded once to T; vu = 0 for an unkept halo row
// and for a row without out-edges, so both get exact zeros
template <typename T, int VB>
__device__ __forceinline__ void src_store(const RgArgs& a, int u, int vi, const float (&vu)[Pack<T, VB>::V],
                                          const float (&A)[Pack<T, VB>::V], const float (&B)[Pack<T, VB>::V]) {
  constexpr int V = Pack<T, VB>::V;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  float dq[V];
#pragma unroll
  for (int k = 0; k < V; ++k) dq[k] = __fmul_rn(vu[k], B[k]);
  st_row<T, VB>(a.out, a.ldo, u, c0, dq, valid);
  st_row<T, VB>(a.out, a.ldo, u, a.half + c0, A, valid);
}

// over the CSC row u (the destinations v of source u), per element: A = sum_v G_v sigmoid(k_v + q_u),
// B = sum_v G_v sigmoid'(k_v + q_u)
template <typename T, int VB>
__device__ __forceinline__ void src_row(const RgArgs& a, int u, int e0, int n, int slot, int vi, int lane) {
  using P = Pack<T, VB>;
  constexpr int V = P::V;
  constexpr int kRgInFlight = rg_in_flight<V, true>();
  const bool live = vi < a.nvec;
  const int c0 = vi * V;
  float qu[V], vu[V], A[V], B[V];
#pragma unroll
  for (int k = 0; k < V; ++k) { qu[k] = vu[k] = A[k] = B[k] = 0.f; }
  if (!rg_kept(a.keep, a.num_in, u)) n = 0;
  if (n > 0 && live) {
    ld_row<T, VB>(a.qv, a.ldqv, u, c0, qu);
    ld_row<T, VB>(a.qv, a.ldqv, u, a.half + c0, vu);
  }
  const T* ks = static_cast<const T*>(a.ks);
  const T* gp = static_cast<const T*>(a.g);
  for (int b = 0; b < n; b += 32) {
    const int32_t vl = b + lane < n ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const int cnt = min(32, n - b);
    for (int j = 0; j < cnt; j += kRgInFlight) {
      typename P::Raw rk[kRgInFlight], rg[kRgInFlight];
#pragma unroll
      for (int i = 0; i < kRgInFlight; ++i) {
        const int v = __shfl_sync(0xffffffffu, vl, min(j + i, cnt - 1));
        if (j + i < cnt && live) {
          rk[i] = ld_vec<VB>(ks + static_cast<int64_t>(v) * a.ldks + c0);
          rg[i] = ld_vec<VB>(gp + static_cast<int64_t>(v) * a.ldg + c0);
        }
      }
#pragma unroll
      for (int i = 0; i < kRgInFlight; ++i) {
        if (j + i < cnt && live) {
          float fk[V], fg[V];
          P::unpack(rk[i], fk);
          P::unpack(rg[i], fg);
#pragma unroll
          for (int k = 0; k < V; ++k) {
            float s, ds;
            rg_gate(__fadd_rn(fk[k], qu[k]), s, ds);
            A[k] = __fmaf_rn(fg[k], s, A[k]);
            B[k] = __fmaf_rn(fg[k], ds, B[k]);
          }
        }
      }
    }
  }
  if (!live) return;
  if (slot < 0) {
    src_store<T, VB>(a, u, vi, vu, A, B);
  } else {
    save_partial<T, VB>(a, slot, c0, 0, A);
    save_partial<T, VB>(a, slot, c0, a.d, B);
  }
}

template <typename T, int VB>
__global__ void __launch_bounds__(kRgWarps * 32) resgated_src_kernel(RgArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kRgWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { src_row<T, VB>(a, u, e0, n, slot, vi, lane); });
}

// a long CSC row: the segments' (A, B) added in segment order (an unkept row's segments hold zeros, and its val is
// not read)
template <typename T, int VB>
__global__ void __launch_bounds__(kRgWarps * 32) resgated_src_fixup_kernel(RgArgs a) {
  constexpr int V = Pack<T, VB>::V;
  const int li = blockIdx.x * kRgWarps + (threadIdx.x >> 5);
  const int vi = blockIdx.y * 32 + (threadIdx.x & 31);
  if (li >= a.w.n_long || vi >= a.nvec) return;
  const int u = a.w.long_row[li], c0 = vi * V;
  float vu[V], A[V], B[V];
  if (rg_kept(a.keep, a.num_in, u)) {
    ld_row<T, VB>(a.qv, a.ldqv, u, a.half + c0, vu);
  } else {
#pragma unroll
    for (int k = 0; k < V; ++k) vu[k] = 0.f;
  }
  add_partials<T, VB>(a, li, c0, 0, A);
  add_partials<T, VB>(a, li, c0, a.d, B);
  src_store<T, VB>(a, u, vi, vu, A, B);
}

// ---------------------------------------------------------------------------------------------------- dispatch
enum RgPass { kAggregate, kDst, kSrc };

template <typename T, int VB>
void preload_vb() {
  cudaFuncAttributes f;
  cudaFuncGetAttributes(&f, resgated_fwd_kernel<T, VB>);
  cudaFuncGetAttributes(&f, resgated_fwd_fixup_kernel<T, VB>);
  cudaFuncGetAttributes(&f, resgated_dst_kernel<T, VB>);
  cudaFuncGetAttributes(&f, resgated_dst_fixup_kernel<T, VB>);
  cudaFuncGetAttributes(&f, resgated_src_kernel<T, VB>);
  cudaFuncGetAttributes(&f, resgated_src_fixup_kernel<T, VB>);
}

template <typename T, int VB>
void launch_vb(RgPass pass, const RgArgs& a, const pg_csr* g, cudaStream_t st) {
  const dim3 grid((g->n_chunks + kRgWarps - 1) / kRgWarps, (a.nvec + 31) / 32);
  const dim3 grid_fix((g->n_long + kRgWarps - 1) / kRgWarps, (a.nvec + 31) / 32);
  const int th = kRgWarps * 32;
  if (pass == kAggregate) {
    if (g->n_chunks > 0) resgated_fwd_kernel<T, VB><<<grid, th, 0, st>>>(a);
    if (g->n_long > 0) resgated_fwd_fixup_kernel<T, VB><<<grid_fix, th, 0, st>>>(a);
  } else if (pass == kDst) {
    if (g->n_chunks > 0) resgated_dst_kernel<T, VB><<<grid, th, 0, st>>>(a);
    if (g->n_long > 0) resgated_dst_fixup_kernel<T, VB><<<grid_fix, th, 0, st>>>(a);
  } else {
    if (g->n_chunks > 0) resgated_src_kernel<T, VB><<<grid, th, 0, st>>>(a);
    if (g->n_long > 0) resgated_src_fixup_kernel<T, VB><<<grid_fix, th, 0, st>>>(a);
  }
}

template <typename T>
void launch_t(int vb, RgPass pass, const RgArgs& a, const pg_csr* g, cudaStream_t st) {
  if (vb == 16) launch_vb<T, 16>(pass, a, g, st);
  else if (vb == 8) launch_vb<T, 8>(pass, a, g, st);
  else if (vb == 4) launch_vb<T, 4>(pass, a, g, st);
  else if constexpr (sizeof(T) == 2) launch_vb<T, 2>(pass, a, g, st);
}

// the widest vector (bytes) that every row of every operand allows: a paired operand's second half included
int rg_vec_bytes(const void* qv, int64_t ldqv, const void* ks, int64_t ldks, const void* gr, int64_t ldg,
                 const void* out, int64_t ldo, bool out_paired, int32_t half, int es) {
  const char* q = static_cast<const char*>(qv);
  const char* k = static_cast<const char*>(ks);
  const char* o = static_cast<const char*>(out);
  const int64_t hb = static_cast<int64_t>(half) * es;
  int vb = std::min({vec_bytes(q, ldqv, es), vec_bytes(q + hb, ldqv, es), vec_bytes(k, ldks, es),
                     vec_bytes(k + hb, ldks, es), vec_bytes(o, ldo, es)});
  if (out_paired) vb = std::min(vb, vec_bytes(o + hb, ldo, es));
  if (gr != nullptr) vb = std::min(vb, vec_bytes(gr, ldg, es));
  return vb;
}

int run(const char* who, RgPass pass, const pg_csr* g, const void* qv, int64_t ldqv, const void* ks, int64_t ldks,
        int32_t half, const void* grad, int64_t ldg, int32_t d, int dtype, const uint8_t* keep, int32_t num_in,
        void* out, int64_t ldo, float* scratch, int64_t ld_scratch, void* stream) {
  if (int rc = check_plan(g, who)) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "%s: unknown dtype %d", who, dtype);
  PG_REQUIRE(d > 0 && half >= d && num_in >= 0, "%s: bad sizes (d %d, half %d)", who, d, half);
  if (g->n_rows == 0) return PG_OK;
  const bool backward = pass != kAggregate;
  PG_REQUIRE(qv && ks && out && (!backward || grad) && (g->n_seg == 0 || scratch), "%s: null argument", who);
  const int es = elem_size(dtype);
  const int vb = rg_vec_bytes(qv, ldqv, ks, ldks, backward ? grad : nullptr, ldg, out, ldo, backward, half, es);
  const int V = vb / es;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  PG_REQUIRE(half >= full && ldqv >= half + full && ldks >= half + full && (!backward || ldg >= full) &&
                 ldo >= (backward ? half + full : full),
             "%s: a row (or half row) shorter than its last %d-byte vector (d %d, half %d)", who, vb, d, half);
  PG_REQUIRE(g->n_seg == 0 || ld_scratch >= (pass == kSrc ? 2 : 1) * static_cast<int64_t>(d),
             "%s: scratch rows shorter than %d d", who, pass == kSrc ? 2 : 1);
  RgArgs a{make_walk(g), qv, ldqv, ks, ldks, grad, ldg, keep, num_in, out, ldo, scratch, ld_scratch, half, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) launch_t<float>(vb, pass, a, g, st);
  else launch_t<__nv_bfloat16>(vb, pass, a, g, st);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

}  // namespace

// CUDA loads kernels lazily, and loading one may wait for the device: see exchange.cu's bns_preload.
static void resgated_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_vb<float, 16>(); preload_vb<float, 8>(); preload_vb<float, 4>();
    preload_vb<__nv_bfloat16, 16>(); preload_vb<__nv_bfloat16, 8>(); preload_vb<__nv_bfloat16, 4>();
    preload_vb<__nv_bfloat16, 2>();
    cudaGetLastError();
  });
}

}  // namespace pg

extern "C" int pg_resgated_preload(void) {
  pg::resgated_preload();
  return PG_OK;
}

extern "C" int pg_resgated_aggregate(const pg_csr* g, const void* qv, int64_t ldqv, const void* ks, int64_t ldks,
                                     int32_t half, int32_t d, int dtype, const uint8_t* keep, int32_t num_in, void* out,
                                     int64_t ldo, float* scratch, int64_t ld_scratch, void* stream) {
  pg::resgated_preload();
  return pg::run("pg_resgated_aggregate", pg::kAggregate, g, qv, ldqv, ks, ldks, half, nullptr, 0, d, dtype, keep,
                 num_in, out, ldo, scratch, ld_scratch, stream);
}

extern "C" int pg_resgated_bwd_dst(const pg_csr* g, const void* qv, int64_t ldqv, const void* ks, int64_t ldks,
                                   int32_t half, const void* grad, int64_t ldg, int32_t d, int dtype,
                                   const uint8_t* keep, int32_t num_in, void* dkg, int64_t lddkg, float* scratch,
                                   int64_t ld_scratch, void* stream) {
  pg::resgated_preload();
  return pg::run("pg_resgated_bwd_dst", pg::kDst, g, qv, ldqv, ks, ldks, half, grad, ldg, d, dtype, keep, num_in, dkg,
                 lddkg, scratch, ld_scratch, stream);
}

extern "C" int pg_resgated_bwd_src(const pg_csr* gt, const void* qv, int64_t ldqv, const void* ks, int64_t ldks,
                                   int32_t half, const void* grad, int64_t ldg, int32_t d, int dtype,
                                   const uint8_t* keep, int32_t num_in, void* dqv, int64_t lddqv, float* scratch,
                                   int64_t ld_scratch, void* stream) {
  pg::resgated_preload();
  return pg::run("pg_resgated_bwd_src", pg::kSrc, gt, qv, ldqv, ks, ldks, half, grad, ldg, d, dtype, keep, num_in, dqv,
                 lddqv, scratch, ld_scratch, stream);
}
