// Gaussian mixture model convolution (Monti et al., "Geometric deep learning on graphs and manifolds using mixture model
// CNNs", CVPR 2017; DGL GMMConv, mean aggregator) on sm_90a, with the degree pseudo-coordinates e_uv = (c[u], c[v]),
// c = clamp(deg, 1)^-1/2.  For the K mixture kernels:
//
//   w_k(e) = exp(-1/2 sum_j ((e_j - mu[k, j]) inv_sigma[k, j])^2)
//
// Two gathers, each in one template with a compile-time direction:
//   gather-K   one gathered row per edge, K fp32 accumulators per element, written as K column slices `slice` apart:
//              forward over the CSR   A[v][k]  = (1/deg_v) sum_u w_k(e_uv) x[u]            (aggregate first)
//              backward over the CSC  dz[u][k] = sum_v (w_k(e_uv) / deg_v) G[v]           (transform first)
//   gather-sum K slices per gathered row, one accumulator:
//              forward over the CSR   out[v]   = (1/deg_v) sum_u sum_k w_k(e_uv) z[u][k] + bias   (transform first)
//              backward over the CSC  dh[u]    = dropout(sum_v (1/deg_v) sum_k w_k(e_uv) dA[v][k]) (aggregate first)
// Both backward passes also produce the gradients of mu and inv_sigma.  With s_k(e) = dL/dw_k(e), the per-edge dot
// product <G[v], z[u][k]> / deg_v or <dA[v][k], h[u]> / deg_v:
//   dmu[k, j]        =  inv_sigma[k, j]^2 sum_e s_k w_k (e_j - mu[k, j])
//   dinv_sigma[k, j] = -inv_sigma[k, j]   sum_e s_k w_k (e_j - mu[k, j])^2
// Each lane keeps the 4K sums of its own columns; after its chunk a warp adds them in a fixed shuffle tree and writes
// one slot of a workspace; a small kernel then adds the slots in a fixed order (fp64) and applies the inv_sigma factors.
//
// The plan walks are genconv.cu's: one warp per (chunk, tile of 32 16-byte vectors), lane l holding vector l of the
// tile.  The lane that loads a column id also loads that row's c (and 1/deg) and computes its K weights; the other lanes
// get them by shuffle.  Sums are fp32 in CSR or CSC order; long rows come as segments whose partials a fix-up adds in
// segment order.  No atomics: the results are the same bits from run to run.  mu and inv_sigma are read from device
// memory, so a captured CUDA graph sees the optimiser's updates.
#include <math.h>

#include <mutex>

#include "chunk_walk.cuh"

namespace pg {
namespace {

// warps per CTA of the plan walks; their __launch_bounds__ also name one resident CTA, without which ptxas spills a
// few registers in some of the small instances (with it no instance spills, K = 8 included)
constexpr int kMoWarps = 4;
constexpr int kMoMaxK = 8;
constexpr int kMoRedThreads = 256;

struct MoArgs {
  Walk w;
  const float* c;                    // [num_all] pseudo-coordinate of every [inner | halo] row
  const float* rdeg;                 // [N_in] 1 / CSR row length (fp32)
  const float* mu; const float* isg; // [K, 2] each
  const void* x; int64_t ldx;        // the gathered rows (K slices `slice` apart for gather-sum)
  const void* aux; int64_t ldaux;    // backward: the row's own operand (z [K slices] for gather-K, h for gather-sum)
  const float* bias;                 // gather-sum forward: [d] or NULL
  DropArg drop;                      // gather-sum backward
  void* out; int64_t ldo;            // K slices for gather-K, one row for gather-sum
  int64_t slice;
  float* scratch; int64_t ldsc;      // [n_seg][ldsc] fp32 partials: K d values (gather-K) or d (gather-sum)
  float* partial; int64_t n_slots;   // backward: [4K][n_slots]
  int32_t d, nvec;
};

// mu at [0, 2K), inv_sigma at [2K, 4K)
template <int K>
__device__ __forceinline__ void load_mix(const MoArgs& a, float* sm) {
  if (threadIdx.x < 2 * K) sm[threadIdx.x] = a.mu[threadIdx.x];
  else if (threadIdx.x < 4 * K) sm[threadIdx.x] = a.isg[threadIdx.x - 2 * K];
  __syncthreads();
}

template <int K>
__device__ __forceinline__ void mix_weights(const float* sm, float e0, float e1, float (&w)[K]) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float t0 = __fmul_rn(__fsub_rn(e0, sm[2 * k]), sm[2 * K + 2 * k]);
    const float t1 = __fmul_rn(__fsub_rn(e1, sm[2 * k + 1]), sm[2 * K + 2 * k + 1]);
    w[k] = expf(__fmul_rn(-0.5f, __fmaf_rn(t0, t0, __fmul_rn(t1, t1))));
  }
}

// per lane: p[k][j] = sum a (e_j - mu_kj), q[k][j] = sum a (e_j - mu_kj)^2 with a = s_k w_k
template <int K> struct MixGrad {
  float p[K][2], q[K][2];
  __device__ __forceinline__ void init() {
#pragma unroll
    for (int k = 0; k < K; ++k) p[k][0] = p[k][1] = q[k][0] = q[k][1] = 0.f;
  }
  __device__ __forceinline__ void add(const float* sm, int k, float a, float e0, float e1) {
    const float d0 = __fsub_rn(e0, sm[2 * k]), d1 = __fsub_rn(e1, sm[2 * k + 1]);
    const float a0 = __fmul_rn(a, d0), a1 = __fmul_rn(a, d1);
    p[k][0] = __fadd_rn(p[k][0], a0);
    p[k][1] = __fadd_rn(p[k][1], a1);
    q[k][0] = __fmaf_rn(a0, d0, q[k][0]);
    q[k][1] = __fmaf_rn(a1, d1, q[k][1]);
  }
  // the warp's sums (a fixed xor tree) into slot `slot` of the workspace
  __device__ __forceinline__ void flush(const MoArgs& a, int64_t slot, int lane) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      float v[4] = {p[k][0], p[k][1], q[k][0], q[k][1]};
#pragma unroll
      for (int m = 0; m < 4; ++m) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[m] = __fadd_rn(v[m], __shfl_xor_sync(0xffffffffu, v[m], o));
        if (lane == 0) a.partial[static_cast<int64_t>(4 * k + m) * a.n_slots + slot] = v[m];
      }
    }
  }
};

template <typename T>
__device__ __forceinline__ const T* row_ptr(const void* base, int64_t ld, int r, int64_t col) {
  return static_cast<const T*>(base) + static_cast<int64_t>(r) * ld + col;
}

// one whole 16-byte vector: the first `valid` values (one rounding each), zeros after them
template <typename T>
__device__ __forceinline__ void st_whole(void* base, int64_t ld, int r, int64_t col, const float (&f)[Vec<T>::V],
                                         int valid) {
  constexpr int V = Vec<T>::V;
  float o[V];
#pragma unroll
  for (int k = 0; k < V; ++k) o[k] = k < valid ? f[k] : 0.f;
  st_vec<16>(static_cast<T*>(base) + static_cast<int64_t>(r) * ld + col, Vec<T>::P::pack(o));
}

// ---------------------------------------------------------------------------------------------------- gather-K
// forward: A[v][k] = acc[k] (1/deg_v); backward: dz[u][k] = acc[k]
template <typename T, int K, bool BWD>
__device__ __forceinline__ void gk_store(const MoArgs& a, int r, int vi, float (&acc)[K][Vec<T>::V]) {
  constexpr int V = Vec<T>::V;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  const float rd = BWD ? 1.f : a.rdeg[r];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (!BWD) {
#pragma unroll
      for (int q = 0; q < V; ++q) acc[k][q] = __fmul_rn(acc[k][q], rd);
    }
    st_whole<T>(a.out, a.ldo, r, k * a.slice + c0, acc[k], valid);
  }
}

template <typename T, int K, bool BWD>
__device__ __forceinline__ void gk_row(const MoArgs& a, const float* sm, int r, int e0, int n, int slot, int vi,
                                       int lane, MixGrad<K>& mg) {
  using P = typename Vec<T>::P;
  constexpr int V = Vec<T>::V;
  constexpr int F = !BWD ? 4 : K * V > 32 ? 1 : 2;     // gathered rows in flight
  const bool live = vi < a.nvec;
  const int c0 = vi * V;
  const int valid = min(V, a.d - c0);   // the dot products leave out the columns past d (their values are arbitrary)
  const float cr = a.c[r];
  float acc[K][V];
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int q = 0; q < V; ++q) acc[k][q] = 0.f;
  typename P::Raw zr[BWD ? K : 1];
  if (BWD && n > 0 && live) {
#pragma unroll
    for (int k = 0; k < K; ++k) zr[k] = ld_vec<16>(row_ptr<T>(a.aux, a.ldaux, r, k * a.slice + c0));
  }
  for (int b = 0; b < n; b += 32) {
    const bool has = b + lane < n;
    const int32_t ul = has ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const float cl = has ? a.c[ul] : 0.f;
    const float rl = BWD && has ? a.rdeg[ul] : 1.f;
    float wl[K];
    mix_weights<K>(sm, BWD ? cr : cl, BWD ? cl : cr, wl);
    const int cnt = min(32, n - b);
    for (int j = 0; j < cnt; j += F) {
      typename P::Raw raw[F];
#pragma unroll
      for (int i = 0; i < F; ++i) {
        const int u = __shfl_sync(0xffffffffu, ul, min(j + i, cnt - 1));
        if (j + i < cnt && live) raw[i] = ld_vec<16>(row_ptr<T>(a.x, a.ldx, u, c0));
      }
#pragma unroll
      for (int i = 0; i < F; ++i) {
        const int src = min(j + i, cnt - 1);
        float ws[K];
#pragma unroll
        for (int k = 0; k < K; ++k) ws[k] = __shfl_sync(0xffffffffu, wl[k], src);
        const float rs = __shfl_sync(0xffffffffu, rl, src);
        const float ce = __shfl_sync(0xffffffffu, cl, src);
        if (j + i >= cnt || !live) continue;
        float f[V];
        P::unpack(raw[i], f);
#pragma unroll
        for (int k = 0; k < K; ++k) {
          const float s = BWD ? __fmul_rn(ws[k], rs) : ws[k];
#pragma unroll
          for (int q = 0; q < V; ++q) acc[k][q] = __fmaf_rn(s, f[q], acc[k][q]);
          if (BWD) {
            float zf[V];
            P::unpack(zr[k], zf);
            float dot = 0.f;
#pragma unroll
            for (int q = 0; q < V; ++q)
              if (q < valid) dot = __fmaf_rn(f[q], zf[q], dot);
            mg.add(sm, k, __fmul_rn(dot, s), cr, ce);
          }
        }
      }
    }
  }
  if (!live) return;
  if (slot < 0) {
    gk_store<T, K, BWD>(a, r, vi, acc);
    return;
  }
  float* p = a.scratch + static_cast<int64_t>(slot) * a.ldsc;
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int q = 0; q < V; ++q)
      if (c0 + q < a.d) p[k * a.d + c0 + q] = acc[k][q];
}

template <typename T, int K, bool BWD>
__global__ void __launch_bounds__(kMoWarps * 32, 1) monet_gk_kernel(MoArgs a) {
  __shared__ float sm[4 * K];
  load_mix<K>(a, sm);
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kMoWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  MixGrad<K> mg;
  if (BWD) mg.init();
  walk_chunk(a.w, c, [&](int r, int e0, int n, int slot) { gk_row<T, K, BWD>(a, sm, r, e0, n, slot, vi, lane, mg); });
  if (BWD) mg.flush(a, static_cast<int64_t>(c) * gridDim.y + blockIdx.y, lane);
}

template <typename T, int K, bool BWD>
__global__ void __launch_bounds__(kMoWarps * 32, 1) monet_gk_fixup_kernel(MoArgs a) {
  constexpr int V = Vec<T>::V;
  const int li = blockIdx.x * kMoWarps + (threadIdx.x >> 5);
  const int vi = blockIdx.y * 32 + (threadIdx.x & 31);
  if (li >= a.w.n_long || vi >= a.nvec) return;
  const int c0 = vi * V;
  float acc[K][V];
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int q = 0; q < V; ++q) acc[k][q] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.ldsc;
#pragma unroll
    for (int k = 0; k < K; ++k)
#pragma unroll
      for (int q = 0; q < V; ++q)
        if (c0 + q < a.d) acc[k][q] = __fadd_rn(acc[k][q], p[k * a.d + c0 + q]);
  }
  gk_store<T, K, BWD>(a, a.w.long_row[li], vi, acc);
}

// ---------------------------------------------------------------------------------------------------- gather-sum
// forward: out[v] = acc (1/deg_v) + bias; backward: dh[u] = dropout(acc)
template <typename T, bool BWD>
__device__ __forceinline__ void gs_store(const MoArgs& a, int r, int vi, float (&acc)[Vec<T>::V]) {
  constexpr int V = Vec<T>::V;
  const int c0 = vi * V, valid = min(V, a.d - c0);
  if (BWD) {
    if (a.drop.thresh16 != 0u)
      drop_apply<V>(acc, static_cast<uint64_t>(r) * a.nvec + vi, a.drop.thresh16, a.drop.scale, a.drop.seed_lo,
                    drop_seed_hi(a.drop));
  } else {
    const float rd = a.rdeg[r];
#pragma unroll
    for (int q = 0; q < V; ++q) {
      acc[q] = __fmul_rn(acc[q], rd);
      if (a.bias != nullptr && q < valid) acc[q] = __fadd_rn(acc[q], a.bias[c0 + q]);
    }
  }
  st_whole<T>(a.out, a.ldo, r, c0, acc, valid);
}

template <typename T, int K, bool BWD>
__device__ __forceinline__ void gs_row(const MoArgs& a, const float* sm, int r, int e0, int n, int slot, int vi,
                                       int lane, MixGrad<K>& mg) {
  using P = typename Vec<T>::P;
  constexpr int V = Vec<T>::V;
  constexpr int F = K <= 4 ? 2 : 1;  // gathered rows in flight (K vectors each)
  const bool live = vi < a.nvec;
  const int c0 = vi * V;
  const int valid = min(V, a.d - c0);   // the dot products leave out the columns past d (their values are arbitrary)
  const float cr = a.c[r];
  float acc[V], hr[BWD ? V : 1];
#pragma unroll
  for (int q = 0; q < V; ++q) acc[q] = 0.f;
  if (BWD && n > 0 && live) P::unpack(ld_vec<16>(row_ptr<T>(a.aux, a.ldaux, r, c0)), hr);
  for (int b = 0; b < n; b += 32) {
    const bool has = b + lane < n;
    const int32_t ul = has ? (a.w.pidx[e0 + b + lane] & kColMask) : 0;
    const float cl = has ? a.c[ul] : 0.f;
    const float rl = BWD && has ? a.rdeg[ul] : 1.f;
    float wl[K];
    mix_weights<K>(sm, BWD ? cr : cl, BWD ? cl : cr, wl);
    const int cnt = min(32, n - b);
    for (int j = 0; j < cnt; j += F) {
      typename P::Raw raw[F][K];
#pragma unroll
      for (int i = 0; i < F; ++i) {
        const int u = __shfl_sync(0xffffffffu, ul, min(j + i, cnt - 1));
        if (j + i < cnt && live) {
#pragma unroll
          for (int k = 0; k < K; ++k) raw[i][k] = ld_vec<16>(row_ptr<T>(a.x, a.ldx, u, k * a.slice + c0));
        }
      }
#pragma unroll
      for (int i = 0; i < F; ++i) {
        const int src = min(j + i, cnt - 1);
        float ws[K];
#pragma unroll
        for (int k = 0; k < K; ++k) ws[k] = __shfl_sync(0xffffffffu, wl[k], src);
        const float rs = __shfl_sync(0xffffffffu, rl, src);
        const float ce = __shfl_sync(0xffffffffu, cl, src);
        if (j + i >= cnt || !live) continue;
#pragma unroll
        for (int k = 0; k < K; ++k) {
          float f[V];
          P::unpack(raw[i][k], f);
          const float s = BWD ? __fmul_rn(ws[k], rs) : ws[k];
#pragma unroll
          for (int q = 0; q < V; ++q) acc[q] = __fmaf_rn(s, f[q], acc[q]);
          if (BWD) {
            float dot = 0.f;
#pragma unroll
            for (int q = 0; q < V; ++q)
              if (q < valid) dot = __fmaf_rn(f[q], hr[q], dot);
            mg.add(sm, k, __fmul_rn(dot, s), cr, ce);
          }
        }
      }
    }
  }
  if (!live) return;
  if (slot < 0) {
    gs_store<T, BWD>(a, r, vi, acc);
    return;
  }
  float* p = a.scratch + static_cast<int64_t>(slot) * a.ldsc;
#pragma unroll
  for (int q = 0; q < V; ++q)
    if (c0 + q < a.d) p[c0 + q] = acc[q];
}

template <typename T, int K, bool BWD>
__global__ void __launch_bounds__(kMoWarps * 32, 1) monet_gs_kernel(MoArgs a) {
  __shared__ float sm[4 * K];
  load_mix<K>(a, sm);
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kMoWarps + (threadIdx.x >> 5);
  if (c >= a.w.n_chunks) return;
  const int vi = blockIdx.y * 32 + lane;
  MixGrad<K> mg;
  if (BWD) mg.init();
  walk_chunk(a.w, c, [&](int r, int e0, int n, int slot) { gs_row<T, K, BWD>(a, sm, r, e0, n, slot, vi, lane, mg); });
  if (BWD) mg.flush(a, static_cast<int64_t>(c) * gridDim.y + blockIdx.y, lane);
}

template <typename T, bool BWD>
__global__ void __launch_bounds__(kMoWarps * 32, 1) monet_gs_fixup_kernel(MoArgs a) {
  constexpr int V = Vec<T>::V;
  const int li = blockIdx.x * kMoWarps + (threadIdx.x >> 5);
  const int vi = blockIdx.y * 32 + (threadIdx.x & 31);
  if (li >= a.w.n_long || vi >= a.nvec) return;
  const int c0 = vi * V;
  float acc[V];
#pragma unroll
  for (int q = 0; q < V; ++q) acc[q] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + static_cast<int64_t>(sg) * a.ldsc;
#pragma unroll
    for (int q = 0; q < V; ++q)
      if (c0 + q < a.d) acc[q] = __fadd_rn(acc[q], p[c0 + q]);
  }
  gs_store<T, BWD>(a, a.w.long_row[li], vi, acc);
}

// ---------------------------------------------------------------------------------------------------- mixture gradient
// block q = 4k + m adds slots [q][0, n_slots) (each thread in stride order, fp64, then a fixed tree):
// m = 0, 1: dmu[k, m] = inv_sigma^2 sum;  m = 2, 3: dinv_sigma[k, m - 2] = -inv_sigma sum
__global__ void __launch_bounds__(kMoRedThreads) monet_mix_reduce_kernel(const float* partial, int64_t n_slots,
                                                                         const float* isg, float* dmu, float* dinv) {
  __shared__ double red[kMoRedThreads];
  const int q = blockIdx.x, k = q / 4, m = q % 4, j = m & 1;
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < n_slots; i += kMoRedThreads) acc += static_cast<double>(partial[q * n_slots + i]);
  red[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int h = kMoRedThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x != 0) return;
  const double s = static_cast<double>(isg[2 * k + j]);
  if (m < 2) dmu[2 * k + j] = static_cast<float>(s * s * red[0]);
  else dinv[2 * k + j] = static_cast<float>(-s * red[0]);
}

// ---------------------------------------------------------------------------------------------------- dispatch
enum MoKind { kGatherK, kGatherSum };

template <typename T, int K>
void preload_tk() {
  cudaFuncAttributes f;
  cudaFuncGetAttributes(&f, monet_gk_kernel<T, K, false>);
  cudaFuncGetAttributes(&f, monet_gk_kernel<T, K, true>);
  cudaFuncGetAttributes(&f, monet_gk_fixup_kernel<T, K, false>);
  cudaFuncGetAttributes(&f, monet_gk_fixup_kernel<T, K, true>);
  cudaFuncGetAttributes(&f, monet_gs_kernel<T, K, false>);
  cudaFuncGetAttributes(&f, monet_gs_kernel<T, K, true>);
}

template <typename T>
void preload_t() {
  preload_tk<T, 1>(); preload_tk<T, 2>(); preload_tk<T, 3>(); preload_tk<T, 4>();
  preload_tk<T, 5>(); preload_tk<T, 6>(); preload_tk<T, 7>(); preload_tk<T, 8>();
  cudaFuncAttributes f;
  cudaFuncGetAttributes(&f, monet_gs_fixup_kernel<T, false>);
  cudaFuncGetAttributes(&f, monet_gs_fixup_kernel<T, true>);
}

template <typename T, int K, bool BWD>
void launch_tkb(MoKind kind, const MoArgs& a, const pg_csr* g, cudaStream_t st) {
  const int tiles = (a.nvec + 31) / 32;
  const dim3 grid((g->n_chunks + kMoWarps - 1) / kMoWarps, tiles);
  const dim3 grid_fix((g->n_long + kMoWarps - 1) / kMoWarps, tiles);
  const int th = kMoWarps * 32;
  if (kind == kGatherK) {
    if (g->n_chunks > 0) monet_gk_kernel<T, K, BWD><<<grid, th, 0, st>>>(a);
    if (g->n_long > 0) monet_gk_fixup_kernel<T, K, BWD><<<grid_fix, th, 0, st>>>(a);
  } else {
    if (g->n_chunks > 0) monet_gs_kernel<T, K, BWD><<<grid, th, 0, st>>>(a);
    if (g->n_long > 0) monet_gs_fixup_kernel<T, BWD><<<grid_fix, th, 0, st>>>(a);
  }
}

template <typename T, bool BWD>
void launch_tb(int k, MoKind kind, const MoArgs& a, const pg_csr* g, cudaStream_t st) {
  switch (k) {
    case 1: launch_tkb<T, 1, BWD>(kind, a, g, st); break;
    case 2: launch_tkb<T, 2, BWD>(kind, a, g, st); break;
    case 3: launch_tkb<T, 3, BWD>(kind, a, g, st); break;
    case 4: launch_tkb<T, 4, BWD>(kind, a, g, st); break;
    case 5: launch_tkb<T, 5, BWD>(kind, a, g, st); break;
    case 6: launch_tkb<T, 6, BWD>(kind, a, g, st); break;
    case 7: launch_tkb<T, 7, BWD>(kind, a, g, st); break;
    default: launch_tkb<T, 8, BWD>(kind, a, g, st); break;
  }
}

int64_t n_slots_of(const pg_csr* g, int32_t d, int dtype) {
  const int V = 16 / elem_size(dtype);
  const int64_t nvec = (static_cast<int64_t>(d) + V - 1) / V;
  return static_cast<int64_t>(g->n_chunks) * ((nvec + 31) / 32);
}

// One pass.  x: the gathered rows; aux: the row's own operand (backward); out: the written rows.  The K slices are
// those of out (gather-K) or of x (gather-sum); in the backward of gather-K aux has them too.
int run(const char* who, MoKind kind, bool bwd, const pg_csr* g, const void* x, int64_t ldx, const void* aux,
        int64_t ldaux, int64_t slice, int32_t d, int dtype, int32_t k, const float* c, const float* rdeg,
        const float* mu, const float* isg, const float* bias, const pg_drop* drop, void* out, int64_t ldo,
        float* scratch, int64_t ld_scratch, float* partial, int64_t n_partial, float* dmu, float* dinv,
        void* stream) {
  if (int rc = check_plan(g, who)) return rc;
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "%s: unknown dtype %d", who, dtype);
  PG_REQUIRE(k >= 1 && k <= kMoMaxK, "%s: %d mixture kernels (1 to %d are compiled)", who, k, kMoMaxK);
  PG_REQUIRE(d > 0, "%s: bad width d %d", who, d);
  PG_REQUIRE(x && out && c && rdeg && mu && isg && (!bwd || (aux && dmu && dinv)) && (g->n_seg == 0 || scratch),
             "%s: null argument", who);
  const int es = elem_size(dtype);
  const int V = 16 / es;
  const int32_t nvec = (d + V - 1) / V;
  const int64_t full = static_cast<int64_t>(nvec) * V;
  const int64_t sliced = (k - 1) * slice + full;   // the columns an operand with K slices spans
  const bool k_slices = kind == kGatherK;
  PG_REQUIRE(slice >= full && (slice * es) % 16 == 0, "%s: slices %lld apart, shorter than the last 16-byte vector of "
             "d %d or not a 16-byte multiple", who, static_cast<long long>(slice), d);
  PG_REQUIRE(ldx >= (k_slices ? full : sliced) && ldo >= (k_slices ? sliced : full) &&
                 (!bwd || ldaux >= (k_slices ? sliced : full)),
             "%s: a row shorter than its last 16-byte vector (d %d, %d slices %lld apart)", who, d, k,
             static_cast<long long>(slice));
  PG_REQUIRE(vec_ok(x, ldx, es) && vec_ok(out, ldo, es) && (!bwd || vec_ok(aux, ldaux, es)),
             "%s: rows must start on 16-byte boundaries with a 16-byte multiple stride", who);
  PG_REQUIRE(g->n_seg == 0 || ld_scratch >= (k_slices ? k : 1) * static_cast<int64_t>(d), "%s: scratch rows < %d d",
             who, k_slices ? k : 1);
  const int64_t n_slots = n_slots_of(g, d, dtype);
  PG_REQUIRE(!bwd || n_slots == 0 || (partial && n_partial >= 4 * k * n_slots),
             "%s: the mixture workspace needs %lld floats (pg_monet_workspace)", who,
             static_cast<long long>(4 * k * n_slots));
  MoArgs a{make_walk(g), c, rdeg, mu, isg, x, ldx, aux, ldaux, bias, make_drop(drop), out, ldo, slice,
           scratch, ld_scratch, partial, n_slots, d, nvec};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (g->n_rows > 0) {
    if (dtype == PG_F32) {
      if (bwd) launch_tb<float, true>(k, kind, a, g, st);
      else launch_tb<float, false>(k, kind, a, g, st);
    } else {
      if (bwd) launch_tb<__nv_bfloat16, true>(k, kind, a, g, st);
      else launch_tb<__nv_bfloat16, false>(k, kind, a, g, st);
    }
  }
  if (bwd) monet_mix_reduce_kernel<<<4 * k, kMoRedThreads, 0, st>>>(partial, g->n_rows > 0 ? n_slots : 0, isg, dmu, dinv);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

}  // namespace

// CUDA loads kernels lazily, and loading one may wait for the device: see exchange.cu's bns_preload.
static void monet_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_t<float>();
    preload_t<__nv_bfloat16>();
    cudaFuncAttributes f;
    cudaFuncGetAttributes(&f, monet_mix_reduce_kernel);
    cudaGetLastError();
  });
}

}  // namespace pg

extern "C" int pg_monet_preload(void) {
  pg::monet_preload();
  return PG_OK;
}

extern "C" int64_t pg_monet_workspace(const pg_csr* gt, int32_t d, int dtype, int32_t k) {
  if (gt == nullptr || d <= 0 || k < 1) return 0;
  return 4 * static_cast<int64_t>(k) * pg::n_slots_of(gt, d, dtype);
}

extern "C" int pg_monet_agg_k(const pg_csr* g, const void* x, int64_t ldx, int32_t d, int dtype, int32_t k,
                              const float* c, const float* rdeg, const float* mu, const float* inv_sigma, void* out,
                              int64_t ldo, int64_t slice, float* scratch, int64_t ld_scratch, void* stream) {
  pg::monet_preload();
  return pg::run("pg_monet_agg_k", pg::kGatherK, false, g, x, ldx, nullptr, 0, slice, d, dtype, k, c, rdeg, mu,
                 inv_sigma, nullptr, nullptr, out, ldo, scratch, ld_scratch, nullptr, 0, nullptr, nullptr, stream);
}

extern "C" int pg_monet_agg_sum(const pg_csr* g, const void* z, int64_t ldz, int64_t slice, int32_t d, int dtype,
                                int32_t k, const float* c, const float* rdeg, const float* mu, const float* inv_sigma,
                                const float* bias, void* out, int64_t ldo, float* scratch, int64_t ld_scratch,
                                void* stream) {
  pg::monet_preload();
  return pg::run("pg_monet_agg_sum", pg::kGatherSum, false, g, z, ldz, nullptr, 0, slice, d, dtype, k, c, rdeg, mu,
                 inv_sigma, bias, nullptr, out, ldo, scratch, ld_scratch, nullptr, 0, nullptr, nullptr, stream);
}

extern "C" int pg_monet_bwd_k(const pg_csr* gt, const void* grad, int64_t ldg, const void* z, int64_t ldz,
                              int64_t slice, int32_t d, int dtype, int32_t k, const float* c, const float* rdeg,
                              const float* mu, const float* inv_sigma, void* dz, int64_t lddz, float* scratch,
                              int64_t ld_scratch, float* partial, int64_t n_partial, float* dmu, float* dinv_sigma,
                              void* stream) {
  pg::monet_preload();
  return pg::run("pg_monet_bwd_k", pg::kGatherK, true, gt, grad, ldg, z, ldz, slice, d, dtype, k, c, rdeg, mu,
                 inv_sigma, nullptr, nullptr, dz, lddz, scratch, ld_scratch, partial, n_partial, dmu, dinv_sigma,
                 stream);
}

extern "C" int pg_monet_bwd_sum(const pg_csr* gt, const void* da, int64_t ldda, int64_t slice, const void* h,
                                int64_t ldh, int32_t d, int dtype, int32_t k, const float* c, const float* rdeg,
                                const float* mu, const float* inv_sigma, const pg_drop* drop, void* dh, int64_t lddh,
                                float* scratch, int64_t ld_scratch, float* partial, int64_t n_partial, float* dmu,
                                float* dinv_sigma, void* stream) {
  pg::monet_preload();
  return pg::run("pg_monet_bwd_sum", pg::kGatherSum, true, gt, da, ldda, h, ldh, slice, d, dtype, k, c, rdeg, mu,
                 inv_sigma, nullptr, drop, dh, lddh, scratch, ld_scratch, partial, n_partial, dmu, dinv_sigma, stream);
}
