// Graph attention (GAT, DGL GATConv semantics) on sm_90a: attention scores, the edge-softmax aggregate and its two
// backward passes, and the fixed-order column reductions of the attention-vector gradients.  The GATv2 (GATv2Conv)
// aggregate and its two backward passes share the chunk walk, the keep test and the forward fix-up (section GATv2).
//
// One warp owns one (row, head) pair: lane l holds the columns l, l + 32, ... of the head's D columns, so every
// per-head dot product is one warp butterfly (all lanes end with the same bits: IEEE addition commutes).  Edges are
// taken 32 at a time: lane i scores edge i, the batch's maximum / sum are warp reductions, and the gathered rows are
// then accumulated edge by edge in CSR order.  The rows are walked through the chunk table of the pg_csr plan (the
// chunked aggregate's): long rows come as segments that write fp32 partials to `scratch`, and a fix-up merges each
// long row's partials in segment order.  No atomics, no per-edge storage: every result is the same bits run to run.
#include <algorithm>
#include <math.h>
#include <mutex>

#include "common.cuh"

namespace pg {
namespace {

constexpr int kGatWarps = 4;              // warps per CTA
constexpr float kNegSlope = 0.2f;         // LeakyReLU negative slope of GATConv
constexpr int32_t kColMask = 0x7fffffff;  // pidx bit 31 is the "hot row" hint

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}
__device__ __forceinline__ float warp_max(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, o));
  return x;
}

__device__ __forceinline__ float ldf(const float* p) { return __ldg(p); }
__device__ __forceinline__ float ldf(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
template <typename T> __device__ __forceinline__ T from_f(float x);
template <> __device__ __forceinline__ float from_f<float>(float x) { return x; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float x) { return __float2bfloat16_rn(x); }

__device__ __forceinline__ bool is_kept(const uint8_t* keep, int32_t num_in, int32_t u) {
  return keep == nullptr || u < num_in || keep[u - num_in] != 0;
}

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

// ---------------------------------------------------------------------------------------------------- scores
template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32)
gat_scores_kernel(const T* __restrict__ z, int64_t ldz, int32_t n_rows, int32_t n_er, int32_t H, int32_t D,
                  const float* __restrict__ attn_l, const float* __restrict__ attn_r, float* __restrict__ el,
                  float* __restrict__ er) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (r >= n_rows) return;
  const T* zr = z + static_cast<int64_t>(r) * ldz + static_cast<int64_t>(k) * D;
  const bool want_r = r < n_er;
  float sl = 0.f, sr = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < D) {
      const float x = ldf(zr + col);
      sl = fmaf(x, attn_l[k * D + col], sl);
      if (want_r) sr = fmaf(x, attn_r[k * D + col], sr);
    }
  }
  sl = warp_sum(sl);
  if (want_r) sr = warp_sum(sr);
  if (lane == 0) {
    el[static_cast<int64_t>(r) * H + k] = sl;
    if (want_r) er[static_cast<int64_t>(r) * H + k] = sr;
  }
}

// ---------------------------------------------------------------------------------------------------- forward
struct FwdArgs {
  Walk w;
  const void* z; int64_t ldz;
  const float* el; const float* er; const float* bias;
  const uint8_t* keep; int32_t num_in;
  void* out; int64_t ldo;
  float* m; float* s;
  float* scratch;          // [n_seg][H][D + 2] = (m, s, acc[D]) of every long-row segment
  int32_t H, D;
};

template <typename T, int NJ>
__device__ __forceinline__ void fwd_store(const FwdArgs& a, int v, int k, int lane, float m, float s,
                                          const float (&acc)[NJ]) {
  T* o = static_cast<T*>(a.out) + static_cast<int64_t>(v) * a.ldo + static_cast<int64_t>(k) * a.D;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < a.D) {
      const float b = a.bias != nullptr ? a.bias[k * a.D + col] : 0.f;
      o[col] = from_f<T>((s > 0.f ? __fdiv_rn(acc[j], s) : 0.f) + b);
    }
  }
  if (lane == 0) {
    a.m[static_cast<int64_t>(v) * a.H + k] = m;
    a.s[static_cast<int64_t>(v) * a.H + k] = s;
  }
}

// online softmax of one row (or segment) for head k: running max m, running sum s, rescaled accumulator
template <typename T, int NJ>
__device__ __forceinline__ void fwd_row(const FwdArgs& a, const Walk& w, int v, int e0, int n, int slot, int k,
                                        int lane) {
  const T* z = static_cast<const T*>(a.z);
  const int H = a.H, D = a.D;
  const float erv = a.er[static_cast<int64_t>(v) * H + k];
  float m = -INFINITY, s = 0.f, acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  for (int b = 0; b < n; b += 32) {
    const int i = b + lane;
    int u = 0;
    float e = -INFINITY;
    if (i < n) {
      u = w.pidx[e0 + i] & kColMask;
      if (is_kept(a.keep, a.num_in, u)) {
        const float x = a.el[static_cast<int64_t>(u) * H + k] + erv;
        e = x > 0.f ? x : x * kNegSlope;
      }
    }
    const float bm = warp_max(e);
    if (bm == -INFINITY) continue;           // no kept source in this batch
    const float mn = fmaxf(m, bm);
    const float sc = expf(m - mn);
    const float p = e == -INFINITY ? 0.f : expf(e - mn);
    s = fmaf(s, sc, warp_sum(p));
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[j] *= sc;
    const int cnt = min(32, n - b);
    for (int t = 0; t < cnt; ++t) {
      const float pt = __shfl_sync(0xffffffffu, p, t);
      const int ut = __shfl_sync(0xffffffffu, u, t);
      if (pt == 0.f) continue;               // warp-uniform: unkept sources are never read
      const T* zr = z + static_cast<int64_t>(ut) * a.ldz + static_cast<int64_t>(k) * D;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int col = lane + 32 * j;
        if (col < D) acc[j] = fmaf(pt, ldf(zr + col), acc[j]);
      }
    }
    m = mn;
  }
  if (slot < 0) {
    fwd_store<T, NJ>(a, v, k, lane, m, s, acc);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * H + k) * (D + 2);
    if (lane == 0) { p[0] = m; p[1] = s; }
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) p[2 + col] = acc[j];
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gat_fwd_kernel(FwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { fwd_row<T, NJ>(a, a.w, v, e0, n, slot, k, lane); });
}

// merge the (m, s, acc) partials ([n_seg][H][D + 2]) of long row li, head k, in segment order
template <int NJ>
__device__ __forceinline__ void fwd_merge(const Walk& w, const float* scratch, int li, int k, int H, int D, int lane,
                                          float& m, float& s, float (&acc)[NJ]) {
  m = -INFINITY;
  s = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  for (int sg = w.long_seg_ptr[li]; sg < w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = scratch + (static_cast<int64_t>(sg) * H + k) * (D + 2);
    const float mi = p[0];
    if (mi == -INFINITY) continue;
    const float mn = fmaxf(m, mi);
    const float ca = expf(m - mn), cb = expf(mi - mn);
    s = fmaf(s, ca, p[1] * cb);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) acc[j] = fmaf(acc[j], ca, p[2 + col] * cb);
    }
    m = mn;
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gat_fwd_fixup_kernel(FwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  float m, s, acc[NJ];
  fwd_merge<NJ>(a.w, a.scratch, li, k, a.H, a.D, lane, m, s, acc);
  fwd_store<T, NJ>(a, a.w.long_row[li], k, lane, m, s, acc);
}

// ---------------------------------------------------------------------------------------------------- backward
struct BwdArgs {
  Walk w;
  const void* z; int64_t ldz;
  const void* g; int64_t ldg;
  const float* el; const float* er; const float* m; const float* s;
  const float* dv;                        // source pass: D[v, k] = <g[v, k], out[v, k] - bias[k]>
  const float* der;                       // source pass: der of the inner rows
  const float* attn_l; const float* attn_r;
  const uint8_t* keep; int32_t num_in;
  float* der_out; float* dv_out;          // destination pass
  void* dz; int64_t lddz; float* del_out; // source pass
  float* scratch;
  int32_t H, D;
};

// softmax weight and LeakyReLU slope of edge u -> v for head k (0 for an unkept source or an empty softmax)
__device__ __forceinline__ void edge_weight(const BwdArgs& a, int u, int v, int k, float& w, float& slope) {
  const int64_t vk = static_cast<int64_t>(v) * a.H + k;
  const float x = a.el[static_cast<int64_t>(u) * a.H + k] + a.er[vk];
  const float e = x > 0.f ? x : x * kNegSlope;
  const float s = a.s[vk];
  w = s > 0.f ? __fdiv_rn(expf(e - a.m[vk]), s) : 0.f;
  slope = x > 0.f ? 1.f : kNegSlope;
}

// der[v, k] = sum_u a_uv (<g_v, z_u> - D_v) LeakyReLU'(x_uv) over the forward CSR row v, with
// D_v = <g_v, out_v - bias> = sum_u a_uv <g_v, z_u> taken from the same products as the first term (not from the stored
// output: with bf16 storage its rounding would not cancel), in one pass: der = A - D_v B with A = sum a dot slope and
// B = sum a slope.  A segment of a long row writes its partial (A, B, D) to scratch.
template <typename T, int NJ>
__device__ __forceinline__ void dst_row(const BwdArgs& a, const Walk& w, int v, int e0, int n, int slot, int k,
                                        int lane) {
  const T* z = static_cast<const T*>(a.z);
  const int D = a.D;
  const T* gv = static_cast<const T*>(a.g) + static_cast<int64_t>(v) * a.ldg + static_cast<int64_t>(k) * D;
  float gr[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    gr[j] = col < D ? ldf(gv + col) : 0.f;
  }
  float sa = 0.f, sb = 0.f, sd = 0.f;
  for (int b = 0; b < n; b += 32) {
    const int i = b + lane;
    int u = 0;
    float wt = 0.f, sl = 0.f;
    if (i < n) {
      u = w.pidx[e0 + i] & kColMask;
      if (is_kept(a.keep, a.num_in, u)) edge_weight(a, u, v, k, wt, sl);
    }
    const int cnt = min(32, n - b);
    for (int t = 0; t < cnt; ++t) {
      const float at = __shfl_sync(0xffffffffu, wt, t);
      const int ut = __shfl_sync(0xffffffffu, u, t);
      const float st = __shfl_sync(0xffffffffu, sl, t);
      if (at == 0.f) continue;
      const T* zr = z + static_cast<int64_t>(ut) * a.ldz + static_cast<int64_t>(k) * D;
      float dp = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int col = lane + 32 * j;
        if (col < D) dp = fmaf(gr[j], ldf(zr + col), dp);
      }
      const float ad = at * warp_sum(dp);
      sd += ad;
      sa = fmaf(ad, st, sa);
      sb = fmaf(at, st, sb);
    }
  }
  if (lane == 0) {
    const int64_t vk = static_cast<int64_t>(v) * a.H + k;
    if (slot < 0) {
      a.der_out[vk] = fmaf(-sd, sb, sa);
      a.dv_out[vk] = sd;
    } else {
      float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + k) * 3;
      p[0] = sa; p[1] = sb; p[2] = sd;
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gat_bwd_dst_kernel(BwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { dst_row<T, NJ>(a, a.w, v, e0, n, slot, k, lane); });
}

__global__ void gat_bwd_dst_fixup_kernel(BwdArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.w.n_long * a.H) return;
  const int li = i / a.H, k = i % a.H;
  float sa = 0.f, sb = 0.f, sd = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + (static_cast<int64_t>(sg) * a.H + k) * 3;
    sa += p[0]; sb += p[1]; sd += p[2];
  }
  const int64_t vk = static_cast<int64_t>(a.w.long_row[li]) * a.H + k;
  a.der_out[vk] = fmaf(-sd, sb, sa);
  a.dv_out[vk] = sd;
}

template <typename T, int NJ>
__device__ __forceinline__ void src_store(const BwdArgs& a, int u, int k, int lane, float del, const float (&acc)[NJ]) {
  const int D = a.D;
  const float der = u < a.num_in ? a.der[static_cast<int64_t>(u) * a.H + k] : 0.f;
  T* o = static_cast<T*>(a.dz) + static_cast<int64_t>(u) * a.lddz + static_cast<int64_t>(k) * D;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < D) o[col] = from_f<T>(fmaf(der, a.attn_r[k * D + col], fmaf(del, a.attn_l[k * D + col], acc[j])));
  }
  if (lane == 0) a.del_out[static_cast<int64_t>(u) * a.H + k] = del;
}

// dz[u, k] = sum_v a_uv g_v (+ del attn_l + der attn_r), del[u, k] = sum_v a_uv (<g_v, z_u> - D_v) LeakyReLU'(x_uv)
// over the CSC row u (the destinations v of source u)
template <typename T, int NJ>
__device__ __forceinline__ void src_row(const BwdArgs& a, const Walk& w, int u, int e0, int n, int slot, int k,
                                        int lane) {
  const int D = a.D;
  float zr[NJ], acc[NJ], del = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) { zr[j] = 0.f; acc[j] = 0.f; }
  if (is_kept(a.keep, a.num_in, u)) {
    const T* zu = static_cast<const T*>(a.z) + static_cast<int64_t>(u) * a.ldz + static_cast<int64_t>(k) * D;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) zr[j] = ldf(zu + col);
    }
    for (int b = 0; b < n; b += 32) {
      const int i = b + lane;
      int v = 0;
      float wt = 0.f, sl = 0.f, dv = 0.f;
      if (i < n) {
        v = w.pidx[e0 + i] & kColMask;
        edge_weight(a, u, v, k, wt, sl);
        dv = a.dv[static_cast<int64_t>(v) * a.H + k];
      }
      const int cnt = min(32, n - b);
      for (int t = 0; t < cnt; ++t) {
        const float at = __shfl_sync(0xffffffffu, wt, t);
        const int vt = __shfl_sync(0xffffffffu, v, t);
        const float st = __shfl_sync(0xffffffffu, sl, t);
        const float dt = __shfl_sync(0xffffffffu, dv, t);
        if (at == 0.f) continue;
        const T* gv = static_cast<const T*>(a.g) + static_cast<int64_t>(vt) * a.ldg + static_cast<int64_t>(k) * D;
        float dp = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const int col = lane + 32 * j;
          if (col < D) {
            const float gj = ldf(gv + col);
            dp = fmaf(gj, zr[j], dp);
            acc[j] = fmaf(at, gj, acc[j]);
          }
        }
        del = fmaf(at * (warp_sum(dp) - dt), st, del);
      }
    }
  }
  if (slot < 0) {
    src_store<T, NJ>(a, u, k, lane, del, acc);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + k) * (D + 1);
    if (lane == 0) p[0] = del;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) p[1 + col] = acc[j];
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gat_bwd_src_kernel(BwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { src_row<T, NJ>(a, a.w, u, e0, n, slot, k, lane); });
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gat_bwd_src_fixup_kernel(BwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  const int D = a.D;
  float del = 0.f, acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + (static_cast<int64_t>(sg) * a.H + k) * (D + 1);
    del += p[0];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) acc[j] += p[1 + col];
    }
  }
  src_store<T, NJ>(a, a.w.long_row[li], k, lane, del, acc);
}

// ---------------------------------------------------------------------------------------------------- column sums
// stage 1: CTA b sums rows [b * R, (b + 1) * R) of 32 columns, 8 row lanes, merged in row-lane order
template <typename T>
__global__ void __launch_bounds__(256) gat_colsum_kernel(const T* __restrict__ x, int64_t ldx, int32_t n_rows,
                                                         int32_t H, int32_t D, const float* __restrict__ coef,
                                                         int32_t rows_per, float* __restrict__ partial) {
  __shared__ float red[8][33];
  const int n_cols = H * D;
  const int col = blockIdx.y * 32 + threadIdx.x;
  const int r0 = blockIdx.x * rows_per, r1 = min(n_rows, r0 + rows_per);
  float acc = 0.f;
  if (col < n_cols) {
    const int k = col / D;
    for (int r = r0 + threadIdx.y; r < r1; r += 8) {
      const float v = ldf(x + static_cast<int64_t>(r) * ldx + col);
      acc = coef != nullptr ? fmaf(coef[static_cast<int64_t>(r) * H + k], v, acc) : acc + v;
    }
  }
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && col < n_cols) {
    float s = red[0][threadIdx.x];
#pragma unroll
    for (int i = 1; i < 8; ++i) s += red[i][threadIdx.x];
    partial[static_cast<int64_t>(blockIdx.x) * n_cols + col] = s;
  }
}

__global__ void gat_colsum_final_kernel(const float* __restrict__ partial, int32_t n_blocks, int32_t n_cols,
                                        float* __restrict__ out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= n_cols) return;
  float s = 0.f;
  for (int b = 0; b < n_blocks; ++b) s += partial[static_cast<int64_t>(b) * n_cols + col];
  out[col] = s;
}

int colsum_blocks(int32_t n_rows) {
  return static_cast<int>(std::max<int64_t>(1, std::min<int64_t>((n_rows + 255) / 256, 2 * sm_count())));
}

// ---------------------------------------------------------------------------------------------------- GATv2
// GATv2Conv: e_uv = <attn[k], LeakyReLU(zs[u, k] + zd[v, k])>.  The score is no longer two per-node scalars, so every
// edge needs a D-wide sum in the forward and in both backward passes.  A warp still owns one (row, head) pair with lane
// l holding the columns l, l + 32, ..., but it takes E edges at a time: E row gathers in flight, and the per-lane
// partial sums of all of them reduced together by warp_sum_n (2E values in 4E - 1 + log2(32 / 2E) shuffles instead
// of 10E).  Every sum is taken over warp_sum's tree (offsets 16, 8, 4, 2, 1; IEEE addition commutes), so a score or a
// dot has the same bits in every pass and in every slot of a batch: the backward recomputes a_uv exactly.
// edges in flight per warp: the most that every pass compiles with at NJ columns per lane without local-memory spills
template <int NJ> __host__ __device__ constexpr int v2_edges() { return NJ <= 2 ? 2 : NJ <= 4 ? 4 : NJ <= 8 ? 2 : 1; }

// x[i] <- the warp sum of x[i], on every lane (N a power of two <= 32)
template <int N>
__device__ __forceinline__ void warp_sum_n(float (&x)[N], int lane) {
  // step o keeps half of the live values: the half selected by lane bit o, plus the partner's copy of the same half
#pragma unroll
  for (int n = N, o = 16; n > 1; n >>= 1, o >>= 1) {
    const bool hi = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      const float send = hi ? x[i] : x[i + n / 2];
      const float own = hi ? x[i + n / 2] : x[i];
      x[i] = own + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
#pragma unroll
  for (int o = 16 / N; o > 0; o >>= 1) x[0] += __shfl_xor_sync(0xffffffffu, x[0], o);
  // value t now sits on the lanes whose bit o of every halving step is bit n / 2 of t
  const float r = x[0];
#pragma unroll
  for (int t = 0; t < N; ++t) {
    int src = 0;
#pragma unroll
    for (int n = N, o = 16; n > 1; n >>= 1, o >>= 1) src |= (t & (n / 2)) ? o : 0;
    x[t] = __shfl_sync(0xffffffffu, r, src);
  }
}

__device__ __forceinline__ float lrelu(float x) { return x > 0.f ? x : x * kNegSlope; }

// the D columns of head k of one row: lane l takes l, l + 32, ... (0 past D)
template <typename T, int NJ>
__device__ __forceinline__ void load_head(const T* row, int D, int lane, float (&r)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    r[j] = col < D ? ldf(row + col) : 0.f;
  }
}
template <int NJ>
__device__ __forceinline__ void load_head_f32(const float* row, int D, int lane, float (&r)[NJ]) {
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    r[j] = col < D ? row[col] : 0.f;
  }
}

// the per-lane partial of <attn, LeakyReLU(zs_u + zd_v)> (zs_u + zd_v in that order in every pass)
template <int NJ>
__device__ __forceinline__ float score_part(const float (&zs)[NJ], const float (&zd)[NJ], const float (&at)[NJ]) {
  float p = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) p = fmaf(at[j], lrelu(zs[j] + zd[j]), p);
  return p;
}

// the per-lane partial of <g_v, zs_u>
template <int NJ>
__device__ __forceinline__ float dot_part(const float (&g)[NJ], const float (&zs)[NJ]) {
  float p = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) p = fmaf(g[j], zs[j], p);
  return p;
}

struct V2Args {
  Walk w;
  const void* zs; int64_t ldzs;           // [num_all, H * D]
  const void* zd; int64_t ldzd;           // [N_in, H * D]
  const void* g; int64_t ldg;             // backward: dL/d out [N_in, H * D]
  const float* attn;                      // [H * D]
  const float* m; const float* s;         // [N_in, H]
  const float* dv;                        // source pass: D_v [N_in, H]
  const uint8_t* keep; int32_t num_in;
  void* out; int64_t ldo;                 // forward: out; destination pass: d zd; source pass: d zs
  float* m_out; float* s_out;             // forward
  float* dv_out; float* pattn; int64_t ldp;  // destination pass
  float* scratch;
  int32_t H, D;
};

// the forward's (m, s, acc) partials and their fix-up are GAT's (FwdArgs, gat_fwd_fixup_kernel, no bias)
__host__ __device__ FwdArgs v2_fwd_args(const V2Args& a) {
  return FwdArgs{a.w, a.zs, a.ldzs, nullptr, nullptr, nullptr, a.keep, a.num_in, a.out, a.ldo, a.m_out, a.s_out,
                 a.scratch, a.H, a.D};
}

// online softmax of one row (or segment) for head k, E in-edges at a time
template <typename T, int NJ>
__device__ __forceinline__ void v2_fwd_row(const V2Args& a, const FwdArgs& f, int v, int e0, int n, int slot, int k,
                                           int lane) {
  constexpr int E = v2_edges<NJ>();
  const int D = a.D;
  const T* zs = static_cast<const T*>(a.zs) + static_cast<int64_t>(k) * D;
  float zdv[NJ], at[NJ], acc[NJ];
  load_head<T, NJ>(static_cast<const T*>(a.zd) + static_cast<int64_t>(v) * a.ldzd + static_cast<int64_t>(k) * D, D,
                   lane, zdv);
  load_head_f32<NJ>(a.attn + k * D, D, lane, at);
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  float m = -INFINITY, s = 0.f;
  for (int b = 0; b < n; b += E) {
    int u[E];
    float x[E][NJ], p[E];
#pragma unroll
    for (int t = 0; t < E; ++t) {
      u[t] = -1;
      if (b + t < n) {
        const int ut = a.w.pidx[e0 + b + t] & kColMask;
        if (is_kept(a.keep, a.num_in, ut)) u[t] = ut;
      }
    }
#pragma unroll
    for (int t = 0; t < E; ++t) {
      if (u[t] >= 0) {
        load_head<T, NJ>(zs + static_cast<int64_t>(u[t]) * a.ldzs, D, lane, x[t]);
      } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) x[t][j] = 0.f;
      }
    }
#pragma unroll
    for (int t = 0; t < E; ++t) p[t] = score_part<NJ>(x[t], zdv, at);
    warp_sum_n<E>(p, lane);
    float bm = -INFINITY;
#pragma unroll
    for (int t = 0; t < E; ++t) if (u[t] >= 0) bm = fmaxf(bm, p[t]);
    if (bm == -INFINITY) continue;            // warp-uniform: no kept source in this batch
    const float mn = fmaxf(m, bm);
    const float sc = expf(m - mn);
    s *= sc;
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[j] *= sc;
#pragma unroll
    for (int t = 0; t < E; ++t) {
      if (u[t] < 0) continue;
      const float pt = expf(p[t] - mn);
      s += pt;
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[j] = fmaf(pt, x[t][j], acc[j]);
    }
    m = mn;
  }
  if (slot < 0) {
    fwd_store<T, NJ>(f, v, k, lane, m, s, acc);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + k) * (D + 2);
    if (lane == 0) { p[0] = m; p[1] = s; }
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) p[2 + col] = acc[j];
    }
  }
}

template <typename T, int NJ>
// no __launch_bounds__: with it ptxas spills the bf16 NJ = 4 instance (launched with kGatWarps * 32 threads as well)
__global__ void gatv2_fwd_kernel(V2Args a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  const FwdArgs f = v2_fwd_args(a);
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { v2_fwd_row<T, NJ>(a, f, v, e0, n, slot, k, lane); });
}

// destination pass results of row v, head k from the sums over its in-edges (the weights w = a_uv, ad = a_uv dot_uv):
//   sd = D_v = sum ad,  A = sum ad σ',  B = sum w σ',  C = sum ad LeakyReLU(t),  Q = sum w LeakyReLU(t)  (per column)
//   d zd = attn (A - D_v B),  d attn contribution = C - D_v Q,  since de_uv = a_uv dot_uv - a_uv D_v
template <typename T, int NJ>
__device__ __forceinline__ void v2_dst_store(const V2Args& a, int v, int k, int lane, float sd, const float (&A)[NJ],
                                             const float (&B)[NJ], const float (&C)[NJ], const float (&Q)[NJ]) {
  const int D = a.D;
  T* o = static_cast<T*>(a.out) + static_cast<int64_t>(v) * a.ldo + static_cast<int64_t>(k) * D;
  float* pa = a.pattn + static_cast<int64_t>(v) * a.ldp + static_cast<int64_t>(k) * D;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < D) {
      o[col] = from_f<T>(a.attn[k * D + col] * fmaf(-sd, B[j], A[j]));
      pa[col] = fmaf(-sd, Q[j], C[j]);
    }
  }
  if (lane == 0) a.dv_out[static_cast<int64_t>(v) * a.H + k] = sd;
}

// scratch of a long-row segment: [H][4 D + 1] = (sd, A[D], B[D], C[D], Q[D])
template <typename T, int NJ>
__device__ __forceinline__ void v2_dst_row(const V2Args& a, int v, int e0, int n, int slot, int k, int lane) {
  constexpr int E = v2_edges<NJ>();
  const int D = a.D;
  const T* zs = static_cast<const T*>(a.zs) + static_cast<int64_t>(k) * D;
  float zdv[NJ], at[NJ], gv[NJ], A[NJ], B[NJ], C[NJ], Q[NJ];
  load_head<T, NJ>(static_cast<const T*>(a.zd) + static_cast<int64_t>(v) * a.ldzd + static_cast<int64_t>(k) * D, D,
                   lane, zdv);
  load_head<T, NJ>(static_cast<const T*>(a.g) + static_cast<int64_t>(v) * a.ldg + static_cast<int64_t>(k) * D, D,
                   lane, gv);
  load_head_f32<NJ>(a.attn + k * D, D, lane, at);
#pragma unroll
  for (int j = 0; j < NJ; ++j) { A[j] = 0.f; B[j] = 0.f; C[j] = 0.f; Q[j] = 0.f; }
  float sd = 0.f;
  const int64_t vk = static_cast<int64_t>(v) * a.H + k;
  const float mv = a.m[vk], sv = a.s[vk];
  for (int b = 0; sv > 0.f && b < n; b += E) {
    int u[E];
    float x[E][NJ], p[2 * E];
#pragma unroll
    for (int t = 0; t < E; ++t) {
      u[t] = -1;
      if (b + t < n) {
        const int ut = a.w.pidx[e0 + b + t] & kColMask;
        if (is_kept(a.keep, a.num_in, ut)) u[t] = ut;
      }
    }
#pragma unroll
    for (int t = 0; t < E; ++t) {
      if (u[t] >= 0) {
        load_head<T, NJ>(zs + static_cast<int64_t>(u[t]) * a.ldzs, D, lane, x[t]);
      } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) x[t][j] = 0.f;
      }
    }
#pragma unroll
    for (int t = 0; t < E; ++t) {
      p[t] = score_part<NJ>(x[t], zdv, at);
      p[E + t] = dot_part<NJ>(gv, x[t]);
    }
    warp_sum_n<2 * E>(p, lane);
#pragma unroll
    for (int t = 0; t < E; ++t) {
      if (u[t] < 0) continue;
      const float w = __fdiv_rn(expf(p[t] - mv), sv);
      const float ad = w * p[E + t];
      sd += ad;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float tt = x[t][j] + zdv[j];
        const float sl = tt > 0.f ? 1.f : kNegSlope, lr = lrelu(tt);
        A[j] = fmaf(ad, sl, A[j]);
        B[j] = fmaf(w, sl, B[j]);
        C[j] = fmaf(ad, lr, C[j]);
        Q[j] = fmaf(w, lr, Q[j]);
      }
    }
  }
  if (slot < 0) {
    v2_dst_store<T, NJ>(a, v, k, lane, sd, A, B, C, Q);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + k) * (4 * D + 1);
    if (lane == 0) p[0] = sd;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) { p[1 + col] = A[j]; p[1 + D + col] = B[j]; p[1 + 2 * D + col] = C[j]; p[1 + 3 * D + col] = Q[j]; }
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gatv2_bwd_dst_kernel(V2Args a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { v2_dst_row<T, NJ>(a, v, e0, n, slot, k, lane); });
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gatv2_bwd_dst_fixup_kernel(V2Args a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  const int D = a.D;
  float sd = 0.f, A[NJ], B[NJ], C[NJ], Q[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) { A[j] = 0.f; B[j] = 0.f; C[j] = 0.f; Q[j] = 0.f; }
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + (static_cast<int64_t>(sg) * a.H + k) * (4 * D + 1);
    sd += p[0];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) { A[j] += p[1 + col]; B[j] += p[1 + D + col]; C[j] += p[1 + 2 * D + col]; Q[j] += p[1 + 3 * D + col]; }
    }
  }
  v2_dst_store<T, NJ>(a, a.w.long_row[li], k, lane, sd, A, B, C, Q);
}

template <typename T, int NJ>
__device__ __forceinline__ void v2_src_store(const V2Args& a, int u, int k, int lane, const float (&acc)[NJ]) {
  T* o = static_cast<T*>(a.out) + static_cast<int64_t>(u) * a.ldo + static_cast<int64_t>(k) * a.D;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < a.D) o[col] = from_f<T>(acc[j]);
  }
}

// d zs[u, k] = sum_v a_uv g_v + de_uv attn ⊙ σ'(t_uv) over the CSC row u (the destinations v of source u), with
// de_uv = a_uv (<g_v, zs_u> - D_v); an unkept source gets 0.  Scratch of a long-row segment: [H][D].
template <typename T, int NJ>
__device__ __forceinline__ void v2_src_row(const V2Args& a, int u, int e0, int n, int slot, int k, int lane) {
  constexpr int E = v2_edges<NJ>();
  const int D = a.D;
  float acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  if (is_kept(a.keep, a.num_in, u)) {
    const T* zd = static_cast<const T*>(a.zd) + static_cast<int64_t>(k) * D;
    const T* g = static_cast<const T*>(a.g) + static_cast<int64_t>(k) * D;
    float zsu[NJ], at[NJ];
    load_head<T, NJ>(static_cast<const T*>(a.zs) + static_cast<int64_t>(u) * a.ldzs + static_cast<int64_t>(k) * D, D,
                     lane, zsu);
    load_head_f32<NJ>(a.attn + k * D, D, lane, at);
    for (int b = 0; b < n; b += E) {
      int v[E];
      float y[E][NJ], gg[E][NJ], p[2 * E], mv[E], sv[E], dv[E];
#pragma unroll
      for (int t = 0; t < E; ++t) v[t] = b + t < n ? a.w.pidx[e0 + b + t] & kColMask : -1;
#pragma unroll
      for (int t = 0; t < E; ++t) {
        if (v[t] >= 0) {
          load_head<T, NJ>(zd + static_cast<int64_t>(v[t]) * a.ldzd, D, lane, y[t]);
          load_head<T, NJ>(g + static_cast<int64_t>(v[t]) * a.ldg, D, lane, gg[t]);
          const int64_t vk = static_cast<int64_t>(v[t]) * a.H + k;
          mv[t] = a.m[vk]; sv[t] = a.s[vk]; dv[t] = a.dv[vk];
        } else {
#pragma unroll
          for (int j = 0; j < NJ; ++j) { y[t][j] = 0.f; gg[t][j] = 0.f; }
          mv[t] = 0.f; sv[t] = 0.f; dv[t] = 0.f;
        }
      }
#pragma unroll
      for (int t = 0; t < E; ++t) {
        p[t] = score_part<NJ>(zsu, y[t], at);
        p[E + t] = dot_part<NJ>(gg[t], zsu);
      }
      warp_sum_n<2 * E>(p, lane);
#pragma unroll
      for (int t = 0; t < E; ++t) {
        if (!(sv[t] > 0.f)) continue;         // also the slots past the row's end
        const float w = __fdiv_rn(expf(p[t] - mv[t]), sv[t]);
        const float de = w * (p[E + t] - dv[t]);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          const float tt = zsu[j] + y[t][j];
          acc[j] = fmaf(w, gg[t][j], acc[j]);
          acc[j] = fmaf(tt > 0.f ? de : de * kNegSlope, at[j], acc[j]);
        }
      }
    }
  }
  if (slot < 0) {
    v2_src_store<T, NJ>(a, u, k, lane, acc);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + k) * D;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) p[col] = acc[j];
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gatv2_bwd_src_kernel(V2Args a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { v2_src_row<T, NJ>(a, u, e0, n, slot, k, lane); });
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) gatv2_bwd_src_fixup_kernel(V2Args a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  const int D = a.D;
  float acc[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + (static_cast<int64_t>(sg) * a.H + k) * D;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) acc[j] += p[col];
    }
  }
  v2_src_store<T, NJ>(a, a.w.long_row[li], k, lane, acc);
}

// ---------------------------------------------------------------------------------------------------- transformer
// Graph transformer (PyG TransformerConv, concat=True, beta=False, root_weight=True): per head k,
//   e_uv = scale <q[v, k], k[u, k]>,  a_uv = softmax over u of e_uv,  out[v, k] = sum_u a_uv v[u, k] + skip[v, k].
// The warp layout and the E-edges-at-a-time batches are GATv2's.  Every score is dot_part(q_v, k_u) summed over
// warp_sum's tree (through warp_sum_n) and then multiplied by scale with __fmul_rn, so no pass can contract it into a
// later subtraction: e_uv has the same bits in all three passes and the backward recomputes a_uv exactly from (m, s).
// edges in flight per warp: the most that every pass compiles with at NJ columns per lane without local-memory spills
template <int NJ> __host__ __device__ constexpr int tc_edges() { return NJ <= 4 ? 4 : 2; }

struct TcArgs {
  Walk w;
  const void* q; int64_t ldq;             // [N_in, H * D]
  const void* k; int64_t ldk;             // [num_all, H * D]
  const void* v; int64_t ldv;             // [num_all, H * D]
  const void* skip; int64_t ldskip;       // forward: [N_in, H * D]
  const void* g; int64_t ldg;             // backward: dL/d out [N_in, H * D]
  const float* m; const float* s;         // backward: softmax statistics [N_in, H]
  const float* delta;                     // source pass: delta_v [N_in, H]
  const uint8_t* keep; int32_t num_in;
  void* out; int64_t ldo;                 // forward: out; destination pass: dq; source pass: dk
  void* out2; int64_t ldo2;               // destination pass: the copy of g; source pass: dv
  float* m_out; float* s_out;             // forward
  float* delta_out;                       // destination pass
  float* scratch;
  float scale;
  int32_t H, D;
};

template <typename T>
__device__ __forceinline__ const T* head_row(const void* base, int64_t ld, int r, int k, int D) {
  return static_cast<const T*>(base) + static_cast<int64_t>(r) * ld + static_cast<int64_t>(k) * D;
}
template <typename T>
__device__ __forceinline__ T* head_row_out(void* base, int64_t ld, int r, int k, int D) {
  return static_cast<T*>(base) + static_cast<int64_t>(r) * ld + static_cast<int64_t>(k) * D;
}

// the batch of E in-edges of row v from entry e0 + b: kept sources in u (else -1), their k rows in x and v rows in y
template <typename T, int NJ, int E>
__device__ __forceinline__ void tc_gather(const TcArgs& a, int e0, int b, int n, int kh, int lane, int (&u)[E],
                                          float (&x)[E][NJ], float (&y)[E][NJ]) {
#pragma unroll
  for (int t = 0; t < E; ++t) {
    u[t] = -1;
    if (b + t < n) {
      const int ut = a.w.pidx[e0 + b + t] & kColMask;
      if (is_kept(a.keep, a.num_in, ut)) u[t] = ut;
    }
  }
#pragma unroll
  for (int t = 0; t < E; ++t) {
    if (u[t] >= 0) {
      load_head<T, NJ>(head_row<T>(a.k, a.ldk, u[t], kh, a.D), a.D, lane, x[t]);
      load_head<T, NJ>(head_row<T>(a.v, a.ldv, u[t], kh, a.D), a.D, lane, y[t]);
    } else {
#pragma unroll
      for (int j = 0; j < NJ; ++j) { x[t][j] = 0.f; y[t][j] = 0.f; }
    }
  }
}

template <typename T, int NJ>
__device__ __forceinline__ void tc_fwd_store(const TcArgs& a, int v, int kh, int lane, float m, float s,
                                             const float (&acc)[NJ]) {
  const T* sk = head_row<T>(a.skip, a.ldskip, v, kh, a.D);
  T* o = head_row_out<T>(a.out, a.ldo, v, kh, a.D);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < a.D) o[col] = from_f<T>((s > 0.f ? __fdiv_rn(acc[j], s) : 0.f) + ldf(sk + col));
  }
  if (lane == 0) {
    a.m_out[static_cast<int64_t>(v) * a.H + kh] = m;
    a.s_out[static_cast<int64_t>(v) * a.H + kh] = s;
  }
}

// online softmax of one row (or segment) for head kh, E in-edges at a time; a segment writes GAT's (m, s, acc) partial
template <typename T, int NJ>
__device__ __forceinline__ void tc_fwd_row(const TcArgs& a, int v, int e0, int n, int slot, int kh, int lane) {
  constexpr int E = tc_edges<NJ>();
  const int D = a.D;
  float qv[NJ], acc[NJ];
  load_head<T, NJ>(head_row<T>(a.q, a.ldq, v, kh, D), D, lane, qv);
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
  float m = -INFINITY, s = 0.f;
  for (int b = 0; b < n; b += E) {
    int u[E];
    float x[E][NJ], y[E][NJ], p[E];
    tc_gather<T, NJ, E>(a, e0, b, n, kh, lane, u, x, y);
#pragma unroll
    for (int t = 0; t < E; ++t) p[t] = dot_part<NJ>(qv, x[t]);
    warp_sum_n<E>(p, lane);
    float bm = -INFINITY;
#pragma unroll
    for (int t = 0; t < E; ++t) {
      p[t] = __fmul_rn(p[t], a.scale);
      if (u[t] >= 0) bm = fmaxf(bm, p[t]);
    }
    if (bm == -INFINITY) continue;            // warp-uniform: no kept source in this batch
    const float mn = fmaxf(m, bm);
    const float sc = expf(m - mn);
    s *= sc;
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc[j] *= sc;
#pragma unroll
    for (int t = 0; t < E; ++t) {
      if (u[t] < 0) continue;
      const float pt = expf(p[t] - mn);
      s += pt;
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[j] = fmaf(pt, y[t][j], acc[j]);
    }
    m = mn;
  }
  if (slot < 0) {
    tc_fwd_store<T, NJ>(a, v, kh, lane, m, s, acc);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + kh) * (D + 2);
    if (lane == 0) { p[0] = m; p[1] = s; }
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) p[2 + col] = acc[j];
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) tconv_fwd_kernel(TcArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { tc_fwd_row<T, NJ>(a, v, e0, n, slot, k, lane); });
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) tconv_fwd_fixup_kernel(TcArgs a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  float m, s, acc[NJ];
  fwd_merge<NJ>(a.w, a.scratch, li, k, a.H, a.D, lane, m, s, acc);
  tc_fwd_store<T, NJ>(a, a.w.long_row[li], k, lane, m, s, acc);
}

// destination pass of row v, head kh, from the sums over its in-edges (w = a_uv, gd = <g_v, v_u>, ad = w gd):
//   delta = sum ad,  A = sum ad k_u,  B = sum w k_u  (per column),  dq = scale (A - delta B),
// since dq_v = scale sum_u a_uv (gd_uv - delta_v) k_u.  The copy of g_v goes next to dq (the input-gradient GEMM reads
// [dq | g] as one operand).
template <typename T, int NJ>
__device__ __forceinline__ void tc_dst_store(const TcArgs& a, int v, int kh, int lane, float sd, const float (&A)[NJ],
                                             const float (&B)[NJ], const float (&gv)[NJ]) {
  T* dq = head_row_out<T>(a.out, a.ldo, v, kh, a.D);
  T* gc = head_row_out<T>(a.out2, a.ldo2, v, kh, a.D);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < a.D) {
      dq[col] = from_f<T>(a.scale * fmaf(-sd, B[j], A[j]));
      gc[col] = from_f<T>(gv[j]);
    }
  }
  if (lane == 0) a.delta_out[static_cast<int64_t>(v) * a.H + kh] = sd;
}

// scratch of a long-row segment: [H][2 D + 1] = (delta, A[D], B[D])
template <typename T, int NJ>
__device__ __forceinline__ void tc_dst_row(const TcArgs& a, int v, int e0, int n, int slot, int kh, int lane) {
  constexpr int E = tc_edges<NJ>();
  const int D = a.D;
  float qv[NJ], gv[NJ], A[NJ], B[NJ];
  load_head<T, NJ>(head_row<T>(a.q, a.ldq, v, kh, D), D, lane, qv);
  load_head<T, NJ>(head_row<T>(a.g, a.ldg, v, kh, D), D, lane, gv);
#pragma unroll
  for (int j = 0; j < NJ; ++j) { A[j] = 0.f; B[j] = 0.f; }
  float sd = 0.f;
  const int64_t vk = static_cast<int64_t>(v) * a.H + kh;
  const float mv = a.m[vk], sv = a.s[vk];
  for (int b = 0; sv > 0.f && b < n; b += E) {
    int u[E];
    float x[E][NJ], y[E][NJ], p[2 * E];
    tc_gather<T, NJ, E>(a, e0, b, n, kh, lane, u, x, y);
#pragma unroll
    for (int t = 0; t < E; ++t) {
      p[t] = dot_part<NJ>(qv, x[t]);
      p[E + t] = dot_part<NJ>(gv, y[t]);
    }
    warp_sum_n<2 * E>(p, lane);
#pragma unroll
    for (int t = 0; t < E; ++t) {
      if (u[t] < 0) continue;
      const float w = __fdiv_rn(expf(__fmul_rn(p[t], a.scale) - mv), sv);
      const float ad = w * p[E + t];
      sd += ad;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        A[j] = fmaf(ad, x[t][j], A[j]);
        B[j] = fmaf(w, x[t][j], B[j]);
      }
    }
  }
  if (slot < 0) {
    tc_dst_store<T, NJ>(a, v, kh, lane, sd, A, B, gv);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + kh) * (2 * D + 1);
    if (lane == 0) p[0] = sd;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) { p[1 + col] = A[j]; p[1 + D + col] = B[j]; }
    }
  }
}

template <typename T, int NJ>
// no __launch_bounds__: with it ptxas spills the NJ = 2 instances (launched with kGatWarps * 32 threads as well)
__global__ void tconv_bwd_dst_kernel(TcArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int v, int e0, int n, int slot) { tc_dst_row<T, NJ>(a, v, e0, n, slot, k, lane); });
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) tconv_bwd_dst_fixup_kernel(TcArgs a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  const int D = a.D, v = a.w.long_row[li];
  float sd = 0.f, A[NJ], B[NJ], gv[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) { A[j] = 0.f; B[j] = 0.f; }
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + (static_cast<int64_t>(sg) * a.H + k) * (2 * D + 1);
    sd += p[0];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) { A[j] += p[1 + col]; B[j] += p[1 + D + col]; }
    }
  }
  load_head<T, NJ>(head_row<T>(a.g, a.ldg, v, k, D), D, lane, gv);
  tc_dst_store<T, NJ>(a, v, k, lane, sd, A, B, gv);
}

template <typename T, int NJ>
__device__ __forceinline__ void tc_src_store(const TcArgs& a, int u, int kh, int lane, const float (&dk)[NJ],
                                             const float (&dv)[NJ]) {
  T* ok = head_row_out<T>(a.out, a.ldo, u, kh, a.D);
  T* ov = head_row_out<T>(a.out2, a.ldo2, u, kh, a.D);
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int col = lane + 32 * j;
    if (col < a.D) {
      ok[col] = from_f<T>(a.scale * dk[j]);
      ov[col] = from_f<T>(dv[j]);
    }
  }
}

// over the CSC row u (the destinations v of source u), with c_uv = a_uv (<g_v, v_u> - delta_v):
//   dv_u = sum_v a_uv g_v,  dk_u = scale sum_v c_uv q_v;  an unkept source gets 0.  Scratch of a segment: [H][2 D].
template <typename T, int NJ>
__device__ __forceinline__ void tc_src_row(const TcArgs& a, int u, int e0, int n, int slot, int kh, int lane) {
  constexpr int E = tc_edges<NJ>();
  const int D = a.D;
  float dk[NJ], dv[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) { dk[j] = 0.f; dv[j] = 0.f; }
  if (is_kept(a.keep, a.num_in, u)) {
    float ku[NJ], vu[NJ];
    load_head<T, NJ>(head_row<T>(a.k, a.ldk, u, kh, D), D, lane, ku);
    load_head<T, NJ>(head_row<T>(a.v, a.ldv, u, kh, D), D, lane, vu);
    for (int b = 0; b < n; b += E) {
      int v[E];
      float x[E][NJ], y[E][NJ], p[2 * E], mv[E], sv[E], dl[E];
#pragma unroll
      for (int t = 0; t < E; ++t) v[t] = b + t < n ? a.w.pidx[e0 + b + t] & kColMask : -1;
#pragma unroll
      for (int t = 0; t < E; ++t) {
        if (v[t] >= 0) {
          load_head<T, NJ>(head_row<T>(a.q, a.ldq, v[t], kh, D), D, lane, x[t]);
          load_head<T, NJ>(head_row<T>(a.g, a.ldg, v[t], kh, D), D, lane, y[t]);
          const int64_t vk = static_cast<int64_t>(v[t]) * a.H + kh;
          mv[t] = a.m[vk]; sv[t] = a.s[vk]; dl[t] = a.delta[vk];
        } else {
#pragma unroll
          for (int j = 0; j < NJ; ++j) { x[t][j] = 0.f; y[t][j] = 0.f; }
          mv[t] = 0.f; sv[t] = 0.f; dl[t] = 0.f;
        }
      }
#pragma unroll
      for (int t = 0; t < E; ++t) {
        p[t] = dot_part<NJ>(x[t], ku);        // the forward's <q_v, k_u>, column for column
        p[E + t] = dot_part<NJ>(y[t], vu);    // the destination pass's <g_v, v_u>
      }
      warp_sum_n<2 * E>(p, lane);
#pragma unroll
      for (int t = 0; t < E; ++t) {
        if (!(sv[t] > 0.f)) continue;         // also the slots past the row's end
        const float w = __fdiv_rn(expf(__fmul_rn(p[t], a.scale) - mv[t]), sv[t]);
        const float c = w * (p[E + t] - dl[t]);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          dv[j] = fmaf(w, y[t][j], dv[j]);
          dk[j] = fmaf(c, x[t][j], dk[j]);
        }
      }
    }
  }
  if (slot < 0) {
    tc_src_store<T, NJ>(a, u, kh, lane, dk, dv);
  } else {
    float* p = a.scratch + (static_cast<int64_t>(slot) * a.H + kh) * (2 * D);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) { p[col] = dk[j]; p[D + col] = dv[j]; }
    }
  }
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) tconv_bwd_src_kernel(TcArgs a) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (c >= a.w.n_chunks) return;
  walk_chunk(a.w, c, [&](int u, int e0, int n, int slot) { tc_src_row<T, NJ>(a, u, e0, n, slot, k, lane); });
}

template <typename T, int NJ>
__global__ void __launch_bounds__(kGatWarps * 32) tconv_bwd_src_fixup_kernel(TcArgs a) {
  const int lane = threadIdx.x & 31;
  const int li = blockIdx.x * kGatWarps + (threadIdx.x >> 5);
  const int k = blockIdx.y;
  if (li >= a.w.n_long) return;
  const int D = a.D;
  float dk[NJ], dv[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) { dk[j] = 0.f; dv[j] = 0.f; }
  for (int sg = a.w.long_seg_ptr[li]; sg < a.w.long_seg_ptr[li + 1]; ++sg) {
    const float* p = a.scratch + (static_cast<int64_t>(sg) * a.H + k) * (2 * D);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int col = lane + 32 * j;
      if (col < D) { dk[j] += p[col]; dv[j] += p[D + col]; }
    }
  }
  tc_src_store<T, NJ>(a, a.w.long_row[li], k, lane, dk, dv);
}

// ---------------------------------------------------------------------------------------------------- dispatch
int nj_of(int32_t D) { return D <= 32 ? 1 : D <= 64 ? 2 : D <= 128 ? 4 : D <= 256 ? 8 : D <= 512 ? 16 : 0; }

#define PG_GAT_NJ(T, KERNEL, GRID, ST, ...)                                              \
  switch (nj) {                                                                          \
    case 1: KERNEL<T, 1><<<GRID, kGatWarps * 32, 0, ST>>>(__VA_ARGS__); break;           \
    case 2: KERNEL<T, 2><<<GRID, kGatWarps * 32, 0, ST>>>(__VA_ARGS__); break;           \
    case 4: KERNEL<T, 4><<<GRID, kGatWarps * 32, 0, ST>>>(__VA_ARGS__); break;           \
    case 8: KERNEL<T, 8><<<GRID, kGatWarps * 32, 0, ST>>>(__VA_ARGS__); break;           \
    default: KERNEL<T, 16><<<GRID, kGatWarps * 32, 0, ST>>>(__VA_ARGS__); break;         \
  }

template <typename T, int NJ>
void preload_t() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, gat_scores_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gat_fwd_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gat_fwd_fixup_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gat_bwd_dst_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gat_bwd_src_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gat_bwd_src_fixup_kernel<T, NJ>);
}
template <typename T, int NJ>
void preload_v2_t() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, gatv2_fwd_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gat_fwd_fixup_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gatv2_bwd_dst_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gatv2_bwd_dst_fixup_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gatv2_bwd_src_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, gatv2_bwd_src_fixup_kernel<T, NJ>);
}
template <typename T>
void preload_v2_all() {
  preload_v2_t<T, 1>(); preload_v2_t<T, 2>(); preload_v2_t<T, 4>(); preload_v2_t<T, 8>(); preload_v2_t<T, 16>();
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, gat_colsum_kernel<T>);
}
template <typename T, int NJ>
void preload_tc_t() {
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, tconv_fwd_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, tconv_fwd_fixup_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, tconv_bwd_dst_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, tconv_bwd_dst_fixup_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, tconv_bwd_src_kernel<T, NJ>);
  cudaFuncGetAttributes(&a, tconv_bwd_src_fixup_kernel<T, NJ>);
}
template <typename T>
void preload_tc_all() {
  preload_tc_t<T, 1>(); preload_tc_t<T, 2>(); preload_tc_t<T, 4>(); preload_tc_t<T, 8>(); preload_tc_t<T, 16>();
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, gat_colsum_kernel<T>);
}
template <typename T>
void preload_all() {
  preload_t<T, 1>(); preload_t<T, 2>(); preload_t<T, 4>(); preload_t<T, 8>(); preload_t<T, 16>();
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, gat_colsum_kernel<T>);
}

int check_plan(const pg_csr* g, const char* who) {
  PG_REQUIRE(g != nullptr, "%s: null plan", who);
  PG_REQUIRE(g->n_rows == 0 || (g->chunks != nullptr && g->pidx != nullptr && g->prow != nullptr),
             "%s: the plan has no chunk table (build it with sorted rows and chunks enabled)", who);
  PG_REQUIRE(g->n_seg == 0 || (g->long_row && g->long_seg_ptr && g->seg_long), "%s: the plan has no long-row split", who);
  return PG_OK;
}

}  // namespace

// CUDA loads kernels lazily, and loading one may wait for the device: see exchange.cu's bns_preload.
static void gat_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_all<float>();
    preload_all<__nv_bfloat16>();
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, gat_bwd_dst_fixup_kernel);
    cudaFuncGetAttributes(&a, gat_colsum_final_kernel);
    cudaGetLastError();
  });
}

static void gatv2_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_v2_all<float>();
    preload_v2_all<__nv_bfloat16>();
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, gat_colsum_final_kernel);
    cudaGetLastError();
  });
}

static void tconv_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    preload_tc_all<float>();
    preload_tc_all<__nv_bfloat16>();
    cudaFuncAttributes a;
    cudaFuncGetAttributes(&a, gat_colsum_final_kernel);
    cudaGetLastError();
  });
}

}  // namespace pg

using pg::kGatWarps;

extern "C" int pg_gat_preload(void) {
  pg::gat_preload();
  return PG_OK;
}

extern "C" int pg_gat_scores(const void* z, int64_t ldz, int32_t n_rows, int32_t n_er, int32_t H, int32_t D,
                             int dtype, const float* attn_l, const float* attn_r, float* el, float* er, void* stream) {
  pg::gat_preload();
  PG_REQUIRE(n_rows >= 0 && n_er >= 0 && n_er <= n_rows && H > 0 && D > 0 && ldz >= static_cast<int64_t>(H) * D,
             "pg_gat_scores: bad sizes");
  const int nj = pg::nj_of(D);
  PG_REQUIRE(nj > 0, "pg_gat_scores: head width %d > 512", D);
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(z && attn_l && el && (n_er == 0 || (attn_r && er)), "pg_gat_scores: null argument");
  const dim3 grid((n_rows + kGatWarps - 1) / kGatWarps, H);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32) {
    PG_GAT_NJ(float, pg::gat_scores_kernel, grid, st, static_cast<const float*>(z), ldz, n_rows,
                                                                         n_er, H, D, attn_l, attn_r, el, er);
  } else if (dtype == PG_BF16) {
    PG_GAT_NJ(__nv_bfloat16, pg::gat_scores_kernel, grid, st,
        static_cast<const __nv_bfloat16*>(z), ldz, n_rows, n_er, H, D, attn_l, attn_r, el, er);
  } else {
    pg::set_error("pg_gat_scores: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gat_aggregate(const pg_csr* g, const void* z, int64_t ldz, int32_t H, int32_t D, int dtype,
                                const float* el, const float* er, const float* bias, const uint8_t* keep,
                                int32_t num_in, void* out, int64_t ldo, float* m, float* s, float* scratch,
                                void* stream) {
  pg::gat_preload();
  if (int rc = pg::check_plan(g, "pg_gat_aggregate")) return rc;
  const int nj = pg::nj_of(D);
  PG_REQUIRE(H > 0 && nj > 0 && ldz >= static_cast<int64_t>(H) * D && ldo >= static_cast<int64_t>(H) * D,
             "pg_gat_aggregate: bad sizes (H %d, D %d)", H, D);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(z && el && er && out && m && s && (g->n_seg == 0 || scratch), "pg_gat_aggregate: null argument");
  pg::FwdArgs a{pg::make_walk(g), z, ldz, el, er, bias, keep, num_in, out, ldo, m, s, scratch, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((g->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (g->n_chunks) PG_GAT_NJ(float, pg::gat_fwd_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(float, pg::gat_fwd_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (g->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::gat_fwd_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(__nv_bfloat16, pg::gat_fwd_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_gat_aggregate: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gat_bwd_dst(const pg_csr* g, const void* z, int64_t ldz, const void* grad, int64_t ldg, int32_t H,
                              int32_t D, int dtype, const float* el, const float* er, const float* m, const float* s,
                              const uint8_t* keep, int32_t num_in, float* der, float* dv, float* scratch,
                              void* stream) {
  pg::gat_preload();
  if (int rc = pg::check_plan(g, "pg_gat_bwd_dst")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && nj > 0 && ldz >= hd && ldg >= hd, "pg_gat_bwd_dst: bad sizes (H %d, D %d)", H, D);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(z && grad && el && er && m && s && der && dv && (g->n_seg == 0 || scratch),
             "pg_gat_bwd_dst: null argument");
  pg::BwdArgs a{pg::make_walk(g), z, ldz, grad, ldg, el, er, m, s, nullptr, nullptr, nullptr, nullptr,
                keep, num_in, der, dv, nullptr, 0, nullptr, scratch, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (g->n_chunks) PG_GAT_NJ(float, pg::gat_bwd_dst_kernel, grid, st, a);
  } else if (dtype == PG_BF16) {
    if (g->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::gat_bwd_dst_kernel, grid, st, a);
  } else {
    pg::set_error("pg_gat_bwd_dst: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  if (g->n_long) {
    const int n = g->n_long * H;
    pg::gat_bwd_dst_fixup_kernel<<<(n + 255) / 256, 256, 0, st>>>(a);
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gat_bwd_src(const pg_csr* gt, const void* z, int64_t ldz, const void* grad, int64_t ldg, int32_t H,
                              int32_t D, int dtype, const float* el, const float* er, const float* m, const float* s,
                              const float* dv, const float* der, const float* attn_l, const float* attn_r,
                              const uint8_t* keep, int32_t num_in, void* dz, int64_t lddz, float* del,
                              float* scratch, void* stream) {
  pg::gat_preload();
  if (int rc = pg::check_plan(gt, "pg_gat_bwd_src")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && nj > 0 && ldz >= hd && ldg >= hd && lddz >= hd && num_in >= 0,
             "pg_gat_bwd_src: bad sizes (H %d, D %d)", H, D);
  if (gt->n_rows == 0) return PG_OK;
  PG_REQUIRE(z && grad && el && er && m && s && dv && (num_in == 0 || der) && attn_l && attn_r && dz && del &&
                 (gt->n_seg == 0 || scratch),
             "pg_gat_bwd_src: null argument");
  pg::BwdArgs a{pg::make_walk(gt), z, ldz, grad, ldg, el, er, m, s, dv, der, attn_l, attn_r,
                keep, num_in, nullptr, nullptr, dz, lddz, del, scratch, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((gt->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((gt->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (gt->n_chunks) PG_GAT_NJ(float, pg::gat_bwd_src_kernel, grid, st, a);
    if (gt->n_long) PG_GAT_NJ(float, pg::gat_bwd_src_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (gt->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::gat_bwd_src_kernel, grid, st, a);
    if (gt->n_long) PG_GAT_NJ(__nv_bfloat16, pg::gat_bwd_src_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_gat_bwd_src: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gat_colsum_blocks(int32_t n_rows) { return pg::colsum_blocks(n_rows); }

extern "C" int pg_gat_colsum(const void* x, int64_t ldx, int32_t n_rows, int32_t H, int32_t D, int dtype,
                             const float* coef, float* out, float* partial, void* stream) {
  pg::gat_preload();
  const int n_cols = H * D;
  PG_REQUIRE(n_rows >= 0 && H > 0 && D > 0 && ldx >= n_cols && out && partial, "pg_gat_colsum: bad arguments");
  PG_REQUIRE(n_rows == 0 || x, "pg_gat_colsum: null input");
  const int nb = pg::colsum_blocks(n_rows);
  const int rows_per = static_cast<int>((static_cast<int64_t>(n_rows) + nb - 1) / nb);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(nb, (n_cols + 31) / 32), block(32, 8);
  if (dtype == PG_F32) {
    pg::gat_colsum_kernel<float><<<grid, block, 0, st>>>(static_cast<const float*>(x), ldx, n_rows, H, D, coef,
                                                         rows_per, partial);
  } else if (dtype == PG_BF16) {
    pg::gat_colsum_kernel<__nv_bfloat16><<<grid, block, 0, st>>>(static_cast<const __nv_bfloat16*>(x), ldx, n_rows,
                                                                 H, D, coef, rows_per, partial);
  } else {
    pg::set_error("pg_gat_colsum: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  pg::gat_colsum_final_kernel<<<(n_cols + 255) / 256, 256, 0, st>>>(partial, nb, n_cols, out);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gatv2_preload(void) {
  pg::gatv2_preload();
  return PG_OK;
}

extern "C" int pg_gatv2_aggregate(const pg_csr* g, const void* zs, int64_t ldzs, const void* zd, int64_t ldzd,
                                  int32_t H, int32_t D, int dtype, const float* attn, const uint8_t* keep,
                                  int32_t num_in, void* out, int64_t ldo, float* m, float* s, float* scratch,
                                  void* stream) {
  pg::gatv2_preload();
  if (int rc = pg::check_plan(g, "pg_gatv2_aggregate")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && nj > 0 && ldzs >= hd && ldzd >= hd && ldo >= hd, "pg_gatv2_aggregate: bad sizes (H %d, D %d)",
             H, D);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(zs && zd && attn && out && m && s && (g->n_seg == 0 || scratch), "pg_gatv2_aggregate: null argument");
  pg::V2Args a{pg::make_walk(g), zs, ldzs, zd, ldzd, nullptr, 0, attn, nullptr, nullptr, nullptr, keep, num_in,
               out, ldo, m, s, nullptr, nullptr, 0, scratch, H, D};
  const pg::FwdArgs f = pg::v2_fwd_args(a);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((g->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (g->n_chunks) PG_GAT_NJ(float, pg::gatv2_fwd_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(float, pg::gat_fwd_fixup_kernel, grid_fix, st, f);
  } else if (dtype == PG_BF16) {
    if (g->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::gatv2_fwd_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(__nv_bfloat16, pg::gat_fwd_fixup_kernel, grid_fix, st, f);
  } else {
    pg::set_error("pg_gatv2_aggregate: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gatv2_bwd_dst(const pg_csr* g, const void* zs, int64_t ldzs, const void* zd, int64_t ldzd,
                                const void* grad, int64_t ldg, int32_t H, int32_t D, int dtype, const float* attn,
                                const float* m, const float* s, const uint8_t* keep, int32_t num_in, void* dzd,
                                int64_t lddzd, float* dv, float* pattn, int64_t ldp, float* scratch, void* stream) {
  pg::gatv2_preload();
  if (int rc = pg::check_plan(g, "pg_gatv2_bwd_dst")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && nj > 0 && ldzs >= hd && ldzd >= hd && ldg >= hd && lddzd >= hd && ldp >= hd,
             "pg_gatv2_bwd_dst: bad sizes (H %d, D %d)", H, D);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(zs && zd && grad && attn && m && s && dzd && dv && pattn && (g->n_seg == 0 || scratch),
             "pg_gatv2_bwd_dst: null argument");
  pg::V2Args a{pg::make_walk(g), zs, ldzs, zd, ldzd, grad, ldg, attn, m, s, nullptr, keep, num_in,
               dzd, lddzd, nullptr, nullptr, dv, pattn, ldp, scratch, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((g->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (g->n_chunks) PG_GAT_NJ(float, pg::gatv2_bwd_dst_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(float, pg::gatv2_bwd_dst_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (g->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::gatv2_bwd_dst_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(__nv_bfloat16, pg::gatv2_bwd_dst_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_gatv2_bwd_dst: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gatv2_bwd_src(const pg_csr* gt, const void* zs, int64_t ldzs, const void* zd, int64_t ldzd,
                                const void* grad, int64_t ldg, int32_t H, int32_t D, int dtype, const float* attn,
                                const float* m, const float* s, const float* dv, const uint8_t* keep, int32_t num_in,
                                void* dzs, int64_t lddzs, float* scratch, void* stream) {
  pg::gatv2_preload();
  if (int rc = pg::check_plan(gt, "pg_gatv2_bwd_src")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && nj > 0 && ldzs >= hd && ldzd >= hd && ldg >= hd && lddzs >= hd && num_in >= 0,
             "pg_gatv2_bwd_src: bad sizes (H %d, D %d)", H, D);
  if (gt->n_rows == 0) return PG_OK;
  PG_REQUIRE(zs && (num_in == 0 || (zd && grad && m && s && dv)) && attn && dzs && (gt->n_seg == 0 || scratch),
             "pg_gatv2_bwd_src: null argument");
  pg::V2Args a{pg::make_walk(gt), zs, ldzs, zd, ldzd, grad, ldg, attn, m, s, dv, keep, num_in,
               dzs, lddzs, nullptr, nullptr, nullptr, nullptr, 0, scratch, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((gt->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((gt->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (gt->n_chunks) PG_GAT_NJ(float, pg::gatv2_bwd_src_kernel, grid, st, a);
    if (gt->n_long) PG_GAT_NJ(float, pg::gatv2_bwd_src_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (gt->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::gatv2_bwd_src_kernel, grid, st, a);
    if (gt->n_long) PG_GAT_NJ(__nv_bfloat16, pg::gatv2_bwd_src_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_gatv2_bwd_src: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_tconv_preload(void) {
  pg::tconv_preload();
  return PG_OK;
}

extern "C" int pg_tconv_aggregate(const pg_csr* g, const void* q, int64_t ldq, const void* k, int64_t ldk,
                                  const void* v, int64_t ldv, const void* skip, int64_t ldskip, int32_t H, int32_t D,
                                  int dtype, float scale, const uint8_t* keep, int32_t num_in, void* out, int64_t ldo,
                                  float* m, float* s, float* scratch, void* stream) {
  pg::tconv_preload();
  if (int rc = pg::check_plan(g, "pg_tconv_aggregate")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && D > 0 && nj > 0 && ldq >= hd && ldk >= hd && ldv >= hd && ldskip >= hd && ldo >= hd,
             "pg_tconv_aggregate: bad sizes (H %d, D %d; D must be in 1..512)", H, D);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(q && k && v && skip && out && m && s && (g->n_seg == 0 || scratch), "pg_tconv_aggregate: null argument");
  pg::TcArgs a{pg::make_walk(g), q, ldq, k, ldk, v, ldv, skip, ldskip, nullptr, 0, nullptr, nullptr, nullptr, keep,
               num_in, out, ldo, nullptr, 0, m, s, nullptr, scratch, scale, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((g->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (g->n_chunks) PG_GAT_NJ(float, pg::tconv_fwd_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(float, pg::tconv_fwd_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (g->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::tconv_fwd_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(__nv_bfloat16, pg::tconv_fwd_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_tconv_aggregate: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_tconv_bwd_dst(const pg_csr* g, const void* q, int64_t ldq, const void* k, int64_t ldk,
                                const void* v, int64_t ldv, const void* grad, int64_t ldg, int32_t H, int32_t D,
                                int dtype, float scale, const float* m, const float* s, const uint8_t* keep,
                                int32_t num_in, void* dq, int64_t lddq, void* gcopy, int64_t ldgc, float* delta,
                                float* scratch, void* stream) {
  pg::tconv_preload();
  if (int rc = pg::check_plan(g, "pg_tconv_bwd_dst")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && D > 0 && nj > 0 && ldq >= hd && ldk >= hd && ldv >= hd && ldg >= hd && lddq >= hd && ldgc >= hd,
             "pg_tconv_bwd_dst: bad sizes (H %d, D %d; D must be in 1..512)", H, D);
  if (g->n_rows == 0) return PG_OK;
  PG_REQUIRE(q && k && v && grad && m && s && dq && gcopy && delta && (g->n_seg == 0 || scratch),
             "pg_tconv_bwd_dst: null argument");
  pg::TcArgs a{pg::make_walk(g), q, ldq, k, ldk, v, ldv, nullptr, 0, grad, ldg, m, s, nullptr, keep,
               num_in, dq, lddq, gcopy, ldgc, nullptr, nullptr, delta, scratch, scale, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((g->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((g->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (g->n_chunks) PG_GAT_NJ(float, pg::tconv_bwd_dst_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(float, pg::tconv_bwd_dst_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (g->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::tconv_bwd_dst_kernel, grid, st, a);
    if (g->n_long) PG_GAT_NJ(__nv_bfloat16, pg::tconv_bwd_dst_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_tconv_bwd_dst: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_tconv_bwd_src(const pg_csr* gt, const void* q, int64_t ldq, const void* k, int64_t ldk,
                                const void* v, int64_t ldv, const void* grad, int64_t ldg, int32_t H, int32_t D,
                                int dtype, float scale, const float* m, const float* s, const float* delta,
                                const uint8_t* keep, int32_t num_in, void* dk, int64_t lddk, void* dv, int64_t lddv,
                                float* scratch, void* stream) {
  pg::tconv_preload();
  if (int rc = pg::check_plan(gt, "pg_tconv_bwd_src")) return rc;
  const int nj = pg::nj_of(D);
  const int64_t hd = static_cast<int64_t>(H) * D;
  PG_REQUIRE(H > 0 && D > 0 && nj > 0 && ldq >= hd && ldk >= hd && ldv >= hd && ldg >= hd && lddk >= hd &&
                 lddv >= hd && num_in >= 0,
             "pg_tconv_bwd_src: bad sizes (H %d, D %d; D must be in 1..512)", H, D);
  if (gt->n_rows == 0) return PG_OK;
  PG_REQUIRE(k && v && (num_in == 0 || (q && grad && m && s && delta)) && dk && dv && (gt->n_seg == 0 || scratch),
             "pg_tconv_bwd_src: null argument");
  pg::TcArgs a{pg::make_walk(gt), q, ldq, k, ldk, v, ldv, nullptr, 0, grad, ldg, m, s, delta, keep,
               num_in, dk, lddk, dv, lddv, nullptr, nullptr, nullptr, scratch, scale, H, D};
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((gt->n_chunks + kGatWarps - 1) / kGatWarps, H), grid_fix((gt->n_long + kGatWarps - 1) / kGatWarps, H);
  if (dtype == PG_F32) {
    if (gt->n_chunks) PG_GAT_NJ(float, pg::tconv_bwd_src_kernel, grid, st, a);
    if (gt->n_long) PG_GAT_NJ(float, pg::tconv_bwd_src_fixup_kernel, grid_fix, st, a);
  } else if (dtype == PG_BF16) {
    if (gt->n_chunks) PG_GAT_NJ(__nv_bfloat16, pg::tconv_bwd_src_kernel, grid, st, a);
    if (gt->n_long) PG_GAT_NJ(__nv_bfloat16, pg::tconv_bwd_src_fixup_kernel, grid_fix, st, a);
  } else {
    pg::set_error("pg_tconv_bwd_src: unknown dtype %d", dtype);
    return PG_ERR_INVALID;
  }
  PG_LAUNCH_CHECK();
  return PG_OK;
}
