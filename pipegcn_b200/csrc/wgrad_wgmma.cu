// Weight gradients of the GraphSAGE layer on the Hopper tensor cores (SURVEY.md K10, row B3):
//
//   D[n, k] = sum_s sum_m  G_s[m, n] * X_s[m, k]            n <= 256 outputs, k <= 256 inputs, m = rows (10^5..10^6)
//
// i.e. gW1 = g^T feat[:N_in] and gW2 = g^T ah of the autograd of the reference's module/layer.py:51 (one call each),
// bf16 operands; fp32 activations come as six bf16 pairs (fp32 = b0 + b1 + b2 in bf16:
// b0*b0 + b0*b1 + b1*b0 + b0*b2 + b2*b0 + b1*b1).
//
// Both operands are row-major [m, .]: the contraction index m is the SLOW index, so the tiles are MN-major for the
// tensor core (wgmma's transpose bits for A and B, which exist for 16-bit operands only -- hence no tf32 form).  A TMA
// box of [128 bytes of n] x [64 rows of m] with the 128-byte swizzle is exactly one column of the canonical MN-major
// SWIZZLE_128B layout ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units: SBO = 8 rows * 128 B, LBO = one box.
// Split-K over m: CTA (x, y) owns a contiguous range x of rows and the 128 outputs y of D (a 128 x 256 fp32
// accumulator is what the registers of two warpgroups hold), accumulates its partial D and writes it to a workspace;
// a second kernel sums the partials in split order (deterministic).  With n > 128 the two CTAs of a row range read
// the same X rows at the same time, the second one from L2.
//   warpgroup 0: TMA producer (one thread)   warpgroups 1-2: wgmma m64nNTk16 on 64 outputs each, then the store
#include <algorithm>

#include "tc_common.cuh"

namespace pg {

constexpr int kWgThreads = 384;
constexpr int kWgStages = 4;
constexpr int kWgMaxSrc = 6;
constexpr int kWgRows = 64;              // rows of m per pipeline stage
constexpr int kWgBox = kWgRows * 128;    // bytes of one TMA box: 64 elements of n or k x 64 rows of m
constexpr int kWgTileN = 128;            // outputs (rows of D) per CTA
constexpr int kWgMaxSplits = 132;

struct WgradMaps {
  CUtensorMap a[kWgMaxSrc];   // G_s: dims {n, m}, box {128 B of n, 64 rows}
  CUtensorMap b[kWgMaxSrc];   // X_s: dims {k, m}, box {128 B of k, 64 rows}
};

struct WgradArgs {
  int m;
  int n_src;
  int k_pad;                 // row length of the partials: k rounded up to 16
  int rows_pad;              // rows of one partial: gridDim.y * 128
  int rows_per_split;        // multiple of kWgRows
  float* partial;            // [splits][rows_pad][k_pad]
};

template <int NT>
__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_wgmma_kernel(const __grid_constant__ WgradMaps maps, const WgradArgs p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kABytes = (kWgTileN / 64) * kWgBox, kBBytes = (NT / 64) * kWgBox;
  constexpr int kStageBytes = kABytes + kBBytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kWgStages * kStageBytes);
  uint64_t* full_bar = bars;                 // [kWgStages]
  uint64_t* empty_bar = bars + kWgStages;    // [kWgStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row_begin = blockIdx.x * p.rows_per_split;
  const int row_end = min(p.m, row_begin + p.rows_per_split);
  const int n_kb = row_end > row_begin ? (row_end - row_begin + kWgRows - 1) / kWgRows : 0;
  const int total_it = n_kb * p.n_src;
  const int n0 = blockIdx.y * kWgTileN;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < p.n_src; ++s) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.a[s])) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.b[s])) : "memory");
    }
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kWgStages; ++s) {
      mbar_init(smem_u32(full_bar + s), 1);
      mbar_init(smem_u32(empty_bar + s), 8);   // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    set_max_regs_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int it = 0; it < total_it; ++it) {
        const int kb = it / p.n_src, src = it % p.n_src;
        const int m0 = row_begin + kb * kWgRows;
        mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
        const uint32_t fb = smem_u32(full_bar + stage);
        mbar_expect_tx(fb, static_cast<uint32_t>(kStageBytes));
        const uint32_t sa = smem_u32(smem + stage * kStageBytes);
        const uint32_t sb = sa + kABytes;
        for (int blk = 0; blk < kWgTileN / 64; ++blk) tma_load_2d(sa + blk * kWgBox, &maps.a[src], fb, n0 + blk * 64, m0);
        for (int blk = 0; blk < NT / 64; ++blk) tma_load_2d(sb + blk * kWgBox, &maps.b[src], fb, blk * 64, m0);
        if (++stage == kWgStages) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    set_max_regs_inc<232>();
    const int wg = (warp >> 2) - 1;                        // outputs [n0 + 64 wg, n0 + 64 wg + 64): one box of A
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;         // a CTA without rows writes zeros
    for (int it = 0; it < total_it; ++it) {
      mbar_wait(smem_u32(full_bar + stage), phase);
      const uint32_t sa = smem_u32(smem + stage * kStageBytes) + wg * kWgBox;
      const uint32_t sb = smem_u32(smem + stage * kStageBytes) + kABytes;
      fence_accum(acc);
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < kWgRows / 16; ++ks) {          // 16 rows of m per MMA
        const uint64_t ad = smem_desc_sw128(sa + ks * 16 * 128, kWgBox);
        const uint64_t bd = smem_desc_sw128(sb + ks * 16 * 128, kWgBox);
        Wgmma<NT>::template bf16<1, 1>(acc, ad, bd, (it > 0 || ks > 0) ? 1u : 0u);
      }
      wgmma_commit();
      fence_accum(acc);
      if (prev >= 0) {                                     // the previous stage's MMAs have retired: free it
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(smem_u32(empty_bar + prev));
      }
      prev = stage;
      if (++stage == kWgStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    fence_accum(acc);
    // this thread's rows of D (accumulator layout in tc_common.cuh), all 128 rows of the tile are written
    const int q = lane & 3;
    const int row = n0 + (warp - 4) * 16 + (lane >> 2);
    float* out = p.partial + (static_cast<int64_t>(blockIdx.x) * p.rows_pad + row) * p.k_pad;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      const int col = 8 * j + 2 * q;
      if (col < p.k_pad) {
        *reinterpret_cast<float2*>(out + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(out + static_cast<int64_t>(8) * p.k_pad + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
  }
}

// out[n, k] = sum over splits of partial[split][n][k], in split order (eight partials in flight per thread)
__global__ void __launch_bounds__(256)
wgrad_reduce_kernel(const float* __restrict__ partial, int splits, int rows_pad, int k_pad, float* __restrict__ out,
                    int64_t ldo, int n, int k) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * k) return;
  const int r = idx / k, c = idx % k;
  const float* p = partial + static_cast<int64_t>(r) * k_pad + c;
  const int64_t stride = static_cast<int64_t>(rows_pad) * k_pad;
  float s = 0.f;
  int sp = 0;
  for (; sp + 8 <= splits; sp += 8) {
    float t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) t[u] = __ldcs(p + (sp + u) * stride);
#pragma unroll
    for (int u = 0; u < 8; ++u) s += t[u];
  }
  for (; sp < splits; ++sp) s += __ldcs(p + sp * stride);
  out[static_cast<int64_t>(r) * ldo + c] = s;
}

// [rows m, cols] row-major bf16 operand, box = [128 bytes of cols, 64 rows], 128B swizzle, zero fill out of bounds
static int make_mn_map(CUtensorMap* map, const void* ptr, int64_t ld, int m, int cols) {
  EncodeTiledFn enc = get_encode();
  if (enc == nullptr) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return PG_ERR_UNSUPPORTED; }
  PG_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "pg_wgrad: operand base must be 16-byte aligned");
  PG_REQUIRE((ld * 2) % 16 == 0, "pg_wgrad: operand row stride (%lld elements) must be a multiple of 16 bytes", (long long)ld);
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(m)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {64, kWgRows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) m=%d cols=%d ld=%lld", (int)r, m, cols, (long long)ld); return PG_ERR_CUDA; }
  return PG_OK;
}

// row ranges: at least 8 stages per CTA, at most `max_splits` ranges
static int wgrad_splits(int m, int max_splits, int* rows_per_split) {
  const int n_kb = (m + kWgRows - 1) / kWgRows;
  int splits = std::min(max_splits, std::max(1, n_kb / 8));
  const int kb_per = (n_kb + splits - 1) / splits;
  splits = (n_kb + kb_per - 1) / kb_per;
  *rows_per_split = kb_per * kWgRows;
  return splits;
}

// one CTA per SM over both halves of D; without a device (workspace query) the largest count any device gets
static int wgrad_max_splits(int n_tiles, bool query_device) {
  const int sms = query_device ? std::min(sm_count(), kWgMaxSplits) : kWgMaxSplits;
  return std::max(1, sms / n_tiles);
}

template <int NT>
static int launch_wgrad(dim3 grid, cudaStream_t st, const WgradMaps& maps, const WgradArgs& p) {
  const size_t smem = static_cast<size_t>(kWgStages) * (kWgTileN / 64 + NT / 64) * kWgBox + 256 /*barriers*/ + 1024 /*align*/;
  static bool attr_set = false;       // once: opt in to the full 227 KB of shared memory (not a stream operation)
  if (!attr_set) {
    PG_CHECK_CUDA(cudaFuncSetAttribute(wgrad_wgmma_kernel<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_set = true;
  }
  wgrad_wgmma_kernel<NT><<<grid, kWgThreads, smem, st>>>(maps, p);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

}  // namespace pg

extern "C" int64_t pg_wgrad_workspace(int32_t m, int32_t n, int32_t k, int dtype_in) {
  using namespace pg;
  if (m <= 0 || n <= 0 || k <= 0 || dtype_in != PG_BF16) return 0;
  const int n_tiles = (n + kWgTileN - 1) / kWgTileN;
  int rps = 0;
  const int splits = wgrad_splits(m, wgrad_max_splits(n_tiles, false), &rps);
  return static_cast<int64_t>(splits) * n_tiles * kWgTileN * round_up(k, 16);
}

extern "C" int pg_wgrad(int dtype_in, const pg_gemm_src* srcs, int32_t n_src, float* out, int64_t ldo, int32_t m,
                        int32_t n, int32_t k, float* workspace, int64_t workspace_floats, void* stream) {
  using namespace pg;
  PG_REQUIRE(srcs && out, "pg_wgrad: null operand");
  PG_REQUIRE(n_src >= 1 && n_src <= kWgMaxSrc, "pg_wgrad: 1..%d operand pairs, got %d", kWgMaxSrc, n_src);
  PG_REQUIRE(m >= 0 && n > 0 && n <= 256 && k > 0 && k <= 256, "pg_wgrad: unsupported shape m=%d n=%d k=%d (n, k <= 256)", m, n, k);
  if (dtype_in != PG_BF16) {
    set_error("pg_wgrad: bf16 operands only (the tensor core transposes 16-bit operands only); pass fp32 as bf16 terms");
    return PG_ERR_UNSUPPORTED;
  }
  PG_REQUIRE(ldo >= k, "pg_wgrad: ldo < k");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (m == 0) {
    PG_CHECK_CUDA(cudaMemset2DAsync(out, ldo * sizeof(float), 0, k * sizeof(float), n, st));
    return PG_OK;
  }
  WgradArgs p;
  WgradMaps maps;
  const int n_tiles = (n + kWgTileN - 1) / kWgTileN;
  p.m = m; p.n_src = n_src;
  p.k_pad = static_cast<int>(round_up(k, 16));
  p.rows_pad = n_tiles * kWgTileN;
  const int splits = wgrad_splits(m, wgrad_max_splits(n_tiles, true), &p.rows_per_split);
  const int64_t need = static_cast<int64_t>(splits) * p.rows_pad * p.k_pad;
  PG_REQUIRE(workspace != nullptr && workspace_floats >= need,
             "pg_wgrad: workspace too small (%lld floats, need %lld: pg_wgrad_workspace)", (long long)workspace_floats,
             (long long)need);
  p.partial = workspace;
  int rc;
  for (int s = 0; s < kWgMaxSrc; ++s) {
    if (s < n_src) {
      PG_REQUIRE(srcs[s].a && srcs[s].b, "pg_wgrad: operand pair %d is empty", s);
      if ((rc = make_mn_map(&maps.a[s], srcs[s].a, srcs[s].lda, m, n)) != PG_OK) return rc;
      if ((rc = make_mn_map(&maps.b[s], srcs[s].b, srcs[s].ldb, m, k)) != PG_OK) return rc;
    } else {
      maps.a[s] = maps.a[0];
      maps.b[s] = maps.b[0];
    }
  }
  const dim3 grid(splits, n_tiles);
  switch (tile_n(k)) {
    case 64: rc = launch_wgrad<64>(grid, st, maps, p); break;
    case 128: rc = launch_wgrad<128>(grid, st, maps, p); break;
    case 192: rc = launch_wgrad<192>(grid, st, maps, p); break;
    default: rc = launch_wgrad<256>(grid, st, maps, p); break;
  }
  if (rc != PG_OK) return rc;
  const int total = n * k;
  wgrad_reduce_kernel<<<(total + 255) / 256, 256, 0, st>>>(workspace, splits, p.rows_pad, p.k_pad, out, ldo, n, k);
  PG_LAUNCH_CHECK();
  return PG_OK;
}
