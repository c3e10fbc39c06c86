// Dense part of the GraphSAGE layer on the Hopper tensor cores (SURVEY.md K8/K10):
//
//   C[M,N] = sum_s A_s[M,K_s] * B_s[N,K_s]^T  (+ bias[N])  (/ row_div[M])          1 <= s <= 6 operand pairs
//
// i.e. `linear1(feat[:N_in]) + linear2(ah)` of the reference's module/layer.py:51 as ONE kernel
// (pair 0 = inner rows x W1, pair 1 = neighbour mean x W2, bias = b1 + b2), with a single pair the dX
// GEMMs of its backward (row_div = in_deg fuses the `/ degs` gradient), and with three pairs per product
// the split-fp32 "3xTF32" evaluation (hi*hi + hi*lo + lo*hi) used for fp32 activations.
//
// Grouped form: up to kMaxProb problems share the A operands (every source's A) and each has its own B operands, bias,
// row scale, output and dropout -- the two dX products g W1 and (g W2) / deg of a layer backward.  The grid is a
// multiple of the problem count and CTA b serves problem b % n_prob on M tiles b / n_prob, b / n_prob + gridDim /
// n_prob, ...: the CTAs that multiply the same 128 rows of A are adjacent and run side by side, so every A tile after
// the first comes from L2 and A is read from HBM once instead of once per problem.  A tile computes exactly what a
// lone launch computes for it (same K order, same epilogue).
//
// Persistent, warp-specialised, sm_90a only, three warpgroups:
//   warpgroup 0     one thread is the TMA producer: 128-byte-swizzled K-major tiles of A (128 rows) and B (NT rows)
//                   into a 4-stage shared-memory ring, completion on mbarriers; its registers go to the consumers
//   warpgroups 1-2  consumers: each owns 64 of the tile's 128 rows, issues wgmma.mma_async (m64nNTk16 bf16 / m64nNTk8
//                   tf32, fp32 accumulators in registers, one group in flight while the next stage is waited for) and
//                   then runs its own epilogue: bias / row scale / dropout, convert, 128B-swizzled shared-memory slab,
//                   TMA store (cp.async.bulk.tensor) -- every global write is a full line.  The producer keeps filling
//                   the ring with the next tile's stages while the epilogue runs.
// M is tiled by 128 (TMA zero-fills the tail and clips the store); N <= 256 is one tile, NT = N rounded up to 64, 128,
// 192 or 256 (TMA zero-fills the weight rows beyond N); K tails are zero-filled by TMA.
#include <algorithm>

#include "tc_common.cuh"

namespace pg {

constexpr int kBlockM = 128;
constexpr int kRowBytes = 128;          // one swizzle-128B row: 64 bf16 or 32 tf32 of K
constexpr int kStages = 4;
constexpr int kGemmThreads = 384;       // producer warpgroup + 2 consumer warpgroups
constexpr int kABytes = kBlockM * kRowBytes;   // 16 KB per stage

constexpr int kMaxSrc = 6;              // 2 operands pairs x 3 passes of the split-fp32 (3xTF32) product
constexpr int kMaxProb = 4;             // problems of one grouped launch
constexpr int kMaxB = 12;               // B operands of one launch: problems x sources

struct GemmMaps {
  CUtensorMap a[kMaxSrc];    // shared by every problem
  CUtensorMap b[kMaxB];      // problem q, source s: b[q * n_src + s]
  CUtensorMap c[kMaxProb];   // outputs, box = [16 rows, 128 bytes], used by the TMA-store epilogue
};
constexpr int kSlabRows = 16;                         // rows of the accumulator one warp holds
constexpr int kSlabBytes = kSlabRows * kRowBytes;     // one staging slab: 16 rows x 128 B
constexpr int kSlabsTotal = 8 /*consumer warps*/ * 2 * kSlabBytes;

struct GemmOut {
  const float* bias;         // [n] or null
  const float* row_div;      // [m] or null
  void* c;
  int64_t ldc;
  int tma_store;             // 1: epilogue stages through shared memory and stores with TMA
  DropArg drop;              // dropout applied to the output as it is written (thresh16 == 0: none)
  int64_t drop_row0;         // row index of c's first row in the tensor the mask is defined on
};

struct GemmArgs {
  int m, n;
  int n_src;
  int n_prob;
  int kb_end[kMaxSrc];       // prefix sums of the k-blocks (of 128 bytes) of every source
  int k_elems;               // elements per k-block
  int out_bf16;              // 1: bf16 output, 0: fp32 output
  int epi_slabs;             // 1 | 2 staging slabs per epilogue warp
  int drop_nvec;             // 16-byte vectors per row of the tensor a dropout mask is defined on
  GemmOut out[kMaxProb];
};

// Epilogue of one consumer warp: its 16 rows x NT columns of the accumulator.  This thread holds rows `row` and
// `row + 8` (the layout in tc_common.cuh).  kOutBf16 ? bf16 : fp32 output.
template <int NT, bool kOutBf16>
__device__ __forceinline__ void epilogue_tma(const CUtensorMap* map_c, const GemmArgs& p, const GemmOut& o,
                                             float (&acc)[NT / 2], const float* s_bias, uint8_t* warp_slabs,
                                             uint32_t& ck, int row0, int lane, uint32_t drop_hi) {
  constexpr int kCpc = kOutBf16 ? 64 : 32;                 // columns per 128-byte chunk
  const int q = lane & 3, rl = lane >> 2;                  // column pair and row inside the warp's 16 rows
  // read once: `o` lives in parameter memory, which the compiler cannot tell apart from the slab stores below
  const uint32_t thresh16 = o.drop.thresh16, seed_lo = o.drop.seed_lo;
  const float drop_scale = o.drop.scale;
  const int64_t drop_row0 = o.drop_row0;
  float scale[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + rl + 8 * h;
    scale[h] = (o.row_div != nullptr && row < p.m) ? 1.f / __ldg(o.row_div + row) : 1.f;
  }
#pragma unroll
  for (int ch = 0; ch < NT / kCpc; ++ch) {
    const int c0 = ch * kCpc;
    if (c0 >= p.n) break;
    // two staging slabs per warp: the TMA store of a chunk reads one while the next chunk is written to the other
    // (epi_slabs == 1: one slab, every chunk waits for the previous store to have read it)
    const bool two = p.epi_slabs == 2;
    uint8_t* slab = warp_slabs + ((two ? (ck & 1u) : 0u) * kSlabBytes);
    if (lane == 0) {                                       // the slab about to be written is free again
      if (two) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      else asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
    __syncwarp();
#pragma unroll
    for (int jj = 0; jj < kCpc / 8; ++jj) {
      const int j = c0 / 8 + jj;                           // 8-column block of the accumulator
      const int col = 8 * j + 2 * q;
      const float2 b2 = *reinterpret_cast<const float2*>(s_bias + col);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = (acc[4 * j + 2 * h] + b2.x) * scale[h];
        float v1 = (acc[4 * j + 2 * h + 1] + b2.y) * scale[h];
        const int r = rl + 8 * h;
        if (thresh16 != 0u) {
          // mask of the (rounded) output, per 16-byte vector: what pg_dropout_rows would make of c
          const uint64_t ibase = static_cast<uint64_t>(drop_row0 + row0 + r) * p.drop_nvec;
          if (kOutBf16) {
            v0 = __bfloat162float(__float2bfloat16_rn(v0));
            v1 = __bfloat162float(__float2bfloat16_rn(v1));
            drop_pair(v0, v1, ibase + (col >> 3), q, thresh16, drop_scale, seed_lo, drop_hi);
          } else {
            drop_pair(v0, v1, ibase + (col >> 2), q & 1, thresh16, drop_scale, seed_lo, drop_hi);
          }
        }
        // 128B swizzle of the slab: 16-byte chunk index XOR (row & 7)
        uint8_t* my = slab + r * kRowBytes;
        if (kOutBf16) {
          *reinterpret_cast<__nv_bfloat162*>(my + ((jj ^ (r & 7)) << 4) + 4 * q) = __floats2bfloat162_rn(v0, v1);
        } else {
          *reinterpret_cast<float2*>(my + (((2 * jj + (q >> 1)) ^ (r & 7)) << 4) + 8 * (q & 1)) = make_float2(v0, v1);
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (lane == 0) {
      if (row0 < p.m) tma_store_2d(map_c, smem_u32(slab), c0, row0);
      // one group per chunk, empty or not: the slab parity (ck & 1) and the group count stay in step
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    ++ck;
  }
}

// output rows that are not 16-byte aligned: plain stores from the accumulator registers
template <int NT>
__device__ __forceinline__ void epilogue_direct(const GemmArgs& p, const GemmOut& o, float (&acc)[NT / 2],
                                                const float* s_bias, int row0, int lane) {
  const int q = lane & 3, rl = lane >> 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + rl + 8 * h;
    if (row >= p.m) continue;
    const float scale = o.row_div != nullptr ? 1.f / __ldg(o.row_div + row) : 1.f;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * j + 2 * q + e;
        if (col >= p.n) continue;
        const float v = (acc[4 * j + 2 * h + e] + s_bias[col]) * scale;
        if (p.out_bf16) static_cast<__nv_bfloat16*>(o.c)[static_cast<int64_t>(row) * o.ldc + col] = __float2bfloat16_rn(v);
        else static_cast<float*>(o.c)[static_cast<int64_t>(row) * o.ldc + col] = v;
      }
    }
  }
}

template <bool kTf32, int NT>
__global__ void __launch_bounds__(kGemmThreads, 1)
linear_wgmma_kernel(const __grid_constant__ GemmMaps maps, const __grid_constant__ GemmArgs p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte alignment of the swizzled tiles
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int kBBytes = NT * kRowBytes;
  constexpr int kStageBytes = kABytes + kBBytes;
  uint8_t* slabs = smem + kStages * kStageBytes;                          // 8 warps x 2 x 2 KB, 1024-byte aligned
  float* s_bias = reinterpret_cast<float*>(slabs + kSlabsTotal);          // [256]
  uint64_t* bars = reinterpret_cast<uint64_t*>(slabs + kSlabsTotal + 1024);
  uint64_t* full_bar = bars;                    // [kStages]
  uint64_t* empty_bar = bars + kStages;         // [kStages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = (p.m + kBlockM - 1) / kBlockM;
  const int kb_total = p.kb_end[p.n_src - 1];
  const int prob = blockIdx.x % p.n_prob;                   // this CTA's problem (gridDim.x is a multiple of n_prob)
  const int tile0 = blockIdx.x / p.n_prob, tile_step = gridDim.x / p.n_prob;
  const GemmOut& o = p.out[prob];
  const CUtensorMap* map_b = maps.b + prob * p.n_src;

  if (warp == 0 && lane == 0) {
    for (int s = 0; s < p.n_src; ++s) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&maps.a[s])) : "memory");
      asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map_b + s)) : "memory");
    }
  }
  for (int i = threadIdx.x; i < 256; i += kGemmThreads)
    s_bias[i] = (o.bias != nullptr && i < p.n) ? __ldg(o.bias + i) : 0.f;
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(smem_u32(full_bar + s), 1);
      mbar_init(smem_u32(empty_bar + s), 8);      // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    set_max_regs_dec<40>();
    if (warp == 0 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = tile0; tile < n_tiles; tile += tile_step) {
        const int m0 = tile * kBlockM;
        int src = 0, kb_begin = 0;
        for (int kb = 0; kb < kb_total; ++kb) {
          while (kb >= p.kb_end[src]) { kb_begin = p.kb_end[src]; ++src; }
          mbar_wait(smem_u32(empty_bar + stage), phase ^ 1);
          const uint32_t fb = smem_u32(full_bar + stage);
          mbar_expect_tx(fb, static_cast<uint32_t>(kStageBytes));
          const uint32_t sa = smem_u32(smem + stage * kStageBytes);
          const uint32_t sb = sa + kABytes;
          tma_load_2d(sa, &maps.a[src], fb, (kb - kb_begin) * p.k_elems, m0);
          tma_load_2d(sb, map_b + src, fb, (kb - kb_begin) * p.k_elems, 0);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== consumers: MMA + epilogue =====================
    set_max_regs_inc<232>();
    const int wg = (warp >> 2) - 1;                          // 0 | 1: rows [64 wg, 64 wg + 64) of the tile
    const int cw = warp - 4;                                 // consumer warp 0..7: rows [16 cw, 16 cw + 16)
    uint8_t* warp_slabs = slabs + cw * 2 * kSlabBytes;
    const uint32_t drop_hi = drop_seed_hi(o.drop);
    const int tma_store = o.tma_store;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t ck = 0;                                         // chunks stored by this warp
    float acc[NT / 2];
    for (int tile = tile0; tile < n_tiles; tile += tile_step) {
      int prev = -1;                                         // stage whose MMAs are still in flight
      for (int kb = 0; kb < kb_total; ++kb) {
        mbar_wait(smem_u32(full_bar + stage), phase);
        const uint32_t sa = smem_u32(smem + stage * kStageBytes) + wg * 64 * kRowBytes;
        const uint32_t sb = smem_u32(smem + stage * kStageBytes) + kABytes;
        fence_accum(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kRowBytes / 32; ++k) {           // 32 bytes of K per MMA (16 bf16 / 8 tf32)
          const uint64_t ad = smem_desc_sw128(sa + k * 32);
          const uint64_t bd = smem_desc_sw128(sb + k * 32);
          const uint32_t accumulate = (kb > 0 || k > 0) ? 1u : 0u;
          if constexpr (kTf32) Wgmma<NT>::tf32(acc, ad, bd, accumulate);
          else Wgmma<NT>::template bf16<0, 0>(acc, ad, bd, accumulate);
        }
        wgmma_commit();
        fence_accum(acc);
        if (prev >= 0) {                                     // the previous stage's MMAs have retired: free it
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(smem_u32(empty_bar + prev));
        }
        prev = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_accum(acc);
      if (lane == 0 && prev >= 0) mbar_arrive(smem_u32(empty_bar + prev));
      const int row0 = tile * kBlockM + cw * kSlabRows;
      if (tma_store) {
        if (p.out_bf16) epilogue_tma<NT, true>(&maps.c[prob], p, o, acc, s_bias, warp_slabs, ck, row0, lane, drop_hi);
        else epilogue_tma<NT, false>(&maps.c[prob], p, o, acc, s_bias, warp_slabs, ck, row0, lane, drop_hi);
      } else {
        epilogue_direct<NT>(p, o, acc, s_bias, row0, lane);
      }
    }
    if (tma_store && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// ---- host side -----------------------------------------------------------------------------------
// rows x k row-major matrix, box = [box_rows, 128 bytes of k], 128B swizzle, zero fill out of bounds
static int make_map(CUtensorMap* map, const void* ptr, int64_t ld, int rows, int k, int box_rows, bool tf32) {
  EncodeTiledFn enc = get_encode();
  if (enc == nullptr) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return PG_ERR_UNSUPPORTED; }
  const int es = tf32 ? 4 : 2;
  PG_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0, "pg_linear: operand base must be 16-byte aligned");
  PG_REQUIRE((ld * es) % 16 == 0, "pg_linear: operand row stride (%lld elements) must be a multiple of 16 bytes", (long long)ld);
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * es};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(kRowBytes / es), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, tf32 ? CU_TENSOR_MAP_DATA_TYPE_TFLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                   const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d) rows=%d k=%d ld=%lld", (int)r, rows, k, (long long)ld); return PG_ERR_CUDA; }
  return PG_OK;
}

int g_gemm_epi_slabs = 2;     // pg_set_option("gemm_epi_slabs", 1|2)

template <bool kTf32, int NT>
static int launch_linear_nt(int grid, size_t smem, cudaStream_t st, const GemmMaps& maps, const GemmArgs& p) {
  static bool attr_set = false;       // once: opt in to the full 227 KB of shared memory (not a stream operation)
  if (!attr_set) {
    PG_CHECK_CUDA(cudaFuncSetAttribute(linear_wgmma_kernel<kTf32, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448));
    attr_set = true;
  }
  linear_wgmma_kernel<kTf32, NT><<<grid, kGemmThreads, smem, st>>>(maps, p);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

template <bool kTf32>
static int launch_linear(int nt, int grid, size_t smem, cudaStream_t st, const GemmMaps& maps, const GemmArgs& p) {
  switch (nt) {
    case 64: return launch_linear_nt<kTf32, 64>(grid, smem, st, maps, p);
    case 128: return launch_linear_nt<kTf32, 128>(grid, smem, st, maps, p);
    case 192: return launch_linear_nt<kTf32, 192>(grid, smem, st, maps, p);
    default: return launch_linear_nt<kTf32, 256>(grid, smem, st, maps, p);
  }
}

}  // namespace pg

extern "C" int pg_linear(int dtype_in, int dtype_out, const pg_gemm_src* srcs, int32_t n_src, const float* bias,
                         const float* row_div, void* c, int64_t ldc, int32_t m, int32_t n, void* stream) {
  return pg_linear_drop(dtype_in, dtype_out, srcs, n_src, bias, row_div, c, ldc, m, n, nullptr, 0, stream);
}

extern "C" int pg_linear_drop(int dtype_in, int dtype_out, const pg_gemm_src* srcs, int32_t n_src, const float* bias,
                              const float* row_div, void* c, int64_t ldc, int32_t m, int32_t n, const pg_drop* drop,
                              int64_t drop_row0, void* stream) {
  const pg_gemm_out out{bias, row_div, c, ldc, drop, drop_row0};
  return pg_linear_group(dtype_in, dtype_out, srcs, n_src, 1, &out, m, n, stream);
}

extern "C" int pg_linear_group(int dtype_in, int dtype_out, const pg_gemm_src* srcs, int32_t n_src, int32_t n_prob,
                               const pg_gemm_out* outs, int32_t m, int32_t n, void* stream) {
  using namespace pg;
  PG_REQUIRE(srcs && outs, "pg_linear: null operand");
  PG_REQUIRE(n_src >= 1 && n_src <= kMaxSrc, "pg_linear: 1..%d operand pairs, got %d", kMaxSrc, n_src);
  PG_REQUIRE(n_prob >= 1 && n_prob <= kMaxProb && n_prob * n_src <= kMaxB,
             "pg_linear_group: 1..%d problems of at most %d operand pairs in all, got %d x %d", kMaxProb, kMaxB, n_prob,
             n_src);
  PG_REQUIRE(m >= 0 && n > 0 && n <= 256, "pg_linear: unsupported shape m=%d n=%d (n <= 256)", m, n);
  PG_REQUIRE(dtype_in == PG_F32 || dtype_in == PG_BF16, "pg_linear: bad input dtype");
  PG_REQUIRE(dtype_out == PG_F32 || dtype_out == PG_BF16, "pg_linear: bad output dtype");
  for (int q = 0; q < n_prob; ++q) {
    PG_REQUIRE(outs[q].c, "pg_linear: null output %d", q);
    PG_REQUIRE(outs[q].ldc >= n, "pg_linear: ldc < n");
  }
  if (m == 0) return PG_OK;
  const bool tf32 = dtype_in == PG_F32;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GemmArgs p;
  GemmMaps maps;
  p.m = m; p.n = n;
  const int nt = tile_n(n);
  p.n_src = n_src;
  p.n_prob = n_prob;
  p.k_elems = kRowBytes / (tf32 ? 4 : 2);
  int kb = 0, rc;
  for (int s = 0; s < kMaxSrc; ++s) {
    if (s < n_src) {
      PG_REQUIRE(srcs[s].a && srcs[s].k > 0, "pg_linear: operand pair %d is empty", s);
      kb += (srcs[s].k + p.k_elems - 1) / p.k_elems;
      if ((rc = make_map(&maps.a[s], srcs[s].a, srcs[s].lda, m, srcs[s].k, kBlockM, tf32)) != PG_OK) return rc;
    } else {
      maps.a[s] = maps.a[0];
    }
    p.kb_end[s] = kb;
  }
  for (int i = 0; i < kMaxB; ++i) {
    if (i < n_prob * n_src) {
      const pg_gemm_src& src = srcs[i];
      const pg_gemm_src& first = srcs[i % n_src];
      PG_REQUIRE(src.b, "pg_linear: operand pair %d is empty", i);
      PG_REQUIRE(src.a == first.a && src.lda == first.lda && src.k == first.k,
                 "pg_linear_group: problem %d, pair %d does not share problem 0's A operand", i / n_src, i % n_src);
      if ((rc = make_map(&maps.b[i], src.b, src.ldb, n, src.k, nt, tf32)) != PG_OK) return rc;
    } else {
      maps.b[i] = maps.b[0];
    }
  }
  p.out_bf16 = dtype_out == PG_BF16;
  p.epi_slabs = g_gemm_epi_slabs;
  const int eso = p.out_bf16 ? 2 : 4;
  p.drop_nvec = static_cast<int>(round_up(n, p.out_bf16 ? 8 : 4) / (p.out_bf16 ? 8 : 4));
  for (int q = 0; q < kMaxProb; ++q) {
    GemmOut& o = p.out[q];
    if (q >= n_prob) {
      o = p.out[0];
      maps.c[q] = maps.c[0];
      continue;
    }
    const pg_gemm_out& in = outs[q];
    o.bias = in.bias; o.row_div = in.row_div; o.c = in.c; o.ldc = in.ldc;
    // TMA-store epilogue when the output rows are 16-byte aligned (always true for engine buffers)
    o.tma_store = ((reinterpret_cast<uintptr_t>(in.c) & 15) == 0 && (in.ldc * eso) % 16 == 0) ? 1 : 0;
    if (o.tma_store) {
      EncodeTiledFn enc = get_encode();
      cuuint64_t gdim[2] = {static_cast<cuuint64_t>(n), static_cast<cuuint64_t>(m)};
      cuuint64_t gstride[1] = {static_cast<cuuint64_t>(in.ldc) * eso};
      cuuint32_t box[2] = {static_cast<cuuint32_t>(kRowBytes / eso), kSlabRows};
      cuuint32_t estr[2] = {1, 1};
      CUresult r = enc(&maps.c[q], p.out_bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                       in.c, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                       CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(output) failed (%d)", (int)r); return PG_ERR_CUDA; }
    } else {
      maps.c[q] = maps.a[0];
    }
    o.drop = make_drop(in.drop);
    o.drop_row0 = in.drop_row0;
    PG_REQUIRE(o.drop.thresh16 == 0u || o.tma_store, "pg_linear_drop: the fused dropout needs 16-byte aligned output rows");
  }
  // a multiple of n_prob CTAs: CTA b serves problem b % n_prob only, and the n_prob CTAs of one M tile are adjacent
  const int n_tiles = (m + kBlockM - 1) / kBlockM;
  const int grid = std::min(n_tiles, std::max(1, sm_count() / n_prob)) * n_prob;
  const size_t smem = static_cast<size_t>(kStages) * (kABytes + nt * kRowBytes) + kSlabsTotal /*staging*/ +
                      1024 /*bias*/ + 256 /*barriers*/ + 1024 /*align*/;
  return tf32 ? launch_linear<true>(nt, grid, smem, st, maps, p) : launch_linear<false>(nt, grid, smem, st, maps, p);
}

// hi = x with the 13 low mantissa bits cleared (exactly a tf32), lo = x - hi (exact in fp32)
namespace pg {
__global__ void __launch_bounds__(256)
split_tf32_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ hi, float* __restrict__ lo, int64_t ld,
                  int rows, int d) {
  const int64_t total = static_cast<int64_t>(rows) * d;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / d), c = static_cast<int>(i % d);
    const float v = x[static_cast<int64_t>(r) * ldx + c];
    const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    hi[static_cast<int64_t>(r) * ld + c] = h;
    lo[static_cast<int64_t>(r) * ld + c] = v - h;
  }
}
}  // namespace pg

extern "C" int pg_split_tf32(const float* x, int64_t ldx, float* hi, float* lo, int64_t ld, int32_t rows, int32_t d,
                             void* stream) {
  PG_REQUIRE(x && hi && lo, "pg_split_tf32: null argument");
  PG_REQUIRE(rows >= 0 && d > 0 && ldx >= d && ld >= d, "pg_split_tf32: bad sizes");
  const int64_t total = static_cast<int64_t>(rows) * d;
  if (total == 0) return PG_OK;
  const unsigned blocks = static_cast<unsigned>((total + 255) / 256 < pg::sm_count() * 16 ? (total + 255) / 256 : pg::sm_count() * 16);
  pg::split_tf32_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, ldx, hi, lo, ld, rows, d);
  PG_LAUNCH_CHECK();
  return PG_OK;
}
