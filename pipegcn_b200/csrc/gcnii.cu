// Row kernels of GCNII (--model gcnii) for sm_90a: the parts of a training step that neither pg_linear nor the
// residual aggregate (pg_aggregate_scaled_res, aggregate.cu) can do.
//
//   pg_gcnii_relu_drop : h0 = ReLU(z) and, under a dropout key, hd = dropout(h0) -- one read of z, two stores
//   pg_gcnii_teleport  : acc = alpha * ds  or  acc = fma(alpha, ds, acc)  -- fp32, the gradient every convolution
//                        sends to h0, summed in the order of the calls
//   pg_gcnii_relu_bwd  : dz = (h0 > 0) ? g + acc : 0  in fp32 (acc on the first n_acc rows only), one rounding
//
// One thread per 16-byte vector of a row; rows are 16-byte aligned and padded to the vector (alloc_rows), and the pad
// columns of every output are written as 0.  No atomics, no reductions: every element is a function of its inputs.
#include "common.cuh"

namespace pg {

static unsigned vec_grid(int64_t total) {
  const int64_t need = (total + 255) / 256;
  return static_cast<unsigned>(need < sm_count() * 16 ? (need > 0 ? need : 1) : sm_count() * 16);
}

template <typename T>
__global__ void __launch_bounds__(256)
gcnii_relu_drop_kernel(const T* __restrict__ z, int64_t ldz, T* __restrict__ h0, int64_t ldh, T* __restrict__ hd,
                       int64_t ldd, int n_rows, int d, int nvec, DropArg drop) {
  using P = Pack<T, 16>;
  constexpr int V = P::V;
  const uint32_t seed_hi = drop_seed_hi(drop);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / nvec), vi = static_cast<int>(i % nvec);
    const int64_t o = static_cast<int64_t>(vi) * V;
    float f[V];
    P::unpack(*reinterpret_cast<const typename P::Raw*>(z + r * ldz + o), f);
#pragma unroll
    for (int k = 0; k < V; ++k) f[k] = (o + k < d && !(f[k] < 0.f)) ? f[k] : 0.f;   // NaN stays NaN
    st_vec<16>(h0 + r * ldh + o, P::pack(f));
    if (hd != nullptr) {
      if (drop.thresh16 != 0u) drop_apply<V>(f, static_cast<uint64_t>(i), drop.thresh16, drop.scale, drop.seed_lo, seed_hi);
      st_vec<16>(hd + r * ldd + o, P::pack(f));
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
gcnii_teleport_kernel(const T* __restrict__ ds, int64_t ldd, float* __restrict__ acc, int64_t lda, int n_rows, int d,
                      int nvec, float alpha, int accumulate) {
  using P = Pack<T, 16>;
  constexpr int V = P::V;
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / nvec), vi = static_cast<int>(i % nvec);
    const int64_t o = static_cast<int64_t>(vi) * V;
    float f[V];
    P::unpack(*reinterpret_cast<const typename P::Raw*>(ds + r * ldd + o), f);
    float* ap = acc + r * lda + o;
#pragma unroll
    for (int k = 0; k < V; ++k)
      if (o + k < d) ap[k] = accumulate ? __fmaf_rn(alpha, f[k], ap[k]) : __fmul_rn(alpha, f[k]);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
gcnii_relu_bwd_kernel(const T* __restrict__ g, int64_t ldg, const T* __restrict__ h0, int64_t ldh,
                      const float* __restrict__ acc, int64_t lda, int n_acc, T* __restrict__ dz, int64_t ldz, int n_rows,
                      int d, int nvec) {
  using P = Pack<T, 16>;
  constexpr int V = P::V;
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / nvec), vi = static_cast<int>(i % nvec);
    const int64_t o = static_cast<int64_t>(vi) * V;
    float f[V], h[V];
    P::unpack(*reinterpret_cast<const typename P::Raw*>(g + r * ldg + o), f);
    P::unpack(*reinterpret_cast<const typename P::Raw*>(h0 + r * ldh + o), h);
    const float* ap = acc + r * lda + o;
#pragma unroll
    for (int k = 0; k < V; ++k) {
      float v = f[k];
      if (r < n_acc && o + k < d) v = __fadd_rn(v, __ldg(ap + k));
      f[k] = (o + k < d && h[k] > 0.f) ? v : 0.f;
    }
    st_vec<16>(dz + r * ldz + o, P::pack(f));
  }
}

// rows of `ld` elements of `es` bytes at `p`: 16-byte aligned and wide enough for nvec whole vectors
static bool rows_ok(const void* p, int64_t ld, int es, int d) {
  const int v = 16 / es;
  return p != nullptr && vec_bytes(p, ld, es) == 16 && round_up(d, v) <= ld;
}

}  // namespace pg

extern "C" int pg_gcnii_relu_drop(const void* z, int64_t ldz, void* h0, int64_t ldh, void* hd, int64_t ldd,
                                  int32_t n_rows, int32_t d, int dtype, const pg_drop* drop, void* stream) {
  using namespace pg;
  PG_REQUIRE(n_rows >= 0 && d > 0 && (dtype == PG_F32 || dtype == PG_BF16), "pg_gcnii_relu_drop: bad sizes or dtype");
  const int es = elem_size(dtype), v = 16 / es;
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(rows_ok(z, ldz, es, d) && rows_ok(h0, ldh, es, d) && (hd == nullptr || rows_ok(hd, ldd, es, d)),
             "pg_gcnii_relu_drop: rows must be 16-byte aligned and padded to the vector width");
  PG_REQUIRE(drop == nullptr || (drop->p >= 0.f && drop->p < 1.f), "pg_gcnii_relu_drop: dropout p outside [0, 1)");
  const DropArg da = make_drop(drop);
  const int nvec = static_cast<int>(round_up(d, v) / v);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32)
    gcnii_relu_drop_kernel<float><<<vec_grid(total), 256, 0, st>>>(static_cast<const float*>(z), ldz, static_cast<float*>(h0), ldh,
                                                                   static_cast<float*>(hd), ldd, n_rows, d, nvec, da);
  else
    gcnii_relu_drop_kernel<__nv_bfloat16><<<vec_grid(total), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(z), ldz, static_cast<__nv_bfloat16*>(h0), ldh, static_cast<__nv_bfloat16*>(hd), ldd,
        n_rows, d, nvec, da);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gcnii_teleport(const void* ds, int64_t ldd, float* acc, int64_t lda, int32_t n_rows, int32_t d, int dtype,
                                 float alpha, int accumulate, void* stream) {
  using namespace pg;
  PG_REQUIRE(n_rows >= 0 && d > 0 && (dtype == PG_F32 || dtype == PG_BF16), "pg_gcnii_teleport: bad sizes or dtype");
  const int es = elem_size(dtype), v = 16 / es;
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(rows_ok(ds, ldd, es, d) && acc != nullptr && lda >= d, "pg_gcnii_teleport: bad rows");
  const int nvec = static_cast<int>(round_up(d, v) / v);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32)
    gcnii_teleport_kernel<float><<<vec_grid(total), 256, 0, st>>>(static_cast<const float*>(ds), ldd, acc, lda, n_rows, d, nvec,
                                                                  alpha, accumulate);
  else
    gcnii_teleport_kernel<__nv_bfloat16><<<vec_grid(total), 256, 0, st>>>(static_cast<const __nv_bfloat16*>(ds), ldd, acc, lda,
                                                                          n_rows, d, nvec, alpha, accumulate);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_gcnii_relu_bwd(const void* g, int64_t ldg, const void* h0, int64_t ldh, const float* acc, int64_t lda,
                                 int32_t n_acc, void* dz, int64_t ldz, int32_t n_rows, int32_t d, int dtype, void* stream) {
  using namespace pg;
  PG_REQUIRE(n_rows >= 0 && d > 0 && n_acc >= 0 && n_acc <= n_rows && (dtype == PG_F32 || dtype == PG_BF16),
             "pg_gcnii_relu_bwd: bad sizes or dtype");
  const int es = elem_size(dtype), v = 16 / es;
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(rows_ok(g, ldg, es, d) && rows_ok(h0, ldh, es, d) && rows_ok(dz, ldz, es, d) &&
             (n_acc == 0 || (acc != nullptr && lda >= d)), "pg_gcnii_relu_bwd: bad rows");
  const int nvec = static_cast<int>(round_up(d, v) / v);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dtype == PG_F32)
    gcnii_relu_bwd_kernel<float><<<vec_grid(total), 256, 0, st>>>(static_cast<const float*>(g), ldg, static_cast<const float*>(h0),
                                                                  ldh, acc, lda, n_acc, static_cast<float*>(dz), ldz, n_rows, d, nvec);
  else
    gcnii_relu_bwd_kernel<__nv_bfloat16><<<vec_grid(total), 256, 0, st>>>(
        static_cast<const __nv_bfloat16*>(g), ldg, static_cast<const __nv_bfloat16*>(h0), ldh, acc, lda, n_acc,
        static_cast<__nv_bfloat16*>(dz), ldz, n_rows, d, nvec);
  PG_LAUNCH_CHECK();
  return PG_OK;
}
