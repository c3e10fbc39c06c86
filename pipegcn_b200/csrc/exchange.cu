// Halo exchange kernels (SURVEY.md K1/K3/K12/K13) for sm_90a: in-kernel P2P stores over
// NVLink/NVSwitch into peer-mapped buffers, sender-side EMA mirror, flag publish / wait,
// and the ordered boundary add.  These replace the gather -> pinned host -> gloo -> pinned
// host -> device path of PipeGCN/helper/feature_buffer.py:165-194.
#include <algorithm>
#include <string.h>
#include "common.cuh"

namespace pg {

constexpr int kPushRows = 32;      // rows per CTA
constexpr int kPushThreads = 256;  // 8 warps, one row per warp at a time

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// One launch moves every message of one (layer, direction): CTA -> message by cta_begin.
template <typename T, int VB>
__global__ void __launch_bounds__(kPushThreads)
halo_push_kernel(const pg_msg* __restrict__ msgs, int n_msgs, const T* __restrict__ src, int64_t ld_src, int nvec,
                 float momentum, float one_minus, uint32_t value, const uint32_t* __restrict__ value_dev, DropArg drop) {
  if (value_dev != nullptr) value += *value_dev;     // epoch counter kept on the device (CUDA-graph replay)
  const uint32_t drop_hi = drop_seed_hi(drop);
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  constexpr int V = P::V;
  // locate the message of this CTA (n_msgs is tiny: P peers + the local copy)
  int m = 0;
  while (m + 1 < n_msgs && static_cast<int>(blockIdx.x) >= msgs[m + 1].cta_begin) ++m;
  const pg_msg msg = msgs[m];
  const int row0 = (static_cast<int>(blockIdx.x) - msg.cta_begin) * kPushRows;
  const int row1 = min(msg.n_rows, row0 + kPushRows);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  T* dst = static_cast<T*>(msg.dst);

  for (int r = row0 + warp; r < row1; r += kPushThreads / 32) {
    const int64_t srow = msg.idx ? static_cast<int64_t>(__ldg(msg.idx + r)) : msg.src_row0 + r;
    const T* sp = src + srow * ld_src;
    T* dp = dst + static_cast<int64_t>(r) * msg.ld_dst;
    if (msg.ema == nullptr) {
      for (int vi = lane; vi < nvec; vi += 32) {
        Raw v = *reinterpret_cast<const Raw*>(sp + static_cast<int64_t>(vi) * V);
        if (drop.thresh16 != 0u) {               // the receiver's dropout of its row dst_row0 + r
          float f[V];
          P::unpack(v, f);
          drop_apply<V>(f, static_cast<uint64_t>(msg.dst_row0 + r) * nvec + vi, drop.thresh16, drop.scale, drop.seed_lo, drop_hi);
          v = P::pack(f);
        }
        st_vec<VB>(dp + static_cast<int64_t>(vi) * V, v);
      }
    } else {
      float* ep = msg.ema + static_cast<int64_t>(r) * msg.ld_ema;
      for (int vi = lane; vi < nvec; vi += 32) {
        float f[V];
        P::unpack(*reinterpret_cast<const Raw*>(sp + static_cast<int64_t>(vi) * V), f);
        float* e = ep + static_cast<int64_t>(vi) * V;
#pragma unroll
        for (int i = 0; i < V; ++i) {
          // t *= m; t += (1 - m) * recv   (feature_buffer.py:189-191): two roundings, no FMA
          const float t = __fmul_rn(e[i], momentum);
          f[i] = __fadd_rn(t, __fmul_rn(one_minus, f[i]));
          e[i] = f[i];
        }
        if (drop.thresh16 != 0u) {               // the mirror stays clean; what travels is dropout(round(ema))
          const Raw c = P::pack(f);
          P::unpack(c, f);
          drop_apply<V>(f, static_cast<uint64_t>(msg.dst_row0 + r) * nvec + vi, drop.thresh16, drop.scale, drop.seed_lo, drop_hi);
        }
        st_vec<VB>(dp + static_cast<int64_t>(vi) * V, P::pack(f));
      }
    }
  }

  // messages without rows have no CTA of their own: the first CTA of the launch publishes their flags
  if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < n_msgs) {
    const pg_msg& em = msgs[threadIdx.x];
    if (em.n_rows == 0 && em.flag != nullptr) st_release_sys(em.flag, value);
  }
  if (msg.flag != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const int n_ctas = (msg.n_rows + kPushRows - 1) / kPushRows;
      __threadfence_system();                        // my CTA's rows are visible system-wide
      const unsigned prev = atomicAdd(msg.counter, 1u);
      if (prev == static_cast<unsigned>(n_ctas - 1)) {
        *msg.counter = 0u;                           // ready for the next launch on this stream
        __threadfence_system();
        st_release_sys(msg.flag, value);
      }
    }
  }
}

__global__ void halo_flag_only_kernel(const pg_msg* __restrict__ msgs, int n_msgs, uint32_t value,
                                      const uint32_t* __restrict__ value_dev) {
  if (value_dev != nullptr) value += *value_dev;
  // messages with zero rows still have to publish their flag
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m < n_msgs && msgs[m].n_rows == 0 && msgs[m].flag != nullptr) st_release_sys(msgs[m].flag, value);
}

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// wait_ns (optional): the nanoseconds this launch spent spinning are ADDED to *wait_ns -- the exposed
// communication of the epoch, measurable inside a replayed CUDA graph where host-side events are not
__global__ void halo_wait_kernel(const uint32_t* const* __restrict__ flags, int n_flags, uint32_t value,
                                 const uint32_t* __restrict__ value_dev, long long timeout_cycles, int* status,
                                 unsigned long long* wait_ns) {
  if (value_dev != nullptr) value += *value_dev;
  const int i = threadIdx.x;
  const unsigned long long g0 = (wait_ns != nullptr && i == 0) ? globaltimer_ns() : 0ull;
  if (i < n_flags) {
    const uint32_t* f = flags[i];
    const long long t0 = clock64();
    unsigned ns = 20;
    // flags count epochs monotonically; compare as a signed distance so wrap-around is harmless
    while (static_cast<int32_t>(ld_acquire_sys(f) - value) < 0) {
      __nanosleep(ns);
      if (ns < 1000) ns *= 2;
      if (clock64() - t0 > timeout_cycles) {
        if (status) atomicExch(status, PG_ERR_TIMEOUT);
        break;
      }
    }
  }
  if (wait_ns != nullptr) {
    __syncthreads();                       // every flag of this launch has arrived (or timed out)
    if (i == 0) atomicAdd(wait_ns, globaltimer_ns() - g0);
  }
}

template <typename T, int VB>
__global__ void __launch_bounds__(256)
boundary_add_kernel(T* __restrict__ grad, int64_t ld_grad, const T* __restrict__ recv, int64_t ld_recv, int nvec,
                    const int32_t* __restrict__ urow, const int32_t* __restrict__ uptr,
                    const int32_t* __restrict__ usrc, int n_urow) {
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  constexpr int V = P::V;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_urow) return;
  T* gp = grad + static_cast<int64_t>(__ldg(urow + w)) * ld_grad;
  const int k0 = __ldg(uptr + w), k1 = __ldg(uptr + w + 1);
  for (int vi = lane; vi < nvec; vi += 32) {
    float g[V];
    P::unpack(*reinterpret_cast<const Raw*>(gp + static_cast<int64_t>(vi) * V), g);
    for (int k = k0; k < k1; ++k) {
      float f[V];
      P::unpack(ld_vec<VB>(recv + static_cast<int64_t>(__ldg(usrc + k)) * ld_recv + static_cast<int64_t>(vi) * V), f);
#pragma unroll
      for (int i = 0; i < V; ++i) g[i] += f[i];
      if (sizeof(T) == 2) {   // the reference adds peer by peer in the tensor dtype: round like it does
        Raw t = P::pack(g);
        P::unpack(t, g);
      }
    }
    st_vec<VB>(gp + static_cast<int64_t>(vi) * V, P::pack(g));
  }
}

// dst = c * src, c from the number k of EMA updates a constant message has seen (static layer-0 shortcut)
template <typename T, int VB>
__global__ void __launch_bounds__(256)
scale_rows_kernel(const T* __restrict__ src, int64_t lds, T* __restrict__ dst, int64_t ldd, int n_rows, int nvec,
                  float m, int corr, int k, const uint32_t* __restrict__ k_dev) {
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  constexpr int V = P::V;
  if (k_dev != nullptr) k += static_cast<int>(*k_dev);
  float c = 0.f;
  if (k > 0) c = corr ? static_cast<float>(1.0 - pow(static_cast<double>(m), static_cast<double>(k))) : 1.f;
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / nvec, vi = i % nvec;
    Raw raw = *reinterpret_cast<const Raw*>(src + r * lds + vi * V);
    if (c != 1.f) {
      float f[V];
      P::unpack(raw, f);
#pragma unroll
      for (int j = 0; j < V; ++j) f[j] *= c;
      raw = P::pack(f);
    }
    st_vec<VB>(dst + r * ldd + vi * V, raw);
  }
}

static int common_vec(int d, int es, int vb, std::initializer_list<int64_t> lds) {
  while (vb > es) {
    const int v = vb / es;
    const int64_t dp = round_up(d, v);
    bool room = true;
    for (int64_t ld : lds) room = room && dp <= ld;
    if (d % v == 0 || room) break;
    vb >>= 1;
  }
  return vb;
}

template <typename T>
static int halo_push_t(const pg_msg* msgs, int n_msgs, int n_ctas, const void* src, int64_t ld_src, int d,
                       int vb, float momentum, float one_minus, uint32_t value, const uint32_t* value_dev, const DropArg& da,
                       cudaStream_t st) {
  const int es = sizeof(T);
  const int v = vb / es;
  const int nvec = static_cast<int>(round_up(d, v) / v);
  const T* sp = static_cast<const T*>(src);
  if (n_ctas > 0) {
    switch (vb) {
      case 16: halo_push_kernel<T, 16><<<n_ctas, kPushThreads, 0, st>>>(msgs, n_msgs, sp, ld_src, nvec, momentum, one_minus, value, value_dev, da); break;
      case 8: halo_push_kernel<T, 8><<<n_ctas, kPushThreads, 0, st>>>(msgs, n_msgs, sp, ld_src, nvec, momentum, one_minus, value, value_dev, da); break;
      case 4: halo_push_kernel<T, 4><<<n_ctas, kPushThreads, 0, st>>>(msgs, n_msgs, sp, ld_src, nvec, momentum, one_minus, value, value_dev, da); break;
      default: set_error("pg_halo_push: unsupported vector width %d", vb); return PG_ERR_INVALID;
    }
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

}  // namespace pg

extern "C" int pg_push_rows_per_cta(void) { return pg::kPushRows; }

// `vec_hint` is folded into ld_src's alignment: all message buffers are allocated by
// Buffer.init_buffer with the same padded stride, the host passes d and strides, and the
// widest vector legal for src is used; destinations must be at least as aligned.
extern "C" int pg_halo_push(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const void* src, int64_t ld_src,
                            int32_t d, int dtype, float momentum, float one_minus, uint32_t value, const uint32_t* value_dev,
                            void* stream) {
  return pg_halo_push_drop(msgs, n_msgs, n_ctas, src, ld_src, d, dtype, momentum, one_minus, value, value_dev, nullptr, stream);
}

extern "C" int pg_halo_push_drop(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const void* src, int64_t ld_src,
                                 int32_t d, int dtype, float momentum, float one_minus, uint32_t value,
                                 const uint32_t* value_dev, const pg_drop* drop, void* stream) {
  PG_REQUIRE(msgs && n_msgs > 0 && n_msgs <= pg::kPushThreads, "pg_halo_push: 1..%d messages per launch", pg::kPushThreads);
  PG_REQUIRE(src != nullptr || n_ctas == 0, "pg_halo_push: null source");
  PG_REQUIRE(d > 0 && ld_src >= d, "pg_halo_push: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int es = pg::elem_size(dtype);
  // destination strides equal the padded source stride by construction; use what src allows
  int vb = pg::vec_bytes(src, ld_src, es);
  vb = pg::common_vec(d, es, vb, {ld_src});
  const pg::DropArg da = pg::make_drop(drop);
  PG_REQUIRE(da.thresh16 == 0u || vb == 16, "pg_halo_push_drop: the dropout mask is defined on 16-byte vectors (rows must be 16-byte aligned)");
  int rc;
  if (dtype == PG_F32) rc = pg::halo_push_t<float>(msgs, n_msgs, n_ctas, src, ld_src, d, vb, momentum, one_minus, value, value_dev, da, st);
  else if (dtype == PG_BF16) rc = pg::halo_push_t<__nv_bfloat16>(msgs, n_msgs, n_ctas, src, ld_src, d, vb, momentum, one_minus, value, value_dev, da, st);
  else { pg::set_error("pg_halo_push: unknown dtype %d", dtype); return PG_ERR_INVALID; }
  if (rc != PG_OK) return rc;
  if (n_ctas == 0) {      // every message is empty: nobody else publishes the flags
    pg::halo_flag_only_kernel<<<(n_msgs + 63) / 64, 64, 0, st>>>(msgs, n_msgs, value, value_dev);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

extern "C" int pg_halo_wait(const uint32_t* const* flags, int32_t n_flags, uint32_t value, const uint32_t* value_dev,
                            int32_t timeout_ms, int32_t* status, uint64_t* wait_ns, void* stream) {
  PG_REQUIRE(n_flags >= 0 && n_flags <= 1024, "pg_halo_wait: bad flag count %d", n_flags);
  if (n_flags == 0) return PG_OK;
  PG_REQUIRE(flags != nullptr, "pg_halo_wait: null flags");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  // clock64 ticks at the SM clock (<= ~2 GHz): a generous upper bound keeps the spin finite
  const long long cycles = static_cast<long long>(timeout_ms) * 2000000ll;
  pg::halo_wait_kernel<<<1, ((n_flags + 31) / 32) * 32, 0, st>>>(flags, n_flags, value, value_dev, cycles, status,
                                                                    reinterpret_cast<unsigned long long*>(wait_ns));
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_boundary_add(void* grad, int64_t ld_grad, const void* recv, int64_t ld_recv, int32_t d, int dtype,
                               const int32_t* urow, const int32_t* uptr, const int32_t* usrc, int32_t n_urow,
                               void* stream) {
  if (n_urow == 0) return PG_OK;
  PG_REQUIRE(grad && recv && urow && uptr && usrc, "pg_boundary_add: null argument");
  PG_REQUIRE(d > 0 && ld_grad >= d && ld_recv >= d, "pg_boundary_add: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int es = pg::elem_size(dtype);
  int vb = min(pg::vec_bytes(grad, ld_grad, es), pg::vec_bytes(recv, ld_recv, es));
  vb = pg::common_vec(d, es, vb, {ld_grad, ld_recv});
  const int v = vb / es;
  const int nvec = static_cast<int>(pg::round_up(d, v) / v);
  const unsigned blocks = (static_cast<unsigned>(n_urow) * 32u + 255u) / 256u;
#define PG_BADD(T_, VB_) pg::boundary_add_kernel<T_, VB_><<<blocks, 256, 0, st>>>(static_cast<T_*>(grad), ld_grad, static_cast<const T_*>(recv), ld_recv, nvec, urow, uptr, usrc, n_urow)
  if (dtype == PG_F32) {
    if (vb == 16) PG_BADD(float, 16); else if (vb == 8) PG_BADD(float, 8); else PG_BADD(float, 4);
  } else if (dtype == PG_BF16) {
    if (vb == 16) PG_BADD(__nv_bfloat16, 16); else if (vb == 8) PG_BADD(__nv_bfloat16, 8);
    else if (vb == 4) PG_BADD(__nv_bfloat16, 4);
    else { pg::set_error("pg_boundary_add: bf16 rows must be 4-byte aligned"); return PG_ERR_INVALID; }
  } else { pg::set_error("pg_boundary_add: unknown dtype %d", dtype); return PG_ERR_INVALID; }
#undef PG_BADD
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_scale_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int32_t n_rows, int32_t d,
                             int dtype, float momentum, int corr, int32_t k_host, const uint32_t* k_dev, void* stream) {
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(src && dst, "pg_scale_rows: null argument");
  PG_REQUIRE(n_rows > 0 && d > 0 && ld_src >= d && ld_dst >= d, "pg_scale_rows: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int es = pg::elem_size(dtype);
  int vb = min(pg::vec_bytes(src, ld_src, es), pg::vec_bytes(dst, ld_dst, es));
  vb = pg::common_vec(d, es, vb, {ld_src, ld_dst});
  const int v = vb / es;
  const int nvec = static_cast<int>(pg::round_up(d, v) / v);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, pg::sm_count() * 16));
#define PG_SCALE(T_, VB_) pg::scale_rows_kernel<T_, VB_><<<blocks, 256, 0, st>>>(static_cast<const T_*>(src), ld_src, static_cast<T_*>(dst), ld_dst, n_rows, nvec, momentum, corr, k_host, k_dev)
  if (dtype == PG_F32) {
    if (vb == 16) PG_SCALE(float, 16); else if (vb == 8) PG_SCALE(float, 8); else PG_SCALE(float, 4);
  } else if (dtype == PG_BF16) {
    if (vb == 16) PG_SCALE(__nv_bfloat16, 16); else if (vb == 8) PG_SCALE(__nv_bfloat16, 8);
    else if (vb == 4) PG_SCALE(__nv_bfloat16, 4); else PG_SCALE(__nv_bfloat16, 2);
  } else { pg::set_error("pg_scale_rows: unknown dtype %d", dtype); return PG_ERR_INVALID; }
#undef PG_SCALE
  PG_LAUNCH_CHECK();
  return PG_OK;
}

// ---- symmetric heap + CUDA IPC --------------------------------------------------------------
extern "C" int pg_heap_alloc(size_t bytes, void** ptr) {
  PG_REQUIRE(ptr != nullptr && bytes > 0, "pg_heap_alloc: bad arguments");
  PG_CHECK_CUDA(cudaMalloc(ptr, bytes));
  PG_CHECK_CUDA(cudaMemset(*ptr, 0, bytes));
  PG_CHECK_CUDA(cudaDeviceSynchronize());
  return PG_OK;
}
extern "C" int pg_heap_free(void* ptr) {
  if (ptr) PG_CHECK_CUDA(cudaFree(ptr));
  return PG_OK;
}
extern "C" int pg_ipc_export(void* ptr, unsigned char* handle) {
  PG_REQUIRE(ptr && handle, "pg_ipc_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == PG_IPC_HANDLE_BYTES, "IPC handle size");
  cudaIpcMemHandle_t h;
  PG_CHECK_CUDA(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle, &h, sizeof(h));
  return PG_OK;
}
extern "C" int pg_ipc_import(const unsigned char* handle, void** ptr) {
  PG_REQUIRE(ptr && handle, "pg_ipc_import: null argument");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle, sizeof(h));
  PG_CHECK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return PG_OK;
}
extern "C" int pg_ipc_close(void* ptr) {
  if (ptr) PG_CHECK_CUDA(cudaIpcCloseMemHandle(ptr));
  return PG_OK;
}
extern "C" int pg_enable_peer_access(int peer_device) {
  int dev = 0, can = 0;
  PG_CHECK_CUDA(cudaGetDevice(&dev));
  if (dev == peer_device) return PG_OK;
  PG_CHECK_CUDA(cudaDeviceCanAccessPeer(&can, dev, peer_device));
  if (!can) { pg::set_error("device %d cannot access peer %d", dev, peer_device); return PG_ERR_UNSUPPORTED; }
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
    pg::set_error("cudaDeviceEnablePeerAccess(%d): %s", peer_device, cudaGetErrorString(e));
    return PG_ERR_CUDA;
  }
  cudaGetLastError();
  return PG_OK;
}
