// Halo exchange kernels (SURVEY.md K1/K3/K12/K13) for sm_90a: in-kernel P2P stores over
// NVLink/NVSwitch into peer-mapped buffers, sender-side EMA mirror, flag publish / wait,
// and the ordered boundary add.  These replace the gather -> pinned host -> gloo -> pinned
// host -> device path of PipeGCN/helper/feature_buffer.py:165-194.
#include <algorithm>
#include <mutex>
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

// ---- boundary-node sampling ------------------------------------------------------------------------------------------
// this epoch's keep mask of the halo rows (one byte per row) and the sampled in-degree of every inner row: a warp per
// row walks the row's column ids (coalesced) and counts the kept sources
__global__ void __launch_bounds__(256)
bns_sample_kernel(pg_bns s, int rank, const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                  int num_in, int n_halo, uint8_t* __restrict__ mask, float* __restrict__ deg) {
  const uint32_t key = bns_key(s.seed, bns_epoch(s), static_cast<uint32_t>(rank));
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nth = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t h = tid; h < n_halo; h += nth)
    mask[h] = bns_keep(key, static_cast<uint32_t>(num_in + h), s.thresh) ? 1 : 0;
  const int lane = threadIdx.x & 31;
  for (int64_t v = tid >> 5; v < num_in; v += nth >> 5) {       // the whole warp holds the same v
    const int e0 = __ldg(indptr + v), e1 = __ldg(indptr + v + 1);
    int cnt = 0;
    for (int e = e0 + lane; e < e1; e += 32) {
      const int u = __ldg(indices + e);
      cnt += (u < num_in || bns_keep(key, static_cast<uint32_t>(u), s.thresh)) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) deg[v] = static_cast<float>(cnt);
  }
}

// halo_push_kernel without the EMA, for the sampled rows only: an unkept row is neither loaded nor stored
template <typename T, int VB>
__global__ void __launch_bounds__(kPushThreads)
halo_push_bns_kernel(const pg_msg* __restrict__ msgs, int n_msgs, const int32_t* __restrict__ keys,
                     const T* __restrict__ src, int64_t ld_src, int nvec, uint32_t value,
                     const uint32_t* __restrict__ value_dev, DropArg drop, pg_bns s) {
  if (value_dev != nullptr) value += *value_dev;
  const uint32_t drop_hi = drop_seed_hi(drop);
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  constexpr int V = P::V;
  int m = 0;
  while (m + 1 < n_msgs && static_cast<int>(blockIdx.x) >= msgs[m + 1].cta_begin) ++m;
  const pg_msg msg = msgs[m];
  const uint32_t key = bns_key(s.seed, bns_epoch(s), static_cast<uint32_t>(__ldg(keys + 2 * m)));
  const uint32_t key_row0 = static_cast<uint32_t>(__ldg(keys + 2 * m + 1));
  const int row0 = (static_cast<int>(blockIdx.x) - msg.cta_begin) * kPushRows;
  const int row1 = min(msg.n_rows, row0 + kPushRows);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  T* dst = static_cast<T*>(msg.dst);

  for (int r = row0 + warp; r < row1; r += kPushThreads / 32) {
    if (!bns_keep(key, key_row0 + static_cast<uint32_t>(r), s.thresh)) continue;     // warp-uniform
    const int64_t srow = msg.idx ? static_cast<int64_t>(__ldg(msg.idx + r)) : msg.src_row0 + r;
    const T* sp = src + srow * ld_src;
    T* dp = dst + static_cast<int64_t>(r) * msg.ld_dst;
    for (int vi = lane; vi < nvec; vi += 32) {
      Raw v = *reinterpret_cast<const Raw*>(sp + static_cast<int64_t>(vi) * V);
      if (drop.thresh16 != 0u) {
        float f[V];
        P::unpack(v, f);
        drop_apply<V>(f, static_cast<uint64_t>(msg.dst_row0 + r) * nvec + vi, drop.thresh16, drop.scale, drop.seed_lo, drop_hi);
        v = P::pack(f);
      }
      st_vec<VB>(dp + static_cast<int64_t>(vi) * V, v);
    }
  }

  // flags exactly as halo_push_kernel publishes them
  if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < n_msgs) {
    const pg_msg& em = msgs[threadIdx.x];
    if (em.n_rows == 0 && em.flag != nullptr) st_release_sys(em.flag, value);
  }
  if (msg.flag != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const int n_ctas = (msg.n_rows + kPushRows - 1) / kPushRows;
      __threadfence_system();
      const unsigned prev = atomicAdd(msg.counter, 1u);
      if (prev == static_cast<unsigned>(n_ctas - 1)) {
        *msg.counter = 0u;
        __threadfence_system();
        st_release_sys(msg.flag, value);
      }
    }
  }
}

// boundary_add_kernel over the slots the receiving peers kept
template <typename T, int VB>
__global__ void __launch_bounds__(256)
boundary_add_bns_kernel(T* __restrict__ grad, int64_t ld_grad, const T* __restrict__ recv, int64_t ld_recv, int nvec,
                        const int32_t* __restrict__ urow, const int32_t* __restrict__ uptr,
                        const int32_t* __restrict__ usrc, int n_urow, const int32_t* __restrict__ slot_keys, pg_bns s) {
  using P = Pack<T, VB>;
  using Raw = typename P::Raw;
  constexpr int V = P::V;
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_urow) return;
  const uint32_t t = bns_epoch(s);
  T* gp = grad + static_cast<int64_t>(__ldg(urow + w)) * ld_grad;
  const int k0 = __ldg(uptr + w), k1 = __ldg(uptr + w + 1);
  uint32_t kept = 0u;                         // bit k - k0: slot usrc[k] was kept (a row has at most P - 1 slots)
  for (int k = k0; k < k1 && k - k0 < 32; ++k) {
    const int sl = __ldg(usrc + k);
    if (bns_keep(bns_key(s.seed, t, static_cast<uint32_t>(__ldg(slot_keys + 2 * sl))),
                 static_cast<uint32_t>(__ldg(slot_keys + 2 * sl + 1)), s.thresh))
      kept |= 1u << (k - k0);
  }
  if (kept == 0u) return;
  for (int vi = lane; vi < nvec; vi += 32) {
    float g[V];
    P::unpack(*reinterpret_cast<const Raw*>(gp + static_cast<int64_t>(vi) * V), g);
    for (int k = k0; k < k1; ++k) {
      if (!((kept >> (k - k0)) & 1u)) continue;
      float f[V];
      P::unpack(ld_vec<VB>(recv + static_cast<int64_t>(__ldg(usrc + k)) * ld_recv + static_cast<int64_t>(vi) * V), f);
#pragma unroll
      for (int i = 0; i < V; ++i) g[i] += f[i];
      if (sizeof(T) == 2) {
        Raw t2 = P::pack(g);
        P::unpack(t2, g);
      }
    }
    st_vec<VB>(gp + static_cast<int64_t>(vi) * V, P::pack(g));
  }
}

// dst = mask ? src : 0 (src == nullptr: zero the unkept rows, leave the kept ones)
template <typename T, int VB>
__global__ void __launch_bounds__(256)
bns_mask_rows_kernel(const T* __restrict__ src, int64_t lds, T* __restrict__ dst, int64_t ldd, int n_rows, int nvec,
                     const uint8_t* __restrict__ mask) {
  using Raw = typename RawVec<VB>::type;
  constexpr int V = VB / static_cast<int>(sizeof(T));
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t r = i / nvec, vi = i % nvec;
    if (__ldg(mask + r)) {
      if (src != nullptr) st_vec<VB>(dst + r * ldd + vi * V, *reinterpret_cast<const Raw*>(src + r * lds + vi * V));
    } else {
      Raw z;
      memset(&z, 0, sizeof(z));
      st_vec<VB>(dst + r * ldd + vi * V, z);
    }
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

// ---- boundary-node sampling -------------------------------------------------------------------
namespace pg {
// CUDA loads kernels lazily, and loading one may wait for the device.  The ranks of a one-GPU LocalWorld launch their
// flag waits before the peers' pushes, so no first launch may happen while a wait spins: the first call of any pg_bns
// entry point loads every kernel of the sampled path.
static void bns_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncAttributes a;
#define PG_LOAD(F) cudaFuncGetAttributes(&a, F)
    PG_LOAD(bns_sample_kernel);
    PG_LOAD((halo_push_bns_kernel<float, 16>)); PG_LOAD((halo_push_bns_kernel<float, 8>)); PG_LOAD((halo_push_bns_kernel<float, 4>));
    PG_LOAD((halo_push_bns_kernel<__nv_bfloat16, 16>)); PG_LOAD((halo_push_bns_kernel<__nv_bfloat16, 8>));
    PG_LOAD((halo_push_bns_kernel<__nv_bfloat16, 4>));
    PG_LOAD((boundary_add_bns_kernel<float, 16>)); PG_LOAD((boundary_add_bns_kernel<float, 8>)); PG_LOAD((boundary_add_bns_kernel<float, 4>));
    PG_LOAD((boundary_add_bns_kernel<__nv_bfloat16, 16>)); PG_LOAD((boundary_add_bns_kernel<__nv_bfloat16, 8>));
    PG_LOAD((boundary_add_bns_kernel<__nv_bfloat16, 4>));
    PG_LOAD((bns_mask_rows_kernel<float, 16>)); PG_LOAD((bns_mask_rows_kernel<float, 8>)); PG_LOAD((bns_mask_rows_kernel<float, 4>));
    PG_LOAD((bns_mask_rows_kernel<__nv_bfloat16, 16>)); PG_LOAD((bns_mask_rows_kernel<__nv_bfloat16, 8>));
    PG_LOAD((bns_mask_rows_kernel<__nv_bfloat16, 4>)); PG_LOAD((bns_mask_rows_kernel<__nv_bfloat16, 2>));
    PG_LOAD(halo_flag_only_kernel);
#undef PG_LOAD
    cudaGetLastError();
  });
}
}  // namespace pg

extern "C" int pg_bns_sample(const pg_bns* s, int32_t rank, const int32_t* indptr, const int32_t* indices,
                             int32_t num_in, int32_t num_all, uint8_t* mask, float* deg, void* stream) {
  pg::bns_preload();
  PG_REQUIRE(s != nullptr && num_in >= 0 && num_all >= num_in, "pg_bns_sample: bad arguments");
  const int n_halo = num_all - num_in;
  PG_REQUIRE((n_halo == 0 || mask) && (num_in == 0 || (indptr && indices && deg)), "pg_bns_sample: null argument");
  const int64_t work = std::max<int64_t>(n_halo, static_cast<int64_t>(num_in) * 32);
  if (work == 0) return PG_OK;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((work + 255) / 256, pg::sm_count() * 16));
  pg::bns_sample_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(*s, rank, indptr, indices, num_in,
                                                                              n_halo, mask, deg);
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_halo_push_bns(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const int32_t* keys,
                                const void* src, int64_t ld_src, int32_t d, int dtype, uint32_t value,
                                const uint32_t* value_dev, const pg_drop* drop, const pg_bns* s, void* stream) {
  pg::bns_preload();
  PG_REQUIRE(msgs && n_msgs > 0 && n_msgs <= pg::kPushThreads, "pg_halo_push_bns: 1..%d messages per launch", pg::kPushThreads);
  PG_REQUIRE(keys != nullptr && s != nullptr, "pg_halo_push_bns: null keys / sample");
  PG_REQUIRE(src != nullptr || n_ctas == 0, "pg_halo_push_bns: null source");
  PG_REQUIRE(d > 0 && ld_src >= d, "pg_halo_push_bns: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int es = pg::elem_size(dtype);
  int vb = pg::vec_bytes(src, ld_src, es);
  vb = pg::common_vec(d, es, vb, {ld_src});
  const pg::DropArg da = pg::make_drop(drop);
  PG_REQUIRE(da.thresh16 == 0u || vb == 16, "pg_halo_push_bns: the dropout mask is defined on 16-byte vectors (rows must be 16-byte aligned)");
  const int nvec = static_cast<int>(pg::round_up(d, vb / es) / (vb / es));
  if (n_ctas > 0) {
#define PG_PUSH_BNS(T_, VB_) pg::halo_push_bns_kernel<T_, VB_><<<n_ctas, pg::kPushThreads, 0, st>>>(msgs, n_msgs, keys, static_cast<const T_*>(src), ld_src, nvec, value, value_dev, da, *s)
    if (dtype == PG_F32) {
      if (vb == 16) PG_PUSH_BNS(float, 16); else if (vb == 8) PG_PUSH_BNS(float, 8); else PG_PUSH_BNS(float, 4);
    } else if (dtype == PG_BF16) {
      if (vb == 16) PG_PUSH_BNS(__nv_bfloat16, 16); else if (vb == 8) PG_PUSH_BNS(__nv_bfloat16, 8);
      else if (vb == 4) PG_PUSH_BNS(__nv_bfloat16, 4);
      else { pg::set_error("pg_halo_push_bns: bf16 rows must be 4-byte aligned"); return PG_ERR_INVALID; }
    } else { pg::set_error("pg_halo_push_bns: unknown dtype %d", dtype); return PG_ERR_INVALID; }
#undef PG_PUSH_BNS
    PG_LAUNCH_CHECK();
  } else {      // every message is empty: nobody else publishes the flags
    pg::halo_flag_only_kernel<<<(n_msgs + 63) / 64, 64, 0, st>>>(msgs, n_msgs, value, value_dev);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

extern "C" int pg_boundary_add_bns(void* grad, int64_t ld_grad, const void* recv, int64_t ld_recv, int32_t d, int dtype,
                                   const int32_t* urow, const int32_t* uptr, const int32_t* usrc, int32_t n_urow,
                                   const int32_t* slot_keys, const pg_bns* s, void* stream) {
  pg::bns_preload();
  if (n_urow == 0) return PG_OK;
  PG_REQUIRE(grad && recv && urow && uptr && usrc && slot_keys && s, "pg_boundary_add_bns: null argument");
  PG_REQUIRE(d > 0 && ld_grad >= d && ld_recv >= d, "pg_boundary_add_bns: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int es = pg::elem_size(dtype);
  int vb = min(pg::vec_bytes(grad, ld_grad, es), pg::vec_bytes(recv, ld_recv, es));
  vb = pg::common_vec(d, es, vb, {ld_grad, ld_recv});
  const int v = vb / es;
  const int nvec = static_cast<int>(pg::round_up(d, v) / v);
  const unsigned blocks = (static_cast<unsigned>(n_urow) * 32u + 255u) / 256u;
#define PG_BADD(T_, VB_) pg::boundary_add_bns_kernel<T_, VB_><<<blocks, 256, 0, st>>>(static_cast<T_*>(grad), ld_grad, static_cast<const T_*>(recv), ld_recv, nvec, urow, uptr, usrc, n_urow, slot_keys, *s)
  if (dtype == PG_F32) {
    if (vb == 16) PG_BADD(float, 16); else if (vb == 8) PG_BADD(float, 8); else PG_BADD(float, 4);
  } else if (dtype == PG_BF16) {
    if (vb == 16) PG_BADD(__nv_bfloat16, 16); else if (vb == 8) PG_BADD(__nv_bfloat16, 8);
    else if (vb == 4) PG_BADD(__nv_bfloat16, 4);
    else { pg::set_error("pg_boundary_add_bns: bf16 rows must be 4-byte aligned"); return PG_ERR_INVALID; }
  } else { pg::set_error("pg_boundary_add_bns: unknown dtype %d", dtype); return PG_ERR_INVALID; }
#undef PG_BADD
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_bns_mask_rows(const void* src, int64_t ld_src, void* dst, int64_t ld_dst, int32_t n_rows, int32_t d,
                                int dtype, const uint8_t* mask, void* stream) {
  pg::bns_preload();
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(dst && mask, "pg_bns_mask_rows: null argument");
  PG_REQUIRE(n_rows > 0 && d > 0 && ld_dst >= d && (src == nullptr || ld_src >= d), "pg_bns_mask_rows: bad sizes");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int es = pg::elem_size(dtype);
  int vb = pg::vec_bytes(dst, ld_dst, es);
  if (src != nullptr) vb = min(vb, pg::vec_bytes(src, ld_src, es));
  vb = src != nullptr ? pg::common_vec(d, es, vb, {ld_src, ld_dst}) : pg::common_vec(d, es, vb, {ld_dst});
  const int v = vb / es;
  const int nvec = static_cast<int>(pg::round_up(d, v) / v);
  const int64_t total = static_cast<int64_t>(n_rows) * nvec;
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((total + 255) / 256, pg::sm_count() * 16));
#define PG_MASK(T_, VB_) pg::bns_mask_rows_kernel<T_, VB_><<<blocks, 256, 0, st>>>(static_cast<const T_*>(src), ld_src, static_cast<T_*>(dst), ld_dst, n_rows, nvec, mask)
  if (dtype == PG_F32) {
    if (vb == 16) PG_MASK(float, 16); else if (vb == 8) PG_MASK(float, 8); else PG_MASK(float, 4);
  } else if (dtype == PG_BF16) {
    if (vb == 16) PG_MASK(__nv_bfloat16, 16); else if (vb == 8) PG_MASK(__nv_bfloat16, 8);
    else if (vb == 4) PG_MASK(__nv_bfloat16, 4); else PG_MASK(__nv_bfloat16, 2);
  } else { pg::set_error("pg_bns_mask_rows: unknown dtype %d", dtype); return PG_ERR_INVALID; }
#undef PG_MASK
  PG_LAUNCH_CHECK();
  return PG_OK;
}

// ---- quantised halo messages (--halo-bits) ----------------------------------------------------
// A lane owns chunks of 8 consecutive elements: 8 codes are 8 bytes (8-bit) or 4 bytes (4-bit), one vector store.
namespace pg {
constexpr int kQChunk = 8;

// elements [e0, e0 + 8) of a row; VEC: 16-byte loads (the row is 16-byte aligned and padded to 8 elements),
// else scalar loads of the elements < d.  Elements >= d read as 0.
template <typename T, bool VEC>
__device__ __forceinline__ void load8(const T* p, int e0, int d, float (&f)[kQChunk]) {
  if constexpr (VEC) {
    using P = Pack<T, 16>;
#pragma unroll
    for (int h = 0; h < kQChunk / P::V; ++h)
      P::unpack(*reinterpret_cast<const typename P::Raw*>(p + e0 + h * P::V), f + h * P::V);
#pragma unroll
    for (int i = 0; i < kQChunk; ++i) if (e0 + i >= d) f[i] = 0.f;
  } else {
#pragma unroll
    for (int i = 0; i < kQChunk; ++i) {
      float x = 0.f;
      if (e0 + i < d) {
        if constexpr (sizeof(T) == 2) x = __bfloat162float(p[e0 + i]);
        else x = p[e0 + i];
      }
      f[i] = x;
    }
  }
}
// the inverse; VEC stores the whole chunk (the caller keeps elements >= d as they were)
template <typename T, bool VEC>
__device__ __forceinline__ void store8(T* p, int e0, int d, const float (&f)[kQChunk]) {
  if constexpr (VEC) {
    using P = Pack<T, 16>;
#pragma unroll
    for (int h = 0; h < kQChunk / P::V; ++h) st_vec<16>(p + e0 + h * P::V, P::pack(f + h * P::V));
  } else {
#pragma unroll
    for (int i = 0; i < kQChunk; ++i) {
      if (e0 + i < d) {
        if constexpr (sizeof(T) == 2) p[e0 + i] = __float2bfloat16_rn(f[i]);
        else p[e0 + i] = f[i];
      }
    }
  }
}
template <typename T>
__device__ __forceinline__ float round_to(float x) {
  if constexpr (sizeof(T) == 2) return __bfloat162float(__float2bfloat16_rn(x));
  else return x;
}

template <int BITS> struct Codes;
template <> struct Codes<8> {
  using Raw = uint2;
  __device__ __forceinline__ static Raw pack(const uint32_t (&q)[kQChunk]) {
    return make_uint2(q[0] | q[1] << 8 | q[2] << 16 | q[3] << 24, q[4] | q[5] << 8 | q[6] << 16 | q[7] << 24);
  }
  __device__ __forceinline__ static uint32_t get(const Raw& r, int i) { return ((i < 4 ? r.x : r.y) >> (8 * (i & 3))) & 0xffu; }
};
template <> struct Codes<4> {
  using Raw = uint32_t;
  __device__ __forceinline__ static Raw pack(const uint32_t (&q)[kQChunk]) {
    uint32_t w = 0u;
#pragma unroll
    for (int i = 0; i < kQChunk; ++i) w |= q[i] << (4 * i);     // even element in the low nibble of its byte
    return w;
  }
  __device__ __forceinline__ static uint32_t get(const Raw& r, int i) { return (r >> (4 * i)) & 0xfu; }
};

// the decoded chunk c of a code row (elements >= d: 0)
template <int BITS>
__device__ __forceinline__ void decode8(const uint8_t* row, float2 ls, int c, int d, float (&f)[kQChunk]) {
  using Cd = Codes<BITS>;
  const typename Cd::Raw r = *reinterpret_cast<const typename Cd::Raw*>(row + c * (kQChunk * BITS / 8));
#pragma unroll
  for (int i = 0; i < kQChunk; ++i)
    f[i] = (c * kQChunk + i < d) ? __fadd_rn(ls.x, __fmul_rn(static_cast<float>(Cd::get(r, i)), ls.y)) : 0.f;
}
// mirror <- m * mirror + (1 - m) * f (feature_buffer.py:189-191, two roundings), f <- mirror
__device__ __forceinline__ void ema8(float* mp, float m, float one_minus, float (&f)[kQChunk]) {
  float4* p4 = reinterpret_cast<float4*>(mp);
  float4 a = p4[0], b = p4[1];
  float e[kQChunk] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < kQChunk; ++i) f[i] = __fadd_rn(__fmul_rn(e[i], m), __fmul_rn(one_minus, f[i]));
  p4[0] = make_float4(f[0], f[1], f[2], f[3]);
  p4[1] = make_float4(f[4], f[5], f[6], f[7]);
}

template <typename T, int BITS, bool VEC>
__global__ void __launch_bounds__(kPushThreads)
halo_push_q_kernel(const pg_msg* __restrict__ msgs, int n_msgs, const pg_qmsg* __restrict__ qmsgs,
                   const T* __restrict__ src, int64_t ld_src, int d, uint32_t value,
                   const uint32_t* __restrict__ value_dev, pg_quant q) {
  if (value_dev != nullptr) value += *value_dev;
  int m = 0;
  while (m + 1 < n_msgs && static_cast<int>(blockIdx.x) >= msgs[m + 1].cta_begin) ++m;
  // the fields of message m one by one (a copy of the whole descriptor would go through local memory)
  const pg_msg& msg = msgs[m];
  const int32_t* idx = msg.idx;
  const int64_t src_row0 = msg.src_row0, ld_dst = msg.ld_dst, dst_row0 = msg.dst_row0;
  uint8_t* const dst = static_cast<uint8_t*>(msg.dst);
  const uint32_t key = quant_key(q.seed, static_cast<uint32_t>(q.stream), value, static_cast<uint32_t>(qmsgs[m].rank));
  float2* pairs = reinterpret_cast<float2*>(qmsgs[m].pairs);
  const int row0 = (static_cast<int>(blockIdx.x) - msg.cta_begin) * kPushRows;
  const int n_rows = msg.n_rows;
  const int row1 = min(n_rows, row0 + kPushRows);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nch = (d + kQChunk - 1) / kQChunk;
  constexpr float qmax = static_cast<float>((1 << BITS) - 1);
  using Cd = Codes<BITS>;

  for (int r = row0 + warp; r < row1; r += kPushThreads / 32) {
    const int64_t srow = idx ? static_cast<int64_t>(__ldg(idx + r)) : src_row0 + r;
    const T* sp = src + srow * ld_src;
    float lo = INFINITY, hi = -INFINITY;
    bool bad = false;
    for (int c = lane; c < nch; c += 32) {
      float f[kQChunk];
      load8<T, VEC>(sp, c * kQChunk, d, f);
#pragma unroll
      for (int i = 0; i < kQChunk; ++i) {
        if (c * kQChunk + i < d) {
          lo = fminf(lo, f[i]);
          hi = fmaxf(hi, f[i]);
          bad |= !isfinite(f[i]);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    bad = __any_sync(0xffffffffu, bad);
    const float range = __fsub_rn(hi, lo);
    float scale = __fdiv_rn(range, qmax);
    const float inv = __fdiv_rn(qmax, range);                                  // (x - lo) / scale as (x - lo) * inv
    if (bad || !isfinite(scale)) lo = scale = __int_as_float(0x7fc00000);      // NaN: the row decodes to NaN
    const bool coded = scale > 0.f && isfinite(inv);                           // false: constant / NaN rows, q = 0
    const uint32_t rk = quant_row_key(key, static_cast<uint32_t>(dst_row0 + r));
    uint8_t* dp = dst + static_cast<int64_t>(r) * ld_dst;
    for (int c = lane; c < nch; c += 32) {
      float f[kQChunk];
      load8<T, VEC>(sp, c * kQChunk, d, f);
      uint32_t qs[kQChunk];
#pragma unroll
      for (int i = 0; i < kQChunk; ++i) {
        const int e = c * kQChunk + i;
        float t = 0.f;
        if (coded && e < d)
          t = fminf(fmaxf(floorf(__fadd_rn(__fmul_rn(__fsub_rn(f[i], lo), inv), quant_u(rk, static_cast<uint32_t>(e)))), 0.f), qmax);
        qs[i] = static_cast<uint32_t>(t);
      }
      *reinterpret_cast<typename Cd::Raw*>(dp + c * (kQChunk * BITS / 8)) = Cd::pack(qs);
    }
    if (lane == 0) pairs[r] = make_float2(lo, scale);
  }

  // flags exactly as halo_push_kernel publishes them
  if (blockIdx.x == 0 && static_cast<int>(threadIdx.x) < n_msgs) {
    const pg_msg& em = msgs[threadIdx.x];
    if (em.n_rows == 0 && em.flag != nullptr) st_release_sys(em.flag, value);
  }
  if (msg.flag != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const int n_ctas = (n_rows + kPushRows - 1) / kPushRows;
      __threadfence_system();
      const unsigned prev = atomicAdd(msg.counter, 1u);
      if (prev == static_cast<unsigned>(n_ctas - 1)) {
        *msg.counter = 0u;
        __threadfence_system();
        st_release_sys(msg.flag, value);
      }
    }
  }
}

// one warp per row: decode, (EMA), (dropout), store in the activation dtype
template <typename T, int BITS>
__global__ void __launch_bounds__(256)
halo_dequant_kernel(const uint8_t* __restrict__ codes, int64_t ld_codes, const float2* __restrict__ pairs, int n_rows,
                    int d, T* __restrict__ out, int64_t ld_out, float* __restrict__ mirror, int64_t ld_mirror,
                    float momentum, float one_minus, DropArg drop, int64_t drop_row0) {
  const uint32_t drop_hi = drop_seed_hi(drop);
  using P = Pack<T, 16>;
  constexpr int V = P::V;                            // elements per 16-byte vector: the dropout mask's unit
  const int nvec = (d + V - 1) / V;
  const int nch = (d + kQChunk - 1) / kQChunk;
  const int lane = threadIdx.x & 31;
  const int64_t nw = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t r = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; r < n_rows; r += nw) {
    const float2 ls = __ldg(pairs + r);
    const uint8_t* cr = codes + r * ld_codes;
    for (int c = lane; c < nch; c += 32) {
      float f[kQChunk];
      decode8<BITS>(cr, ls, c, d, f);
      if (mirror != nullptr) ema8(mirror + r * ld_mirror + c * kQChunk, momentum, one_minus, f);
      if (drop.thresh16 != 0u) {                   // what pg_dropout_rows makes of the stored (rounded) row
#pragma unroll
        for (int i = 0; i < kQChunk; ++i) f[i] = round_to<T>(f[i]);
#pragma unroll
        for (int h = 0; h < kQChunk / V; ++h) {
          float g[V];
#pragma unroll
          for (int i = 0; i < V; ++i) g[i] = f[h * V + i];
          drop_apply<V>(g, static_cast<uint64_t>(drop_row0 + r) * nvec + c * (kQChunk / V) + h, drop.thresh16, drop.scale,
                        drop.seed_lo, drop_hi);
#pragma unroll
          for (int i = 0; i < V; ++i) f[h * V + i] = g[i];
        }
      }
#pragma unroll
      for (int i = 0; i < kQChunk; ++i) if (c * kQChunk + i >= d) f[i] = 0.f;
      store8<T, true>(out + r * ld_out, c * kQChunk, d, f);
    }
  }
}

template <typename T, int BITS, bool VEC>
__global__ void __launch_bounds__(256)
boundary_add_q_kernel(T* __restrict__ grad, int64_t ld_grad, int d, const uint8_t* __restrict__ codes, int64_t ld_codes,
                      const float2* __restrict__ pairs, const int32_t* __restrict__ urow, const int32_t* __restrict__ uptr,
                      const int32_t* __restrict__ usrc, int n_urow, float* __restrict__ mirror, int64_t ld_mirror,
                      float momentum, float one_minus) {
  const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (w >= n_urow) return;
  T* gp = grad + static_cast<int64_t>(__ldg(urow + w)) * ld_grad;
  const int k0 = __ldg(uptr + w), k1 = __ldg(uptr + w + 1);
  const int nch = (d + kQChunk - 1) / kQChunk;
  for (int c = lane; c < nch; c += 32) {
    float g[kQChunk];
    if constexpr (VEC) {                             // the padding columns are stored back as they were
      using P = Pack<T, 16>;
#pragma unroll
      for (int h = 0; h < kQChunk / P::V; ++h)
        P::unpack(*reinterpret_cast<const typename P::Raw*>(gp + c * kQChunk + h * P::V), g + h * P::V);
    } else {
      load8<T, false>(gp, c * kQChunk, d, g);
    }
    for (int k = k0; k < k1; ++k) {
      const int s = __ldg(usrc + k);
      float f[kQChunk];
      decode8<BITS>(codes + static_cast<int64_t>(s) * ld_codes, __ldg(pairs + s), c, d, f);
      if (mirror != nullptr) ema8(mirror + static_cast<int64_t>(s) * ld_mirror + c * kQChunk, momentum, one_minus, f);
#pragma unroll
      for (int i = 0; i < kQChunk; ++i)
        if (c * kQChunk + i < d) g[i] = round_to<T>(__fadd_rn(g[i], round_to<T>(f[i])));
    }
    store8<T, VEC>(gp, c * kQChunk, d, g);
  }
}

// see bns_preload: no first launch of a quantised-path kernel may happen while a flag wait spins
static void quant_preload() {
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncAttributes a;
#define PG_LOAD(F) cudaFuncGetAttributes(&a, F)
#define PG_LOAD_TB(K, T_, B_) PG_LOAD((K<T_, B_, true>)); PG_LOAD((K<T_, B_, false>))
    PG_LOAD_TB(halo_push_q_kernel, float, 8); PG_LOAD_TB(halo_push_q_kernel, float, 4);
    PG_LOAD_TB(halo_push_q_kernel, __nv_bfloat16, 8); PG_LOAD_TB(halo_push_q_kernel, __nv_bfloat16, 4);
    PG_LOAD_TB(boundary_add_q_kernel, float, 8); PG_LOAD_TB(boundary_add_q_kernel, float, 4);
    PG_LOAD_TB(boundary_add_q_kernel, __nv_bfloat16, 8); PG_LOAD_TB(boundary_add_q_kernel, __nv_bfloat16, 4);
    PG_LOAD((halo_dequant_kernel<float, 8>)); PG_LOAD((halo_dequant_kernel<float, 4>));
    PG_LOAD((halo_dequant_kernel<__nv_bfloat16, 8>)); PG_LOAD((halo_dequant_kernel<__nv_bfloat16, 4>));
    PG_LOAD(halo_flag_only_kernel);
#undef PG_LOAD_TB
#undef PG_LOAD
    cudaGetLastError();
  });
}

// 16-byte aligned rows padded to a multiple of 8 elements: the vector path of load8 / store8
static bool rows8(const void* p, int64_t ld, int d, int es) {
  return vec_bytes(p, ld, es) == 16 && ld >= round_up(d, kQChunk);
}
static int64_t code_bytes(int d, int bits) { return round_up(static_cast<int64_t>(d) * bits, 8) / 8; }
}  // namespace pg

extern "C" int pg_halo_push_q(const pg_msg* msgs, int32_t n_msgs, int32_t n_ctas, const pg_qmsg* qmsgs, const void* src,
                              int64_t ld_src, int32_t d, int dtype, uint32_t value, const uint32_t* value_dev,
                              const pg_quant* q, void* stream) {
  pg::quant_preload();
  PG_REQUIRE(msgs && n_msgs > 0 && n_msgs <= pg::kPushThreads, "pg_halo_push_q: 1..%d messages per launch", pg::kPushThreads);
  PG_REQUIRE(qmsgs != nullptr && q != nullptr && (q->bits == 8 || q->bits == 4), "pg_halo_push_q: bad quantiser");
  PG_REQUIRE(src != nullptr || n_ctas == 0, "pg_halo_push_q: null source");
  PG_REQUIRE(d > 0 && ld_src >= d, "pg_halo_push_q: bad sizes");
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_halo_push_q: unknown dtype %d", dtype);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (n_ctas > 0) {
    const bool vec = pg::rows8(src, ld_src, d, pg::elem_size(dtype));
#define PG_PUSH_Q(T_, B_, V_) pg::halo_push_q_kernel<T_, B_, V_><<<n_ctas, pg::kPushThreads, 0, st>>>(msgs, n_msgs, qmsgs, static_cast<const T_*>(src), ld_src, d, value, value_dev, *q)
#define PG_PUSH_QB(T_, B_) do { if (vec) PG_PUSH_Q(T_, B_, true); else PG_PUSH_Q(T_, B_, false); } while (0)
    if (dtype == PG_F32) { if (q->bits == 8) PG_PUSH_QB(float, 8); else PG_PUSH_QB(float, 4); }
    else { if (q->bits == 8) PG_PUSH_QB(__nv_bfloat16, 8); else PG_PUSH_QB(__nv_bfloat16, 4); }
#undef PG_PUSH_QB
#undef PG_PUSH_Q
    PG_LAUNCH_CHECK();
  } else {      // every message is empty: nobody else publishes the flags
    pg::halo_flag_only_kernel<<<(n_msgs + 63) / 64, 64, 0, st>>>(msgs, n_msgs, value, value_dev);
    PG_LAUNCH_CHECK();
  }
  return PG_OK;
}

extern "C" int pg_halo_dequant(const uint8_t* codes, int64_t ld_codes, const float* pairs, int32_t n_rows, int32_t d,
                               int32_t bits, void* out, int64_t ld_out, int dtype, float* mirror, int64_t ld_mirror,
                               float momentum, float one_minus, const pg_drop* drop, int64_t drop_row0, void* stream) {
  pg::quant_preload();
  if (n_rows == 0) return PG_OK;
  PG_REQUIRE(codes && pairs && out && n_rows > 0 && d > 0 && (bits == 8 || bits == 4), "pg_halo_dequant: bad arguments");
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_halo_dequant: unknown dtype %d", dtype);
  PG_REQUIRE(ld_codes >= pg::code_bytes(d, bits) && ld_codes % 16 == 0 && reinterpret_cast<uintptr_t>(codes) % 16 == 0 &&
             reinterpret_cast<uintptr_t>(pairs) % 8 == 0, "pg_halo_dequant: code rows must be 16-byte aligned and padded");
  PG_REQUIRE(pg::rows8(out, ld_out, d, pg::elem_size(dtype)), "pg_halo_dequant: out rows must be 16-byte aligned and padded to 8 elements");
  PG_REQUIRE(mirror == nullptr || pg::rows8(mirror, ld_mirror, d, 4), "pg_halo_dequant: mirror rows must be 16-byte aligned and padded to 8");
  const pg::DropArg da = pg::make_drop(drop);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned blocks = static_cast<unsigned>(std::min<int64_t>((static_cast<int64_t>(n_rows) * 32 + 255) / 256, pg::sm_count() * 16));
  const float2* pp = reinterpret_cast<const float2*>(pairs);
#define PG_DEQ(T_, B_) pg::halo_dequant_kernel<T_, B_><<<blocks, 256, 0, st>>>(codes, ld_codes, pp, n_rows, d, static_cast<T_*>(out), ld_out, mirror, ld_mirror, momentum, one_minus, da, drop_row0)
  if (dtype == PG_F32) { if (bits == 8) PG_DEQ(float, 8); else PG_DEQ(float, 4); }
  else { if (bits == 8) PG_DEQ(__nv_bfloat16, 8); else PG_DEQ(__nv_bfloat16, 4); }
#undef PG_DEQ
  PG_LAUNCH_CHECK();
  return PG_OK;
}

extern "C" int pg_boundary_add_q(void* grad, int64_t ld_grad, int32_t d, int dtype, const uint8_t* codes, int64_t ld_codes,
                                 const float* pairs, int32_t bits, const int32_t* urow, const int32_t* uptr,
                                 const int32_t* usrc, int32_t n_urow, float* mirror, int64_t ld_mirror, float momentum,
                                 float one_minus, void* stream) {
  pg::quant_preload();
  if (n_urow == 0) return PG_OK;
  PG_REQUIRE(grad && codes && pairs && urow && uptr && usrc && (bits == 8 || bits == 4), "pg_boundary_add_q: null argument");
  PG_REQUIRE(dtype == PG_F32 || dtype == PG_BF16, "pg_boundary_add_q: unknown dtype %d", dtype);
  PG_REQUIRE(d > 0 && ld_grad >= d, "pg_boundary_add_q: bad sizes");
  PG_REQUIRE(ld_codes >= pg::code_bytes(d, bits) && ld_codes % 16 == 0 && reinterpret_cast<uintptr_t>(codes) % 16 == 0 &&
             reinterpret_cast<uintptr_t>(pairs) % 8 == 0, "pg_boundary_add_q: code rows must be 16-byte aligned and padded");
  PG_REQUIRE(mirror == nullptr || pg::rows8(mirror, ld_mirror, d, 4), "pg_boundary_add_q: mirror rows must be 16-byte aligned and padded to 8");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = pg::rows8(grad, ld_grad, d, pg::elem_size(dtype));
  const unsigned blocks = (static_cast<unsigned>(n_urow) * 32u + 255u) / 256u;
  const float2* pp = reinterpret_cast<const float2*>(pairs);
#define PG_BADD_Q(T_, B_, V_) pg::boundary_add_q_kernel<T_, B_, V_><<<blocks, 256, 0, st>>>(static_cast<T_*>(grad), ld_grad, d, codes, ld_codes, pp, urow, uptr, usrc, n_urow, mirror, ld_mirror, momentum, one_minus)
#define PG_BADD_QB(T_, B_) do { if (vec) PG_BADD_Q(T_, B_, true); else PG_BADD_Q(T_, B_, false); } while (0)
  if (dtype == PG_F32) { if (bits == 8) PG_BADD_QB(float, 8); else PG_BADD_QB(float, 4); }
  else { if (bits == 8) PG_BADD_QB(__nv_bfloat16, 8); else PG_BADD_QB(__nv_bfloat16, 4); }
#undef PG_BADD_QB
#undef PG_BADD_Q
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
