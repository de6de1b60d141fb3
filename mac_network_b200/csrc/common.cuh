// Shared device/host helpers for libmac_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include "../../include/mac_b200.h"

#define MAC_CUDA_TRY(expr)                          \
  do {                                              \
    cudaError_t _e = (expr);                        \
    if (_e != cudaSuccess) return (int)_e;          \
  } while (0)
// every kernel launch of the library goes through this: counts it (mac_b200_launch_count) and surfaces launch errors
extern "C" void mac_b200_count_launch_(void);
#define MAC_LAUNCH_CHECK()                          \
  do {                                              \
    mac_b200_count_launch_();                       \
    cudaError_t _e = cudaGetLastError();            \
    if (_e != cudaSuccess) return (int)_e;          \
  } while (0)

static inline bool mac_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// SM count of the current device (cached per device ordinal): the grid-sizing heuristics aim at ~2 CTAs per SM
static inline int mac_num_sms() {
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return sms[dev];
}

namespace mac {

// ------------------------------------------------------------------ activations (ops.py:161-187)
__device__ __forceinline__ float elu_f(float x) { return x > 0.f ? x : expm1f(x); }
__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ float apply_act(int act, float x) {
  switch (act) {
    case MAC_ACT_TANH: return tanhf(x);
    case MAC_ACT_SIGMOID: return sigmoid_f(x);
    case MAC_ACT_ELU: return elu_f(x);
    case MAC_ACT_RELU: return fmaxf(x, 0.f);
    default: return x;
  }
}

// ------------------------------------------------------------------ warp / block reductions
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------ Philox4x32-10 (counter-based dropout RNG)
// counter = (elem/4 lo, elem/4 hi, site, step), key = seed.  u = (x >> 8) * 2^-24 in [0,1).
// keep-mask = [u >= 1 - keep]  (== floor(keep + u), ops.py:1054-1059 / tf.nn.dropout), evaluated on the 24-bit
// integer so that fp32 and the fp64 oracle agree bit-for-bit.
struct Philox4 { uint32_t x, y, z, w; };
__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}
__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint64_t seed, uint64_t idx4, uint32_t site, uint32_t step) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)idx4, c1 = (uint32_t)(idx4 >> 32), c2 = site, c3 = step;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = mulhi32(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = mulhi32(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
__host__ __device__ __forceinline__ uint32_t keep_threshold(float keep) {
  // smallest 24-bit integer t with t * 2^-24 >= 1 - keep (computed in double on either side)
  double thr = (1.0 - (double)keep) * 16777216.0;
  double c = (double)(uint32_t)thr;
  if (c < thr) c += 1.0;
  return (uint32_t)c;
}

// ------------------------------------------------------------------ mbarrier / bulk-copy PTX (TMA engine)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {}
}
// 1-D bulk async copy global -> shared (SASS: UBLKCP); size multiple of 16, both addresses 16-B aligned
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// 2-D tiled TMA load (SASS: UTMALDG)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(smem_dst)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

}  // namespace mac
