// The cell's M <= 128 projections on tensor cores (ops.linear at mac_cell.py:442-448 qInput / qInput{i}, 322 ctrlProj,
// 352 newMemory, 363 gate; ops.py:689 projY):
//
//     Y[M, N] = epilogue( concat_k(x_0 .. x_{nseg-1})[M, K] @ W[K, N] )        M <= 128 (the batch), fp32 in, fp32 out
//
// These are latency problems (33-100 MFLOP against 0.5-2 MB of weights), and they sit on the recurrent state path, so
// they must not lose the state's precision to bf16: the activations are split on the fly into bf16 hi + lo parts and the
// weights are pre-split the same way (mac_pack_weight_bf16_split), and three wgmma products accumulate into one fp32
// accumulator,
//     D = A_hi B_hi + A_lo B_hi + A_hi B_lo        (the dropped A_lo B_lo term is ~2^-18 relative),
// which keeps the result at fp32-class accuracy (~1e-5) while the MACs run on the tensor pipe (wgmma 64 x BN x 16).
// With wt_lo == NULL it is a plain single-pass bf16 product.
//
// One CTA per BN output columns (BN = 32 / 64 -> 16..96 CTAs pull the weights from L2 in parallel).  Roles:
//   warp 8           TMA producer: weight k-blocks [BN x 64] (hi and lo) through a 6-stage ring
//   warpgroups 0, 1  workers: load the fp32 activation k-block [M x 64] with 16-byte loads -- the loads of k-block i+2 are
//                    in flight while k-block i is split into bf16 hi / lo and written in the 128-byte-swizzled K-major layout
//                    (4-stage ring) -- then warpgroup g issues the products of rows [64 g, 64 g + 64) and finally runs the
//                    epilogue of those rows from its accumulator registers (bias, activation / write gate, column split of
//                    the folded write unit).
#pragma once
#include "tc_gemm.cuh"

namespace mac {

constexpr int ST_A_STAGES = 4;
constexpr int ST_B_STAGES = 6;
constexpr int ST_WORKERS = 256;
constexpr int ST_THREADS = ST_WORKERS + 32;
constexpr int ST_F4 = 128 * 16 / ST_WORKERS;  // float4 groups per worker thread and k-block at M = 128
constexpr int ST_A_TILE = 128 * 128;          // [128 rows x 64 bf16]

struct SkinnyTcParams {
  const float* a[4];
  int ak[4];
  int lda[4];
  int nseg;
  int M, N, K;
  int split;               // 1: hi/lo three-pass product
  const float* bias;       // [N] or NULL
  float bias_const;
  int act;
  float* Y;
  int ldy;
  float* Y2;               // columns >= n_split go to Y2[m, n - n_split] (same ldy) when Y2 != NULL
  int n_split;
  const float* gnew;       // write gate (mac_cell.py:358-367) when != NULL: z = sigmoid(t); Y = gnew*z + gold*(1-z)
  const float* gold;
  float* gate_z;
};

template <int BN>
struct StCfg {
  static constexpr int B_TILE = BN * 128;                                 // [BN rows x 64 bf16]
  static constexpr int A_BYTES = ST_A_STAGES * 2 * ST_A_TILE;             // hi + lo per stage
  static constexpr int B_BYTES = ST_B_STAGES * 2 * B_TILE;
  static constexpr int SMEM_BYTES = A_BYTES + B_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};

__device__ __forceinline__ uint32_t bf16_bits_rn(float x) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(x));
}

template <int BN>
__device__ __forceinline__ void wgmma_bf16_bn(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (BN == 64) wgmma_bf16_n64(d, adesc, bdesc, accum);
  else wgmma_bf16_n32(d, adesc, bdesc, accum);
}

// SPLIT: the three-pass hi / lo product (p.split); a template parameter so that the wgmma sequence has no data-dependent branch
template <int BN, bool SPLIT>
__global__ void __launch_bounds__(ST_THREADS, 1)
skinny_tc_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo, const SkinnyTcParams p) {
  using C = StCfg<BN>;
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  const uint32_t pad = (1024u - (base_u32 & 1023u)) & 1023u;
  unsigned char* a_tiles = smem_dyn + pad;                       // [stage][hi | lo]
  unsigned char* b_tiles = a_tiles + C::A_BYTES;                 // [stage][hi | lo]
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_tiles + C::B_BYTES);
  uint64_t* b_full = bars;                         // [6] TMA -> workers
  uint64_t* b_empty = bars + ST_B_STAGES;          // [6] workers -> TMA (8 warp arrivals)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN;
  const int kblocks = p.K / TC_BK;
  const int passes_bytes = (p.split ? 2 : 1) * C::B_TILE;

  if (threadIdx.x == ST_WORKERS) {
    tma_prefetch_desc(&map_hi);
    if (p.split) tma_prefetch_desc(&map_lo);
#pragma unroll
    for (int i = 0; i < ST_B_STAGES; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], ST_WORKERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == ST_WORKERS / 32) {
    if (elect_one()) {
      for (int kb = 0; kb < kblocks; ++kb) {
        const int s = kb % ST_B_STAGES, n = kb / ST_B_STAGES;
        mbar_wait(&b_empty[s], (n & 1) ^ 1);
        mbar_expect_tx(&b_full[s], passes_bytes);
        unsigned char* dst = b_tiles + s * 2 * C::B_TILE;
        tma_load_2d(dst, &map_hi, kb * TC_BK, n0, &b_full[s]);
        if (p.split) tma_load_2d(dst + C::B_TILE, &map_lo, kb * TC_BK, n0, &b_full[s]);
      }
    }
    return;
  }

  // ===================================================== workers: activation split + products, then the epilogue
  const int wt = threadIdx.x;                      // 0..255
  const int g = warp >> 2;                         // warpgroup: rows [64 g, 64 g + 64)
  const int nf4 = p.M * 16;                        // float4 groups of one [M x 64] k-block
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  // k-block -> (segment pointer at that k, leading dimension)
  auto kb_src = [&](int kb, int& ld) -> const float* {
    int k0 = kb * TC_BK, sg = 0;
    while (sg + 1 < p.nseg && k0 >= p.ak[sg]) { k0 -= p.ak[sg]; ++sg; }
    ld = p.lda[sg];
    return p.a[sg] + k0;
  };
  auto load_kb = [&](int kb, float4 (&v)[ST_F4]) {
    int ld;
    const float* src = kb_src(kb, ld);
#pragma unroll
    for (int i = 0; i < ST_F4; ++i) {
      const int e = wt + ST_WORKERS * i;
      if (e < nf4) {
        const uint4 u = ldg_nc_v4(src + (size_t)(e >> 4) * ld + (e & 15) * 4);
        v[i] = make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
      }
    }
  };
  // Stage reuse: the A slot of k-block kb was last read by the products of kb - 4; every worker has passed the named
  // barrier of kb - 1 only after its wait_group(1) retired the products of kb - 2 and earlier.
  auto step_kb = [&](int kb, const float4 (&v)[ST_F4]) {
    const int sa = kb % ST_A_STAGES;
    unsigned char* t_hi = a_tiles + sa * 2 * ST_A_TILE;
    unsigned char* t_lo = t_hi + ST_A_TILE;
#pragma unroll
    for (int i = 0; i < ST_F4; ++i) {
      const int e = wt + ST_WORKERS * i;
      if (e < nf4) {
        const int row = e >> 4, f4 = e & 15;
        const uint32_t off = row * 128 + (((f4 >> 1) ^ (row & 7)) << 4) + (f4 & 1) * 8;
        const uint32_t h0 = bf16_bits_rn(v[i].x), h1 = bf16_bits_rn(v[i].y), h2 = bf16_bits_rn(v[i].z), h3 = bf16_bits_rn(v[i].w);
        *reinterpret_cast<uint2*>(t_hi + off) = make_uint2(h0 | (h1 << 16), h2 | (h3 << 16));
        if constexpr (SPLIT) {
          const uint32_t l0 = bf16_bits_rn(v[i].x - __uint_as_float(h0 << 16)), l1 = bf16_bits_rn(v[i].y - __uint_as_float(h1 << 16));
          const uint32_t l2 = bf16_bits_rn(v[i].z - __uint_as_float(h2 << 16)), l3 = bf16_bits_rn(v[i].w - __uint_as_float(h3 << 16));
          *reinterpret_cast<uint2*>(t_lo + off) = make_uint2(l0 | (l1 << 16), l2 | (l3 << 16));
        }
      }
    }
    fence_proxy_async();                                       // generic-proxy stores -> visible to wgmma
    asm volatile("bar.sync 1, %0;" ::"n"(ST_WORKERS) : "memory");
    const int sb = kb % ST_B_STAGES;
    mbar_wait(&b_full[sb], (kb / ST_B_STAGES) & 1);
    const uint32_t sa_u = smem_u32(t_hi) + g * (64 * 128), sb_u = smem_u32(b_tiles + sb * 2 * C::B_TILE);
    const uint64_t a_hi = make_sw128_kmajor_desc(sa_u), a_lo = make_sw128_kmajor_desc(sa_u + ST_A_TILE);
    const uint64_t b_hi = make_sw128_kmajor_desc(sb_u), b_lo = make_sw128_kmajor_desc(sb_u + C::B_TILE);
    // issued by both warpgroups whatever M is: rows at or above M hold stale data and are never stored
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_bn<BN>(acc, a_hi + 2 * k, b_hi + 2 * k, (kb | k) ? 1u : 0u);
    if constexpr (SPLIT) {
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_bn<BN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_bn<BN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (kb > 0 && lane == 0) mbar_arrive(&b_empty[(kb - 1) % ST_B_STAGES]);
  };
  // three register buffers rotate: k-blocks i+1 and i+2 are in flight while k-block i is converted
  float4 v0[ST_F4], v1[ST_F4], v2[ST_F4];
  load_kb(0, v0);
  if (kblocks > 1) load_kb(1, v1);
  for (int kb = 0; kb < kblocks; kb += 3) {
    if (kb + 2 < kblocks) load_kb(kb + 2, v2);
    step_kb(kb, v0);
    if (kb + 1 < kblocks) {
      if (kb + 3 < kblocks) load_kb(kb + 3, v0);
      step_kb(kb + 1, v1);
    }
    if (kb + 2 < kblocks) {
      if (kb + 4 < kblocks) load_kb(kb + 4, v1);
      step_kb(kb + 2, v2);
    }
  }
  wgmma_wait<0>();
  wgmma_hold(acc);

  // ---- epilogue: acc[4 j + 2 h + e] is row 64 g + 16 (warp & 3) + lane / 4 + 8 h, column 8 j + 2 (lane & 3) + e
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = 64 * g + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    if (row >= p.M) continue;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      float t0 = acc[4 * j + 2 * h] + p.bias_const, t1 = acc[4 * j + 2 * h + 1] + p.bias_const;
      if (p.bias) {
        t0 += __ldg(p.bias + n);
        t1 += __ldg(p.bias + n + 1);
      }
      const size_t o = (size_t)row * p.ldy + n;
      if (p.gnew) {
        const float2 gn = *reinterpret_cast<const float2*>(p.gnew + o), go = *reinterpret_cast<const float2*>(p.gold + o);
        const float z0 = sigmoid_f(t0), z1 = sigmoid_f(t1);
        if (p.gate_z) *reinterpret_cast<float2*>(p.gate_z + o) = make_float2(z0, z1);
        *reinterpret_cast<float2*>(p.Y + o) = make_float2(gn.x * z0 + go.x * (1.f - z0), gn.y * z1 + go.y * (1.f - z1));
      } else {
        float* dst = (p.Y2 && n >= p.n_split) ? p.Y2 + (size_t)row * p.ldy + (n - p.n_split) : p.Y + o;
        *reinterpret_cast<float2*>(dst) = make_float2(apply_act(p.act, t0), apply_act(p.act, t1));
      }
    }
  }
}

// wt_hi / wt_lo: bf16 [N, K] (K-major) halves of the fp32 weight (mac_pack_weight_bf16_split); wt_lo == NULL: single pass
inline int skinny_tc_launch(SkinnyTcParams p, const void* wt_hi, const void* wt_lo, cudaStream_t stream) {
  if (p.M <= 0 || p.M > 128 || p.N <= 0 || p.K <= 0 || p.nseg < 1 || p.nseg > 4) return MAC_ERR_INVALID;
  if ((p.N % 32) || (p.K % TC_BK) || (p.ldy & 3) || (p.Y2 && (p.n_split % 32))) return MAC_ERR_UNSUPPORTED;
  int ksum = 0;
  for (int i = 0; i < p.nseg; ++i) {
    if (!p.a[i] || p.ak[i] <= 0 || (p.ak[i] % TC_BK) || (p.lda[i] & 3)) return MAC_ERR_UNSUPPORTED;
    if (!mac_aligned16(p.a[i])) return MAC_ERR_ALIGN;
    ksum += p.ak[i];
  }
  if (ksum != p.K || !wt_hi || !p.Y || !mac_aligned16(p.Y) || !mac_aligned16(wt_hi)) return MAC_ERR_INVALID;
  p.split = wt_lo ? 1 : 0;
  const int BN = (p.N % 64 == 0 && p.N >= 1024) ? 64 : 32;
  CUtensorMap mhi, mlo;
  int st = make_tmap_2d(&mhi, wt_hi, 1, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K * 2, (uint32_t)BN, TC_BK, 1);
  if (st != MAC_OK) return st;
  if (wt_lo) {
    st = make_tmap_2d(&mlo, wt_lo, 1, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K * 2, (uint32_t)BN, TC_BK, 1);
    if (st != MAC_OK) return st;
  } else {
    mlo = mhi;
  }
  // the shared-memory opt-in belongs to the current device's context: set it on every launch
  auto launch = [&](auto kern, int bn, int smem) -> int {
    MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<p.N / bn, ST_THREADS, smem, stream>>>(mhi, mlo, p);
    return MAC_OK;
  };
  int rc;
  if (BN == 64)
    rc = p.split ? launch(skinny_tc_kernel<64, true>, 64, StCfg<64>::SMEM_BYTES) : launch(skinny_tc_kernel<64, false>, 64, StCfg<64>::SMEM_BYTES);
  else
    rc = p.split ? launch(skinny_tc_kernel<32, true>, 32, StCfg<32>::SMEM_BYTES) : launch(skinny_tc_kernel<32, false>, 32, StCfg<32>::SMEM_BYTES);
  if (rc != MAC_OK) return rc;
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// fp32 [K, N] (in, out) weight -> bf16 hi and lo halves, both [N, K] (out, in): W = hi + lo + O(2^-17 |W|)
__global__ void pack_weight_bf16_split_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ hi,
                                              __nv_bfloat16* __restrict__ lo, int K, int N) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? W[(size_t)k * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K) {
      const float w = tile[threadIdx.x][i];
      const __nv_bfloat16 h = __float2bfloat16_rn(w);
      hi[(size_t)n * K + k] = h;
      lo[(size_t)n * K + k] = __float2bfloat16_rn(w - __bfloat162float(h));
    }
  }
}

}  // namespace mac
