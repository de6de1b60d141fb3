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
// which keeps the result at fp32-class accuracy (~1e-5) while the MACs run on the tensor pipe.
// With wt_lo == NULL it is a plain single-pass bf16 product.
//
// One CTA per BN output columns (BN = 32 / 64 -> 16..96 CTAs pull the weights from L2 in parallel).  Roles:
//   warp 8           TMA producer: per k-block, the fp32 activation block [MR x 64] (MR = 64 at M <= 64, else 128; one
//                    2-D tensor map per segment, rows past M zero-filled) into a ring of its own, and the weight block
//                    [BN x 64] (hi and lo) into the weight ring
//   warpgroups 0, 1  workers: split the fp32 block from shared memory into bf16 hi / lo, written in the 128-byte-swizzled
//                    K-major layout (3-stage ring), then issue the products: at M <= 64 warpgroup g takes columns
//                    [g BN/2, (g + 1) BN/2) of all 64 rows (m64 n(BN/2) k16), above 64 rows [64 g, 64 g + 64) of all BN
//                    columns; finally each runs the epilogue of its accumulator (bias, activation / write gate, column
//                    split of the folded write unit).
// The workers issue no global load inside the k loop, so the proxy fence before the products orders shared-memory stores
// only, and the ring depth alone decides how far the loads run ahead.
#pragma once
#include "tc_gemm.cuh"

namespace mac {

constexpr int ST_A16_STAGES = 3;   // bf16 hi / lo tiles: the slot of k-block kb was last read by the products of kb - 3
constexpr int ST_WORKERS = 256;
constexpr int ST_THREADS = ST_WORKERS + 32;
constexpr int ST_MAX_STAGES = 6;

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
  int mrows;               // rows of one activation block: 64 (M <= 64) or 128
  int a_stages, b_stages;  // depths of the fp32 activation ring and the weight ring (<= ST_MAX_STAGES)
};

// weight halves and one fp32 activation map per segment ({ak, M}, row stride lda * 4, box {64, mrows})
struct SkinnyTcMaps {
  CUtensorMap w_hi, w_lo;
  CUtensorMap a[4];
};

// shared-memory layout (bytes after the 1024-byte alignment): bf16 A ring | weight ring | fp32 A ring | barriers
struct StLayout {
  int a16_tile, b_tile, a32_stage;
  int b_off, a32_off, bar_off, smem_bytes;
  __host__ __device__ StLayout(int bn, int mrows, int a_stages, int b_stages) {
    a16_tile = mrows * 128;                        // [mrows x 64 bf16]
    b_tile = bn * 128;                             // [BN x 64 bf16]
    a32_stage = mrows * 256;                       // [mrows x 64 fp32]
    b_off = ST_A16_STAGES * 2 * a16_tile;
    a32_off = b_off + b_stages * 2 * b_tile;
    bar_off = a32_off + a_stages * a32_stage;
    smem_bytes = bar_off + 1024 /*align*/ + 256 /*barriers*/;
  }
};

__device__ __forceinline__ uint32_t bf16_bits_rn(float x) {
  return (uint32_t)__bfloat16_as_ushort(__float2bfloat16_rn(x));
}

__device__ __forceinline__ void wgmma_bf16_n16(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

template <int WN>
__device__ __forceinline__ void wgmma_bf16_w(float (&d)[WN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  if constexpr (WN == 64) wgmma_bf16_n64(d, adesc, bdesc, accum);
  else if constexpr (WN == 32) wgmma_bf16_n32(d, adesc, bdesc, accum);
  else wgmma_bf16_n16(d, adesc, bdesc, accum);
}

// SPLIT: the three-pass hi / lo product (p.split); COLS: M <= 64, the warpgroups split the columns.  Both are template
// parameters so that the wgmma sequence has no data-dependent branch.
template <int BN, bool SPLIT, bool COLS>
__global__ void __launch_bounds__(ST_THREADS, 1)
skinny_tc_kernel(const __grid_constant__ SkinnyTcMaps maps, const SkinnyTcParams p) {
  constexpr int WN = COLS ? BN / 2 : BN;           // columns of one warpgroup's products
  const StLayout L(BN, p.mrows, p.a_stages, p.b_stages);
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  const uint32_t pad = (1024u - (base_u32 & 1023u)) & 1023u;
  unsigned char* a16 = smem_dyn + pad;                           // [stage][hi | lo]
  unsigned char* b_tiles = a16 + L.b_off;                        // [stage][hi | lo]
  unsigned char* a32 = a16 + L.a32_off;                          // [stage] fp32 [mrows x 64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(a16 + L.bar_off);
  uint64_t* b_full = bars;                                       // TMA -> workers
  uint64_t* b_empty = bars + ST_MAX_STAGES;                      // workers -> TMA (8 warp arrivals)
  uint64_t* a_full = bars + 2 * ST_MAX_STAGES;
  uint64_t* a_empty = bars + 3 * ST_MAX_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BN;
  const int kblocks = p.K / TC_BK;

  if (threadIdx.x == ST_WORKERS) {
    tma_prefetch_desc(&maps.w_hi);
    if (SPLIT) tma_prefetch_desc(&maps.w_lo);
    for (int i = 0; i < p.nseg; ++i) tma_prefetch_desc(&maps.a[i]);
    for (int i = 0; i < p.b_stages; ++i) {
      mbar_init(&b_full[i], 1);
      mbar_init(&b_empty[i], ST_WORKERS / 32);
    }
    for (int i = 0; i < p.a_stages; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], ST_WORKERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == ST_WORKERS / 32) {
    if (elect_one()) {
      const uint32_t b_bytes = (SPLIT ? 2 : 1) * L.b_tile, a_bytes = L.a32_stage;   // zero-filled rows count too
      int sg = 0, k0 = 0, sa = 0, pa = 0, sb = 0, pb = 0;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&a_empty[sa], pa ^ 1);
        mbar_expect_tx(&a_full[sa], a_bytes);
        tma_load_2d(a32 + sa * L.a32_stage, &maps.a[sg], k0, 0, &a_full[sa]);
        if ((k0 += TC_BK) == p.ak[sg]) { k0 = 0; ++sg; }
        mbar_wait(&b_empty[sb], pb ^ 1);
        mbar_expect_tx(&b_full[sb], b_bytes);
        unsigned char* dst = b_tiles + sb * 2 * L.b_tile;
        tma_load_2d(dst, &maps.w_hi, kb * TC_BK, n0, &b_full[sb]);
        if (SPLIT) tma_load_2d(dst + L.b_tile, &maps.w_lo, kb * TC_BK, n0, &b_full[sb]);
        if (++sa == p.a_stages) { sa = 0; pa ^= 1; }
        if (++sb == p.b_stages) { sb = 0; pb ^= 1; }
      }
    }
    return;
  }

  // ===================================================== workers: activation split + products, then the epilogue
  const int wt = threadIdx.x;                      // 0..255
  const int g = warp >> 2;                         // warpgroup
  const int nf4 = p.M * 16;                        // float4 groups of the M live rows of one k-block
  float acc[WN / 2];
#pragma unroll
  for (int i = 0; i < WN / 2; ++i) acc[i] = 0.f;
  // the A rows and B columns this warpgroup multiplies: B rows (output columns) [g BN/2, ...) at COLS, A rows [64 g, ...)
  const uint32_t a_part = COLS ? 0u : (uint32_t)g * (64 * 128), b_part = COLS ? (uint32_t)g * (BN / 2 * 128) : 0u;
  int sa = 0, pa = 0, sb = 0, pb = 0, s16 = 0, sb_prev = 0;
  for (int kb = 0; kb < kblocks; ++kb) {
    // fp32 block -> bf16 hi / lo; rows at or above M are neither read nor written (their products are never stored).
    // Stage reuse: every worker has passed the named barrier of kb - 1 only after its wait_group(1) retired the products
    // of kb - 3 and earlier, the last reader of this A16 slot.
    mbar_wait(&a_full[sa], pa);
    const float* src = reinterpret_cast<const float*>(a32 + sa * L.a32_stage);
    unsigned char* t_hi = a16 + s16 * 2 * L.a16_tile;
    unsigned char* t_lo = t_hi + L.a16_tile;
#pragma unroll
    for (int i = 0; i < 128 * 16 / ST_WORKERS; ++i) {
      const int e = wt + ST_WORKERS * i;
      if (e < nf4) {
        const int row = e >> 4, f4 = e & 15;
        const float4 v = *reinterpret_cast<const float4*>(src + row * TC_BK + f4 * 4);
        const uint32_t off = row * 128 + (((f4 >> 1) ^ (row & 7)) << 4) + (f4 & 1) * 8;
        const uint32_t h0 = bf16_bits_rn(v.x), h1 = bf16_bits_rn(v.y), h2 = bf16_bits_rn(v.z), h3 = bf16_bits_rn(v.w);
        *reinterpret_cast<uint2*>(t_hi + off) = make_uint2(h0 | (h1 << 16), h2 | (h3 << 16));
        if constexpr (SPLIT) {
          const uint32_t l0 = bf16_bits_rn(v.x - __uint_as_float(h0 << 16)), l1 = bf16_bits_rn(v.y - __uint_as_float(h1 << 16));
          const uint32_t l2 = bf16_bits_rn(v.z - __uint_as_float(h2 << 16)), l3 = bf16_bits_rn(v.w - __uint_as_float(h3 << 16));
          *reinterpret_cast<uint2*>(t_lo + off) = make_uint2(l0 | (l1 << 16), l2 | (l3 << 16));
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&a_empty[sa]);                  // this warp's reads of the fp32 slot are done
    fence_proxy_async();                                       // generic-proxy stores -> visible to wgmma
    asm volatile("bar.sync 1, %0;" ::"n"(ST_WORKERS) : "memory");
    mbar_wait(&b_full[sb], pb);
    const uint32_t sa_u = smem_u32(t_hi) + a_part, sb_u = smem_u32(b_tiles + sb * 2 * L.b_tile) + b_part;
    const uint64_t a_hi = make_sw128_kmajor_desc(sa_u), a_lo = make_sw128_kmajor_desc(sa_u + L.a16_tile);
    const uint64_t b_hi = make_sw128_kmajor_desc(sb_u), b_lo = make_sw128_kmajor_desc(sb_u + L.b_tile);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_w<WN>(acc, a_hi + 2 * k, b_hi + 2 * k, (kb | k) ? 1u : 0u);
    if constexpr (SPLIT) {
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_w<WN>(acc, a_lo + 2 * k, b_hi + 2 * k, 1u);
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_w<WN>(acc, a_hi + 2 * k, b_lo + 2 * k, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (kb > 0 && lane == 0) mbar_arrive(&b_empty[sb_prev]);
    sb_prev = sb;
    if (++sa == p.a_stages) { sa = 0; pa ^= 1; }
    if (++sb == p.b_stages) { sb = 0; pb ^= 1; }
    if (++s16 == ST_A16_STAGES) s16 = 0;
  }
  wgmma_wait<0>();
  wgmma_hold(acc);

  // ---- epilogue: acc[4 j + 2 h + e] is row r0 + 16 (warp & 3) + lane / 4 + 8 h, column c0 + 8 j + 2 (lane & 3) + e
  const int r0 = COLS ? 0 : 64 * g, c0 = n0 + (COLS ? g * (BN / 2) : 0);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r0 + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    if (row >= p.M) continue;
#pragma unroll
    for (int j = 0; j < WN / 8; ++j) {
      const int n = c0 + 8 * j + 2 * (lane & 3);
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

// The arguments skinny_tc_launch cannot serve, checked on the host alone (no CUDA call, so mac_linear_tc_small_fwd runs it
// before its device check): what the tiles do not take (UNSUPPORTED), a missing operand, an output region its stride
// cannot hold or a segment wider than its row stride (INVALID), misalignment (ALIGN).
// The epilogue writes rows [0, M) of y at stride ldy: columns [0, N), or [0, n_split) and y2's [0, N - n_split); the write
// gate reads gnew / gold and writes gate_z over y's columns.  The gate and the column split are one epilogue each.
inline int skinny_tc_check(const SkinnyTcParams& p, const void* wt_hi, const void* wt_lo) {
  if (p.M <= 0 || p.M > 128 || p.N <= 0 || p.K <= 0 || p.nseg < 1 || p.nseg > 4) return MAC_ERR_INVALID;
  if ((p.N % 32) || (p.K % TC_BK) || (p.ldy & 3) || (p.Y2 && (p.n_split % 32))) return MAC_ERR_UNSUPPORTED;
  if (p.Y2 && p.gnew) return MAC_ERR_UNSUPPORTED;
  if (p.gate_z && !p.gnew) return MAC_ERR_INVALID;
  if (p.Y2 ? (p.n_split <= 0 || p.n_split >= p.N || p.ldy < p.n_split || p.ldy < p.N - p.n_split) : p.ldy < p.N)
    return MAC_ERR_INVALID;
  int ksum = 0;
  for (int i = 0; i < p.nseg; ++i) {
    if (!p.a[i] || p.ak[i] <= 0 || (p.ak[i] % TC_BK) || (p.lda[i] & 3)) return MAC_ERR_UNSUPPORTED;
    if (p.lda[i] < p.ak[i]) return MAC_ERR_INVALID;
    if (!mac_aligned16(p.a[i])) return MAC_ERR_ALIGN;
    ksum += p.ak[i];
  }
  if (ksum != p.K || !wt_hi || !p.Y || !mac_aligned16(p.Y) || !mac_aligned16(wt_hi)) return MAC_ERR_INVALID;
  if ((wt_lo && !mac_aligned16(wt_lo)) || (p.Y2 && !mac_aligned16(p.Y2)) || (p.gnew && !mac_aligned16(p.gnew)) ||
      (p.gold && !mac_aligned16(p.gold)) || (p.gate_z && !mac_aligned16(p.gate_z)))
    return MAC_ERR_ALIGN;
  return MAC_OK;
}

// wt_hi / wt_lo: bf16 [N, K] (K-major) halves of the fp32 weight (mac_pack_weight_bf16_split); wt_lo == NULL: single pass.
// p has passed skinny_tc_check.
inline int skinny_tc_launch(SkinnyTcParams p, const void* wt_hi, const void* wt_lo, cudaStream_t stream) {
  p.split = wt_lo ? 1 : 0;
  const int BN = (p.N % 64 == 0 && p.N >= 1024) ? 64 : 32;
  const bool cols = p.M <= 64;
  // ring depths: at 64 rows 4 activation and 6 weight stages (<= 208 KB); at 128 rows the activation blocks are twice as
  // large, so 2 and 4 (<= 225 KB)
  p.mrows = cols ? 64 : 128;
  p.a_stages = cols ? 4 : 2;
  p.b_stages = cols ? 6 : 4;
  SkinnyTcMaps m;
  int st = make_tmap_2d(&m.w_hi, wt_hi, 1, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K * 2, (uint32_t)BN, TC_BK, 1);
  if (st != MAC_OK) return st;
  if (wt_lo) {
    st = make_tmap_2d(&m.w_lo, wt_lo, 1, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)p.K * 2, (uint32_t)BN, TC_BK, 1);
    if (st != MAC_OK) return st;
  } else {
    m.w_lo = m.w_hi;
  }
  for (int i = 0; i < 4; ++i) {
    if (i >= p.nseg) { m.a[i] = m.a[0]; continue; }
    st = make_tmap_2d(&m.a[i], p.a[i], 0, (uint64_t)p.M, (uint64_t)p.ak[i], (uint64_t)p.lda[i] * 4, (uint32_t)p.mrows,
                      TC_BK, 0);
    if (st != MAC_OK) return st;
  }
  const int smem = StLayout(BN, p.mrows, p.a_stages, p.b_stages).smem_bytes;
  // the shared-memory opt-in belongs to the current device's context: set it on every launch
  auto launch = [&](auto kern) -> int {
    MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    kern<<<p.N / BN, ST_THREADS, smem, stream>>>(m, p);
    return MAC_OK;
  };
  int rc;
  if (BN == 64) {
    if (cols) rc = p.split ? launch(skinny_tc_kernel<64, true, true>) : launch(skinny_tc_kernel<64, false, true>);
    else rc = p.split ? launch(skinny_tc_kernel<64, true, false>) : launch(skinny_tc_kernel<64, false, false>);
  } else {
    if (cols) rc = p.split ? launch(skinny_tc_kernel<32, true, true>) : launch(skinny_tc_kernel<32, false, true>);
    else rc = p.split ? launch(skinny_tc_kernel<32, true, false>) : launch(skinny_tc_kernel<32, false, false>);
  }
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
