// The image stem's inference forward in e4m3 (FP8) on wgmma: the patch-matrix quantisation and the GEMM of one 3x3
// convolution layer (Stem(prec="fp8"), mac_im2col3x3_fp8 / mac_linear_fp8_fwd in mac_b200.h).
//
// Scaling (every scale is fp32; e4m3 = round-to-nearest-even, saturating at +-448):
//   amax_m = max |x| over the in-image pixels of output pixel m's 3x3 window      (zero padding contributes nothing)
//   sA_m   = amax_m / 448;  cols8[m, tap*C + c] = e4m3(x[pixel m shifted by tap, c] * (448 / amax_m))   (0 when amax_m == 0)
//   W8     = e4m3(W / sW_n), sW_n = max_k |W[k, n]| / 448      per output column (mac_pack_weight_fp8, read_step_fp8.cuh)
//   y      = act(acc * sA_m * sW_n + b_n),  acc = cols8[m, :] . W8[n, :]                    fp32 [M, n_out]
// oracle/fp8_stem_oracle.py restates this with the same fp32 operations for sA and the quantisation.
//
// The GEMM keeps tc_gemm_kernel's shape (tc_gemm.cuh): one CTA per 128 x 128 output tile, two consumer warpgroups of 64
// rows each, one TMA producer warp, 128-byte swizzle, an mbarrier ring.  A 128-element e4m3 k-block is one 128-byte
// swizzle-atom row, so the boxes and shared-memory descriptors are the bf16 kernel's, with twice the K per k-block.
// Each k-block is four wgmma m64n128k32 e4m3 x e4m3 into a fresh register accumulator, which the CUDA cores then add into
// the fp32 master accumulator: Hopper's e4m3 wgmma adds its products into the accumulator with fewer mantissa bits than
// fp32, and over K = 9216 (72 k-blocks) that loss would grow with K; two-level accumulation bounds it to one k-block.
#pragma once
#include "tc_gemm.cuh"
#include "read_step_fp8.cuh"     // float2_to_e4m3x2

namespace mac {

constexpr int F8_BK = 128;                                  // e4m3 per k-block: 128 bytes, one swizzle atom row
constexpr int F8_STAGES = 6;
constexpr int F8_A_BYTES = TC_BM * F8_BK;                   // 16 KB
constexpr int F8_B_BYTES = TC_BN * F8_BK;                   // 16 KB
constexpr int F8_STAGE_BYTES = F8_A_BYTES + F8_B_BYTES;
constexpr int F8_SMEM_BYTES = F8_STAGES * F8_STAGE_BYTES + 1024 /*align*/ + 128 /*barriers*/;
static_assert(F8_SMEM_BYTES <= 232448, "over the sm_90 per-block shared memory opt-in limit");

// D[64 x 128] (+)= A[64 x 32] B[32 x 128], e4m3 operands (both K-major) from shared memory, fp32 accumulators
__device__ __forceinline__ void wgmma_e4m3_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

struct LinearFp8Params {
  int M, N, K;
  const float* sa;         // [M] row scales of the A operand
  const float* sw;         // [N] column scales of the packed weight
  const float* bias;       // [N] or NULL
  float* y;                // [M, N] fp32
};

template <int ACT>
__global__ void __launch_bounds__(TC_THREADS, 1)
linear_fp8_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                  const LinearFp8Params p) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  unsigned char* tiles = smem_dyn + ((1024u - (base_u32 & 1023u)) & 1023u);          // 1024-byte aligned operand ring
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + F8_STAGES * F8_STAGE_BYTES);  // [STAGES] TMA -> consumers
  uint64_t* empty = full + F8_STAGES;                                                // [STAGES] consumers -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x, mt = blockIdx.y;
  const int kblocks = p.K / F8_BK;

  if (threadIdx.x == TC_CONSUMERS) {
    tma_prefetch_desc(&map_a);
    tma_prefetch_desc(&map_b);
#pragma unroll
    for (int i = 0; i < F8_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], TC_CONSUMERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == TC_CONSUMERS / 32) {
    // ===================================================== TMA producer (rows past M arrive as zero fill)
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        unsigned char* sa = tiles + stage * F8_STAGE_BYTES;
        mbar_expect_tx(&full[stage], F8_STAGE_BYTES);
        tma_load_2d(sa, &map_a, kb * F8_BK, mt * TC_BM, &full[stage]);
        tma_load_2d(sa + F8_A_BYTES, &map_b, kb * F8_BK, nt * TC_BN, &full[stage]);
        if (++stage == F8_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================================================== consumers: one k-block per wgmma group, then the fp32 add
  const int g = warp >> 2;                                  // warpgroup: rows [64 g, 64 g + 64) of the tile
  float acc[64], blk[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = blk[i] = 0.f;
  {
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(tiles + stage * F8_STAGE_BYTES);
      const uint64_t adesc = make_sw128_kmajor_desc(sa + g * (64 * 128));
      const uint64_t bdesc = make_sw128_kmajor_desc(sa + F8_A_BYTES);
      wgmma_fence();                                        // blk was read by the previous k-block's add
#pragma unroll
      for (int k = 0; k < F8_BK / 32; ++k) wgmma_e4m3_n128(blk, adesc + 2 * k, bdesc + 2 * k, k ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(blk);
      if (lane == 0) mbar_arrive(&empty[stage]);            // this warp's products have retired: the slot may refill
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] += blk[i];
      if (++stage == F8_STAGES) { stage = 0; phase ^= 1; }
    }
  }

  // ===================================================== epilogue: acc[4 j + 2 h + e] is row (16 * (warp & 3) + lane / 4 + 8 h)
  // of the warpgroup's 64, column 8 j + 2 (lane & 3) + e
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = mt * TC_BM + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    if (row >= p.M) continue;
    const float sa = __ldg(p.sa + row);
    float* yr = p.y + (size_t)row * p.N;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = nt * TC_BN + 8 * j + cq;
      const float2 sw = __ldg(reinterpret_cast<const float2*>(p.sw + n));
      float x0 = acc[4 * j + 2 * h] * sa * sw.x, x1 = acc[4 * j + 2 * h + 1] * sa * sw.y;
      if (p.bias) {
        x0 += __ldg(p.bias + n);
        x1 += __ldg(p.bias + n + 1);
      }
      *reinterpret_cast<float2*>(yr + n) = make_float2(act_ct<ACT>(x0), act_ct<ACT>(x1));
    }
  }
}

template <int ACT>
inline int linear_fp8_launch_t(const CUtensorMap& ma, const CUtensorMap& mb, const LinearFp8Params& p, cudaStream_t stream) {
  auto kern = linear_fp8_kernel<ACT>;
  // the shared-memory opt-in belongs to the current device's context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, F8_SMEM_BYTES));
  kern<<<dim3(p.N / TC_BN, (p.M + TC_BM - 1) / TC_BM), TC_THREADS, F8_SMEM_BYTES, stream>>>(ma, mb, p);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

inline bool linear_fp8_act_supported(int act) { return act == MAC_ACT_NON || act == MAC_ACT_ELU || act == MAC_ACT_RELU; }

// a8 [M, K] e4m3 row-major with row scales sa [M]; w8 [N, K] e4m3 (mac_pack_weight_fp8) with column scales sw [N];
// K % 128 == 0, N % 128 == 0 (checked by the caller)
inline int linear_fp8_launch(const void* a8, const float* sa, const void* w8, const float* sw, const float* bias, int act,
                             float* y, int M, int K, int N, cudaStream_t stream) {
  CUtensorMap ma, mb;
  int st = make_tmap_2d(&ma, a8, 2, (uint64_t)M, (uint64_t)K, (uint64_t)K, (uint32_t)TC_BM, F8_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mb, w8, 2, (uint64_t)N, (uint64_t)K, (uint64_t)K, (uint32_t)TC_BN, F8_BK, 1);
  if (st != MAC_OK) return st;
  LinearFp8Params p{M, N, K, sa, sw, bias, y};
  switch (act) {
    case MAC_ACT_NON: return linear_fp8_launch_t<MAC_ACT_NON>(ma, mb, p, stream);
    case MAC_ACT_ELU: return linear_fp8_launch_t<MAC_ACT_ELU>(ma, mb, p, stream);
    case MAC_ACT_RELU: return linear_fp8_launch_t<MAC_ACT_RELU>(ma, mb, p, stream);
  }
  return MAC_ERR_UNSUPPORTED;
}

// ---------------------------------------------------------------------------------------------------------------
// The patch matrix in e4m3.  Pass 1: pa[p] = max_c |x[p, c]| per input pixel (one warp per pixel, the workspace).
// Pass 2: one thread per 16 channels of one tap of one output pixel: the window amax from the nine pa values (L1 hits),
// then 64 bytes of x in and 16 e4m3 bytes out.  C % 128 == 0.
__global__ void __launch_bounds__(256) pixel_amax_kernel(const float* __restrict__ x, float* __restrict__ pa, long long P,
                                                         int C) {
  const long long px = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (px >= P) return;
  const float4* r = reinterpret_cast<const float4*>(x + px * C);
  float m = 0.f;
  for (int i = lane; i < C / 4; i += 32) {
    const float4 v = __ldg(r + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  m = warp_max(m);
  if (lane == 0) pa[px] = m;
}

__device__ __forceinline__ uint32_t e4m3x4(float4 v, float s) {
  return float2_to_e4m3x2(v.x * s, v.y * s) | (float2_to_e4m3x2(v.z * s, v.w * s) << 16);
}

__global__ void __launch_bounds__(256) im2col3x3_e4m3_kernel(const float* __restrict__ x, const float* __restrict__ pa,
                                                             uint8_t* __restrict__ cols8, float* __restrict__ sA, int B,
                                                             int H, int W, int C) {
  const int c16n = C / 16;
  const long long total = (long long)B * H * W * 9 * c16n;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c16 = (int)(i % c16n);
  const long long r = i / c16n;
  const int tap = (int)(r % 9);
  const long long m = r / 9;
  const int w = (int)(m % W), h = (int)((m / W) % H);
  const long long b = m / ((long long)W * H);
  float am = 0.f;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int hs = h + t / 3 - 1, wsrc = w + t % 3 - 1;
    if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W) am = fmaxf(am, __ldg(pa + (b * H + hs) * W + wsrc));
  }
  if (tap == 0 && c16 == 0) sA[m] = am / 448.f;
  const float inv = am > 0.f ? 448.f / am : 0.f;
  const int hs = h + tap / 3 - 1, wsrc = w + tap % 3 - 1;
  uint4 o = make_uint4(0u, 0u, 0u, 0u);
  if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W) {
    const float4* src = reinterpret_cast<const float4*>(x + ((b * H + hs) * W + wsrc) * C + c16 * 16);
    o = make_uint4(e4m3x4(__ldg(src), inv), e4m3x4(__ldg(src + 1), inv), e4m3x4(__ldg(src + 2), inv),
                   e4m3x4(__ldg(src + 3), inv));
  }
  *reinterpret_cast<uint4*>(cols8 + (m * 9 + tap) * C + c16 * 16) = o;
}

inline size_t im2col3x3_fp8_workspace_bytes(long long P) { return ((size_t)P * 4 + 255) & ~(size_t)255; }

inline int im2col3x3_fp8_launch(const float* x, void* cols8, float* sA, void* ws, int B, int H, int W, int C,
                                cudaStream_t stream) {
  const long long P = (long long)B * H * W;
  float* pa = reinterpret_cast<float*>(ws);
  pixel_amax_kernel<<<(unsigned)((P + 7) / 8), 256, 0, stream>>>(x, pa, P, C);
  MAC_LAUNCH_CHECK();
  const long long total = P * 9 * (C / 16);
  im2col3x3_e4m3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, pa, reinterpret_cast<uint8_t*>(cols8), sA, B,
                                                                             H, W, C);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac
