// One reasoning step of the read unit in inference form with e4m3 (FP8) operands on wgmma: the same function as
// read_step_kernel (read_step.cuh), in its 64-row form (64 knowledge-base rows per CTA, packed across sample boundaries; one
// TMA producer warp and two consumer warpgroups that each own 256 output columns; P*y, H and the logits stay on the SM;
// kb_attend on the bf16 knowledge base is the tail), but both GEMMs are m64n256k32 e4m3 x e4m3 -> fp32.  A weight k-block of
// 64 KB holds 128 input rows instead of 64, so each GEMM streams half the weight bytes and waits on half as many ring slots.
//
// Scaling (every scale is fp32; e4m3 = round-to-nearest-even, saturating at +-448):
//   P8  = e4m3(P / sP_r),  sP_r = max|P_r| / 448                     per knowledge-base row, once per forward (inv)
//   W8  = e4m3(W / sW_c),  sW_c = max_k |W[k, c]| / 448             per output column of Wm[0:d] and Wm2 (packed weights)
//   A8  = e4m3(P8 * (y_b / ay_b)),  ay_b = max|y_b|                  per sample, computed here for the tile's samples
//   H   = ELU(acc1 * sP_r * ay_b * sW1_c + Q)                       Q = P @ Wm[d:2d] + bm stays bf16 (GEMM 1's addend)
//   H8  = e4m3(H / sH_r),  sH_r = max|H_r| / 448                     row amax over both warpgroups' halves
//   I1  = acc2 * sH_r * sW2_c + bm2;  then control, ELU, wr and the logits as in read_step_kernel
// oracle/fp8_read_oracle.py restates this in fp64 (the reference of tests/test_gpu_read_step_fp8.py).
//
// Shared memory: A [64 x 512] e4m3 as 4 K-major 128-byte-swizzled [64 x 128] blocks (32 KB): H8, the A operand of GEMM 2.
// B: 2 stages x 72 KB, one mbarrier ring of 9 slots per tile: slots 0..3 each carry k-block j of Wm[0:d] ([512 x 128] e4m3,
// 64 KB) and k-block j of the P8 tile ([64 x 128], 8 KB); slot 4 the tile's bf16 Q rows (64 KB, 8 [64 x 64] blocks);
// slots 5..8 the k-blocks of Wm2.  Three 72 KB stages beside the A tile would need 248 KB, over the 227 KB opt-in limit.
// y / ay_b of the tile's first two samples is staged in shared memory (rows of later samples, only present when N < 64, are
// read from global memory and scaled by 1 / ay_b): sixteen y values per 16-byte P8 chunk do not fit in registers beside the
// 128 accumulators.
#pragma once
#include <cuda_fp8.h>
#include <cuda_fp16.h>
#include "read_step.cuh"

namespace mac {

constexpr int R8_BK = 128;                        // e4m3 per k-block: 128 bytes, one swizzle atom row
constexpr int R8_KB = RS_D / R8_BK;               // 4 k-blocks
constexpr int R8_BLK = RS_BM * R8_BK;             // one [64 x 128] e4m3 A block: 8 KB
constexpr int R8_A_BYTES = R8_KB * R8_BLK;        // 32 KB
constexpr int R8_B_HALF = 256 * R8_BK;            // [256 x 128] e4m3: 32 KB
constexpr int R8_W_BYTES = 2 * R8_B_HALF;         // one weight k-block: 64 KB
constexpr int R8_STAGE = R8_W_BYTES + R8_BLK;     // 72 KB
constexpr int R8_STAGES = 2;
constexpr int R8_Q_SLOT = R8_KB;                  // ring slot of the bf16 Q tile
constexpr int R8_SLOTS = R8_Q_SLOT + 1 + R8_KB;   // 9 ring slots per tile
constexpr int R8_SMEM_BYTES = R8_A_BYTES + R8_STAGES * R8_STAGE + 1024 /*align*/ + 64 /*barriers*/ +
                              2 * RS_BM * 4 /*logit halves*/ + 2 * RS_BM * 4 /*H amax halves*/ +
                              2 * RS_D * 4 /*control of <= 2 samples*/ + 2 * RS_D * 4 /*y / ay of <= 2 samples*/ +
                              4 * RS_D * 4 /*bm2, wr, sW1, sW2*/ + 2 * RS_BM * 4 /*ay, 1 / ay per sample*/;
static_assert(RS_A_BYTES <= R8_STAGE, "the bf16 Q tile must fit in one ring stage");
static_assert(R8_SMEM_BYTES <= 232448, "over the sm_90 per-block shared memory opt-in limit");
static_assert(R8_STAGE % 1024 == 0 && R8_A_BYTES % 1024 == 0, "swizzled operands need 1024-byte alignment");

// D[64 x 256] (+)= A[64 x 32] B[32 x 256], e4m3 operands (both K-major) from shared memory, fp32 accumulators
__device__ __forceinline__ void wgmma_e4m3_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k32.f32.e4m3.e4m3 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

__device__ __forceinline__ float2 e4m3x2_to_float2(uint32_t v) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(v & 0xffffu), __NV_E4M3);
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}
__device__ __forceinline__ uint32_t float2_to_e4m3x2(float a, float b) {
  return (uint32_t)__nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
}
// four e4m3 (one 32-bit word, element 0 in the low byte) times y[0..3] * sc, rounded back to e4m3
__device__ __forceinline__ uint32_t scale4_e4m3(uint32_t w, float4 y, float sc) {
  const float2 a = e4m3x2_to_float2(w), b = e4m3x2_to_float2(w >> 16);
  return float2_to_e4m3x2(a.x * (y.x * sc), a.y * (y.y * sc)) | (float2_to_e4m3x2(b.x * (y.z * sc), b.y * (y.w * sc)) << 16);
}

struct ReadStepFp8Params {
  int M, N;
  const float* y;                   // [B, d] memory projection
  const float* ctrl;                // [B, d]
  const float* bm2;                 // [d]
  const float* wr;                  // [d]
  const float* sP;                  // [M] row scales of P8
  const float* sw1;                 // [d] column scales of Wm[0:d]
  const float* sw2;                 // [d] column scales of Wm2
  float* logits;                    // [B*N]  I2 . wr (without br)
};

__global__ void __launch_bounds__(RS_THREADS, 1)
read_step_fp8_kernel(const __grid_constant__ CUtensorMap map_p8, const __grid_constant__ CUtensorMap map_q,
                     const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w2,
                     const ReadStepFp8Params p) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  unsigned char* a_tile = smem_dyn + ((1024u - (base_u32 & 1023u)) & 1023u);
  unsigned char* b_ring = a_tile + R8_A_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(b_ring + R8_STAGES * R8_STAGE);   // [STAGES] TMA -> consumers
  uint64_t* empty = full + R8_STAGES;              // [STAGES] consumers -> TMA (8 warp arrivals)
  float* s_lg = reinterpret_cast<float*>(full + 8);          // [2][64] logit halves
  float* s_hmax = s_lg + 2 * RS_BM;                          // [2][64] max|H| of each row's two column halves
  float* s_ctrl = s_hmax + 2 * RS_BM;                        // [2][d] control of the tile's first two samples
  float* s_ys = s_ctrl + 2 * RS_D;                           // [2][d] y / ay of the tile's first two samples
  float* s_bm2 = s_ys + 2 * RS_D;                            // [d]
  float* s_wr = s_bm2 + RS_D;                                // [d]
  float* s_sw1 = s_wr + RS_D;                                // [d]
  float* s_sw2 = s_sw1 + RS_D;                               // [d]
  float* s_ay = s_sw2 + RS_D;                                // [64] ay_b of the tile's samples
  float* s_iay = s_ay + RS_BM;                               // [64] 1 / ay_b (0 for an all-zero y_b)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * RS_BM;
  const int s_lo = row0 / p.N;                               // first sample of the tile

  if (threadIdx.x == RS_CONSUMERS) {
    tma_prefetch_desc(&map_p8);
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_w1);
    tma_prefetch_desc(&map_w2);
    for (int i = 0; i < R8_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], RS_CONSUMERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == RS_CONSUMERS / 32) {
    // ===================================================== TMA producer
    if (elect_one()) {
      for (int j = 0; j < R8_SLOTS; ++j) {
        const int s = j % R8_STAGES;
        mbar_wait(&empty[s], ((j / R8_STAGES) & 1) ^ 1);
        unsigned char* dst = b_ring + s * R8_STAGE;
        if (j == R8_Q_SLOT) {
          mbar_expect_tx(&full[s], RS_A_BYTES);
          for (int kb = 0; kb < RS_KB; ++kb) tma_load_2d(dst + kb * RS_BLK, &map_q, kb * TC_BK, row0, &full[s]);
          continue;
        }
        const bool g1 = j < R8_Q_SLOT;
        mbar_expect_tx(&full[s], g1 ? R8_W_BYTES + R8_BLK : R8_W_BYTES);
        const CUtensorMap* m = g1 ? &map_w1 : &map_w2;
        const int k0 = (g1 ? j : j - R8_Q_SLOT - 1) * R8_BK;
        if (g1) tma_load_2d(dst + R8_W_BYTES, &map_p8, k0, row0, &full[s]);
        tma_load_2d(dst, m, k0, 0, &full[s]);
        tma_load_2d(dst + R8_B_HALF, m, k0, 256, &full[s]);
      }
    }
    return;
  }

  // ===================================================== consumers
  const int tid = threadIdx.x;
  const int g = warp >> 2;                                   // warpgroup: output columns [256 g, 256 g + 256)
  // acc[4 j + 2 h + e] is tile row 16 (warp & 3) + lane / 4 + 8 h, column 256 g + 8 j + 2 (lane & 3) + e
  const int rl = 16 * (warp & 3) + (lane >> 2);
  const int cq = 256 * g + 2 * (lane & 3);
  // this thread's two 16-byte chunks of each P8 block: rows tid / 8 and tid / 8 + 32, chunk tid % 8 of the swizzled
  // 128-byte row, i.e. columns pcol .. pcol + 15 of the k-block
  const int prow = tid >> 3;
  const int poff = prow * 128 + (tid & 7) * 16;
  const int pcol = ((tid & 7) ^ (prow & 7)) << 4;
  for (int i = tid; i < RS_D; i += RS_CONSUMERS) {
    s_bm2[i] = __ldg(p.bm2 + i);
    s_wr[i] = __ldg(p.wr + i);
    s_sw1[i] = __ldg(p.sw1 + i);
    s_sw2[i] = __ldg(p.sw2 + i);
  }
  const int last_row = min(p.M, row0 + RS_BM) - 1;
  const int nsamp = last_row / p.N - s_lo + 1;
  for (int q = 0; q < min(nsamp, 2); ++q)
    for (int i = tid; i < RS_D; i += RS_CONSUMERS) s_ctrl[q * RS_D + i] = __ldg(p.ctrl + (size_t)(s_lo + q) * RS_D + i);
  // ay_b = max|y_b| of each sample of the tile, one warp per sample
  for (int q = warp; q < nsamp; q += RS_CONSUMERS / 32) {
    const float* yr = p.y + (size_t)(s_lo + q) * RS_D;
    float v[RS_D / 32];
    float m = 0.f;
#pragma unroll
    for (int i = 0; i < RS_D / 32; ++i) {
      v[i] = __ldg(yr + lane + 32 * i);
      m = fmaxf(m, fabsf(v[i]));
    }
    m = warp_max(m);
    const float inv = m > 0.f ? 1.f / m : 0.f;
    if (lane == 0) {
      s_ay[q] = m;
      s_iay[q] = inv;
    }
    if (q < 2) {
#pragma unroll
      for (int i = 0; i < RS_D / 32; ++i) s_ys[q * RS_D + lane + 32 * i] = v[i] * inv;
    }
  }
  rs_consumer_bar();
  // y / ay of this thread's two P8 rows (rows past M are TMA zero fill and stay zero): staged rows scale by 1, rows of later
  // samples are read from global memory and scaled by 1 / ay_b (the same product as the staged value)
  const float* yrow[2];
  float ysc[2];
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int q = min(row0 + prow + 32 * u, p.M - 1) / p.N - s_lo;
    yrow[u] = (q < 2 ? s_ys + q * RS_D : p.y + (size_t)(s_lo + q) * RS_D) + pcol;
    ysc[u] = q < 2 ? 1.f : s_iay[q];
  }

  float acc[128];
  // ---- GEMM 1: P8 block j becomes A8 = e4m3(P8 * y / ay) in place while the MMAs of block j - 1 run, then block j is issued
  for (int j = 0; j < R8_KB; ++j) {
    const int s = j % R8_STAGES;
    unsigned char* stage = b_ring + s * R8_STAGE;
    mbar_wait(&full[s], (j / R8_STAGES) & 1);
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      uint4* c = reinterpret_cast<uint4*>(stage + R8_W_BYTES + poff + u * 32 * 128);
      const uint4 v = *c;
      const float* yr = yrow[u] + j * R8_BK;
      const float4 y0 = *reinterpret_cast<const float4*>(yr), y1 = *reinterpret_cast<const float4*>(yr + 4);
      const float4 y2 = *reinterpret_cast<const float4*>(yr + 8), y3 = *reinterpret_cast<const float4*>(yr + 12);
      *c = make_uint4(scale4_e4m3(v.x, y0, ysc[u]), scale4_e4m3(v.y, y1, ysc[u]), scale4_e4m3(v.z, y2, ysc[u]),
                      scale4_e4m3(v.w, y3, ysc[u]));
    }
    fence_proxy_async();                                   // generic-proxy stores -> visible to wgmma
    rs_consumer_bar();
    const uint64_t adesc = make_sw128_kmajor_desc(smem_u32(stage + R8_W_BYTES));
    const uint64_t bdesc = make_sw128_kmajor_desc(smem_u32(stage + g * R8_B_HALF));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < R8_BK / 32; ++k) wgmma_e4m3_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j || k) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (j && lane == 0) mbar_arrive(&empty[(j - 1) % R8_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  if (lane == 0) mbar_arrive(&empty[(R8_KB - 1) % R8_STAGES]);

  // ---- GEMM 1's epilogue: H = ELU(acc * sP_r * ay_b * sW1_c + Q), kept in acc; the row amax over both halves; then
  //      H8 = e4m3(H / sH_r) into the A tile (K-major, swizzled).  GEMM 1 takes its A operand from the ring, so nothing else
  //      uses the A tile before this.
  constexpr int qs = R8_Q_SLOT % R8_STAGES;
  const unsigned char* q_tile = b_ring + qs * R8_STAGE;
  mbar_wait(&full[qs], (R8_Q_SLOT / R8_STAGES) & 1);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rl + 8 * h, row = row0 + r;
    const int rr = min(row, p.M - 1);
    const float rf = __ldg(p.sP + rr) * s_ay[rr / p.N - s_lo];
    float m = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = cq + 8 * j;
      const int kb = n >> 6, c = (n & 63) >> 3;
      const uint32_t q = *reinterpret_cast<const uint32_t*>(q_tile + kb * RS_BLK + r * 128 + ((c ^ (r & 7)) << 4) + (n & 7) * 2);
      const float2 sw = *reinterpret_cast<const float2*>(s_sw1 + n);
      float h0 = elu_fast(acc[4 * j + 2 * h] * rf * sw.x + bf16lo(q));
      float h1 = elu_fast(acc[4 * j + 2 * h + 1] * rf * sw.y + bf16hi(q));
      if (row >= p.M) h0 = h1 = 0.f;
      acc[4 * j + 2 * h] = h0;
      acc[4 * j + 2 * h + 1] = h1;
      m = fmaxf(m, fmaxf(fabsf(h0), fabsf(h1)));
    }
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    if ((lane & 3) == 0) s_hmax[g * RS_BM + r] = m;
  }
  rs_consumer_bar();
  if (lane == 0) mbar_arrive(&empty[qs]);                  // Q read and used by every thread of this warp
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rl + 8 * h;
    const float am = fmaxf(s_hmax[r], s_hmax[RS_BM + r]);
    const float inv = am > 0.f ? 448.f / am : 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = cq + 8 * j;
      const int kb = n >> 7, c = (n & 127) >> 4;
      *reinterpret_cast<uint16_t*>(a_tile + kb * R8_BLK + r * 128 + ((c ^ (r & 7)) << 4) + (n & 15)) =
          (uint16_t)float2_to_e4m3x2(acc[4 * j + 2 * h] * inv, acc[4 * j + 2 * h + 1] * inv);
    }
  }
  fence_proxy_async();
  rs_consumer_bar();

  // ---- GEMM 2
  const uint32_t a_u = smem_u32(a_tile);
  for (int j = 0; j < R8_KB; ++j) {
    const int jj = R8_Q_SLOT + 1 + j, s = jj % R8_STAGES;
    mbar_wait(&full[s], (jj / R8_STAGES) & 1);
    const uint64_t adesc = make_sw128_kmajor_desc(a_u + j * R8_BLK);
    const uint64_t bdesc = make_sw128_kmajor_desc(smem_u32(b_ring + s * R8_STAGE + g * R8_B_HALF));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < R8_BK / 32; ++k) wgmma_e4m3_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j || k) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (j && lane == 0) mbar_arrive(&empty[(jj - 1) % R8_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  if (lane == 0) mbar_arrive(&empty[(R8_SLOTS - 1) % R8_STAGES]);

  // ---- GEMM 2's epilogue: I1 = acc * sH_r * sW2_c + bm2; I2 = ELU(I1 * control_b); logit half = sum_n I2 * wr
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rl + 8 * h, row = row0 + r;
    const int s = min(row, p.M - 1) / p.N;
    const float* crow = s - s_lo < 2 ? s_ctrl + (s - s_lo) * RS_D : p.ctrl + (size_t)s * RS_D;
    const float sh = fmaxf(s_hmax[r], s_hmax[RS_BM + r]) / 448.f;
    float part = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = cq + 8 * j;
      const float2 cc = *reinterpret_cast<const float2*>(crow + n);
      const float2 bb = *reinterpret_cast<const float2*>(s_bm2 + n);
      const float2 ww = *reinterpret_cast<const float2*>(s_wr + n);
      const float2 sw = *reinterpret_cast<const float2*>(s_sw2 + n);
      const float t0 = elu_fast((acc[4 * j + 2 * h] * sh * sw.x + bb.x) * cc.x);
      const float t1 = elu_fast((acc[4 * j + 2 * h + 1] * sh * sw.y + bb.y) * cc.y);
      part = fmaf(t0, ww.x, part);
      part = fmaf(t1, ww.y, part);
    }
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 2);
    if ((lane & 3) == 0) s_lg[g * RS_BM + r] = part;
  }
  rs_consumer_bar();
  if (tid < RS_BM && row0 + tid < p.M) p.logits[row0 + tid] = s_lg[tid] + s_lg[RS_BM + tid];
}

// ---- packing and the step-invariant part
// fp32 W[K, n_out] (in, out) -> e4m3 Wt[n_out, K] = e4m3(W / s_n), s_n = max_k |W[k, n]| / 448 (an all-zero column packs to
// zeros with s_n = 0): the K-major B operand of read_step_fp8_kernel.  One block per 32 output columns.
__global__ void pack_weight_fp8_kernel(const float* __restrict__ W, uint8_t* __restrict__ Wt, float* __restrict__ col_scale,
                                       int K, int N) {
  __shared__ float tile[32][33];
  __shared__ float s_max[8][32];
  const int n0 = blockIdx.x * 32, tx = threadIdx.x, ty = threadIdx.y;
  float m = 0.f;
  if (n0 + tx < N)
    for (int k = ty; k < K; k += 8) m = fmaxf(m, fabsf(W[(size_t)k * N + n0 + tx]));
  s_max[ty][tx] = m;
  __syncthreads();
  if (ty == 0) {
    for (int i = 1; i < 8; ++i) m = fmaxf(m, s_max[i][tx]);
    s_max[0][tx] = m;
    if (n0 + tx < N) col_scale[n0 + tx] = m / 448.f;
  }
  __syncthreads();
  for (int k0 = 0; k0 < K; k0 += 32) {
    for (int i = ty; i < 32; i += 8) {
      const int k = k0 + i, n = n0 + tx;
      tile[i][tx] = (k < K && n < N) ? W[(size_t)k * N + n] : 0.f;
    }
    __syncthreads();
    for (int i = ty; i < 32; i += 8) {
      const int n = n0 + i, k = k0 + tx;
      const float am = s_max[0][i];
      if (n < N && k < K)
        Wt[(size_t)n * K + k] = am > 0.f ? __nv_cvt_float_to_fp8(tile[tx][i] / (am / 448.f), __NV_SATFINITE, __NV_E4M3) : 0;
    }
    __syncthreads();
  }
}

// P8[m, :] = e4m3(P[m, :] / sP_m), sP_m = max|P[m, :]| / 448 (0 for an all-zero row), d = 512: one warp per row
__global__ void __launch_bounds__(256) quant_rows_e4m3_kernel(const __nv_bfloat16* __restrict__ P, uint8_t* __restrict__ P8,
                                                             float* __restrict__ sP, int M) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  const uint4* src = reinterpret_cast<const uint4*>(P + (size_t)m * RS_D) + 2 * lane;
  const uint4 a = src[0], b = src[1];
  const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
  float v[16];
  float am = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    v[2 * i] = bf16lo(w[i]);
    v[2 * i + 1] = bf16hi(w[i]);
    am = fmaxf(am, fmaxf(fabsf(v[2 * i]), fabsf(v[2 * i + 1])));
  }
  am = warp_max(am);
  const float s = am / 448.f;
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t lo = float2_to_e4m3x2(v[4 * i] / s, v[4 * i + 1] / s);
    const uint32_t hi = float2_to_e4m3x2(v[4 * i + 2] / s, v[4 * i + 3] / s);
    o[i] = am > 0.f ? lo | (hi << 16) : 0u;
  }
  reinterpret_cast<uint4*>(P8 + (size_t)m * RS_D)[lane] = make_uint4(o[0], o[1], o[2], o[3]);
  if (lane == 0) sP[m] = s;
}

// inv = [P8 | sP | Q | logit scratch | P]: P8 [M, d] e4m3, sP [M] fp32, Q [M, d] bf16 (the bf16 path's Q), one logit per row,
// and the bf16 P that P8 and Q are made from; each slab 1 KB aligned
struct Fp8ReadScratch {
  uint8_t* P8;
  float* sP;
  __nv_bfloat16* Q;
  float* parts;
  __nv_bfloat16* P;
};
inline size_t fp8_align1k(size_t b) { return (b + 1023) & ~(size_t)1023; }
inline size_t fp8_read_invariant_bytes(int B, int N, int d) {
  const size_t M = (size_t)B * N;
  return fp8_align1k(M * d) + fp8_align1k(M * 4) + 2 * fp8_align1k(M * d * 2) + fp8_align1k(M * 4) + 1024;
}
inline Fp8ReadScratch fp8_read_scratch(void* inv, int B, int N, int d) {
  const size_t M = (size_t)B * N;
  char* o = tc_align1k(inv);
  Fp8ReadScratch s;
  s.P8 = reinterpret_cast<uint8_t*>(o);
  o += fp8_align1k(M * d);
  s.sP = reinterpret_cast<float*>(o);
  o += fp8_align1k(M * 4);
  s.Q = reinterpret_cast<__nv_bfloat16*>(o);
  o += fp8_align1k(M * d * 2);
  s.parts = reinterpret_cast<float*>(o);
  o += fp8_align1k(M * 4);
  s.P = reinterpret_cast<__nv_bfloat16*>(o);
  return s;
}

// P = KB @ Wx + bx and Q = P @ Wm[d:2d] + bm exactly as tc_read_invariant computes them (bf16), then P8 and sP from P
inline int fp8_read_invariant(const void* kb_bf16, const mac_read_weights* w, void* inv, size_t inv_bytes, int B, int N, int d,
                              cudaStream_t stream) {
  if (!read_step_supported(B, N, d)) return MAC_ERR_UNSUPPORTED;
  if (!kb_bf16 || !w->Wx_bf16 || !w->Wm_bf16) return MAC_ERR_INVALID;
  if (inv_bytes < fp8_read_invariant_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  const Fp8ReadScratch s = fp8_read_scratch(inv, B, N, d);
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N; p.ldo = d;
  p.epi = TC_EPI_ACT; p.act = MAC_ACT_NON; p.bias = w->bx; p.out0 = s.P;
  int st = tc_gemm_launch(kb_bf16, d, nullptr, 0, w->Wx_bf16, p, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bm; p.out0 = s.Q;
  st = tc_gemm_launch(s.P, d, nullptr, 0, reinterpret_cast<const __nv_bfloat16*>(w->Wm_bf16) + d, p, stream, nullptr, 2 * d);
  if (st != MAC_OK) return st;
  quant_rows_e4m3_kernel<<<(M + 7) / 8, 256, 0, stream>>>(s.P, s.P8, s.sP, M);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// one e4m3 read step: inv from fp8_read_invariant; y, control [B, d] fp32; att [B, N], info [B, d]
inline int read_step_fp8_launch(const void* inv, const void* kb_bf16, const float* y, const float* control,
                                const mac_read_weights* w, float* att, float* info, int B, int N, int d, cudaStream_t stream) {
  if (!read_step_supported(B, N, d)) return MAC_ERR_UNSUPPORTED;
  if (!inv || !kb_bf16 || !y || !control || !w->Wm_fp8 || !w->Wm_fp8_scale || !w->Wm2_fp8 || !w->Wm2_fp8_scale || !att || !info)
    return MAC_ERR_INVALID;
  const int M = B * N;
  const Fp8ReadScratch s = fp8_read_scratch(const_cast<void*>(inv), B, N, d);
  CUtensorMap mp, mq, mw1, mw2;
  int st = make_tmap_2d(&mp, s.P8, 2, (uint64_t)M, (uint64_t)d, (uint64_t)d, RS_BM, R8_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mq, s.Q, 1, (uint64_t)M, (uint64_t)d, (uint64_t)d * 2, RS_BM, TC_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw1, w->Wm_fp8, 2, (uint64_t)d, (uint64_t)d, (uint64_t)d, 256, R8_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw2, w->Wm2_fp8, 2, (uint64_t)d, (uint64_t)d, (uint64_t)d, 256, R8_BK, 1);
  if (st != MAC_OK) return st;
  ReadStepFp8Params p{};
  p.M = M; p.N = N; p.y = y; p.ctrl = control; p.bm2 = w->bm2; p.wr = w->wr;
  p.sP = s.sP; p.sw1 = w->Wm_fp8_scale; p.sw2 = w->Wm2_fp8_scale; p.logits = s.parts;
  // the opt-in is per device context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(read_step_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, R8_SMEM_BYTES));
  read_step_fp8_kernel<<<(M + RS_BM - 1) / RS_BM, RS_THREADS, R8_SMEM_BYTES, stream>>>(mp, mq, mw1, mw2, p);
  MAC_LAUNCH_CHECK();
  return mac_kb_attend_fwd(s.parts, 1, w->br, kb_bf16, 1, att, info, B, N, d, stream);
}

}  // namespace mac
