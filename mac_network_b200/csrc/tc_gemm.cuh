// bf16 tensor-core GEMM for sm_90a: wgmma.mma_async (64 x 128 x 16 per warpgroup, fp32 accumulators in registers), operands
// staged by TMA (cp.async.bulk.tensor, 128-byte swizzle) through an mbarrier ring, and the read unit's elementwise work
// fused into the register epilogue.
//
//   C[M,N] = epilogue( A[M,K] @ Wt[N,K]^T )      A, Wt bf16 row-major with K contiguous ("K-major" both)
//
// One CTA per 128 x 128 output tile (x K slice when split-K), 288 threads:
//   warpgroups 0, 1   consumers: rows [64 g, 64 g + 64) of the tile against all 128 columns (64 accumulators per thread);
//                     they issue the wgmma, then run the epilogue straight from the accumulator registers
//   warp 8            TMA producer (one elected lane issues the A and B boxes of each k-block)
// The 3-stage ring takes 96 KB of shared memory.  The epilogues with the most live values (P, LOGITS) need 160+ registers,
// so a CTA of 288 threads has the SM's register file to itself: there is no cross-CTA overlap of epilogue and main loop.
//
// Epilogues (the read-unit chain of mac_cell.py:230-266 / ops.py:668-725, see mac_b200.h):
//   TC_EPI_P       P = acc + bx            -> bf16 P and bf16 P*y[b]            (ops.py:688, 694-703)
//   TC_EPI_ACT     act(acc + b)            -> bf16                               (mac_cell.py:236-238)
//   TC_EPI_LOGITS  I1 = acc + bm2; t = ELU(I1 * control[b]); (dropout); parts[m, ntile] = sum_n t * wr[n]
//                                                                                (ops.py:325-328, mac_cell.py:248-266)
//                  outf != NULL also stores I1 in fp32 at outf[m * N + n] (the tc32 training forward's saved I1)
//   TC_EPI_F32     act(acc + b + bias_const) -> fp32, stored or added (accum)   (generic ops.linear; act in every MAC_ACT_*)
//   TC_EPI_ADDACT  act(acc + b + add[m,n]) -> bf16, add = bf16 [M, N]           (eval-mode read: step-invariant half of
//                                                                                 the memKbProj concat, mac_cell.py:236-238)
//   TC_EPI_ACT_SPLIT  x = act(acc + b + addf[m,n]) (addf fp32, optional) -> bf16 hi at out0[m, n] and bf16 lo = x - hi at
//                     out0[m, N + n] (ldo = 2N): the A operand of the next split-bf16 ("tc32") product; outf != NULL also
//                     stores x in fp32 at outf[m * N + n] (the tc32 training forward's saved H, exactly as computed here)
//   TC_EPI_F32_ADD act(acc + b + addf[m,n]) -> fp32 at outf, addf fp32 [M, ldaf] and possibly outf itself; no split-K
//                  (the location-aware stem's layer 0: the image product added to the location product, stem.py)
#pragma once
#include "common.cuh"
#include "tmap.cuh"
#include <stdlib.h>

namespace mac {

enum { TC_EPI_P = 0, TC_EPI_ACT = 1, TC_EPI_LOGITS = 2, TC_EPI_F32 = 3, TC_EPI_ADDACT = 4, TC_EPI_ACT_SPLIT = 5,
       TC_EPI_F32_ADD = 6 };

struct TcGemmParams {
  int M, N, K;
  int kblocks0;            // k-blocks (of 64) served by tensor map a0; the rest come from a1 (concat along K)
  int epi, act;
  const float* bias;       // [N] or NULL
  __nv_bfloat16* out0;     // bf16 output 0 (P / act / I1-save), may be NULL for TC_EPI_LOGITS
  __nv_bfloat16* out1;     // bf16 output 1 (P*y)
  float* outf;             // fp32 output (TC_EPI_F32)
  const __nv_bfloat16* add;   // TC_EPI_ADDACT: pre-activation addend [M, ldo]
  const float* addf;          // TC_EPI_ACT_SPLIT (optional), TC_EPI_F32_ADD: fp32 pre-activation addend [M, ldaf]
  int ldaf;
  int ldo;
  const float* y;          // [B, N] row scale for TC_EPI_P
  const float* ctrl;       // [B, N] for TC_EPI_LOGITS
  const float* wr;         // [N]
  float* parts;            // [M, N / TC_BN]
  int rows_per_batch;
  uint32_t e_thresh;       // dropout on the logits' input (0 = none)
  float e_scale;
  uint64_t seed;
  int e_site, step;
  int ksplit;              // split-K (TC_EPI_F32 only): the K range is cut into `ksplit` equal slices (grid z), each writing
  long long split_stride;  //   its fp32 partial to outf + slice * split_stride; 0 / 1 = off
  float bias_const;        // TC_EPI_F32: added to every pre-activation (ops.linear's bias_const, mac_linear_fwd)
  int accum;               // TC_EPI_F32: outf (+)= act(...) -- the data gradients of mac_linear_bwd_tc with dx_accum
  int promote;             // TC_EPI_F32: two-level accumulation (tc_gemm_kernel's PROMOTE form); 0 = one accumulator
};

// ------------------------------------------------------------------ wgmma PTX wrappers
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulators are register operands of the asynchronous MMA: keep the compiler from touching them before the wait
template <int R>
__device__ __forceinline__ void wgmma_hold(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor of a K-major tile stored as rows of 128 bytes with the 128-byte swizzle (what TMA
// SWIZZLE_128B writes for a [rows x 64 bf16] box): start address >> 4 | LBO (unused for swizzled K-major; 1) |
// SBO = 1024 B between 8-row groups | layout type 1 (SWIZZLE_128B) in bits 62-63.  The tile base must be 1024-byte aligned.
// Advancing 16 bf16 (32 bytes) along K inside the swizzle atom is +2 in the address field.
__device__ __forceinline__ uint64_t make_sw128_kmajor_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // bits [0,14)
  d |= (uint64_t)1 << 16;                        // leading byte offset (16-B units), bits [16,30)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset, bits [32,46)
  d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
  return d;
}

// D[64 x N] (+)= A[64 x 16] B[16 x N], both operands from shared memory; accum == 0 overwrites D
__device__ __forceinline__ void wgmma_bf16_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

__device__ __forceinline__ void wgmma_bf16_n64(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

__device__ __forceinline__ void wgmma_bf16_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}

constexpr int TC_BK = 64;                 // 64 bf16 = 128 B = one swizzle atom row
constexpr int TC_BM = 128;
constexpr int TC_BN = 128;
constexpr int TC_STAGES = 3;
constexpr int TC_A_BYTES = TC_BM * TC_BK * 2;             // 16 KB
constexpr int TC_B_BYTES = TC_BN * TC_BK * 2;             // 16 KB
constexpr int TC_STAGE_BYTES = TC_A_BYTES + TC_B_BYTES;
constexpr int TC_CONSUMERS = 256;                         // two warpgroups
constexpr int TC_THREADS = TC_CONSUMERS + 32;
constexpr int TC_SMEM_BYTES = TC_STAGES * TC_STAGE_BYTES + 1024 /*align*/ + 128 /*barriers*/;

// fast ELU for the tensor-core path: x > 0 ? x : exp(x) - 1 with the SFU exponential (abs error ~1e-7 near 0,
// far below the bf16 rounding of the stored activations)
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float elu_fast(float x) {
  const float e = ex2_ftz(x * 1.4426950408889634f) - 1.f;
  return x > 0.f ? x : e;
}
template <int ACT>
__device__ __forceinline__ float act_ct(float x) {
  if constexpr (ACT == MAC_ACT_TANH) return tanhf(x);
  else if constexpr (ACT == MAC_ACT_SIGMOID) return 1.f / (1.f + __expf(-x));
  else if constexpr (ACT == MAC_ACT_ELU) return elu_fast(x);
  else if constexpr (ACT == MAC_ACT_RELU) return fmaxf(x, 0.f);
  else return x;
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ uint32_t pack_bf16_lo(float a, float b, uint32_t hw) {      // lo of the pair whose hi is `hw`
  return pack_bf16(a - __uint_as_float(hw << 16), b - __uint_as_float(hw & 0xffff0000u));
}

// Two-level accumulation (PROMOTE): every TC_PROMOTE_KB k-blocks go into a fresh register accumulator, which the CUDA
// cores then add into the fp32 master accumulator.  Hopper's bf16 wgmma adds its products into an accumulator with fewer
// mantissa bits than an fp32 add: with one accumulator over the image stem's K = 9 C (9216 at C = 1024, tripled by the
// split's three terms) the loss grows with the accumulator's magnitude, and the split-bf16 stem's output left the fp32
// parity bar once composed with the cell.  Bounding each wgmma sum to 128 products keeps mac_linear_tc32_fwd near an fp32
// dot product (tests/test_gpu_stem_bf16x3.py).  The group's last k-block waits for all of its MMAs before the add.
constexpr int TC_PROMOTE_KB = 2;

// SAVE (TC_EPI_ACT_SPLIT / TC_EPI_LOGITS with outf != NULL): a separate instantiation, so the inference form's kernels
// (outf == NULL) are compiled exactly as without the fp32 store; PROMOTE (TC_EPI_F32 only) likewise
template <int EPI, int ACT, bool SAVE = false, bool PROMOTE = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
               const __grid_constant__ CUtensorMap map_b, const TcGemmParams p) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  const uint32_t pad = (1024u - (base_u32 & 1023u)) & 1023u;
  unsigned char* tiles = smem_dyn + pad;                   // 1024-byte aligned operand ring
  uint64_t* full = reinterpret_cast<uint64_t*>(tiles + TC_STAGES * TC_STAGE_BYTES);   // [STAGES] TMA -> consumers
  uint64_t* empty = full + TC_STAGES;                                                 // [STAGES] consumers -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nt = blockIdx.x, mt = blockIdx.y;
  const int n_tiles = gridDim.x;
  const int kblocks = p.K / TC_BK / (int)gridDim.z;        // k-blocks of this CTA's K slice
  const int kb0 = (int)blockIdx.z * kblocks;

  if (threadIdx.x == TC_CONSUMERS) {
    tma_prefetch_desc(&map_a0);
    tma_prefetch_desc(&map_a1);
    tma_prefetch_desc(&map_b);
#pragma unroll
    for (int i = 0; i < TC_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], TC_CONSUMERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == TC_CONSUMERS / 32) {
    // ===================================================== TMA producer
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb0; kb < kb0 + kblocks; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1);
        unsigned char* sa = tiles + stage * TC_STAGE_BYTES;
        mbar_expect_tx(&full[stage], TC_STAGE_BYTES);
        if (kb < p.kblocks0)
          tma_load_2d(sa, &map_a0, kb * TC_BK, mt * TC_BM, &full[stage]);
        else
          tma_load_2d(sa, &map_a1, (kb - p.kblocks0) * TC_BK, mt * TC_BM, &full[stage]);
        tma_load_2d(sa + TC_A_BYTES, &map_b, kb * TC_BK, nt * TC_BN, &full[stage]);
        if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // ===================================================== consumers: main loop
  const int g = warp >> 2;                                  // warpgroup: rows [64 g, 64 g + 64) of the tile
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  if constexpr (PROMOTE) {
    float blk[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) blk[i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < kblocks; ++kb) {
      const int kg = kb % TC_PROMOTE_KB;                    // place in the current group: 0 starts a fresh accumulator
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(tiles + stage * TC_STAGE_BYTES);
      const uint64_t adesc = make_sw128_kmajor_desc(sa + g * (64 * 128));
      const uint64_t bdesc = make_sw128_kmajor_desc(sa + TC_A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n128(blk, adesc + 2 * k, bdesc + 2 * k, (kg | k) ? 1u : 0u);
      wgmma_commit();
      if (kg == TC_PROMOTE_KB - 1 || kb == kblocks - 1) {
        wgmma_wait<0>();                                    // the group's products have retired
        wgmma_hold(blk);
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] += blk[i];
      } else {
        wgmma_wait<1>();                                    // the previous k-block's products have retired
        wgmma_hold(blk);
      }
      if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
    }
  } else {
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(&full[stage], phase);
      const uint32_t sa = smem_u32(tiles + stage * TC_STAGE_BYTES);
      const uint64_t adesc = make_sw128_kmajor_desc(sa + g * (64 * 128));
      const uint64_t bdesc = make_sw128_kmajor_desc(sa + TC_A_BYTES);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n128(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                                      // the previous k-block's products have retired
      wgmma_hold(acc);
      if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
  }

  // ===================================================== epilogue, straight from the accumulator fragment:
  // acc[4 j + 2 h + e] is row (16 * (warp & 3) + lane / 4 + 8 h) of the warpgroup's 64, column 8 j + 2 (lane & 3) + e
  float* const outf_t = p.outf + (size_t)blockIdx.z * (size_t)p.split_stride;      // split-K partial (slice 0: outf)
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = mt * TC_BM + g * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
    const bool row_ok = row < p.M;
    const int bidx = (row_ok ? row : 0) / p.rows_per_batch;
    float part = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int n = nt * TC_BN + 8 * j + cq;
      float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
      if (p.bias) {
        x0 += __ldg(p.bias + n);
        x1 += __ldg(p.bias + n + 1);
      }
      const size_t o = (size_t)row * p.ldo + n;
      if constexpr (EPI == TC_EPI_P) {
        const float2 yv = __ldg(reinterpret_cast<const float2*>(p.y + (size_t)bidx * p.N + n));
        if (row_ok) {
          *reinterpret_cast<uint32_t*>(p.out0 + o) = pack_bf16(x0, x1);
          *reinterpret_cast<uint32_t*>(p.out1 + o) = pack_bf16(x0 * yv.x, x1 * yv.y);
        }
      } else if constexpr (EPI == TC_EPI_ACT) {
        if (row_ok) *reinterpret_cast<uint32_t*>(p.out0 + o) = pack_bf16(act_ct<ACT>(x0), act_ct<ACT>(x1));
      } else if constexpr (EPI == TC_EPI_ADDACT) {
        if (row_ok) {
          const uint32_t q = __ldg(reinterpret_cast<const unsigned int*>(p.add + o));      // bf16 -> fp32 is a 16-bit shift
          *reinterpret_cast<uint32_t*>(p.out0 + o) =
              pack_bf16(act_ct<ACT>(x0 + __uint_as_float(q << 16)), act_ct<ACT>(x1 + __uint_as_float(q & 0xffff0000u)));
        }
      } else if constexpr (EPI == TC_EPI_ACT_SPLIT) {
        if (row_ok) {
          if (p.addf) {
            const float2 a = *reinterpret_cast<const float2*>(p.addf + (size_t)row * p.ldaf + n);
            x0 += a.x;
            x1 += a.y;
          }
          x0 = act_ct<ACT>(x0);
          x1 = act_ct<ACT>(x1);
          if constexpr (SAVE) *reinterpret_cast<float2*>(p.outf + (size_t)row * p.N + n) = make_float2(x0, x1);
          const uint32_t hw = pack_bf16(x0, x1);
          *reinterpret_cast<uint32_t*>(p.out0 + o) = hw;
          *reinterpret_cast<uint32_t*>(p.out0 + o + p.N) =
              pack_bf16(x0 - __uint_as_float(hw << 16), x1 - __uint_as_float(hw & 0xffff0000u));
        }
      } else if constexpr (EPI == TC_EPI_F32) {
        if (row_ok) {
          if (p.bias_const != 0.f) {
            x0 += p.bias_const;
            x1 += p.bias_const;
          }
          float2 v = make_float2(act_ct<ACT>(x0), act_ct<ACT>(x1));
          if (p.accum) {
            const float2 prev = *reinterpret_cast<const float2*>(outf_t + o);
            v.x += prev.x;
            v.y += prev.y;
          }
          *reinterpret_cast<float2*>(outf_t + o) = v;
        }
      } else if constexpr (EPI == TC_EPI_F32_ADD) {
        if (row_ok) {                                       // addf may be outf itself: each element is read, then written
          const float2 a = *reinterpret_cast<const float2*>(p.addf + (size_t)row * p.ldaf + n);
          *reinterpret_cast<float2*>(p.outf + o) = make_float2(act_ct<ACT>(x0 + a.x), act_ct<ACT>(x1 + a.y));
        }
      } else {  // TC_EPI_LOGITS
        const float2 cc = __ldg(reinterpret_cast<const float2*>(p.ctrl + (size_t)bidx * p.N + n));
        const float2 ww = make_float2(__ldg(p.wr + n), __ldg(p.wr + n + 1));
        if (p.out0 && row_ok) *reinterpret_cast<uint32_t*>(p.out0 + o) = pack_bf16(x0, x1);   // I1 kept for backward
        if constexpr (SAVE)
          if (row_ok) *reinterpret_cast<float2*>(p.outf + (size_t)row * p.N + n) = make_float2(x0, x1);
        float t0 = elu_fast(x0 * cc.x), t1 = elu_fast(x1 * cc.y);
        if (p.e_thresh) {
          // one Philox draw per aligned column quad of element index row * N + n (the fp32 path's numbering)
          const uint64_t e = (uint64_t)row * (uint64_t)p.N + (uint64_t)n;
          const Philox4 rr = philox4x32_10(p.seed, e >> 2, (uint32_t)p.e_site, (uint32_t)p.step);
          const uint32_t u0 = (e & 2) ? rr.z : rr.x, u1 = (e & 2) ? rr.w : rr.y;
          t0 = ((u0 >> 8) >= p.e_thresh) ? t0 * p.e_scale : 0.f;
          t1 = ((u1 >> 8) >= p.e_thresh) ? t1 * p.e_scale : 0.f;
        }
        part = fmaf(t0, ww.x, part);
        part = fmaf(t1, ww.y, part);
      }
    }
    if constexpr (EPI == TC_EPI_LOGITS) {
      // the four lanes of a row hold disjoint column pairs: one partial sum per (row, n-tile)
      part += __shfl_xor_sync(0xffffffffu, part, 1);
      part += __shfl_xor_sync(0xffffffffu, part, 2);
      if (row_ok && (lane & 3) == 0) p.parts[(size_t)row * n_tiles + nt] = part;
    }
  }
}

// ------------------------------------------------------------------ host side
inline int tc_num_sms() { return mac_num_sms(); }

template <int EPI, int ACT, bool SAVE = false, bool PROMOTE = false>
inline int tc_gemm_launch_t(const CUtensorMap& ma0, const CUtensorMap& ma1, const CUtensorMap& mb,
                            const TcGemmParams& p, cudaStream_t stream) {
  auto kern = tc_gemm_kernel<EPI, ACT, SAVE, PROMOTE>;
  // the shared-memory opt-in belongs to the current device's context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
  const dim3 grid(p.N / TC_BN, (p.M + TC_BM - 1) / TC_BM, p.ksplit > 1 ? p.ksplit : 1);
  kern<<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(ma0, ma1, mb, p);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

inline int tc_gemm_dispatch(const CUtensorMap& ma0, const CUtensorMap& ma1, const CUtensorMap& mb,
                            const TcGemmParams& p, cudaStream_t stream) {
  if (p.promote && p.epi == TC_EPI_F32_ADD) {
    switch (p.act) {
      case MAC_ACT_NON: return tc_gemm_launch_t<TC_EPI_F32_ADD, MAC_ACT_NON, false, true>(ma0, ma1, mb, p, stream);
      case MAC_ACT_ELU: return tc_gemm_launch_t<TC_EPI_F32_ADD, MAC_ACT_ELU, false, true>(ma0, ma1, mb, p, stream);
      case MAC_ACT_RELU: return tc_gemm_launch_t<TC_EPI_F32_ADD, MAC_ACT_RELU, false, true>(ma0, ma1, mb, p, stream);
    }
    return MAC_ERR_UNSUPPORTED;
  }
  if (p.promote) {
    if (p.epi != TC_EPI_F32) return MAC_ERR_UNSUPPORTED;
    switch (p.act) {
      case MAC_ACT_NON: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_NON, false, true>(ma0, ma1, mb, p, stream);
      case MAC_ACT_ELU: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_ELU, false, true>(ma0, ma1, mb, p, stream);
      case MAC_ACT_RELU: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_RELU, false, true>(ma0, ma1, mb, p, stream);
    }
    return MAC_ERR_UNSUPPORTED;
  }
  switch (p.epi) {
    case TC_EPI_P: return tc_gemm_launch_t<TC_EPI_P, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
    case TC_EPI_ADDACT:
      if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ADDACT, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
      return MAC_ERR_UNSUPPORTED;
    case TC_EPI_LOGITS:
      if (p.outf) return tc_gemm_launch_t<TC_EPI_LOGITS, MAC_ACT_NON, true>(ma0, ma1, mb, p, stream);
      return tc_gemm_launch_t<TC_EPI_LOGITS, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
    case TC_EPI_ACT_SPLIT:
      if (p.outf) {
        if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ACT_SPLIT, MAC_ACT_ELU, true>(ma0, ma1, mb, p, stream);
        return MAC_ERR_UNSUPPORTED;
      }
      if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ACT_SPLIT, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
      if (p.act == MAC_ACT_NON) return tc_gemm_launch_t<TC_EPI_ACT_SPLIT, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
      return MAC_ERR_UNSUPPORTED;
    case TC_EPI_ACT:
      if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ACT, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
      if (p.act == MAC_ACT_NON) return tc_gemm_launch_t<TC_EPI_ACT, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
      return MAC_ERR_UNSUPPORTED;
    case TC_EPI_F32_ADD:
      if (p.ksplit > 1) return MAC_ERR_UNSUPPORTED;
      switch (p.act) {
        case MAC_ACT_NON: return tc_gemm_launch_t<TC_EPI_F32_ADD, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
        case MAC_ACT_ELU: return tc_gemm_launch_t<TC_EPI_F32_ADD, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
        case MAC_ACT_RELU: return tc_gemm_launch_t<TC_EPI_F32_ADD, MAC_ACT_RELU>(ma0, ma1, mb, p, stream);
      }
      return MAC_ERR_UNSUPPORTED;
    case TC_EPI_F32:
      switch (p.act) {
        case MAC_ACT_NON: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
        case MAC_ACT_TANH: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_TANH>(ma0, ma1, mb, p, stream);
        case MAC_ACT_SIGMOID: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_SIGMOID>(ma0, ma1, mb, p, stream);
        case MAC_ACT_ELU: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
        case MAC_ACT_RELU: return tc_gemm_launch_t<TC_EPI_F32, MAC_ACT_RELU>(ma0, ma1, mb, p, stream);
      }
      return MAC_ERR_UNSUPPORTED;
  }
  return MAC_ERR_UNSUPPORTED;
}

// A = [a0 (K0 cols) | a1 (K1 cols)] bf16 row-major (ld = own K), Wt bf16 [N, K0+K1]
inline int tc_gemm_launch(const void* a0, int K0, const void* a1, int K1, const void* wt, TcGemmParams p,
                          cudaStream_t stream, int ldw = 0, int lda0 = 0, int lda1 = 0) {
  if (ldw == 0) ldw = K0 + K1;                  // row pitch of Wt in elements (> K: a column block of a wider weight)
  if (lda0 == 0) lda0 = K0;                     // row pitch of the A segments (> K: a column block of a wider matrix)
  if (lda1 == 0) lda1 = K1;
  if (p.M <= 0 || p.N <= 0 || (p.N % TC_BN) || (K0 % TC_BK) || (K1 % TC_BK) || K0 <= 0) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(a0) || !mac_aligned16(wt)) return MAC_ERR_ALIGN;
  if (p.ksplit > 1 && ((K0 + K1) / TC_BK) % p.ksplit) return MAC_ERR_UNSUPPORTED;
  p.K = K0 + K1;
  p.kblocks0 = K0 / TC_BK;
  CUtensorMap ma0, ma1, mb;
  int st = make_tmap_2d(&ma0, a0, 1, (uint64_t)p.M, (uint64_t)K0, (uint64_t)lda0 * 2, (uint32_t)TC_BM, TC_BK, 1);
  if (st != MAC_OK) return st;
  if (K1 > 0) {
    st = make_tmap_2d(&ma1, a1, 1, (uint64_t)p.M, (uint64_t)K1, (uint64_t)lda1 * 2, (uint32_t)TC_BM, TC_BK, 1);
    if (st != MAC_OK) return st;
  } else {
    ma1 = ma0;
  }
  st = make_tmap_2d(&mb, wt, 1, (uint64_t)p.N, (uint64_t)p.K, (uint64_t)ldw * 2, (uint32_t)TC_BN, TC_BK, 1);
  if (st != MAC_OK) return st;
  return tc_gemm_dispatch(ma0, ma1, mb, p, stream);
}

// fp32 [K, N] (in, out) weight -> bf16 [N, K] (out, in): the K-major B operand of the forward GEMMs
__global__ void pack_weight_bf16_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ Wt, int K, int N) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? W[(size_t)k * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < K) Wt[(size_t)n * K + k] = __float2bfloat16_rn(tile[threadIdx.x][i]);
  }
}

// Activations for a tensor-core weight gradient: fp32 X [K rows, N cols] -> bf16 X^T [N, K] (the contraction index K = B*N rows
// becomes the K-major direction of both wgrad operands), optionally also the row-major bf16 copy (the A operand of the matching
// data gradient) from the same read.  64x64 tiles: 256-byte row reads, 128-byte row writes.
//   MODE 0 plain; 1 x * rowvec[row / rows_per_batch, col] (P * y, ops.py:694-703); 2 dropout(x) with the forward's Philox stream
//   (one draw per aligned column quad, element index row*N + col: mac_dropout_fwd's numbering).      N % 4 == 0, K % 2 == 0.
// ldx is the row pitch of X (elements); Xt rows have pitch ldt >= K, and columns K..ldt-1 of Xt are written as zeros (a
// contraction length padded to the 64-wide k-block).
// Split mode (SEGS = 2 or 3, the operands of the split-bf16 "tc32" weight gradients): every value v is written as hi = bf16(v)
// and lo = bf16(v - hi) into segments of kp columns of an Xt row (pitch ldt = SEGS * kp): [hi | lo] (SEGS 2) or [hi | hi | lo]
// (SEGS 3), each with zero columns K..kp-1; Xrm (if given) receives the row-major [hi | lo] copy [K, 2N].
template <int MODE, int SEGS = 0>
__global__ void __launch_bounds__(256) pack_t_bf16_kernel(const float* __restrict__ X, __nv_bfloat16* __restrict__ Xt,
                                                         __nv_bfloat16* __restrict__ Xrm, int K, int N,
                                                         const float* __restrict__ rowvec, int rows_per_batch, uint32_t thresh,
                                                         float scale, uint64_t seed, int site, int step, int ldx, int ldt,
                                                         int kp = 0) {
  __shared__ float tile[64][65];                              // [col][row]
  const int k0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tq = threadIdx.x & 15, tr = threadIdx.x >> 4;     // 16 column quads x 16 rows per pass
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int kk = tr + 16 * p;
    const int k = k0 + kk, n = n0 + tq * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < K && n < N) {
      v = *reinterpret_cast<const float4*>(X + (size_t)k * ldx + n);
      if (MODE == 1) {
        const float4 y = *reinterpret_cast<const float4*>(rowvec + (size_t)(k / rows_per_batch) * N + n);
        v.x *= y.x; v.y *= y.y; v.z *= y.z; v.w *= y.w;
      }
      if (MODE == 2) {
        const uint64_t e = (uint64_t)k * (uint64_t)N + (uint64_t)n;
        const Philox4 r = philox4x32_10(seed, e >> 2, (uint32_t)site, (uint32_t)step);
        v.x = ((r.x >> 8) >= thresh) ? v.x * scale : 0.f;
        v.y = ((r.y >> 8) >= thresh) ? v.y * scale : 0.f;
        v.z = ((r.z >> 8) >= thresh) ? v.z * scale : 0.f;
        v.w = ((r.w >> 8) >= thresh) ? v.w * scale : 0.f;
      }
      if (Xrm && SEGS == 0) {
        *reinterpret_cast<uint2*>(Xrm + (size_t)k * N + n) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
      } else if (Xrm) {
        const uint32_t h01 = pack_bf16(v.x, v.y), h23 = pack_bf16(v.z, v.w);
        const uint32_t l01 = pack_bf16(v.x - __uint_as_float(h01 << 16), v.y - __uint_as_float(h01 & 0xffff0000u));
        const uint32_t l23 = pack_bf16(v.z - __uint_as_float(h23 << 16), v.w - __uint_as_float(h23 & 0xffff0000u));
        *reinterpret_cast<uint2*>(Xrm + (size_t)k * 2 * N + n) = make_uint2(h01, h23);
        *reinterpret_cast<uint2*>(Xrm + (size_t)k * 2 * N + N + n) = make_uint2(l01, l23);
      }
    }
    tile[tq * 4 + 0][kk] = v.x;
    tile[tq * 4 + 1][kk] = v.y;
    tile[tq * 4 + 2][kk] = v.z;
    tile[tq * 4 + 3][kk] = v.w;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if constexpr (SEGS == 0) {
    for (int r = warp; r < 64; r += 8) {
      const int n = n0 + r, k = k0 + 2 * lane;
      if (n < N && k + 1 < ldt)
        *reinterpret_cast<uint32_t*>(Xt + (size_t)n * ldt + k) = pack_bf16(tile[r][2 * lane], tile[r][2 * lane + 1]);
    }
  } else {
  for (int r = warp; r < 64; r += 8) {
    const int n = n0 + r, k = k0 + 2 * lane;
    if (n < N && k + 1 < kp) {
      const float a = tile[r][2 * lane], b = tile[r][2 * lane + 1];
      const uint32_t hw = pack_bf16(a, b);
      const uint32_t lw = pack_bf16(a - __uint_as_float(hw << 16), b - __uint_as_float(hw & 0xffff0000u));
      __nv_bfloat16* row = Xt + (size_t)n * ldt + k;
      *reinterpret_cast<uint32_t*>(row) = hw;
      *reinterpret_cast<uint32_t*>(row + kp) = SEGS == 3 ? hw : lw;
      if (SEGS == 3) *reinterpret_cast<uint32_t*>(row + 2 * kp) = lw;
    }
  }
  }
}

struct PackTArgs {
  const float* rowvec = nullptr;
  int rows_per_batch = 1;
  uint32_t thresh = 0;
  float scale = 1.f;
  uint64_t seed = 0;
  int site = 0, step = 0;
};

// ldx: row pitch of X (0: N); ldt: row pitch of Xt (0: K), >= K and even -- columns K..ldt-1 are written as zeros
inline int pack_t_bf16_launch(int mode, const float* X, void* Xt, void* Xrm, int K, int N, const PackTArgs& a,
                              cudaStream_t stream, int ldx = 0, int ldt = 0) {
  if (ldx == 0) ldx = N;
  if (ldt == 0) ldt = K;
  if (!X || !Xt || K <= 0 || N <= 0 || (N & 3) || (ldx & 3) || ldx < N || (ldt & 1) || ldt < K) return MAC_ERR_INVALID;
  dim3 grid((N + 63) / 64, (ldt + 63) / 64);
  __nv_bfloat16* t = reinterpret_cast<__nv_bfloat16*>(Xt);
  __nv_bfloat16* r = reinterpret_cast<__nv_bfloat16*>(Xrm);
  if (mode == 0)
    pack_t_bf16_kernel<0><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, 0u, 1.f, 0, 0, 0, ldx, ldt);
  else if (mode == 1)
    pack_t_bf16_kernel<1><<<grid, 256, 0, stream>>>(X, t, r, K, N, a.rowvec, a.rows_per_batch, 0u, 1.f, 0, 0, 0, ldx, ldt);
  else
    pack_t_bf16_kernel<2><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, a.thresh, a.scale, a.seed, a.site, a.step, ldx,
                                                    ldt);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// split mode of pack_t_bf16 (see the kernel): X [K, N] (pitch N) -> Xt [N, segs * kp] with kp = K rounded up to 64, segs 2
// ([hi | lo], modes 0, 1, 2: the activations) or 3 ([hi | hi | lo], mode 0: the gradients), row pitch segs * kp; Xrm (may
// be NULL): [K, 2N] [hi | lo]
inline int pack_t_split_launch(int mode, const float* X, void* Xt, void* Xrm, int K, int N, int segs, const PackTArgs& a,
                               cudaStream_t stream) {
  if (!X || !Xt || K <= 0 || N <= 0 || (N & 3) || (segs != 2 && segs != 3) || mode < 0 || mode > 2 || (segs == 3 && mode))
    return MAC_ERR_INVALID;
  const int kp = (K + 63) & ~63;
  const int ldt = segs * kp;
  dim3 grid((N + 63) / 64, kp / 64);
  __nv_bfloat16* t = reinterpret_cast<__nv_bfloat16*>(Xt);
  __nv_bfloat16* r = reinterpret_cast<__nv_bfloat16*>(Xrm);
  if (segs == 3)
    pack_t_bf16_kernel<0, 3><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, 0u, 1.f, 0, 0, 0, N, ldt, kp);
  else if (mode == 0)
    pack_t_bf16_kernel<0, 2><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, 0u, 1.f, 0, 0, 0, N, ldt, kp);
  else if (mode == 1)
    pack_t_bf16_kernel<1, 2><<<grid, 256, 0, stream>>>(X, t, r, K, N, a.rowvec, a.rows_per_batch, 0u, 1.f, 0, 0, 0, N, ldt,
                                                       kp);
  else
    pack_t_bf16_kernel<2, 2><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, a.thresh, a.scale, a.seed, a.site, a.step,
                                                       N, ldt, kp);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// bf16 -> fp32 widening of up to three equally long slabs in one launch (the activations the tensor-core training forward
// leaves in bf16, read in fp32 by the backward kernels)
__global__ void __launch_bounds__(256) widen3_bf16_kernel(const uint4* __restrict__ s0, const uint4* __restrict__ s1,
                                                         const uint4* __restrict__ s2, float4* __restrict__ d0,
                                                         float4* __restrict__ d1, float4* __restrict__ d2, long long n8) {
  const uint4* s = blockIdx.y == 0 ? s0 : blockIdx.y == 1 ? s1 : s2;
  float4* d = blockIdx.y == 0 ? d0 : blockIdx.y == 1 ? d1 : d2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
    const uint4 v = s[i];
    d[2 * i] = make_float4(__uint_as_float(v.x << 16), __uint_as_float(v.x & 0xffff0000u), __uint_as_float(v.y << 16),
                           __uint_as_float(v.y & 0xffff0000u));
    d[2 * i + 1] = make_float4(__uint_as_float(v.z << 16), __uint_as_float(v.z & 0xffff0000u), __uint_as_float(v.w << 16),
                               __uint_as_float(v.w & 0xffff0000u));
  }
}
// dst[i][0, n) = fp32(src[i][0, n)) for nslab <= 3 slabs: n % 8 == 0, every pointer 16-byte aligned
inline int widen3_bf16_launch(const void* const* src, float* const* dst, int nslab, long long n, cudaStream_t stream) {
  const uint4* s[3] = {nullptr, nullptr, nullptr};
  float4* d[3] = {nullptr, nullptr, nullptr};
  for (int i = 0; i < nslab; ++i) {
    s[i] = reinterpret_cast<const uint4*>(src[i]);
    d[i] = reinterpret_cast<float4*>(dst[i]);
  }
  const long long n8 = n / 8;
  const unsigned gx = (unsigned)std::min<long long>((n8 + 255) / 256, (long long)mac_num_sms() * 16);
  widen3_bf16_kernel<<<dim3(gx, nslab), 256, 0, stream>>>(s[0], s[1], s[2], d[0], d[1], d[2], n8);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

inline char* tc_align1k(void* p) {
  return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

// ---------------------------------------------------------------------------------------------------------------
// Weight gradients on tensor cores: dW[in, out] (+)= X^T[in, M] @ G^T[out, M]^T with K = M = B*N (12 544 at the headline shape)
// and only (in/128) x (out/256) = 8-16 output tiles: one K loop of 196 k-blocks per CTA left 130+ SMs idle (44.7 us per
// launch, 12 % of a tensor-core training step).  Split-K: the K range is cut into S slices, every (slice, tile) is a tile of the
// persistent kernel and writes its fp32 partial; the partials are summed in slice order (deterministic) into dW.
__global__ void splitk_accum_kernel(const float4* __restrict__ part, float4* __restrict__ dst, long long n4, int S,
                                    long long stride4, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  float4 a = accumulate ? dst[i] : make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s_ = 0; s_ < S; ++s_) {
    const float4 v = part[i + s_ * stride4];
    a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
  }
  dst[i] = a;
}

// largest S <= 28 that divides K / 64, keeps >= 2 k-blocks per slice and at most two CTAs per SM
inline int tc_pick_ksplit(int K, int out_tiles) {
  const int kblocks = K / TC_BK;
  int best = 1;
  for (int S = 2; S <= 28; ++S)
    if (kblocks % S == 0 && kblocks / S >= 2 && out_tiles * S <= 2 * tc_num_sms()) best = S;
  return best;
}
inline size_t tc_wgrad_partial_bytes(int in_dim, int out_dim) { return (size_t)28 * in_dim * out_dim * 4; }

// dW[in, out] += xT[in, K] @ gT[out, K]^T   (both bf16, K-major); `partial` holds tc_wgrad_partial_bytes(in, out)
inline int tc_wgrad_splitk(const void* xT, const void* gT, float* dW, float* partial, int in_dim, int out_dim, int K,
                           cudaStream_t stream) {
  if ((in_dim % 128) || (out_dim % 128) || (K % TC_BK)) return MAC_ERR_UNSUPPORTED;
  TcGemmParams p{};
  p.M = in_dim; p.N = out_dim; p.act = MAC_ACT_NON; p.bias = nullptr; p.ldo = out_dim; p.rows_per_batch = 1;
  p.epi = TC_EPI_F32; p.outf = partial;
  const int out_tiles = (in_dim / TC_BM) * (out_dim / TC_BN);
  const int S = tc_pick_ksplit(K, out_tiles);
  p.ksplit = S; p.split_stride = (long long)in_dim * out_dim;
  int st = tc_gemm_launch(xT, K, nullptr, 0, gT, p, stream);
  if (st != MAC_OK) return st;
  const long long n4 = (long long)in_dim * out_dim / 4;
  splitk_accum_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(partial),
                                                                       reinterpret_cast<float4*>(dW), n4, S, n4, 1);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// "tc32": [B*N, .] products as SPLIT-bf16 products on the tensor cores (the read unit's, read_fwd.cuh, and their gradients),
// for the <= 1e-4 parity bar of BASELINE.json (the plain bf16 path is at ~1e-3).  Every fp32 operand x is carried as two bf16 values x_hi = bf16(x),
// x_lo = bf16(x - x_hi) and the product uses three of the four partial products, accumulated in ONE fp32 accumulator:
//     A W  ~=  A_hi W_hi + A_lo W_hi + A_hi W_lo                      (A_lo W_lo ~ 2^-16 relative is dropped)
// With A' = [A_hi | A_lo] ([M, 2K]) and W' = [W_hi | W_hi | W_lo] ([N, 3K], K-major) this is the existing two-segment GEMM:
// segment 0 = A'[:, 0:2K] against W'[:, 0:2K], segment 1 = A'[:, 0:K] against W'[:, 2K:3K] -- K triples, nothing else
// changes.  Producers write their outputs directly as hi | lo pairs (TC_EPI_ACT_SPLIT) or as fp32 (TC_EPI_F32).
// ---------------------------------------------------------------------------------------------------------------
// fp32 W[R, C] row-major -> bf16 W3[R, 3C] = [hi | hi | lo] per row, no transpose: the B operand of a split data gradient
// dX = G @ W^T with W in its own [in, out] layout (rows = in = the output columns of dX, K = out).  C % 4 == 0.
__global__ void split3_rows_kernel(const float4* __restrict__ W, uint2* __restrict__ W3, int C, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int c4n = C / 4;
  const long long r = i / c4n;
  const int c4 = (int)(i - r * c4n);
  const float4 u = W[i];
  const uint32_t h01 = pack_bf16(u.x, u.y), h23 = pack_bf16(u.z, u.w);
  const uint32_t l01 = pack_bf16(u.x - __uint_as_float(h01 << 16), u.y - __uint_as_float(h01 & 0xffff0000u));
  const uint32_t l23 = pack_bf16(u.z - __uint_as_float(h23 << 16), u.w - __uint_as_float(h23 & 0xffff0000u));
  uint2* row = W3 + r * (3 * c4n);
  row[c4] = make_uint2(h01, h23);
  row[c4n + c4] = make_uint2(h01, h23);
  row[2 * c4n + c4] = make_uint2(l01, l23);
}

// fp32 W[K, N] (rows k0 .. k0+K of a wider [*, N] weight are passed as W + k0*N) -> bf16 Wt3[N, 3K] = [hi | hi | lo]
__global__ void pack_weight_split3_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ Wt3, int K, int N) {
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
      __nv_bfloat16* row = Wt3 + (size_t)n * 3 * K;
      row[k] = h;
      row[K + k] = h;
      row[2 * K + k] = __float2bfloat16_rn(w - __bfloat162float(h));
    }
  }
}

// C = epilogue(A W) with A' = [A_hi | A_lo] ([M, 2K] bf16) and W' = [W_hi | W_hi | W_lo] ([N, 3K] bf16)
inline int tc3_gemm(const void* a_split, int K, const void* wt3, TcGemmParams p, cudaStream_t stream) {
  return tc_gemm_launch(a_split, 2 * K, a_split, K, wt3, p, stream, 3 * K, 2 * K, 2 * K);
}

// Split-bf16 weight gradient dW[in, out] += X^T G over a contraction of kp (= M rounded up to 64) rows:
//   xT2 = [X_hi^T | X_lo^T] [in, 2kp], gT3 = [G_hi^T | G_hi^T | G_lo^T] [out, 3kp] (pack_t_split_launch, zero columns M..kp-1)
// is tc3_gemm's two-segment product (X_hi G_hi + X_lo G_hi + X_hi G_lo) as ONE split-K launch over K = 3kp, whose slices are
// summed in slice order (deterministic).  `partial` holds tc_wgrad_partial_bytes(in, out).
inline int tc3_wgrad_splitk(const void* xT2, const void* gT3, float* dW, float* partial, int in_dim, int out_dim, int kp,
                            cudaStream_t stream) {
  if ((in_dim % 128) || (out_dim % 128) || (kp % TC_BK)) return MAC_ERR_UNSUPPORTED;
  TcGemmParams p{};
  p.M = in_dim; p.N = out_dim; p.act = MAC_ACT_NON; p.bias = nullptr; p.ldo = out_dim; p.rows_per_batch = 1;
  p.epi = TC_EPI_F32; p.outf = partial;
  const int S = tc_pick_ksplit(3 * kp, (in_dim / TC_BM) * (out_dim / TC_BN));
  p.ksplit = S; p.split_stride = (long long)in_dim * out_dim;
  int st = tc3_gemm(xT2, kp, gT3, p, stream);
  if (st != MAC_OK) return st;
  const long long n4 = (long long)in_dim * out_dim / 4;
  splitk_accum_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(partial),
                                                                       reinterpret_cast<float4*>(dW), n4, S, n4, 1);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac
