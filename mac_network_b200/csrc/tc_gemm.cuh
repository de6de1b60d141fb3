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
//   TC_EPI_F32     act(acc + b)            -> fp32                               (generic ops.linear)
//   TC_EPI_ADDACT  act(acc + b + add[m,n]) -> bf16, add = bf16 [M, N]           (eval-mode read: step-invariant half of
//                                                                                 the memKbProj concat, mac_cell.py:236-238)
//   TC_EPI_ACT_SPLIT  x = act(acc + b + addf[m,n]) (addf fp32, optional) -> bf16 hi at out0[m, n] and bf16 lo = x - hi at
//                     out0[m, N + n] (ldo = 2N): the A operand of the next split-bf16 ("tc32") product
#pragma once
#include "common.cuh"
#include "tmap.cuh"
#include <stdlib.h>

namespace mac {

enum { TC_EPI_P = 0, TC_EPI_ACT = 1, TC_EPI_LOGITS = 2, TC_EPI_F32 = 3, TC_EPI_ADDACT = 4, TC_EPI_ACT_SPLIT = 5 };

struct TcGemmParams {
  int M, N, K;
  int kblocks0;            // k-blocks (of 64) served by tensor map a0; the rest come from a1 (concat along K)
  int epi, act;
  const float* bias;       // [N] or NULL
  __nv_bfloat16* out0;     // bf16 output 0 (P / act / I1-save), may be NULL for TC_EPI_LOGITS
  __nv_bfloat16* out1;     // bf16 output 1 (P*y)
  float* outf;             // fp32 output (TC_EPI_F32)
  const __nv_bfloat16* add;   // TC_EPI_ADDACT: pre-activation addend [M, ldo]
  const float* addf;          // TC_EPI_ACT_SPLIT: optional fp32 pre-activation addend [M, ldaf]
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

template <int EPI, int ACT>
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
  {
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
          const uint32_t hw = pack_bf16(x0, x1);
          *reinterpret_cast<uint32_t*>(p.out0 + o) = hw;
          *reinterpret_cast<uint32_t*>(p.out0 + o + p.N) =
              pack_bf16(x0 - __uint_as_float(hw << 16), x1 - __uint_as_float(hw & 0xffff0000u));
        }
      } else if constexpr (EPI == TC_EPI_F32) {
        if (row_ok) *reinterpret_cast<float2*>(outf_t + o) = make_float2(act_ct<ACT>(x0), act_ct<ACT>(x1));
      } else {  // TC_EPI_LOGITS
        const float2 cc = __ldg(reinterpret_cast<const float2*>(p.ctrl + (size_t)bidx * p.N + n));
        const float2 ww = make_float2(__ldg(p.wr + n), __ldg(p.wr + n + 1));
        if (p.out0 && row_ok) *reinterpret_cast<uint32_t*>(p.out0 + o) = pack_bf16(x0, x1);   // I1 kept for backward
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

template <int EPI, int ACT>
inline int tc_gemm_launch_t(const CUtensorMap& ma0, const CUtensorMap& ma1, const CUtensorMap& mb,
                            const TcGemmParams& p, cudaStream_t stream) {
  auto kern = tc_gemm_kernel<EPI, ACT>;
  // the shared-memory opt-in belongs to the current device's context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES));
  const dim3 grid(p.N / TC_BN, (p.M + TC_BM - 1) / TC_BM, p.ksplit > 1 ? p.ksplit : 1);
  kern<<<grid, TC_THREADS, TC_SMEM_BYTES, stream>>>(ma0, ma1, mb, p);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

inline int tc_gemm_dispatch(const CUtensorMap& ma0, const CUtensorMap& ma1, const CUtensorMap& mb,
                            const TcGemmParams& p, cudaStream_t stream) {
  switch (p.epi) {
    case TC_EPI_P: return tc_gemm_launch_t<TC_EPI_P, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
    case TC_EPI_ADDACT:
      if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ADDACT, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
      return MAC_ERR_UNSUPPORTED;
    case TC_EPI_LOGITS: return tc_gemm_launch_t<TC_EPI_LOGITS, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
    case TC_EPI_ACT_SPLIT:
      if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ACT_SPLIT, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
      if (p.act == MAC_ACT_NON) return tc_gemm_launch_t<TC_EPI_ACT_SPLIT, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
      return MAC_ERR_UNSUPPORTED;
    case TC_EPI_ACT:
      if (p.act == MAC_ACT_ELU) return tc_gemm_launch_t<TC_EPI_ACT, MAC_ACT_ELU>(ma0, ma1, mb, p, stream);
      if (p.act == MAC_ACT_NON) return tc_gemm_launch_t<TC_EPI_ACT, MAC_ACT_NON>(ma0, ma1, mb, p, stream);
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
                          cudaStream_t stream, int* nparts_per_row = nullptr, int ldw = 0, int lda0 = 0, int lda1 = 0) {
  if (ldw == 0) ldw = K0 + K1;                  // row pitch of Wt in elements (> K: a column block of a wider weight)
  if (lda0 == 0) lda0 = K0;                     // row pitch of the A segments (> K: a column block of a wider matrix)
  if (lda1 == 0) lda1 = K1;
  if (p.M <= 0 || p.N <= 0 || (p.N % TC_BN) || (K0 % TC_BK) || (K1 % TC_BK) || K0 <= 0) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(a0) || !mac_aligned16(wt)) return MAC_ERR_ALIGN;
  if (p.ksplit > 1 && ((K0 + K1) / TC_BK) % p.ksplit) return MAC_ERR_UNSUPPORTED;
  if (nparts_per_row) *nparts_per_row = p.N / TC_BN;
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
template <int MODE>
__global__ void __launch_bounds__(256) pack_t_bf16_kernel(const float* __restrict__ X, __nv_bfloat16* __restrict__ Xt,
                                                         __nv_bfloat16* __restrict__ Xrm, int K, int N,
                                                         const float* __restrict__ rowvec, int rows_per_batch, uint32_t thresh,
                                                         float scale, uint64_t seed, int site, int step) {
  __shared__ float tile[64][65];                              // [col][row]
  const int k0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tq = threadIdx.x & 15, tr = threadIdx.x >> 4;     // 16 column quads x 16 rows per pass
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int kk = tr + 16 * p;
    const int k = k0 + kk, n = n0 + tq * 4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k < K && n < N) {
      v = *reinterpret_cast<const float4*>(X + (size_t)k * N + n);
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
      if (Xrm) *reinterpret_cast<uint2*>(Xrm + (size_t)k * N + n) = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
    }
    tile[tq * 4 + 0][kk] = v.x;
    tile[tq * 4 + 1][kk] = v.y;
    tile[tq * 4 + 2][kk] = v.z;
    tile[tq * 4 + 3][kk] = v.w;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < 64; r += 8) {
    const int n = n0 + r, k = k0 + 2 * lane;
    if (n < N && k + 1 < K)
      *reinterpret_cast<uint32_t*>(Xt + (size_t)n * K + k) = pack_bf16(tile[r][2 * lane], tile[r][2 * lane + 1]);
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

inline int pack_t_bf16_launch(int mode, const float* X, void* Xt, void* Xrm, int K, int N, const PackTArgs& a,
                              cudaStream_t stream) {
  if (!X || !Xt || K <= 0 || N <= 0 || (N & 3) || (K & 1)) return MAC_ERR_INVALID;
  dim3 grid((N + 63) / 64, (K + 63) / 64);
  __nv_bfloat16* t = reinterpret_cast<__nv_bfloat16*>(Xt);
  __nv_bfloat16* r = reinterpret_cast<__nv_bfloat16*>(Xrm);
  if (mode == 0)
    pack_t_bf16_kernel<0><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, 0u, 1.f, 0, 0, 0);
  else if (mode == 1)
    pack_t_bf16_kernel<1><<<grid, 256, 0, stream>>>(X, t, r, K, N, a.rowvec, a.rows_per_batch, 0u, 1.f, 0, 0, 0);
  else
    pack_t_bf16_kernel<2><<<grid, 256, 0, stream>>>(X, t, r, K, N, nullptr, 1, a.thresh, a.scale, a.seed, a.site, a.step);
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

// training mode: bf16 copy of dropout(KB) for this step (ops.py:678), same Philox stream as the fp32 path
__global__ void dropout_cast_bf16_kernel(const float4* __restrict__ x, uint2* __restrict__ out, uint32_t thresh,
                                         float scale, uint64_t seed, int site, int step, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = x[i];
  const Philox4 r = philox4x32_10(seed, (uint64_t)i, (uint32_t)site, (uint32_t)step);
  const float a = ((r.x >> 8) >= thresh) ? v.x * scale : 0.f, b = ((r.y >> 8) >= thresh) ? v.y * scale : 0.f;
  const float c = ((r.z >> 8) >= thresh) ? v.z * scale : 0.f, d = ((r.w >> 8) >= thresh) ? v.w * scale : 0.f;
  out[i] = make_uint2(pack_bf16(a, b), pack_bf16(c, d));
}

// extra workspace of the bf16 read chain: P, P*y, H (+ I1 when saving for backward), each [B*N, d] bf16
inline size_t tc_read_extra_workspace_bytes(int B, int N, int d) {
  return (size_t)5 * (((size_t)B * N * d * 2 + 1023) & ~(size_t)1023) + 1024;     // P, P*y, H, I1, dropout(KB)
}

// The read unit's three projections on tensor cores (see mac_read_fwd in mac_b200.h).
inline int tc_read_chain(const float* kb_f32, const void* kb_bf16, const float* y, const float* control, const mac_read_weights* w,
                         uint32_t thr, float scale, uint64_t seed, int step, float* /*P_f32*/, float* /*H_f32*/,
                         float* /*I1_f32*/, float* parts, int* nparts, void* ws, size_t ws_bytes, int B, int N, int d,
                         bool save, cudaStream_t stream) {
  if (!kb_bf16 || !w->Wx_bf16 || !w->Wm_bf16 || !w->Wm2_bf16) return MAC_ERR_INVALID;
  if (d % 128) return MAC_ERR_UNSUPPORTED;
  if (ws_bytes < tc_read_extra_workspace_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  const size_t slab = (((size_t)M * d * 2 + 1023) & ~(size_t)1023);
  char* base = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws) + 1023) & ~(uintptr_t)1023);
  __nv_bfloat16* P = reinterpret_cast<__nv_bfloat16*>(base);
  __nv_bfloat16* PY = reinterpret_cast<__nv_bfloat16*>(base + slab);
  __nv_bfloat16* H = reinterpret_cast<__nv_bfloat16*>(base + 2 * slab);
  __nv_bfloat16* I1 = save ? reinterpret_cast<__nv_bfloat16*>(base + 3 * slab) : nullptr;
  if (thr != 0) {
    // A operand of the first projection = dropout(KB) (ops.py:678): TMA cannot mask in flight, so make this step's copy
    __nv_bfloat16* kbd = reinterpret_cast<__nv_bfloat16*>(base + 4 * slab);
    const long long n4 = (long long)M * d / 4;
    dropout_cast_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(
        reinterpret_cast<const float4*>(kb_f32), reinterpret_cast<uint2*>(kbd), thr, scale, seed, MAC_SITE_READ_KB, step, n4);
    MAC_LAUNCH_CHECK();
    kb_bf16 = kbd;
  }
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N; p.ldo = d; p.seed = seed; p.step = step;
  // P = KB @ Wx + bx ; also P*y
  p.epi = TC_EPI_P; p.bias = w->bx; p.out0 = P; p.out1 = PY; p.y = y;
  int st = tc_gemm_launch(kb_bf16, d, nullptr, 0, w->Wx_bf16, p, stream);
  if (st != MAC_OK) return st;
  // H = ELU([P*y, P] @ Wm + bm)
  p.epi = TC_EPI_ACT; p.act = MAC_ACT_ELU; p.bias = w->bm; p.out0 = H; p.out1 = nullptr;
  st = tc_gemm_launch(PY, d, P, d, w->Wm_bf16, p, stream);
  if (st != MAC_OK) return st;
  // logits parts = sum_n ELU((H @ Wm2 + bm2) * control) * wr
  p.epi = TC_EPI_LOGITS; p.bias = w->bm2; p.out0 = I1; p.ctrl = control; p.wr = w->wr; p.parts = parts;
  p.e_thresh = thr; p.e_scale = scale; p.e_site = MAC_SITE_READ_INTER;
  st = tc_gemm_launch(H, d, nullptr, 0, w->Wm2_bf16, p, stream, nparts);
  if (st != MAC_OK) return st;
  return MAC_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Eval-mode read (readDropout == 1): dropout(KB) == KB at every step and the read weights are shared over the steps
// (mac_cell.py:209-277 is called with the same variables for each of the netLength cells), so
//   P = KB @ Wx + bx                (ops.py:688)                       and
//   Q = P @ Wm[d:2d, :] + bm        (the projected-KB half of the [P*y, P] concat, mac_cell.py:236-238)
// do not depend on the step.  They are computed once per forward into `inv` = [P | Q] (bf16), and each step runs
//   PY = P * y_b ;  H = ELU(PY @ Wm[0:d, :] + Q) ;  logits = ... (unchanged)
// i.e. 2 x d instead of 4 x d MACs per knowledge-base element and step.
// [P | Q] bf16 slabs, then the scratch of the fused read step (read_step.cuh): P*y and H slabs, the logit partial sums
// [B*N, d / TC_BN] and y [B, d]
inline size_t tc_read_invariant_bytes(int B, int N, int d) {
  const size_t slab = (((size_t)B * N * d * 2 + 1023) & ~(size_t)1023);
  const size_t parts = (((size_t)B * N * (d / TC_BN) * 4 + 1023) & ~(size_t)1023);
  return 4 * slab + parts + (size_t)B * d * 4 + 1024;
}

// PY[m, :] = P[m, :] * y[m / rows_per_batch, :]   (8 bf16 per thread)
__global__ void scale_rows_bf16_kernel(const uint4* __restrict__ P, const float* __restrict__ y, uint4* __restrict__ out,
                                       int rows_per_batch, int d, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const long long e = i * 8;
  const int c = (int)(e % d);
  const long long b = (e / d) / rows_per_batch;
  const uint4 v = P[i];
  const float4 y0 = __ldg(reinterpret_cast<const float4*>(y + b * d + c));
  const float4 y1 = __ldg(reinterpret_cast<const float4*>(y + b * d + c + 4));
  auto lo = [](uint32_t w) { return __uint_as_float(w << 16); };
  auto hi = [](uint32_t w) { return __uint_as_float(w & 0xffff0000u); };
  out[i] = make_uint4(pack_bf16(lo(v.x) * y0.x, hi(v.x) * y0.y), pack_bf16(lo(v.y) * y0.z, hi(v.y) * y0.w),
                      pack_bf16(lo(v.z) * y1.x, hi(v.z) * y1.y), pack_bf16(lo(v.w) * y1.z, hi(v.w) * y1.w));
}

inline char* tc_align1k(void* p) {
  return reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

struct TcReadScratch {
  __nv_bfloat16 *P, *Q, *PY, *H;
  float *parts, *y;
};
inline TcReadScratch tc_read_scratch(void* inv, int B, int N, int d) {
  const size_t slab = (((size_t)B * N * d * 2 + 1023) & ~(size_t)1023);
  const size_t parts = (((size_t)B * N * (d / TC_BN) * 4 + 1023) & ~(size_t)1023);
  char* base = tc_align1k(inv);
  TcReadScratch s;
  s.P = reinterpret_cast<__nv_bfloat16*>(base);
  s.Q = reinterpret_cast<__nv_bfloat16*>(base + slab);
  s.PY = reinterpret_cast<__nv_bfloat16*>(base + 2 * slab);
  s.H = reinterpret_cast<__nv_bfloat16*>(base + 3 * slab);
  s.parts = reinterpret_cast<float*>(base + 4 * slab);
  s.y = reinterpret_cast<float*>(base + 4 * slab + parts);
  return s;
}

inline int tc_read_invariant(const void* kb_bf16, const mac_read_weights* w, void* inv, size_t inv_bytes, int B, int N,
                             int d, cudaStream_t stream) {
  if (!kb_bf16 || !w->Wx_bf16 || !w->Wm_bf16 || !inv) return MAC_ERR_INVALID;
  if (d % 128) return MAC_ERR_UNSUPPORTED;
  if (inv_bytes < tc_read_invariant_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  const size_t slab = (((size_t)M * d * 2 + 1023) & ~(size_t)1023);
  char* base = tc_align1k(inv);
  __nv_bfloat16* P = reinterpret_cast<__nv_bfloat16*>(base);
  __nv_bfloat16* Q = reinterpret_cast<__nv_bfloat16*>(base + slab);
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N; p.ldo = d;
  p.epi = TC_EPI_ACT; p.act = MAC_ACT_NON; p.bias = w->bx; p.out0 = P;
  int st = tc_gemm_launch(kb_bf16, d, nullptr, 0, w->Wx_bf16, p, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bm; p.out0 = Q;
  return tc_gemm_launch(P, d, nullptr, 0, reinterpret_cast<const __nv_bfloat16*>(w->Wm_bf16) + d, p, stream, nullptr, 2 * d);
}

inline int tc_read_chain_inv(const void* inv, const float* y, const float* control, const mac_read_weights* w, float* parts,
                             int* nparts, void* ws, size_t ws_bytes, int B, int N, int d, cudaStream_t stream) {
  if (!inv || !w->Wm_bf16 || !w->Wm2_bf16) return MAC_ERR_INVALID;
  if (d % 128) return MAC_ERR_UNSUPPORTED;
  if (ws_bytes < tc_read_extra_workspace_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  const size_t slab = (((size_t)M * d * 2 + 1023) & ~(size_t)1023);
  const char* ibase = tc_align1k(const_cast<void*>(inv));
  const __nv_bfloat16* P = reinterpret_cast<const __nv_bfloat16*>(ibase);
  const __nv_bfloat16* Q = reinterpret_cast<const __nv_bfloat16*>(ibase + slab);
  char* base = tc_align1k(ws);
  __nv_bfloat16* PY = reinterpret_cast<__nv_bfloat16*>(base + slab);
  __nv_bfloat16* H = reinterpret_cast<__nv_bfloat16*>(base + 2 * slab);
  const long long n8 = (long long)M * d / 8;
  scale_rows_bf16_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const uint4*>(P), y, reinterpret_cast<uint4*>(PY), N, d, n8);
  MAC_LAUNCH_CHECK();
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N; p.ldo = d;
  int st;
  static const bool q_hoist = !(getenv("MAC_READ_QHOIST") && atoi(getenv("MAC_READ_QHOIST")) == 0);
  if (q_hoist) {
    // H = ELU(PY @ Wm[0:d] + Q)      (bm is inside Q)
    p.epi = TC_EPI_ADDACT; p.act = MAC_ACT_ELU; p.bias = nullptr; p.out0 = H; p.add = Q;
    st = tc_gemm_launch(PY, d, nullptr, 0, w->Wm_bf16, p, stream, nullptr, 2 * d);
  } else {
    // experiment switch: keep the concatenated K = 2d form, H = ELU([PY, P] @ Wm + bm), with only P hoisted
    p.epi = TC_EPI_ACT; p.act = MAC_ACT_ELU; p.bias = w->bm; p.out0 = H;
    st = tc_gemm_launch(PY, d, P, d, w->Wm_bf16, p, stream);
  }
  if (st != MAC_OK) return st;
  p.epi = TC_EPI_LOGITS; p.act = MAC_ACT_NON; p.bias = w->bm2; p.out0 = nullptr; p.add = nullptr;
  p.ctrl = control; p.wr = w->wr; p.parts = parts;
  return tc_gemm_launch(H, d, nullptr, 0, w->Wm2_bf16, p, stream, nparts);
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
// "tc32": the read unit's three [B*N, .] projections as SPLIT-bf16 products on the tensor cores, for the <= 1e-4 parity bar
// of BASELINE.json (the plain bf16 path is at ~1e-3).  Every fp32 operand x is carried as two bf16 values x_hi = bf16(x),
// x_lo = bf16(x - x_hi) and the product uses three of the four partial products, accumulated in ONE fp32 accumulator:
//     A W  ~=  A_hi W_hi + A_lo W_hi + A_hi W_lo                      (A_lo W_lo ~ 2^-16 relative is dropped)
// With A' = [A_hi | A_lo] ([M, 2K]) and W' = [W_hi | W_hi | W_lo] ([N, 3K], K-major) this is the existing two-segment GEMM:
// segment 0 = A'[:, 0:2K] against W'[:, 0:2K], segment 1 = A'[:, 0:K] against W'[:, 2K:3K] -- K triples, nothing else
// changes.  Producers write their outputs directly as hi | lo pairs (TC_EPI_ACT_SPLIT) or as fp32 (TC_EPI_F32).
// Inference form only (P, Q hoisted, mac_read_invariant): inv = [P fp32 | Q fp32 | scratch [M, 2d] bf16].
// ---------------------------------------------------------------------------------------------------------------
// out[m, c] = hi(x[m, c] * y[m / rows_per_batch, c]), out[m, d + c] = lo(...)     (y == NULL: plain split); 4 columns / thread
__global__ void split_rows_kernel(const float4* __restrict__ x, const float* __restrict__ y, uint2* __restrict__ out,
                                  int rows_per_batch, int d, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int d4 = d / 4;
  const long long m = i / d4;
  const int c4 = (int)(i - m * d4);
  float4 v = x[i];
  if (y) {
    const float4 s = __ldg(reinterpret_cast<const float4*>(y + (m / rows_per_batch) * d) + c4);
    v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
  }
  const uint32_t h01 = pack_bf16(v.x, v.y), h23 = pack_bf16(v.z, v.w);
  const uint32_t l01 = pack_bf16(v.x - __uint_as_float(h01 << 16), v.y - __uint_as_float(h01 & 0xffff0000u));
  const uint32_t l23 = pack_bf16(v.z - __uint_as_float(h23 << 16), v.w - __uint_as_float(h23 & 0xffff0000u));
  uint2* row = out + m * (2 * d4);
  row[c4] = make_uint2(h01, h23);
  row[d4 + c4] = make_uint2(l01, l23);
}
inline int split_rows_launch(const float* x, const float* y, void* out, int rows_per_batch, int d, long long M,
                             cudaStream_t stream) {
  const long long n4 = M * d / 4;
  split_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(x), y,
                                                                      reinterpret_cast<uint2*>(out), rows_per_batch, d, n4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
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

inline size_t tc3_slab(int B, int N, int d) { return (((size_t)B * N * 2 * d * 2 + 1023) & ~(size_t)1023); }   // [M, 2d] bf16
inline size_t tc3_invariant_bytes(int B, int N, int d) {
  return (size_t)2 * B * N * d * 4 + tc3_slab(B, N, d) + 2048;
}
inline size_t tc3_extra_workspace_bytes(int B, int N, int d) { return 2 * tc3_slab(B, N, d) + 1024; }

// C = epilogue(A W) with A' = [A_hi | A_lo] ([M, 2K] bf16) and W' = [W_hi | W_hi | W_lo] ([N, 3K] bf16)
inline int tc3_gemm(const void* a_split, int K, const void* wt3, TcGemmParams p, cudaStream_t stream, int* nparts = nullptr) {
  return tc_gemm_launch(a_split, 2 * K, a_split, K, wt3, p, stream, nparts, 3 * K, 2 * K, 2 * K);
}

inline int tc3_read_invariant(const float* kb, const mac_read_weights* w, void* inv, size_t inv_bytes, int B, int N, int d,
                              cudaStream_t stream) {
  if (!kb || !w->Wx_s3 || !w->Wmb_s3 || !inv) return MAC_ERR_INVALID;
  if (d % 128) return MAC_ERR_UNSUPPORTED;
  if (inv_bytes < tc3_invariant_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  float* P = reinterpret_cast<float*>(inv);
  float* Q = P + (size_t)M * d;
  void* scratch = tc_align1k(Q + (size_t)M * d);
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N; p.ldo = d; p.epi = TC_EPI_F32; p.act = MAC_ACT_NON;
  int st = split_rows_launch(kb, nullptr, scratch, N, d, M, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bx; p.outf = P;
  st = tc3_gemm(scratch, d, w->Wx_s3, p, stream);                       // P = KB @ Wx + bx            (ops.py:688)
  if (st != MAC_OK) return st;
  st = split_rows_launch(P, nullptr, scratch, N, d, M, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bm; p.outf = Q;
  return tc3_gemm(scratch, d, w->Wmb_s3, p, stream);                    // Q = P @ Wm[d:2d] + bm       (mac_cell.py:236-238)
}

inline int tc3_read_chain_inv(const void* inv, const float* y, const float* control, const mac_read_weights* w, float* parts,
                              int* nparts, void* ws, size_t ws_bytes, int B, int N, int d, cudaStream_t stream) {
  if (!inv || !w->Wma_s3 || !w->Wm2_s3) return MAC_ERR_INVALID;
  if (d % 128) return MAC_ERR_UNSUPPORTED;
  if (ws_bytes < tc3_extra_workspace_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  const float* P = reinterpret_cast<const float*>(inv);
  const float* Q = P + (size_t)M * d;
  char* base = tc_align1k(ws);
  void* PYs = base;
  __nv_bfloat16* Hs = reinterpret_cast<__nv_bfloat16*>(base + tc3_slab(B, N, d));
  int st = split_rows_launch(P, y, PYs, N, d, M, stream);                // (P * y_b) as hi | lo       (ops.py:694-703)
  if (st != MAC_OK) return st;
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N;
  p.epi = TC_EPI_ACT_SPLIT; p.act = MAC_ACT_ELU; p.bias = nullptr; p.addf = Q; p.ldaf = d; p.out0 = Hs; p.ldo = 2 * d;
  st = tc3_gemm(PYs, d, w->Wma_s3, p, stream);                           // H = ELU((P*y) @ Wm[0:d] + Q) as hi | lo
  if (st != MAC_OK) return st;
  p.epi = TC_EPI_LOGITS; p.act = MAC_ACT_NON; p.bias = w->bm2; p.addf = nullptr; p.out0 = nullptr; p.ldo = d;
  p.ctrl = control; p.wr = w->wr; p.parts = parts;
  return tc3_gemm(Hs, d, w->Wm2_s3, p, stream, nparts);                  // logits partial sums         (mac_cell.py:248-266)
}

}  // namespace mac
