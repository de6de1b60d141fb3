// The read unit's step-invariant products at d = 512 in one launch (mac_read_invariant's bf16 and fp8 forms):
//
//   P = KB @ Wx + bx              -> bf16   (ops.py:688)
//   Q = P @ Wm[d:2d, :] + bm      -> bf16   (the un-scaled half of the concat, mac_cell.py:236-238)
//
// read_invariant_kernel runs both products of a 128-row tile (rows packed across sample boundaries: ceil(B*N / 128) CTAs,
// independent of N) on read_step_kernel's CTA layout: 384 threads, a TMA producer warpgroup at 40 registers and two
// consumer warpgroups of 64 rows at 232, the A operand [128 x 512] bf16 as 8 swizzled [128 x 64] blocks (128 KB) and a
// 3 x 32 KB ring of [256 x 64] weight half-blocks that both warpgroups consume.  P never leaves the SM between the two
// products: GEMM 1's first 256-column half ends in P0 = bf16(acc + bx), held in registers while the second half
// accumulates; then P0 and P1 are written over the dead knowledge-base tile and are GEMM 2's A operand, and each P block
// is stored to global memory while GEMM 2's MMAs on it run.  GEMM 2 ends the same way, with Q written over P and stored.
// Each tile streams 1 MB of weights from L2 instead of the 2 x 4 tiles of A and W that tc_gemm streams per 128 rows.
//
// Knowledge-base input:
//   bf16 (F32 = false): the tile goes straight into the A region by TMA, one mbarrier per block.
//   fp32 (F32 = true):  each [128 x 64] fp32 block (32 KB: one ring slot) comes through the ring, interleaved with GEMM 1's
//                       first half-blocks; each warpgroup rounds its 64 rows to bf16 (round-to-nearest-even, the bits of
//                       mac_cast_bf16) into A block j while the MMAs of block j - 1 run, and stores those bf16 rows to
//                       kb_bf16, which kb_attend reads at every step.  The producer first asks L2 for all 8 blocks of
//                       the tile, so the ring's loads of them do not wait on HBM.
// The products are those of tc_gemm's TC_EPI_ACT chain bit for bit: the same k order (64-wide k-blocks, k16 steps
// ascending, one fp32 accumulator), the same roundings (bf16 of acc + bias) and the same bf16 P as GEMM 2's A operand.
#pragma once
#include "read_step.cuh"

namespace mac {

constexpr int RI_KB_SLOTS = RS_KB;                        // fp32 form: the knowledge-base blocks' ring slots
// ring slots per tile: GEMM 1 (2 halves x 8 half-blocks), GEMM 2 (the same), and the fp32 form's 8 knowledge-base blocks
template <bool F32>
__host__ __device__ constexpr int ri_slots() { return 4 * RS_KB + (F32 ? RI_KB_SLOTS : 0); }
// ring slot of weight half-block w (0..31: GEMM 1 columns [0, 256) blocks 0..7, [256, 512), then GEMM 2 likewise).  In the
// fp32 form knowledge-base block j takes slot 2 j and GEMM 1's first half-block j slot 2 j + 1.
template <bool F32>
__device__ __forceinline__ int ri_wslot(int w) { return F32 ? (w < RS_KB ? 2 * w + 1 : w + RI_KB_SLOTS) : w; }

__device__ __forceinline__ void tma_prefetch_l2_2d(const void* tmap, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}

// one warpgroup's 256-column half of a GEMM on the A region (read_step.cuh's rs128_gemm_half with the ring slots of this
// kernel).  afull (or NULL): A block j's barrier, waited on before its MMAs; after_issue(j) runs under block j's MMAs
template <bool F32, typename F>
__device__ __forceinline__ void ri_gemm_half(float (&acc)[128], uint32_t a_u, uint32_t ring_u, uint64_t* full,
                                             uint64_t* empty, uint64_t* afull, int w0, int lane, F&& after_issue) {
  for (int j = 0; j < RS_KB; ++j) {
    const int t = ri_wslot<F32>(w0 + j), s = t % RS128_STAGES;
    if (afull) mbar_wait(&afull[j], 0);
    mbar_wait(&full[s], (t / RS128_STAGES) & 1);
    const uint64_t adesc = make_sw128_kmajor_desc(a_u + j * RS128_BLK);
    const uint64_t bdesc = make_sw128_kmajor_desc(ring_u + s * RS128_STAGE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j || k) ? 1u : 0u);
    wgmma_commit();
    after_issue(j);
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (j && lane == 0) mbar_arrive(&empty[ri_wslot<F32>(w0 + j - 1) % RS128_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  if (lane == 0) mbar_arrive(&empty[ri_wslot<F32>(w0 + RS_KB - 1) % RS128_STAGES]);
}

// bf16(acc + bias) of the 256-column half at column c0, as the accumulator fragment's column pairs: out[2 j + h] is
// warpgroup row rl + 8 h, columns c0 + 8 j + cq and the one after it
__device__ __forceinline__ void ri_round_half(const float (&acc)[128], const float* __restrict__ bias, int cq,
                                              uint32_t (&out)[64]) {
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int n = cq + 8 * j;
    const float b0 = __ldg(bias + n), b1 = __ldg(bias + n + 1);
#pragma unroll
    for (int h = 0; h < 2; ++h) out[2 * j + h] = pack_bf16(acc[4 * j + 2 * h] + b0, acc[4 * j + 2 * h + 1] + b1);
  }
}

// the warpgroup's 64 rows of A block j -> dst rows [rowg, rowg + 64) (those below M), 16-byte chunks, a warp per 4 rows
__device__ __forceinline__ void ri_store_block(const unsigned char* a_wg, __nv_bfloat16* dst, int j, int rowg, int M,
                                               int wt) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int f = wt + 128 * i, r = f >> 3, c = f & 7;
    const uint4 v = *reinterpret_cast<const uint4*>(a_wg + j * RS128_BLK + r * 128 + ((c ^ (r & 7)) << 4));
    if (rowg + r < M) *reinterpret_cast<uint4*>(dst + (size_t)(rowg + r) * RS_D + TC_BK * j + 8 * c) = v;
  }
}

struct ReadInvParams {
  int M;
  const float* bx;                  // [d]
  const float* bm;                  // [d]
  __nv_bfloat16* kb_bf16;           // F32: [M, d] bf16 copy of the knowledge base (written)
  __nv_bfloat16* P;                 // [M, d]
  __nv_bfloat16* Q;                 // [M, d]
};

template <bool F32>
__global__ void __launch_bounds__(RS128_THREADS, 1)
read_invariant_kernel(const __grid_constant__ CUtensorMap map_kb, const __grid_constant__ CUtensorMap map_w1,
                      const __grid_constant__ CUtensorMap map_w2, const ReadInvParams p) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  unsigned char* a_tile = smem_dyn + ((1024u - (base_u32 & 1023u)) & 1023u);
  unsigned char* ring = a_tile + RS128_A_BYTES;
  uint64_t* afull = reinterpret_cast<uint64_t*>(ring + RS128_STAGES * RS128_STAGE);   // [8] bf16 form: A block j landed
  uint64_t* full = afull + RS_KB;                  // [STAGES] TMA -> consumers
  uint64_t* empty = full + RS128_STAGES;           // [STAGES] consumers -> TMA (8 warp arrivals)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * RS128_BM;

  if (threadIdx.x == RS128_CONSUMERS) {
    tma_prefetch_desc(&map_kb);
    tma_prefetch_desc(&map_w1);
    tma_prefetch_desc(&map_w2);
    for (int i = 0; i < RS_KB; ++i) mbar_init(&afull[i], 1);
    for (int i = 0; i < RS128_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], RS128_CONSUMERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= RS128_CONSUMERS / 32) {
    // ===================================================== TMA producer warpgroup
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(RS128_PRODUCER_REGS));
    if (warp == RS128_CONSUMERS / 32 && elect_one()) {
      auto load_a = [&](int j) {
        mbar_expect_tx(&afull[j], RS128_BLK);
        tma_load_2d(a_tile + j * RS128_BLK, &map_kb, j * TC_BK, row0, &afull[j]);
      };
      if constexpr (F32)
        for (int j = 0; j < RS_KB; ++j) tma_prefetch_l2_2d(&map_kb, j * TC_BK, row0);
      for (int t = 0; t < ri_slots<F32>(); ++t) {
        if constexpr (!F32) {                        // the first A blocks interleaved with the first weight slots
          if (t < RS128_STAGES) load_a(t);
          else if (t == RS128_STAGES)
            for (int j = RS128_STAGES; j < RS_KB; ++j) load_a(j);
        }
        const int s = t % RS128_STAGES;
        mbar_wait(&empty[s], ((t / RS128_STAGES) & 1) ^ 1);
        unsigned char* dst = ring + s * RS128_STAGE;
        mbar_expect_tx(&full[s], RS128_STAGE);
        if (F32 && t < 2 * RI_KB_SLOTS && !(t & 1)) {
          tma_load_2d(dst, &map_kb, (t >> 1) * TC_BK, row0, &full[s]);          // fp32 knowledge-base block t / 2
        } else {
          const int w = F32 ? (t < 2 * RI_KB_SLOTS ? t >> 1 : t - RI_KB_SLOTS) : t;
          const int half = (w / RS_KB) & 1, u = w % RS_KB;
          tma_load_2d(dst, w < 2 * RS_KB ? &map_w1 : &map_w2, u * TC_BK, 256 * half, &full[s]);
        }
      }
    }
    return;
  }

  // ===================================================== consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(RS128_CONSUMER_REGS));
  const int g = warp >> 2;                                   // warpgroup: tile rows [64 g, 64 g + 64)
  const int wt = threadIdx.x & 127;
  // acc[4 j + 2 h + e] is warpgroup row rl + 8 h, column 256 half + 8 j + 2 (lane & 3) + e
  const int rl = 16 * (warp & 3) + (lane >> 2);
  const int cq = 2 * (lane & 3);
  const int rowg = row0 + 64 * g;                           // first row of this warpgroup
  unsigned char* a_wg = a_tile + g * (RS128_BM / 2) * 128;  // this warpgroup's rows of every A block
  const uint32_t a_u = smem_u32(a_wg), ring_u = smem_u32(ring);

  float acc[128];
  // ---- GEMM 1, columns [0, 256)
  if constexpr (F32) {
    // fp32 block j (ring slot 2 j) -> bf16 A block j and kb_bf16, while the MMAs of block j - 1 run; then its MMAs
    for (int j = 0; j < RS_KB; ++j) {
      const int s = (2 * j) % RS128_STAGES;
      mbar_wait(&full[s], ((2 * j) / RS128_STAGES) & 1);
      const unsigned char* src = ring + s * RS128_STAGE + g * (RS128_BM / 2) * (TC_BK * 4);
#pragma unroll
      for (int i = 0; i < 8; ++i) {                          // 64 rows x 16 float4 per warpgroup
        const int f = wt + 128 * i, r = f >> 4, c4 = f & 15;
        const float4 v = *reinterpret_cast<const float4*>(src + r * (TC_BK * 4) + c4 * 16);
        const uint2 o = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
        *reinterpret_cast<uint2*>(a_wg + rs128_sw_off(r, TC_BK * j + 4 * c4, RS128_BLK)) = o;
        if (rowg + r < p.M) *reinterpret_cast<uint2*>(p.kb_bf16 + (size_t)(rowg + r) * RS_D + TC_BK * j + 4 * c4) = o;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);                 // this warp's reads of the fp32 block are done
      fence_proxy_async();                                   // generic-proxy stores -> visible to wgmma
      rs128_wg_bar(g);
      const int t = ri_wslot<true>(j), sw = t % RS128_STAGES;
      mbar_wait(&full[sw], (t / RS128_STAGES) & 1);
      const uint64_t adesc = make_sw128_kmajor_desc(a_u + j * RS128_BLK);
      const uint64_t bdesc = make_sw128_kmajor_desc(ring_u + sw * RS128_STAGE);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j || k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_hold(acc);
      if (j && lane == 0) mbar_arrive(&empty[ri_wslot<true>(j - 1) % RS128_STAGES]);
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
    if (lane == 0) mbar_arrive(&empty[ri_wslot<true>(RS_KB - 1) % RS128_STAGES]);
  } else {
    ri_gemm_half<F32>(acc, a_u, ring_u, full, empty, afull, 0, lane, [](int) {});
  }
  uint32_t lo[64];                                           // P0, then Q0
  ri_round_half(acc, p.bx, cq, lo);

  // ---- GEMM 1, columns [256, 512), on the same knowledge-base blocks
  ri_gemm_half<F32>(acc, a_u, ring_u, full, empty, nullptr, RS_KB, lane, [](int) {});

  // ---- the knowledge-base tile is dead once every warp of the warpgroup is past its MMAs: P0 and P1 into the A region
  auto write_a = [&](const uint32_t (&v)[64], int c0) {
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 32; ++j)
        *reinterpret_cast<uint32_t*>(a_wg + rs128_sw_off(rl + 8 * h, c0 + cq + 8 * j, RS128_BLK)) = v[2 * j + h];
  };
  rs128_wg_bar(g);
  write_a(lo, 0);
  ri_round_half(acc, p.bx + 256, cq, lo);
  write_a(lo, 256);
  fence_proxy_async();
  rs128_wg_bar(g);

  // ---- GEMM 2, columns [0, 256); P block j goes to global memory under its MMAs
  ri_gemm_half<F32>(acc, a_u, ring_u, full, empty, nullptr, 2 * RS_KB, lane,
                    [&](int j) { ri_store_block(a_wg, p.P, j, rowg, p.M, wt); });
  ri_round_half(acc, p.bm, cq, lo);

  // ---- GEMM 2, columns [256, 512); then Q over P and out
  ri_gemm_half<F32>(acc, a_u, ring_u, full, empty, nullptr, 3 * RS_KB, lane, [](int) {});
  rs128_wg_bar(g);
  write_a(lo, 0);
  ri_round_half(acc, p.bm + 256, cq, lo);
  write_a(lo, 256);
  rs128_wg_bar(g);
#pragma unroll
  for (int j = 0; j < RS_KB; ++j) ri_store_block(a_wg, p.Q, j, rowg, p.M, wt);
}

// P, Q bf16 [M, RS_D] from the knowledge base: kb (fp32, then kb_bf16 is written) or kb_bf16 (read).  Wx_bf16 [d, d] and
// Wm_bf16 [d, 2d] are the packed K-major weights.  The caller has checked every pointer and d == RS_D.
inline int read_invariant_launch(const float* kb, void* kb_bf16, const mac_read_weights* w, void* P, void* Q, int M,
                                 cudaStream_t stream) {
  constexpr int d = RS_D;
  CUtensorMap mkb, mw1, mw2;
  int st = kb ? make_tmap_2d(&mkb, kb, 0, (uint64_t)M, d, (uint64_t)d * 4, RS128_BM, TC_BK, 0)
              : make_tmap_2d(&mkb, kb_bf16, 1, (uint64_t)M, d, (uint64_t)d * 2, RS128_BM, TC_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw1, w->Wx_bf16, 1, d, d, (uint64_t)d * 2, 256, TC_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw2, reinterpret_cast<const __nv_bfloat16*>(w->Wm_bf16) + d, 1, d, d, (uint64_t)2 * d * 2, 256,
                    TC_BK, 1);                                                       // Wm[d:2d] of [d, 2d]
  if (st != MAC_OK) return st;
  ReadInvParams p{};
  p.M = M; p.bx = w->bx; p.bm = w->bm; p.kb_bf16 = reinterpret_cast<__nv_bfloat16*>(kb_bf16);
  p.P = reinterpret_cast<__nv_bfloat16*>(P); p.Q = reinterpret_cast<__nv_bfloat16*>(Q);
  auto kern = kb ? read_invariant_kernel<true> : read_invariant_kernel<false>;
  // the opt-in is per device context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, RS128_SMEM_BYTES));
  kern<<<(M + RS128_BM - 1) / RS128_BM, RS128_THREADS, RS128_SMEM_BYTES, stream>>>(mkb, mw1, mw2, p);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac
