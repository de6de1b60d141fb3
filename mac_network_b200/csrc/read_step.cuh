// One reasoning step of the read unit in inference form (mac_cell.py:209-277 with readDropout == 1), P and Q hoisted:
//
//   H      = ELU((P * y_b) @ Wm[0:d, :] + Q)            (ops.py:694-703 MUL, mac_cell.py:236-238; P, Q step-invariant)
//   I2     = ELU((H @ Wm2 + bm2) * control_b)           (ops.py:325-328, mac_cell.py:248-250, 262)
//   logit  = I2 . wr + br                               (mac_cell.py:266, ops.py:316-317)
//   att    = softmax_n(logit);  info = sum_n att * KB   (ops.py:143, 149-150; original KB, mac_cell.py:271-275)
//
// read_step_kernel computes the logits of 128-row tiles of the knowledge base (rows packed across sample boundaries, so
// ceil(B*N / 128) tiles) with P*y, H and I2 never leaving the SM; kb_attend (attend.cu) then does the per-sample softmax and
// weighted sum.  Two launches per step instead of the four of scale_rows_bf16 + tc_gemm<ADDACT> + tc_gemm<LOGITS> + kb_attend,
// and none of the P*y / H round trips through L2 and HBM (4 x B*N*d bf16).
//
// The kernel is bound by its weight stream: every tile streams all of Wm[0:d] and Wm2 (1 MB) from L2.  With 128 rows per CTA
// each [256 x 64] weight half-block feeds both consumer warpgroups, so a knowledge-base row costs half the weight bytes of a
// 64-row tile.  CTA = 384 threads: warpgroup 2 is the TMA producer (setmaxnreg down to 40 registers, one elected thread
// issues); consumer warpgroup g in {0, 1} owns tile rows [64 g, 64 g + 64) (setmaxnreg up to 232) and computes all d = 512
// output columns of them, one 256-column half at a time (wgmma m64n256k16, a 64 x 256 fp32 accumulator in 128 registers).
// Shared memory:
//   A   [128 x 512] bf16 as 8 K-major 128-byte-swizzled [128 x 64] blocks (128 KB).  The producer loads the P tile straight
//       into it (one mbarrier per block); each warpgroup scales its own 64 rows of block j by y in place (P*y, rounded to
//       bf16) while the MMAs of block j - 1 run.  Once GEMM 1 is done it holds H, GEMM 2's A operand.  A warpgroup only
//       reads and writes its own rows, so all A-side synchronisation is a 128-thread named barrier of that warpgroup.
//   B   3 stages x 32 KB, one mbarrier ring of 36 slots per tile, each slot a [256 x 64] weight half-block or two [128 x 64]
//       Q blocks: GEMM 1 columns [0, 256) (8 slots), their Q (2), GEMM 1 columns [256, 512) (8), their Q (2), GEMM 2 columns
//       [0, 256) (8), GEMM 2 columns [256, 512) (8).  Both warpgroups consume every slot.
// GEMM 1's first half ends in H0 = ELU(acc + Q), packed to bf16 and held in registers (64 per thread) while the second half
// accumulates; after the second half's MMAs P*y is dead, and H0 and H1 = ELU(acc + Q) are written into the A region.
// Epilogue 2 reduces ELU((acc + bm2) * control) . wr over each 256-column half (bm2, wr and control through L1) and adds the
// two halves' sums as half0 + half1.  Every output element takes the same operations in the same order as in the 64-row
// form (wgmma shape and k order, P*y and H roundings, fmaf order, half sums), so the results do not depend on the tiling.
//
// read_step_fp8_kernel (read_step_fp8.cuh) keeps the 64-row form and its RS_* constants: 288 threads, one producer warp and
// two consumer warpgroups that each own one 256-column half of a 64-row tile, at most 168 registers per thread.
#pragma once
#include "tc_gemm.cuh"

namespace mac {

constexpr int RS_D = 512;                       // d of the shipped configurations
constexpr int RS_BM = 64;                       // knowledge-base rows per CTA of the 64-row form
constexpr int RS_KB = RS_D / TC_BK;             // 8 k-blocks
constexpr int RS_BLK = RS_BM * TC_BK * 2;       // one [64 x 64] bf16 A block: 8 KB
constexpr int RS_A_BYTES = RS_KB * RS_BLK;      // 64 KB
constexpr int RS_B_HALF = 256 * TC_BK * 2;      // [256 x 64] bf16: 32 KB
constexpr int RS_CONSUMERS = 256;
constexpr int RS_THREADS = RS_CONSUMERS + 32;

// read_step_kernel: 128 rows per CTA
constexpr int RS128_BM = 128;
constexpr int RS128_BLK = RS128_BM * TC_BK * 2;          // one [128 x 64] bf16 A block: 16 KB
constexpr int RS128_A_BYTES = RS_KB * RS128_BLK;         // 128 KB
constexpr int RS128_STAGE = RS_B_HALF;                   // 32 KB: a weight half-block or two Q blocks
constexpr int RS128_STAGES = 3;
constexpr int RS128_Q0 = RS_KB;                          // ring slots of the Q blocks of columns [0, 256)
constexpr int RS128_G1B = RS128_Q0 + 2;                  // GEMM 1, columns [256, 512)
constexpr int RS128_Q1 = RS128_G1B + RS_KB;              // Q of columns [256, 512)
constexpr int RS128_G2A = RS128_Q1 + 2;                  // GEMM 2, columns [0, 256)
constexpr int RS128_G2B = RS128_G2A + RS_KB;             // GEMM 2, columns [256, 512)
constexpr int RS128_SLOTS = RS128_G2B + RS_KB;           // 36 ring slots per tile
constexpr int RS128_CONSUMERS = 256;
constexpr int RS128_THREADS = RS128_CONSUMERS + 128;
constexpr int RS128_SMEM_BYTES = RS128_A_BYTES + RS128_STAGES * RS128_STAGE + 1024 /*align*/ +
                                 8 * (RS_KB + 2 * RS128_STAGES) /*barriers*/;
static_assert(RS128_SMEM_BYTES <= 232448, "over the sm_90 per-block shared memory opt-in limit");
static_assert(RS128_BLK % 1024 == 0 && RS128_STAGE % 1024 == 0 && (RS128_BM / 2) * 128 % 1024 == 0,
              "swizzled operands need 1024-byte alignment");
static_assert(2 * RS128_BLK == RS128_STAGE, "a ring slot holds two Q blocks");
// registers per thread of the producer and consumer warpgroups: 40 + 2 x 232 = 3 x 168, the launch allocation of 384 threads
constexpr int RS128_PRODUCER_REGS = 40;
constexpr int RS128_CONSUMER_REGS = 232;
static_assert(RS128_PRODUCER_REGS + 2 * RS128_CONSUMER_REGS <= 3 * (65536 / RS128_THREADS / 8 * 8), "register budget");

__device__ __forceinline__ float bf16lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }

__device__ __forceinline__ void wgmma_bf16_n256(float (&d)[128], uint64_t adesc, uint64_t bdesc, uint32_t accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
// can the read step take this shape?  (B < 2^22: the kernel indexes y [B, d] with 32-bit offsets)
inline bool read_step_supported(int B, int N, int d) {
  return d == RS_D && N >= 1 && N <= 256 && B >= 1 && B < (1 << 22);
}

struct ReadStepParams {
  int M, N;
  const float* y;                   // [B, d] memory projection
  const float* ctrl;                // [B, d]
  const float* bm2;                 // [d]
  const float* wr;                  // [d]
  float* logits;                    // [B*N]  I2 . wr (without br)
};

__device__ __forceinline__ void rs_consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(RS_CONSUMERS) : "memory"); }

// named barrier of one consumer warpgroup (ids 1 and 2; 0 is __syncthreads)
__device__ __forceinline__ void rs128_wg_bar(int g) { asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory"); }

// one warpgroup's 256-column half of a GEMM: acc = A[64 x 512] @ (the [256 x 64] half-blocks in ring slots t0 .. t0 + 7)^T,
// A block j at a_u + j * RS128_BLK.  Releases each slot once its MMAs are done.
__device__ __forceinline__ void rs128_gemm_half(float (&acc)[128], uint32_t a_u, uint32_t ring_u, uint64_t* full,
                                                uint64_t* empty, int t0, int lane) {
  for (int j = 0; j < RS_KB; ++j) {
    const int t = t0 + j, s = t % RS128_STAGES;
    mbar_wait(&full[s], (t / RS128_STAGES) & 1);
    const uint64_t adesc = make_sw128_kmajor_desc(a_u + j * RS128_BLK);
    const uint64_t bdesc = make_sw128_kmajor_desc(ring_u + s * RS128_STAGE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j || k) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (j && lane == 0) mbar_arrive(&empty[(t - 1) % RS128_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  if (lane == 0) mbar_arrive(&empty[(t0 + RS_KB - 1) % RS128_STAGES]);
}

// byte offset of (row r, column n) in a K-major 128-byte-swizzled stack of [rows x 64] bf16 blocks of blk bytes each
__device__ __forceinline__ int rs128_sw_off(int r, int n, int blk) {
  return (n >> 6) * blk + r * 128 + ((((n & 63) >> 3) ^ (r & 7)) << 4) + (n & 7) * 2;
}

__global__ void __launch_bounds__(RS128_THREADS, 1)
read_step_kernel(const __grid_constant__ CUtensorMap map_p, const __grid_constant__ CUtensorMap map_q,
                 const __grid_constant__ CUtensorMap map_w1, const __grid_constant__ CUtensorMap map_w2,
                 const ReadStepParams p) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  unsigned char* a_tile = smem_dyn + ((1024u - (base_u32 & 1023u)) & 1023u);
  unsigned char* ring = a_tile + RS128_A_BYTES;
  uint64_t* pfull = reinterpret_cast<uint64_t*>(ring + RS128_STAGES * RS128_STAGE);   // [8] P block j landed
  uint64_t* full = pfull + RS_KB;                  // [STAGES] TMA -> consumers
  uint64_t* empty = full + RS128_STAGES;           // [STAGES] consumers -> TMA (8 warp arrivals)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * RS128_BM;

  if (threadIdx.x == RS128_CONSUMERS) {
    tma_prefetch_desc(&map_p);
    tma_prefetch_desc(&map_q);
    tma_prefetch_desc(&map_w1);
    tma_prefetch_desc(&map_w2);
    for (int i = 0; i < RS_KB; ++i) mbar_init(&pfull[i], 1);
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
      // the P tile goes straight into the A region; its first blocks are interleaved with the first weight slots so
      // GEMM 1 can start once P block 0 and weight slot 0 have landed
      auto load_p = [&](int j) {
        mbar_expect_tx(&pfull[j], RS128_BLK);
        tma_load_2d(a_tile + j * RS128_BLK, &map_p, j * TC_BK, row0, &pfull[j]);
      };
      for (int t = 0; t < RS128_SLOTS; ++t) {
        if (t < RS128_STAGES) load_p(t);
        else if (t == RS128_STAGES)
          for (int j = RS128_STAGES; j < RS_KB; ++j) load_p(j);
        const int s = t % RS128_STAGES;
        mbar_wait(&empty[s], ((t / RS128_STAGES) & 1) ^ 1);
        unsigned char* dst = ring + s * RS128_STAGE;
        mbar_expect_tx(&full[s], RS128_STAGE);
        if (t < RS128_G2A) {
          const int half = t >= RS128_G1B, u = t - half * RS128_G1B;
          if (u < RS_KB) {
            tma_load_2d(dst, &map_w1, u * TC_BK, 256 * half, &full[s]);
          } else {                                       // Q blocks 4 half + 2 (u - 8) and the one after it
            const int kb = 4 * half + 2 * (u - RS_KB);
            tma_load_2d(dst, &map_q, kb * TC_BK, row0, &full[s]);
            tma_load_2d(dst + RS128_BLK, &map_q, (kb + 1) * TC_BK, row0, &full[s]);
          }
        } else {
          const int half = t >= RS128_G2B, u = t - (half ? RS128_G2B : RS128_G2A);
          tma_load_2d(dst, &map_w2, u * TC_BK, 256 * half, &full[s]);
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
  // this thread's four 16-byte chunks of the warpgroup's rows of each P block: rows wt / 8 + 16 u, chunk wt % 8 of the
  // swizzled 128-byte row, i.e. columns pcol .. pcol + 7 of the k-block (the swizzle only depends on row % 8)
  const int prow = wt >> 3;
  const int poff = prow * 128 + (wt & 7) * 16;
  const int pcol = ((wt & 7) ^ (prow & 7)) << 3;
  // y rows of this thread's four P rows (rows past M are TMA zero fill and stay zero)
  int yoff[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) yoff[u] = min(rowg + prow + 16 * u, p.M - 1) / p.N * RS_D + pcol;

  float acc[128];
  // ---- GEMM 1, columns [0, 256): P block j is scaled by y in place (P*y) while the MMAs of block j - 1 run, then issued.
  //      The y of block j + 1 is loaded right after block j's MMAs are issued, so its L2 latency hides under them.  Plain
  //      loads: the compiler schedules __ldg (ld.global.nc) loads of y after the waits, where their latency is exposed
  float4 y0[4], y1[4];
  auto load_y = [&](int j) {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      y0[u] = *reinterpret_cast<const float4*>(p.y + yoff[u] + j * TC_BK);
      y1[u] = *reinterpret_cast<const float4*>(p.y + yoff[u] + j * TC_BK + 4);
    }
  };
  load_y(0);
  for (int j = 0; j < RS_KB; ++j) {
    const int s = j % RS128_STAGES;
    mbar_wait(&pfull[j], 0);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      uint4* c = reinterpret_cast<uint4*>(a_wg + j * RS128_BLK + poff + u * 16 * 128);
      const uint4 v = *c;
      *c = make_uint4(pack_bf16(bf16lo(v.x) * y0[u].x, bf16hi(v.x) * y0[u].y), pack_bf16(bf16lo(v.y) * y0[u].z, bf16hi(v.y) * y0[u].w),
                      pack_bf16(bf16lo(v.z) * y1[u].x, bf16hi(v.z) * y1[u].y), pack_bf16(bf16lo(v.w) * y1[u].z, bf16hi(v.w) * y1[u].w));
    }
    fence_proxy_async();                                   // generic-proxy stores -> visible to wgmma
    rs128_wg_bar(g);
    mbar_wait(&full[s], (j / RS128_STAGES) & 1);
    const uint64_t adesc = make_sw128_kmajor_desc(a_u + j * RS128_BLK);
    const uint64_t bdesc = make_sw128_kmajor_desc(ring_u + s * RS128_STAGE);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j || k) ? 1u : 0u);
    wgmma_commit();
    if (j + 1 < RS_KB) load_y(j + 1);
    wgmma_wait<1>();
    wgmma_hold(acc);
    if (j && lane == 0) mbar_arrive(&empty[(j - 1) % RS128_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  if (lane == 0) mbar_arrive(&empty[(RS_KB - 1) % RS128_STAGES]);

  // ---- H0 = ELU(acc + Q) -> bf16, held in registers.  Q comes through the ring as [128 x 64] blocks in the A layout.
  uint32_t h0[64];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int t = RS128_Q0 + q, s = t % RS128_STAGES;
    mbar_wait(&full[s], (t / RS128_STAGES) & 1);
    const unsigned char* q_tile = ring + s * RS128_STAGE + g * (RS128_BM / 2) * 128 - 2 * q * RS128_BLK;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rl + 8 * h;
      const bool live = rowg + r < p.M;
#pragma unroll
      for (int j = 16 * q; j < 16 * q + 16; ++j) {
        const uint32_t qv = *reinterpret_cast<const uint32_t*>(q_tile + rs128_sw_off(r, cq + 8 * j, RS128_BLK));
        h0[2 * j + h] = live ? pack_bf16(elu_fast(acc[4 * j + 2 * h] + bf16lo(qv)), elu_fast(acc[4 * j + 2 * h + 1] + bf16hi(qv)))
                             : 0u;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);                 // this warp's Q reads are done
  }

  // ---- GEMM 1, columns [256, 512), on the same P*y blocks
  rs128_gemm_half(acc, a_u, ring_u, full, empty, RS128_G1B, lane);

  // ---- P*y is dead once every warp of the warpgroup is past its MMAs: H0, then H1 = ELU(acc + Q), into the A region
  rs128_wg_bar(g);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rl + 8 * h;
#pragma unroll
    for (int j = 0; j < 32; ++j) *reinterpret_cast<uint32_t*>(a_wg + rs128_sw_off(r, cq + 8 * j, RS128_BLK)) = h0[2 * j + h];
  }
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    const int t = RS128_Q1 + q, s = t % RS128_STAGES;
    mbar_wait(&full[s], (t / RS128_STAGES) & 1);
    const unsigned char* q_tile = ring + s * RS128_STAGE + g * (RS128_BM / 2) * 128 - 2 * q * RS128_BLK;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = rl + 8 * h;
      const bool live = rowg + r < p.M;
#pragma unroll
      for (int j = 16 * q; j < 16 * q + 16; ++j) {
        const int n = cq + 8 * j;
        const uint32_t qv = *reinterpret_cast<const uint32_t*>(q_tile + rs128_sw_off(r, n, RS128_BLK));
        *reinterpret_cast<uint32_t*>(a_wg + rs128_sw_off(r, 256 + n, RS128_BLK)) =
            live ? pack_bf16(elu_fast(acc[4 * j + 2 * h] + bf16lo(qv)), elu_fast(acc[4 * j + 2 * h + 1] + bf16hi(qv))) : 0u;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[s]);
  }
  fence_proxy_async();
  rs128_wg_bar(g);

  // ---- GEMM 2, one 256-column half at a time; epilogue: I2 = ELU((acc + bm2) * control_b), sum_n I2 * wr over the half
  float part[2][2];
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    rs128_gemm_half(acc, a_u, ring_u, full, empty, half ? RS128_G2B : RS128_G2A, lane);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = rowg + rl + 8 * h;
      const float* crow = p.ctrl + (size_t)(min(row, p.M - 1) / p.N) * RS_D + 256 * half;
      const float* bm2 = p.bm2 + 256 * half;
      const float* wr = p.wr + 256 * half;
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int n = cq + 8 * j;
        const float2 cc = __ldg(reinterpret_cast<const float2*>(crow + n));
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bm2 + n));
        const float2 ww = __ldg(reinterpret_cast<const float2*>(wr + n));
        const float t0 = elu_fast((acc[4 * j + 2 * h] + bb.x) * cc.x);
        const float t1 = elu_fast((acc[4 * j + 2 * h + 1] + bb.y) * cc.y);
        s = fmaf(t0, ww.x, s);
        s = fmaf(t1, ww.y, s);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      part[half][h] = s;
    }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = rowg + rl + 8 * h;
    if ((lane & 3) == 0 && row < p.M) p.logits[row] = part[0][h] + part[1][h];
  }
}

// inv = [P | Q] (tc_read_invariant); y, control [B, d] fp32; att [B, N], info [B, d]
inline int read_step_launch(const void* inv, const void* kb_bf16, const float* y, const float* control,
                            const mac_read_weights* w, float* att, float* info, int B, int N, int d, cudaStream_t stream) {
  if (!read_step_supported(B, N, d)) return MAC_ERR_UNSUPPORTED;
  if (!inv || !kb_bf16 || !y || !control || !w->Wm_bf16 || !w->Wm2_bf16 || !att || !info) return MAC_ERR_INVALID;
  const int M = B * N;
  const TcReadScratch s = tc_read_scratch(const_cast<void*>(inv), B, N, d);
  CUtensorMap mp, mq, mw1, mw2;
  int st = make_tmap_2d(&mp, s.P, 1, (uint64_t)M, (uint64_t)d, (uint64_t)d * 2, RS128_BM, TC_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mq, s.Q, 1, (uint64_t)M, (uint64_t)d, (uint64_t)d * 2, RS128_BM, TC_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw1, w->Wm_bf16, 1, (uint64_t)d, (uint64_t)d, (uint64_t)2 * d * 2, 256, TC_BK, 1);   // Wm[0:d] of [d, 2d]
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw2, w->Wm2_bf16, 1, (uint64_t)d, (uint64_t)d, (uint64_t)d * 2, 256, TC_BK, 1);
  if (st != MAC_OK) return st;
  ReadStepParams p{};
  p.M = M; p.N = N; p.y = y; p.ctrl = control; p.bm2 = w->bm2; p.wr = w->wr; p.logits = s.parts;
  // the opt-in is per device context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(read_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RS128_SMEM_BYTES));
  read_step_kernel<<<(M + RS128_BM - 1) / RS128_BM, RS128_THREADS, RS128_SMEM_BYTES, stream>>>(mp, mq, mw1, mw2, p);
  MAC_LAUNCH_CHECK();
  return mac_kb_attend_fwd(s.parts, 1, w->br, kb_bf16, 1, att, info, B, N, d, stream);
}

}  // namespace mac
