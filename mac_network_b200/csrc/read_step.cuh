// One reasoning step of the read unit in inference form (mac_cell.py:209-277 with readDropout == 1), P and Q hoisted:
//
//   H      = ELU((P * y_b) @ Wm[0:d, :] + Q)            (ops.py:694-703 MUL, mac_cell.py:236-238; P, Q step-invariant)
//   I2     = ELU((H @ Wm2 + bm2) * control_b)           (ops.py:325-328, mac_cell.py:248-250, 262)
//   logit  = I2 . wr + br                               (mac_cell.py:266, ops.py:316-317)
//   att    = softmax_n(logit);  info = sum_n att * KB   (ops.py:143, 149-150; original KB, mac_cell.py:271-275)
//
// read_step_kernel computes the logits of 64 knowledge-base rows per CTA (rows packed across sample boundaries, so
// ceil(B*N / 64) CTAs) with P*y, H and I2 never leaving the SM; kb_attend (attend.cu) then does the per-sample softmax and
// weighted sum.  Two launches per step instead of the four of scale_rows_bf16 + tc_gemm<ADDACT> + tc_gemm<LOGITS> + kb_attend,
// and none of the P*y / H round trips through L2 and HBM (4 x B*N*d bf16).
//
// CTA = 288 threads: warp 8 is the TMA producer; warpgroups 0 and 1 each own one 256-column half of the d = 512 outputs
// (wgmma m64n256k16, a 64 x 256 fp32 accumulator in 128 registers per thread).  Shared memory:
//   A   [64 x 512] bf16 as 8 K-major 128-byte-swizzled [64 x 64] blocks (64 KB): the P tile (one TMA wave), scaled by y in
//       place into P*y, then overwritten by H = GEMM 1's epilogue, the A operand of GEMM 2
//   B   2 stages x [512 x 64] bf16 (128 KB): the k-blocks of Wm[0:d] and then of Wm2, streamed through one mbarrier ring
// The logits are summed over both halves in shared memory and written as one partial per row.
//
// Whole-step form (mac_step_fused, N > 128 so that a tile touches at most two samples): the CTA first computes, for each
// sample it touches, the previous step's plain write unit m = [m_prev, info_prev] @ Ww + bw (mac_cell.py:339-352) and this
// step's memory projection y = m @ Wy + by (ops.py:689) as matrix-vector products against the bf16 weights (fp32
// activations and accumulation) while the TMA loads are in flight; the CTA that owns a sample's first row writes its m.
// That removes the separate write / projY launch, at the price of every CTA re-reading those weights (opt-in form).
#pragma once
#include "tc_gemm.cuh"

namespace mac {

constexpr int RS_D = 512;                       // d of the shipped configurations
constexpr int RS_BM = 64;                       // knowledge-base rows per CTA
constexpr int RS_KB = RS_D / TC_BK;             // 8 k-blocks
constexpr int RS_BLK = RS_BM * TC_BK * 2;       // one [64 x 64] bf16 A block: 8 KB
constexpr int RS_A_BYTES = RS_KB * RS_BLK;      // 64 KB
constexpr int RS_B_HALF = 256 * TC_BK * 2;      // [256 x 64] bf16: 32 KB
constexpr int RS_STAGE = 2 * RS_B_HALF;         // 64 KB
constexpr int RS_STAGES = 2;
constexpr int RS_CONSUMERS = 256;
constexpr int RS_THREADS = RS_CONSUMERS + 32;
constexpr int RS_SMEM_BYTES = RS_A_BYTES + RS_STAGES * RS_STAGE + 1024 /*align*/ + 64 /*barriers*/ +
                              2 * RS_BM * 4 /*logit halves*/ + 2 * RS_D * 4 /*y of <= 2 samples*/ + 2 * RS_D * 4 /*m*/;

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
// can the read step take this shape?
inline bool read_step_supported(int B, int N, int d) { return d == RS_D && N >= 1 && N <= 256 && B >= 1; }

// whole-step form: the write unit of the previous step and this step's memory projection run in the kernel's prologue
struct WholeStepArgs {
  const float* mem_prev;
  const float* info_prev;           // NULL on the first step (the memory is then mem_prev itself)
  const void* Ww_t_bf16;            // [d, 2d] bf16 (mac_pack_weight_bf16 of write/newMemory)
  const float* bw;
  const void* Wy_t_bf16;            // [d, d] bf16 (mac_pack_weight_bf16 of projY)
  float* mem_out;
};
inline bool whole_step_supported(int B, int N, int d) { return read_step_supported(B, N, d) && N > 128; }

struct ReadStepParams {
  int M, N;
  const float* y;                   // [B, d] memory projection, or NULL in the whole-step form
  const float* ctrl;                // [B, d]
  const float* bm2;                 // [d]
  const float* wr;                  // [d]
  const __nv_bfloat16* Q;           // [B*N, d]  P @ Wm[d:2d] + bm
  float* logits;                    // [B*N]  I2 . wr (without br)
  const float* mem_prev;            // whole-step form (see WholeStepArgs); Wy_t == NULL otherwise
  const float* info_prev;
  const __nv_bfloat16* Ww_t;
  const float* bw;
  const __nv_bfloat16* Wy_t;
  const float* by;
  float* mem_out;
};

// sum_k x[k] * W_t[n, k] over K (K % 256 == 0), one warp per output column
__device__ __forceinline__ float bf16_row_dot(const __nv_bfloat16* row, const float* x, int K, int lane) {
  float a = 0.f;
  for (int k = lane * 8; k < K; k += 256) {
    const uint4 w = ldg_nc_v4(row + k);
    a = fmaf(bf16lo(w.x), x[k], a);     a = fmaf(bf16hi(w.x), x[k + 1], a);
    a = fmaf(bf16lo(w.y), x[k + 2], a); a = fmaf(bf16hi(w.y), x[k + 3], a);
    a = fmaf(bf16lo(w.z), x[k + 4], a); a = fmaf(bf16hi(w.z), x[k + 5], a);
    a = fmaf(bf16lo(w.w), x[k + 6], a); a = fmaf(bf16hi(w.w), x[k + 7], a);
  }
  return warp_sum(a);
}

__device__ __forceinline__ void rs_consumer_bar() { asm volatile("bar.sync 1, %0;" ::"n"(RS_CONSUMERS) : "memory"); }

__global__ void __launch_bounds__(RS_THREADS, 1)
read_step_kernel(const __grid_constant__ CUtensorMap map_p, const __grid_constant__ CUtensorMap map_w1,
                 const __grid_constant__ CUtensorMap map_w2, const ReadStepParams p) {
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base_u32 = smem_u32(smem_dyn);
  unsigned char* a_tile = smem_dyn + ((1024u - (base_u32 & 1023u)) & 1023u);
  unsigned char* b_ring = a_tile + RS_A_BYTES;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(b_ring + RS_STAGES * RS_STAGE);
  uint64_t* full = a_full + 1;                     // [STAGES] TMA -> consumers
  uint64_t* empty = full + RS_STAGES;              // [STAGES] consumers -> TMA (8 warp arrivals)
  float* s_lg = reinterpret_cast<float*>(a_full + 8);       // [2][64] logit halves
  float* s_y = s_lg + 2 * RS_BM;                             // [2][d] y of the samples of the whole-step form
  float* s_m = s_y + 2 * RS_D;                               // [2][d] m

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row0 = blockIdx.x * RS_BM;
  const int s_lo = row0 / p.N;                               // first sample of the tile

  if (threadIdx.x == RS_CONSUMERS) {
    tma_prefetch_desc(&map_p);
    tma_prefetch_desc(&map_w1);
    tma_prefetch_desc(&map_w2);
    mbar_init(a_full, 1);
    for (int i = 0; i < RS_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], RS_CONSUMERS / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == RS_CONSUMERS / 32) {
    // ===================================================== TMA producer
    if (elect_one()) {
      mbar_expect_tx(a_full, RS_A_BYTES);
      for (int kb = 0; kb < RS_KB; ++kb) tma_load_2d(a_tile + kb * RS_BLK, &map_p, kb * TC_BK, row0, a_full);
      for (int j = 0; j < 2 * RS_KB; ++j) {
        const int s = j % RS_STAGES;
        mbar_wait(&empty[s], ((j / RS_STAGES) & 1) ^ 1);
        mbar_expect_tx(&full[s], RS_STAGE);
        const CUtensorMap* m = j < RS_KB ? &map_w1 : &map_w2;
        const int k0 = (j % RS_KB) * TC_BK;
        unsigned char* dst = b_ring + s * RS_STAGE;
        tma_load_2d(dst, m, k0, 0, &full[s]);
        tma_load_2d(dst + RS_B_HALF, m, k0, 256, &full[s]);
      }
    }
    return;
  }

  // ===================================================== consumers
  const int tid = threadIdx.x;
  const int last_row = min(p.M, row0 + RS_BM) - 1;
  const float* y_src = p.y;
  if (p.Wy_t) {
    const int nsamp = last_row / p.N - s_lo + 1;
    for (int q = 0; q < nsamp; ++q) {
      const int s = s_lo + q;
      float* m = s_m + q * RS_D;
      if (p.info_prev) {
        // m[n] = [m_prev, info_prev] . Ww_t[n, :] + bw[n]: x read straight from global (2d floats, L1-resident)
        const float* mp = p.mem_prev + (size_t)s * RS_D;
        const float* ip = p.info_prev + (size_t)s * RS_D;
        for (int n = warp; n < RS_D; n += RS_CONSUMERS / 32) {
          const __nv_bfloat16* row = p.Ww_t + (size_t)n * 2 * RS_D;
          float a = 0.f;
          for (int k = lane * 8; k < 2 * RS_D; k += 256) {
            const uint4 w = ldg_nc_v4(row + k);
            const float* x = k < RS_D ? mp + k : ip + (k - RS_D);
            const float4 x0 = __ldg(reinterpret_cast<const float4*>(x)), x1 = __ldg(reinterpret_cast<const float4*>(x) + 1);
            a = fmaf(bf16lo(w.x), x0.x, a); a = fmaf(bf16hi(w.x), x0.y, a);
            a = fmaf(bf16lo(w.y), x0.z, a); a = fmaf(bf16hi(w.y), x0.w, a);
            a = fmaf(bf16lo(w.z), x1.x, a); a = fmaf(bf16hi(w.z), x1.y, a);
            a = fmaf(bf16lo(w.w), x1.z, a); a = fmaf(bf16hi(w.w), x1.w, a);
          }
          a = warp_sum(a) + __ldg(p.bw + n);
          if (lane == 0) {
            m[n] = a;
            if (s * p.N >= row0) p.mem_out[(size_t)s * RS_D + n] = a;     // the CTA owning the sample's first row
          }
        }
      } else {
        for (int i = tid; i < RS_D; i += RS_CONSUMERS) m[i] = p.mem_prev[(size_t)s * RS_D + i];
      }
    }
    rs_consumer_bar();
    for (int q = 0; q < nsamp; ++q)
      for (int n = warp; n < RS_D; n += RS_CONSUMERS / 32) {
        const float v = bf16_row_dot(p.Wy_t + (size_t)n * RS_D, s_m + q * RS_D, RS_D, lane) + __ldg(p.by + n);
        if (lane == 0) s_y[q * RS_D + n] = v;
      }
    rs_consumer_bar();
  }

  // ---- P -> P*y in place (rows past M are TMA zero fill and stay zero)
  mbar_wait(a_full, 0);
  for (int i = tid; i < RS_KB * RS_BM * 8; i += RS_CONSUMERS) {
    const int kb = i >> 9, r = (i >> 3) & 63, pos = i & 7;
    const int col = kb * TC_BK + ((pos ^ (r & 7)) << 3);
    const int s = min(row0 + r, p.M - 1) / p.N;
    const float* yy = p.Wy_t ? s_y + (s - s_lo) * RS_D + col : y_src + (size_t)s * RS_D + col;
    uint4* ptr = reinterpret_cast<uint4*>(a_tile + kb * RS_BLK + r * 128 + pos * 16);
    const uint4 v = *ptr;
    const float4 y0 = *reinterpret_cast<const float4*>(yy), y1 = *reinterpret_cast<const float4*>(yy + 4);
    *ptr = make_uint4(pack_bf16(bf16lo(v.x) * y0.x, bf16hi(v.x) * y0.y), pack_bf16(bf16lo(v.y) * y0.z, bf16hi(v.y) * y0.w),
                      pack_bf16(bf16lo(v.z) * y1.x, bf16hi(v.z) * y1.y), pack_bf16(bf16lo(v.w) * y1.z, bf16hi(v.w) * y1.w));
  }
  fence_proxy_async();                                       // generic-proxy stores -> visible to wgmma
  rs_consumer_bar();

  const int g = warp >> 2;                                   // warpgroup: output columns [256 g, 256 g + 256)
  float acc[128];
  const uint32_t a_u = smem_u32(a_tile);
  auto gemm = [&](int j0) {
    for (int j = j0; j < j0 + RS_KB; ++j) {
      const int s = j % RS_STAGES;
      mbar_wait(&full[s], (j / RS_STAGES) & 1);
      const uint64_t adesc = make_sw128_kmajor_desc(a_u + (j - j0) * RS_BLK);
      const uint64_t bdesc = make_sw128_kmajor_desc(smem_u32(b_ring + s * RS_STAGE + g * RS_B_HALF));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TC_BK / 16; ++k) wgmma_bf16_n256(acc, adesc + 2 * k, bdesc + 2 * k, (j > j0 || k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      wgmma_hold(acc);
      if (j > j0 && lane == 0) mbar_arrive(&empty[(j - 1) % RS_STAGES]);
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
    if (lane == 0) mbar_arrive(&empty[(j0 + RS_KB - 1) % RS_STAGES]);
  };
  // acc[4 j + 2 h + e] is tile row 16 (warp & 3) + lane / 4 + 8 h, column 256 g + 8 j + 2 (lane & 3) + e
  const int rl = 16 * (warp & 3) + (lane >> 2);
  const int cq = 256 * g + 2 * (lane & 3);

  // ---- GEMM 1 and its epilogue: H = ELU(acc + Q) -> bf16 into the A tile (K-major, swizzled) once both halves are done
  gemm(0);
  rs_consumer_bar();                                         // the other warpgroup has finished reading P*y
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rl + 8 * h, row = row0 + r;
    const __nv_bfloat16* qrow = p.Q + (size_t)min(row, p.M - 1) * RS_D;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = cq + 8 * j;
      const uint32_t q = __ldg(reinterpret_cast<const unsigned int*>(qrow + n));
      const uint32_t hv = row < p.M ? pack_bf16(elu_fast(acc[4 * j + 2 * h] + bf16lo(q)), elu_fast(acc[4 * j + 2 * h + 1] + bf16hi(q)))
                                    : 0u;
      const int kb = n >> 6, c = (n & 63) >> 3;
      *reinterpret_cast<uint32_t*>(a_tile + kb * RS_BLK + r * 128 + ((c ^ (r & 7)) << 4) + (n & 7) * 2) = hv;
    }
  }
  fence_proxy_async();
  rs_consumer_bar();

  // ---- GEMM 2 and its epilogue: I2 = ELU((acc + bm2) * control_b); logit half = sum_n I2 * wr
  gemm(RS_KB);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = rl + 8 * h, row = row0 + r;
    const float* crow = p.ctrl + (size_t)(min(row, p.M - 1) / p.N) * RS_D;
    float part = 0.f;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
      const int n = cq + 8 * j;
      const float2 cc = __ldg(reinterpret_cast<const float2*>(crow + n));
      const float t0 = elu_fast((acc[4 * j + 2 * h] + __ldg(p.bm2 + n)) * cc.x);
      const float t1 = elu_fast((acc[4 * j + 2 * h + 1] + __ldg(p.bm2 + n + 1)) * cc.y);
      part = fmaf(t0, __ldg(p.wr + n), part);
      part = fmaf(t1, __ldg(p.wr + n + 1), part);
    }
    part += __shfl_xor_sync(0xffffffffu, part, 1);
    part += __shfl_xor_sync(0xffffffffu, part, 2);
    if ((lane & 3) == 0) s_lg[g * RS_BM + r] = part;
  }
  rs_consumer_bar();
  if (tid < RS_BM && row0 + tid < p.M) p.logits[row0 + tid] = s_lg[tid] + s_lg[RS_BM + tid];
}

// inv = [P | Q] (tc_read_invariant); y, control [B, d] fp32; att [B, N], info [B, d]
inline int read_step_launch(const void* inv, const void* kb_bf16, const float* y, const float* control,
                            const mac_read_weights* w, float* att, float* info, int B, int N, int d, cudaStream_t stream,
                            const WholeStepArgs* ws = nullptr) {
  if (!read_step_supported(B, N, d)) return MAC_ERR_UNSUPPORTED;
  if (!inv || !kb_bf16 || (!y && !ws) || !control || !w->Wm_bf16 || !w->Wm2_bf16 || !att || !info) return MAC_ERR_INVALID;
  if (ws) {
    if (!whole_step_supported(B, N, d)) return MAC_ERR_UNSUPPORTED;
    if (!ws->mem_prev || !ws->Wy_t_bf16 || !w->by) return MAC_ERR_INVALID;
    if (ws->info_prev && (!ws->Ww_t_bf16 || !ws->bw || !ws->mem_out)) return MAC_ERR_INVALID;
    if (!mac_aligned16(ws->mem_prev) || !mac_aligned16(ws->Wy_t_bf16) || (ws->info_prev && !mac_aligned16(ws->info_prev)) ||
        (ws->Ww_t_bf16 && !mac_aligned16(ws->Ww_t_bf16)))
      return MAC_ERR_ALIGN;
  }
  const int M = B * N;
  const TcReadScratch s = tc_read_scratch(const_cast<void*>(inv), B, N, d);
  CUtensorMap mp, mw1, mw2;
  int st = make_tmap_2d(&mp, s.P, 1, (uint64_t)M, (uint64_t)d, (uint64_t)d * 2, RS_BM, TC_BK, 1);
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw1, w->Wm_bf16, 1, (uint64_t)d, (uint64_t)d, (uint64_t)2 * d * 2, 256, TC_BK, 1);   // Wm[0:d] of [d, 2d]
  if (st != MAC_OK) return st;
  st = make_tmap_2d(&mw2, w->Wm2_bf16, 1, (uint64_t)d, (uint64_t)d, (uint64_t)d * 2, 256, TC_BK, 1);
  if (st != MAC_OK) return st;
  ReadStepParams p{};
  p.M = M; p.N = N; p.y = y; p.ctrl = control; p.bm2 = w->bm2; p.wr = w->wr; p.Q = s.Q; p.logits = s.parts;
  if (ws) {
    p.y = nullptr; p.mem_prev = ws->mem_prev; p.info_prev = ws->info_prev; p.bw = ws->bw; p.by = w->by; p.mem_out = ws->mem_out;
    p.Ww_t = reinterpret_cast<const __nv_bfloat16*>(ws->Ww_t_bf16);
    p.Wy_t = reinterpret_cast<const __nv_bfloat16*>(ws->Wy_t_bf16);
  }
  // the opt-in is per device context: set it on every launch
  MAC_CUDA_TRY(cudaFuncSetAttribute(read_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RS_SMEM_BYTES));
  read_step_kernel<<<(M + RS_BM - 1) / RS_BM, RS_THREADS, RS_SMEM_BYTES, stream>>>(mp, mw1, mw2, p);
  MAC_LAUNCH_CHECK();
  return mac_kb_attend_fwd(s.parts, 1, w->br, kb_bf16, 1, att, info, B, N, d, stream);
}

}  // namespace mac
