// The two HBM-bound attention kernels of the MAC cell.
//
//  K1  control_attend_kernel   mac_cell.py:155-181  (also the write unit's self-attention, 324-330)
//  K3  kb_attend_kernel        ops.py:143, 149-150 at mac_cell.py:266-275  (softmax over the KB + weighted sum)
//
// Both stage their operand through the TMA engine (cp.async.bulk -> shared memory, mbarrier
// completion), reduce with warp shuffles, and read every HBM byte exactly once.
#include "common.cuh"
#include "tmap.cuh"

namespace mac {

// =====================================================================================
// K1: one CTA per (batch row, step group).  The S x d words of the row land in shared
// memory with ONE bulk copy (they are contiguous), then every step of the group reuses them.
// =====================================================================================
constexpr int K1_THREADS = 256;

__global__ void __launch_bounds__(K1_THREADS) control_attend_kernel(
    const float* __restrict__ cc, long long cc_tstride, long long cc_bstride, const float* __restrict__ in_words,
    long long in_bstride, long long in_rstride, const float* __restrict__ out_words, long long out_bstride,
    long long out_rstride, const int32_t* __restrict__ lengths, const float* __restrict__ w_logit, float b_logit,
    float* __restrict__ att, float* __restrict__ out, int nsteps, int B, int S, int d, int steps_per_cta,
    int separate_out) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* s_in = reinterpret_cast<float*>(smem_raw);                  // [S][d]
  float* s_out = separate_out ? s_in + (size_t)S * d : s_in;         // [S][d]
  float* s_cw = s_out + (size_t)S * d;                               // [d]   cc * w_logit
  float* s_att = s_cw + d;                                           // [S]
  __shared__ __align__(8) uint64_t bar;
  __shared__ float s_red[K1_THREADS / 32];

  const int b = blockIdx.x;
  const int t0 = blockIdx.y * steps_per_cta;
  const int t1 = min(nsteps, t0 + steps_per_cta);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = K1_THREADS / 32;

  const uint32_t bytes = (uint32_t)((size_t)S * d * sizeof(float));
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (warp == 0) {
    // rows contiguous (row stride == d): one bulk copy for the whole [S,d] block; otherwise (step-major
    // history buffers of the write unit's self-attention) one bulk copy per row, spread over the warp's lanes
    if (lane == 0) mbar_expect_tx(&bar, separate_out ? 2 * bytes : bytes);
    __syncwarp();
    const uint32_t row_bytes = (uint32_t)(d * sizeof(float));
    if (in_rstride == d) {
      if (lane == 0) bulk_g2s(s_in, in_words + (size_t)b * in_bstride, bytes, &bar);
    } else {
      for (int r = lane; r < S; r += 32)
        bulk_g2s(s_in + (size_t)r * d, in_words + (size_t)b * in_bstride + (size_t)r * in_rstride, row_bytes, &bar);
    }
    if (separate_out) {
      if (out_rstride == d) {
        if (lane == 0) bulk_g2s(s_out, out_words + (size_t)b * out_bstride, bytes, &bar);
      } else {
        for (int r = lane; r < S; r += 32)
          bulk_g2s(s_out + (size_t)r * d, out_words + (size_t)b * out_bstride + (size_t)r * out_rstride, row_bytes, &bar);
      }
    }
  }
  const int len = lengths ? min(max(lengths[b], 0), S) : S;
  bool landed = false;

  for (int t = t0; t < t1; ++t) {
    const float* q = cc + (size_t)t * cc_tstride + (size_t)b * cc_bstride;
    for (int k = tid; k < d; k += K1_THREADS) s_cw[k] = q[k] * __ldg(w_logit + k);
    __syncthreads();
    if (!landed) {
      mbar_wait(&bar, 0);
      landed = true;
    }
    // logits: one warp per word row; lanes stride the feature dim (conflict-free, coalesced in smem)
    for (int s = warp; s < S; s += NW) {
      const float* wrow = s_in + (size_t)s * d;
      float acc = 0.f;
      for (int k = lane; k < d; k += 32) acc = fmaf(wrow[k], s_cw[k], acc);
      acc = warp_sum(acc);
      // expMask (ops.py:243-247): logits + (1 - mask) * (-1e30)
      if (lane == 0) s_att[s] = (s < len) ? (acc + b_logit) : (acc + b_logit) + (-1e30f);
    }
    __syncthreads();
    // softmax over S (block-wide; S is a few dozen)
    float mx = -INFINITY;
    for (int s = tid; s < S; s += K1_THREADS) mx = fmaxf(mx, s_att[s]);
    mx = warp_max(mx);
    if (lane == 0) s_red[warp] = mx;
    __syncthreads();
    mx = s_red[0];
#pragma unroll
    for (int i = 1; i < NW; ++i) mx = fmaxf(mx, s_red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int s = tid; s < S; s += K1_THREADS) {
      const float e = expf(s_att[s] - mx);
      s_att[s] = e;
      sum += e;
    }
    sum = warp_sum(sum);
    if (lane == 0) s_red[warp] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int i = 0; i < NW; ++i) sum += s_red[i];
    const float inv = 1.f / sum;
    for (int s = tid; s < S; s += K1_THREADS) {
      const float a = s_att[s] * inv;
      s_att[s] = a;
      att[((size_t)t * B + b) * S + s] = a;
    }
    __syncthreads();
    // summary: thread per feature column, serial over the S words
    for (int k = tid; k < d; k += K1_THREADS) {
      float acc = 0.f;
#pragma unroll 4
      for (int s = 0; s < S; ++s) acc = fmaf(s_att[s], s_out[(size_t)s * d + k], acc);
      out[((size_t)t * B + b) * d + k] = acc;
    }
    __syncthreads();
  }
}

// =====================================================================================
// K3: grid = (d / DS column slices, B).  Each CTA pulls its [N x DS] slab of the knowledge
// base into shared memory with bulk copies issued up-front (all bytes in flight at once),
// computes the softmax of the row's N logits while they fly, then accumulates the weighted sum.
// KB bytes are read exactly once; logits are re-read per slice (N*4 B, L2 hits).
// =====================================================================================
constexpr int K3_THREADS = 256;

template <typename KT, int DS>
__global__ void __launch_bounds__(K3_THREADS) kb_attend_kernel(
    const float* __restrict__ logit_parts, int nparts, float br, const __grid_constant__ CUtensorMap kb_map,
    float* __restrict__ att, float* __restrict__ info, int B, int N, int d, int rows_per_stage, int nstages, int nbuf, int buf_elems) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  KT* s_kb = reinterpret_cast<KT*>(smem_raw);                                    // [nstages_resident][rows][DS]
  float* s_att = reinterpret_cast<float*>(smem_raw + (size_t)nbuf * buf_elems * sizeof(KT));  // [N]
  float* s_acc = s_att + ((N + 3) & ~3);                                         // [K3_THREADS / DS groups][DS]
  constexpr int MAXBUF = 8;
  __shared__ __align__(8) uint64_t bar[MAXBUF];
  __shared__ float s_red[K3_THREADS / 32];

  const int slice = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = K3_THREADS / 32;
  constexpr int GROUPS = K3_THREADS / DS;       // row groups working on the same columns
  constexpr uint32_t ROW_BYTES = DS * sizeof(KT);

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < MAXBUF; ++i) mbar_init(&bar[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  // producer: ONE tiled TMA request per stage -- box [rows_per_stage x DS] of the [B*N, d] knowledge base at
  // (row b*N + r0, column slice*DS).  A box that runs past this batch row's N rows just brings rows nobody reads
  // (out-of-range rows at the very end are zero-filled); the transaction count is always the full box.
  auto issue = [&](int stage) {
    if (lane == 0) {
      const int buf = stage % nbuf;
      KT* dst = s_kb + (size_t)buf * buf_elems;        // 128-byte aligned (TMA destination)
      mbar_expect_tx(&bar[buf], (uint32_t)rows_per_stage * ROW_BYTES);
      tma_load_2d(dst, &kb_map, slice * DS, b * N + stage * rows_per_stage, &bar[buf]);
    }
  };
  if (warp == 0) {
    // every resident buffer is requested up-front: all of this CTA's bytes are in flight before the softmax starts
    for (int s = 0; s < nstages && s < nbuf; ++s) issue(s);
  }

  // softmax over the N logits of this batch row while the KB slab is in flight
  float mx = -INFINITY;
  for (int n = tid; n < N; n += K3_THREADS) {
    const float* lp = logit_parts + ((size_t)b * N + n) * nparts;
    float l = br;
    for (int p = 0; p < nparts; ++p) l += __ldg(lp + p);
    s_att[n] = l;
    mx = fmaxf(mx, l);
  }
  mx = warp_max(mx);
  if (lane == 0) s_red[warp] = mx;
  __syncthreads();
  mx = s_red[0];
#pragma unroll
  for (int i = 1; i < NW; ++i) mx = fmaxf(mx, s_red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int n = tid; n < N; n += K3_THREADS) {
    const float e = expf(s_att[n] - mx);
    s_att[n] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int i = 0; i < NW; ++i) sum += s_red[i];
  const float inv = 1.f / sum;
  for (int n = tid; n < N; n += K3_THREADS) {
    const float a = s_att[n] * inv;
    s_att[n] = a;
    if (slice == 0) att[(size_t)b * N + n] = a;
  }
  __syncthreads();

  // weighted sum: thread (g, c) accumulates column c over rows g, g+GROUPS, ...
  const int c = tid % DS, g = tid / DS;
  float acc = 0.f;
  for (int stage = 0; stage < nstages; ++stage) {
    mbar_wait(&bar[stage % nbuf], (stage / nbuf) & 1);
    const KT* buf = s_kb + (size_t)(stage % nbuf) * buf_elems;
    const int r0 = stage * rows_per_stage;
    const int nr = min(rows_per_stage, N - r0);
#pragma unroll 4
    for (int r = g; r < nr; r += GROUPS) acc = fmaf(s_att[r0 + r], (float)buf[(size_t)r * DS + c], acc);
    if (stage + nbuf < nstages) {       // refill this buffer (only when the slab does not fit the resident buffers)
      __syncthreads();
      if (warp == 0) issue(stage + nbuf);
    }
  }
  s_acc[g * DS + c] = acc;
  __syncthreads();
  if (tid < DS) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < GROUPS; ++i) t += s_acc[i * DS + tid];
    info[(size_t)b * d + (size_t)slice * DS + tid] = t;
  }
}

template <typename KT, int DS>
static int launch_kb_attend(const float* logit_parts, int nparts, float br, const KT* kb, float* att, float* info,
                            int B, int N, int d, cudaStream_t stream) {
  // stage sizing: the [N x DS] slab is cut into <= 8 boxes that are all requested up-front and consumed as they
  // land (the weighted sum of box i overlaps the flight of boxes i+1..); when the slab exceeds ~100 KB (two CTAs
  // per SM) the boxes are recycled as a ring
  const size_t row_bytes = (size_t)DS * sizeof(KT);
  const size_t budget = 100 * 1024;
  int nstages = N >= 64 ? 4 : 1;
  int rows_per_stage = (N + nstages - 1) / nstages;
  int nbuf = nstages;
  if (rows_per_stage > 256 || (size_t)rows_per_stage * nstages * row_bytes > budget) {
    nbuf = 4;
    rows_per_stage = (int)(budget / nbuf / row_bytes);
    if (rows_per_stage > 256) rows_per_stage = 256;
    nstages = (N + rows_per_stage - 1) / rows_per_stage;
    if (nstages < nbuf) nbuf = nstages;
  }
  CUtensorMap map;
  int st = make_tmap_2d(&map, kb, sizeof(KT) == 4 ? 0 : 1, (uint64_t)B * N, (uint64_t)d, (uint64_t)d * sizeof(KT),
                        (uint32_t)rows_per_stage, (uint32_t)DS, 0);
  if (st != MAC_OK) return st;
  const size_t buf_bytes = ((size_t)rows_per_stage * row_bytes + 127) & ~(size_t)127;
  const size_t smem = (size_t)nbuf * buf_bytes + (size_t)((N + 3) & ~3) * sizeof(float) +
                      (size_t)K3_THREADS * sizeof(float) + 16;
  auto kern = kb_attend_kernel<KT, DS>;
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(d / DS, B);
  kern<<<grid, K3_THREADS, smem, stream>>>(logit_parts, nparts, br, map, att, info, B, N, d, rows_per_stage, nstages, nbuf,
                                           (int)(buf_bytes / sizeof(KT)));
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac

using namespace mac;

extern "C" int mac_control_attend_fwd(const float* cc, long long cc_tstride, long long cc_bstride,
                                      const float* in_words, long long in_bstride, long long in_rstride,
                                      const float* out_words, long long out_bstride, long long out_rstride,
                                      const int32_t* lengths, const float* w_logit, float b_logit, float* att,
                                      float* out, int nsteps, int B, int S, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!cc || !in_words || !out_words || !w_logit || !att || !out) return MAC_ERR_INVALID;
  if (nsteps <= 0 || B <= 0 || S <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  if (!mac_aligned16(in_words) || !mac_aligned16(out_words) || ((in_bstride * 4) & 15) || ((out_bstride * 4) & 15) ||
      ((in_rstride * 4) & 15) || ((out_rstride * 4) & 15))
    return MAC_ERR_ALIGN;
  const int separate = (in_words != out_words) || (in_bstride != out_bstride) || (in_rstride != out_rstride);
  const size_t smem = ((size_t)S * d * (separate ? 2 : 1) + d + S + 8) * sizeof(float);
  if (smem > 220 * 1024) return MAC_ERR_UNSUPPORTED;   // S*d beyond one SM's shared memory (not a MAC shape)
  if ((size_t)S * d * sizeof(float) * 2 >= (1u << 20)) return MAC_ERR_UNSUPPORTED;  // mbarrier tx-count range
  MAC_CUDA_TRY(cudaFuncSetAttribute(control_attend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // B CTAs cannot fill the SMs at B=64: split the steps over gridDim.y so that ~2 CTAs/SM are resident
  int groups = 1;
  if (nsteps > 1) {
    groups = (2 * mac_num_sms() + B - 1) / B;
    if (groups > nsteps) groups = nsteps;
  }
  const int per = (nsteps + groups - 1) / groups;
  groups = (nsteps + per - 1) / per;
  dim3 grid(B, groups);
  control_attend_kernel<<<grid, K1_THREADS, smem, stream>>>(cc, cc_tstride, cc_bstride, in_words, in_bstride,
                                                           in_rstride, out_words, out_bstride, out_rstride, lengths,
                                                           w_logit, b_logit, att, out, nsteps, B, S, d, per, separate);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_kb_attend_fwd(const float* logit_parts, int nparts, float br, const void* kb, int kb_is_bf16,
                                 float* att, float* info, int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!logit_parts || !kb || !att || !info || nparts <= 0 || B <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  if (!mac_aligned16(kb)) return MAC_ERR_ALIGN;
  if (kb_is_bf16) {
    if (d % 128 == 0) return launch_kb_attend<__nv_bfloat16, 128>(logit_parts, nparts, br, (const __nv_bfloat16*)kb, att, info, B, N, d, stream);
    if (d % 64 == 0) return launch_kb_attend<__nv_bfloat16, 64>(logit_parts, nparts, br, (const __nv_bfloat16*)kb, att, info, B, N, d, stream);
    return MAC_ERR_UNSUPPORTED;
  }
  if (d % 128 == 0) return launch_kb_attend<float, 128>(logit_parts, nparts, br, (const float*)kb, att, info, B, N, d, stream);
  if (d % 64 == 0) return launch_kb_attend<float, 64>(logit_parts, nparts, br, (const float*)kb, att, info, B, N, d, stream);
  if (d % 32 == 0) return launch_kb_attend<float, 32>(logit_parts, nparts, br, (const float*)kb, att, info, B, N, d, stream);
  if (d % 16 == 0) return launch_kb_attend<float, 16>(logit_parts, nparts, br, (const float*)kb, att, info, B, N, d, stream);
  return MAC_ERR_UNSUPPORTED;
}
