#pragma once
// Question encoder on Hopper tensor cores (QuestionEncoder(prec="bf16"), DESIGN.md section 9 item 3): the bi-LSTM of
// encoder.cu with every matrix product on wgmma (bf16 operands, fp32 accumulation).  The cell state, the gate
// pre-activations and non-linearities, the outputs, the saved tensors and every element-wise backward step stay fp32.
//
//   input half   mac_embed_fwd_tc writes questionWords (fp32) and bf16 dropout(X) [B*S, Ep] (Ep = E rounded up to 128,
//                zero columns E..Ep) in one pass; gx = mac_linear_tc_fwd(X16, pack of kernel[0:E]) + bias in fp32
//   recurrence   mac_lstm_fwd_tc: ONE launch of a persistent cluster kernel for all S steps of both directions
//   backward     mac_lstm_bwd_tc: BPTT as ONE persistent cluster launch, then dKernel += [X | h_prev]^T dG (tc_wgrad_splitk,
//                K = B*S padded to 64), dBias (fixed-order column sums), dX = dG Wx^T (mac_linear_tc_fwd)
//
// Cluster layout (h = 256 only): 8 CTAs per (direction, 64 batch rows).  CTA `rank` owns hidden units [32 rank, 32 rank+32)
// and with them the 128 columns g*h + 32 rank + u (gate g < 4, u < 32) of the TF kernel.  Its bf16 slice of Wh (64 KB) is
// loaded into shared memory once and stays there for all S steps.  One warpgroup per CTA; the m64n128 accumulator fragment
// of a thread holds all four gates of its (row, unit) pairs, so the cell update needs no shuffle.
#include <cooperative_groups.h>
#include "tc_gemm.cuh"

namespace mac {
namespace cg = cooperative_groups;

constexpr int ET_H = 256;                // hidden units per direction
constexpr int ET_G = 4 * ET_H;           // gate columns per direction
constexpr int ET_CL = 8;                 // CTAs per cluster
constexpr int ET_HU = ET_H / ET_CL;      // units per CTA (32)
constexpr int ET_ROWS = 64;              // batch rows per cluster (the wgmma M)
constexpr int ET_THREADS = 128;          // one warpgroup

inline int et_pad_e(int E) { return (E + 127) & ~127; }
inline int et_pad_m(long long M) { return (int)((M + 63) & ~63LL); }

// byte offset of element (r, c) in a [rows x 64] bf16 tile stored as 128-byte rows with the 128-byte swizzle (the layout
// make_sw128_kmajor_desc describes; the tile base is 1024-byte aligned)
__device__ __forceinline__ uint32_t sw128_off(int r, int c) {
  return (uint32_t)(r * 128 + ((((c >> 3) ^ (r & 7)) << 4) | ((c & 7) << 1)));
}
// generic-proxy writes (local or remote shared memory) made visible to the async proxy that wgmma reads through
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ input half
// words[m, k] = emb row (mac_embed_fwd's out_raw); x16[m, k] = bf16(dropout(words))[m, k] for k < E, 0 for E <= k < Ep.  The
// Philox draw of float4 (m, k4 < E/4) has mac_embed_fwd's element index m*(E/4) + k4, so the masks are the fp32 path's.
__global__ void embed_tc_kernel(const float4* __restrict__ emb, const int32_t* __restrict__ idx, uint32_t thresh, float scale,
                                uint64_t seed, int site, int step, float4* __restrict__ raw, uint2* __restrict__ x16,
                                long long n4p, int E4, int Ep4, int V) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4p) return;
  const long long row = i / Ep4;
  const int k4 = (int)(i - row * Ep4);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (k4 < E4) {
    const int id = idx[row];
    if (id > 0 && id <= V) v = __ldg(emb + (size_t)(id - 1) * E4 + k4);
    const long long i4 = row * E4 + k4;
    raw[i4] = v;
    if (thresh) {
      const Philox4 r = philox4x32_10(seed, (uint64_t)i4, (uint32_t)site, (uint32_t)step);
      v.x = ((r.x >> 8) >= thresh) ? v.x * scale : 0.f;
      v.y = ((r.y >> 8) >= thresh) ? v.y * scale : 0.f;
      v.z = ((r.z >> 8) >= thresh) ? v.z * scale : 0.f;
      v.w = ((r.w >> 8) >= thresh) ? v.w * scale : 0.f;
    }
  }
  x16[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
}

// fp32 W[K, N] -> bf16 Wt[N, Kp], Wt[n, k] = bf16(W[k, n]) for k < K and 0 for K <= k < Kp
__global__ void pack_weight_kpad_kernel(const float* __restrict__ W, __nv_bfloat16* __restrict__ Wt, int K, int Kp, int N) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.y * 32, n0 = blockIdx.x * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, n = n0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < K && n < N) ? W[(size_t)k * N + n] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int n = n0 + i, k = k0 + threadIdx.x;
    if (n < N && k < Kp) Wt[(size_t)n * Kp + k] = __float2bfloat16_rn(tile[threadIdx.x][i]);
  }
}

// ------------------------------------------------------------------------------------------------ recurrence, forward
struct LstmTcFwdParams {
  const float* gx[2];        // [B*S, 4h] fp32: dropout(X) @ kernel[0:E] + bias
  const float* Wh[2];        // [h, 4h] fp32: rows E.. of the TF kernel (packed to bf16 in shared memory by the kernel)
  const int32_t* lengths;
  float forget_bias;
  float* out_seq;            // [B, S, ndir*h]
  float* vecq;               // [B, ndir*h] (may be NULL)
  float* save_gates;         // [ndir, B*S, 4h] activated i, j, f, o (may be NULL: then save_c / save_hprev are too)
  float* save_c;             // [ndir, B*S, h]
  float* save_hprev;         // [ndir, B*S, h] fp32 h the step consumed (its bf16 rounding is the product operand)
  int B, S, ndir;
};

constexpr int ETF_W_BYTES = 4 * 128 * 128;          // Wt [4 k-blocks][128 gate columns][64 units] bf16
constexpr int ETF_H_BYTES = 4 * ET_ROWS * 128;      // h  [4 k-blocks][64 rows][64 units] bf16
constexpr int ETF_SMEM = ETF_W_BYTES + 2 * ETF_H_BYTES + 1024;

// Per step: gates[64 rows, 128 cols] = h(s) [64 x 256] @ Wh slice [256 x 128] (16 wgmma m64n128k16, h from the shared
// A buffer of step s), + gx, then the cell update in the accumulator registers.  The new h goes out as bf16 into the
// CTA's 32 columns of the other A buffer, locally and to the seven peers over DSMEM (16-byte stores), then one cluster
// barrier.  Double-buffered A: a CTA writes buffer (s+1)&1 only after every CTA has passed the barrier of step s-1, i.e.
// after every wgmma that read it.  Rows b >= B carry h = 0; rows past their length carry h and c through (dynamic_rnn).
__global__ void __launch_bounds__(ET_THREADS, 1) lstm_fwd_tc_kernel(const LstmTcFwdParams p) {
  extern __shared__ unsigned char et_smem[];
  unsigned char* base = et_smem + ((1024u - (smem_u32(et_smem) & 1023u)) & 1023u);
  unsigned char* wsm = base;
  unsigned char* hsm = base + ETF_W_BYTES;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.y, b_base = blockIdx.z * ET_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* __restrict__ Wh = (dir ? p.Wh[1] : p.Wh[0]);
  // Wt[n][k] = bf16(Wh[k][col(n)]), col(n) = (n / 32) * h + 32 rank + n % 32: the K-major B operand
  for (int e = tid; e < 128 * ET_H; e += ET_THREADS) {
    const int n = e & 127, k = e >> 7;
    const float v = __ldg(Wh + (size_t)k * ET_G + (n >> 5) * ET_H + rank * ET_HU + (n & 31));
    *reinterpret_cast<__nv_bfloat16*>(wsm + (k >> 6) * (128 * 128) + sw128_off(n, k & 63)) = __float2bfloat16_rn(v);
  }
  for (int e = tid; e < 2 * ETF_H_BYTES / 16; e += ET_THREADS) reinterpret_cast<uint4*>(hsm)[e] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_all();
  cluster.sync();                                // every buffer is zeroed before any remote store can land

  // fragment: acc[4 j + 2 hh + e] = row 16 warp + lane/4 + 8 hh, column 8 j + 2 (lane & 3) + e; j = 4 g + jj, so the
  // thread's units are u = 8 jj + 2 (lane & 3) + e and acc[4 (4 g + jj) + 2 hh + e] is gate g of (row hh, unit (jj, e))
  const int W2 = p.ndir * ET_H;
  const int u0 = 2 * (lane & 3);
  int brow[2], len[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    brow[hh] = b_base + 16 * warp + (lane >> 2) + 8 * hh;
    len[hh] = brow[hh] < p.B ? seq_len(p.lengths, brow[hh], p.S) : 0;
  }
  const float* __restrict__ gxd = (dir ? p.gx[1] : p.gx[0]);
  const size_t dbase = (size_t)dir * p.B * p.S;
  float c[2][4][2], hc[2][4][2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) c[hh][jj][0] = c[hh][jj][1] = hc[hh][jj][0] = hc[hh][jj][1] = 0.f;
  const int kbo = rank >> 1, co = ET_HU * (rank & 1);    // this CTA's units in the A operand: k-block, first column
  float acc[64];

  for (int s = 0; s < p.S; ++s) {
    const uint32_t ha = smem_u32(hsm + (s & 1) * ETF_H_BYTES), wa = smem_u32(wsm);
    fence_proxy_async();                          // the peers' h stores, acquired by the barrier, before the async reads
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < 4; ++kb)
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_bf16_n128(acc, make_sw128_kmajor_desc(ha + kb * (ET_ROWS * 128)) + 2 * k,
                        make_sw128_kmajor_desc(wa + kb * (128 * 128)) + 2 * k, (kb | k) ? 1u : 0u);
    wgmma_commit();
    // the input half of this step's gates, loaded while the products run
    float2 gx[2][4][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const bool live = s < len[hh];
      const int t = dir ? (len[hh] - 1 - s) : s;
      const float* g0 = gxd + ((size_t)brow[hh] * p.S + t) * ET_G + rank * ET_HU + u0;
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          gx[hh][g][jj] = live ? __ldg(reinterpret_cast<const float2*>(g0 + g * ET_H + 8 * jj)) : make_float2(0.f, 0.f);
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
    unsigned char* nb = hsm + ((s + 1) & 1) * ETF_H_BYTES;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int b = brow[hh];
      const bool valid = b < p.B, live = s < len[hh];
      const int t = live ? (dir ? (len[hh] - 1 - s) : s) : s;   // t >= len rows: each written (as zeros) at step s = t
      const size_t rowi = (size_t)b * p.S + t;
      const int r = 16 * warp + (lane >> 2) + 8 * hh;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        float hn[2], gi[2], gj[2], gf[2], go[2], hp[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float ge[4] = {e ? gx[hh][0][jj].y : gx[hh][0][jj].x, e ? gx[hh][1][jj].y : gx[hh][1][jj].x,
                               e ? gx[hh][2][jj].y : gx[hh][2][jj].x, e ? gx[hh][3][jj].y : gx[hh][3][jj].x};
          hp[e] = hc[hh][jj][e];
          gi[e] = gj[e] = gf[e] = go[e] = 0.f;
          hn[e] = hp[e];                                        // dynamic_rnn: state carried through past the end
          if (live) {
            gi[e] = sigmoid_f(acc[4 * (0 + jj) + 2 * hh + e] + ge[0]);
            gj[e] = tanhf(acc[4 * (4 + jj) + 2 * hh + e] + ge[1]);
            gf[e] = sigmoid_f(acc[4 * (8 + jj) + 2 * hh + e] + ge[2] + p.forget_bias);
            go[e] = sigmoid_f(acc[4 * (12 + jj) + 2 * hh + e] + ge[3]);
            c[hh][jj][e] = c[hh][jj][e] * gf[e] + gi[e] * gj[e];
            hn[e] = tanhf(c[hh][jj][e]) * go[e];
          }
          hc[hh][jj][e] = hn[e];
        }
        const int u = 8 * jj + u0, col = rank * ET_HU + u;
        if (valid) {
          const float2 o = live ? make_float2(hn[0], hn[1]) : make_float2(0.f, 0.f);
          *reinterpret_cast<float2*>(p.out_seq + rowi * W2 + dir * ET_H + col) = o;
          if (p.save_gates) {
            float* sg = p.save_gates + (dbase + rowi) * ET_G + col;
            *reinterpret_cast<float2*>(sg) = make_float2(gi[0], gi[1]);
            *reinterpret_cast<float2*>(sg + ET_H) = make_float2(gj[0], gj[1]);
            *reinterpret_cast<float2*>(sg + 2 * ET_H) = make_float2(gf[0], gf[1]);
            *reinterpret_cast<float2*>(sg + 3 * ET_H) = make_float2(go[0], go[1]);
            *reinterpret_cast<float2*>(p.save_c + (dbase + rowi) * ET_H + col) =
                live ? make_float2(c[hh][jj][0], c[hh][jj][1]) : make_float2(0.f, 0.f);
            *reinterpret_cast<float2*>(p.save_hprev + (dbase + rowi) * ET_H + col) =
                live ? make_float2(hp[0], hp[1]) : make_float2(0.f, 0.f);
          }
        }
        *reinterpret_cast<uint32_t*>(nb + kbo * (ET_ROWS * 128) + sw128_off(r, co + u)) = pack_bf16(hn[0], hn[1]);
      }
    }
    __syncthreads();
    // this CTA's [64 rows x 32 units] block (four 16-byte chunks per row, at their swizzled places) to the 7 peers
    for (int e = tid; e < (ET_CL - 1) * ET_ROWS * 4; e += ET_THREADS) {
      const int q = e & 3, r = (e >> 2) & 63, z = e >> 8;
      const int peer = z + (z >= rank ? 1 : 0);
      const uint32_t off = kbo * (ET_ROWS * 128) + r * 128 + ((((co >> 3) + q) ^ (r & 7)) << 4);
      *reinterpret_cast<uint4*>(cluster.map_shared_rank(nb + off, peer)) = *reinterpret_cast<const uint4*>(nb + off);
    }
    fence_proxy_async_all();
    cluster.sync();
  }
  if (p.vecq) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (brow[hh] < p.B)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj)
          *reinterpret_cast<float2*>(p.vecq + (size_t)brow[hh] * W2 + dir * ET_H + rank * ET_HU + 8 * jj + u0) =
              make_float2(hc[hh][jj][0], hc[hh][jj][1]);
  }
}

// ------------------------------------------------------------------------------------------------ BPTT
struct LstmTcBwdParams {
  const float* Wh[2];        // [h, 4h] fp32
  const int32_t* lengths;
  const float* save_gates;   // [ndir, B*S, 4h]
  const float* save_c;       // [ndir, B*S, h]
  const float* d_out_seq;    // [B, S, ndir*h]
  const float* d_vecq;       // [B, ndir*h] (may be NULL = 0)
  float* dG[2];              // [B*S, 4h] fp32 gate gradients (the bias sums)
  __nv_bfloat16* dGT[2];     // [4h, Mp] bf16: the weight gradient's K-major operand
  __nv_bfloat16* dGcat;      // [B*S, ndir*4h] bf16: the data gradient's A operand
  int B, S, ndir, Mp;
};

constexpr int ETB_W_BYTES = 2 * ET_H * 128;         // Wb [2 k-blocks][256 units][64 gate columns] bf16
constexpr int ETB_A_BYTES = 2 * ET_ROWS * 128;      // dG(s+1) [2 k-blocks][64 rows][64 gate columns] bf16
constexpr int ETB_R_BYTES = ET_CL * ET_ROWS * ET_HU * 4;   // partial dh: [8 source ranks][64 rows][32 units] fp32
constexpr int ETB_SMEM = ETB_W_BYTES + ETB_A_BYTES + 2 * ETB_R_BYTES + 1024;

// Per step s (S-1 .. 0): CTA rank multiplies its own 128 gate-gradient columns of step s+1 (bf16, in its shared A buffer)
// by the resident slice Wb[unit][column] = Wh[unit][col(column)] -- the forward's slice, transposed -- as two m64n128
// halves over all 256 units, and pushes each 32-unit block of the fp32 partial dh to the CTA that owns those units
// (slot `rank` of its receive buffer).  After the cluster barrier every CTA sums the eight slots in rank order (a fixed
// order: deterministic), and the gate derivatives of step s are its epilogue.  Receive buffers alternate by step.
__global__ void __launch_bounds__(ET_THREADS, 1) lstm_bwd_tc_kernel(const LstmTcBwdParams p) {
  extern __shared__ unsigned char et_smem[];
  unsigned char* base = et_smem + ((1024u - (smem_u32(et_smem) & 1023u)) & 1023u);
  unsigned char* wsm = base;
  unsigned char* asm_ = base + ETB_W_BYTES;
  float* recv = reinterpret_cast<float*>(base + ETB_W_BYTES + ETB_A_BYTES);
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int dir = blockIdx.y, b_base = blockIdx.z * ET_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* __restrict__ Wh = (dir ? p.Wh[1] : p.Wh[0]);
  for (int e = tid; e < ET_H * 128; e += ET_THREADS) {
    const int k = e & 127, n = e >> 7;                   // n: unit (row of Wh), k: this CTA's gate column
    const float v = __ldg(Wh + (size_t)n * ET_G + (k >> 5) * ET_H + rank * ET_HU + (k & 31));
    *reinterpret_cast<__nv_bfloat16*>(wsm + (k >> 6) * (ET_H * 128) + sw128_off(n, k & 63)) = __float2bfloat16_rn(v);
  }
  for (int e = tid; e < ETB_A_BYTES / 16; e += ET_THREADS) reinterpret_cast<uint4*>(asm_)[e] = make_uint4(0, 0, 0, 0);
  fence_proxy_async_all();
  cluster.sync();

  const int W2 = p.ndir * ET_H;
  const int u0 = 2 * (lane & 3);
  const size_t M = (size_t)p.B * p.S;
  const size_t dbase = (size_t)dir * M;
  int brow[2], len[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    brow[hh] = b_base + 16 * warp + (lane >> 2) + 8 * hh;
    len[hh] = brow[hh] < p.B ? seq_len(p.lengths, brow[hh], p.S) : 0;
  }
  float dcc[2][4][2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) dcc[hh][jj][0] = dcc[hh][jj][1] = 0.f;
  float acc[64];

  for (int s = p.S - 1; s >= 0; --s) {
    float* rb = recv + (s & 1) * (ETB_R_BYTES / 4);
    const uint32_t aa = smem_u32(asm_), wa = smem_u32(wsm);
#pragma unroll
    for (int nh = 0; nh < 2; ++nh) {
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < 2; ++kb)
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_bf16_n128(acc, make_sw128_kmajor_desc(aa + kb * (ET_ROWS * 128)) + 2 * k,
                          make_sw128_kmajor_desc(wa + kb * (ET_H * 128) + nh * (128 * 128)) + 2 * k, (kb | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_hold(acc);
      // acc[4 j + 2 hh + e]: row 16 warp + lane/4 + 8 hh, unit 128 nh + 8 j + u0 + e -> owner 4 nh + j / 4
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float* dst = cluster.map_shared_rank(rb, 4 * nh + (j >> 2)) + rank * (ET_ROWS * ET_HU);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int r = 16 * warp + (lane >> 2) + 8 * hh;
          *reinterpret_cast<float2*>(dst + r * ET_HU + 8 * (j & 3) + u0) = make_float2(acc[4 * j + 2 * hh], acc[4 * j + 2 * hh + 1]);
        }
      }
    }
    cluster.sync();                               // partials delivered; every CTA is done reading its A buffer
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int b = brow[hh];
      const bool valid = b < p.B, live = s < len[hh];
      const int t = live ? (dir ? (len[hh] - 1 - s) : s) : s;
      const size_t rowi = (size_t)b * p.S + t;
      const int r = 16 * warp + (lane >> 2) + 8 * hh;
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int u = 8 * jj + u0, col = rank * ET_HU + u;
        float dg[4][2];
#pragma unroll
        for (int g = 0; g < 4; ++g) dg[g][0] = dg[g][1] = 0.f;
        if (live) {
          float2 dr = make_float2(0.f, 0.f);
#pragma unroll
          for (int z = 0; z < ET_CL; ++z) {
            const float2 v = *reinterpret_cast<const float2*>(rb + z * (ET_ROWS * ET_HU) + r * ET_HU + u);
            dr.x += v.x;
            dr.y += v.y;
          }
          float2 dh = *reinterpret_cast<const float2*>(p.d_out_seq + rowi * W2 + dir * ET_H + col);
          if (s + 1 < len[hh]) {
            dh.x += dr.x;
            dh.y += dr.y;
          } else if (p.d_vecq) {                   // last live step: its h is the final state
            const float2 q = *reinterpret_cast<const float2*>(p.d_vecq + (size_t)b * W2 + dir * ET_H + col);
            dh.x += q.x;
            dh.y += q.y;
          }
          const float* sg = p.save_gates + (dbase + rowi) * ET_G + col;
          const float2 vi = *reinterpret_cast<const float2*>(sg), vj = *reinterpret_cast<const float2*>(sg + ET_H);
          const float2 vf = *reinterpret_cast<const float2*>(sg + 2 * ET_H), vo = *reinterpret_cast<const float2*>(sg + 3 * ET_H);
          const float2 cn = *reinterpret_cast<const float2*>(p.save_c + (dbase + rowi) * ET_H + col);
          float2 cp = make_float2(0.f, 0.f);
          if (s > 0) cp = *reinterpret_cast<const float2*>(p.save_c + (dbase + (size_t)b * p.S + (dir ? t + 1 : t - 1)) * ET_H + col);
          const float dhv[2] = {dh.x, dh.y}, giv[2] = {vi.x, vi.y}, gjv[2] = {vj.x, vj.y}, gfv[2] = {vf.x, vf.y};
          const float gov[2] = {vo.x, vo.y}, cnv[2] = {cn.x, cn.y}, cpv[2] = {cp.x, cp.y};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float tc = tanhf(cnv[e]);
            const float dc = dcc[hh][jj][e] + dhv[e] * gov[e] * (1.f - tc * tc);
            dg[0][e] = dc * gjv[e] * giv[e] * (1.f - giv[e]);
            dg[1][e] = dc * giv[e] * (1.f - gjv[e] * gjv[e]);
            dg[2][e] = dc * cpv[e] * gfv[e] * (1.f - gfv[e]);
            dg[3][e] = dhv[e] * tc * gov[e] * (1.f - gov[e]);
            dcc[hh][jj][e] = dc * gfv[e];
          }
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const uint32_t pk = pack_bf16(dg[g][0], dg[g][1]);
          const int lc = g * ET_HU + u;                   // this CTA's gate column
          *reinterpret_cast<uint32_t*>(asm_ + (lc >> 6) * (ET_ROWS * 128) + sw128_off(r, lc & 63)) = pk;
          if (valid) {
            const int n = g * ET_H + col;
            *reinterpret_cast<float2*>((dir ? p.dG[1] : p.dG[0]) + rowi * ET_G + n) = make_float2(dg[g][0], dg[g][1]);
            *reinterpret_cast<uint32_t*>(p.dGcat + rowi * (size_t)(p.ndir * ET_G) + dir * ET_G + n) = pk;
            __nv_bfloat16* gt = (dir ? p.dGT[1] : p.dGT[0]) + (size_t)n * p.Mp + rowi;
            gt[0] = __ushort_as_bfloat16((unsigned short)(pk & 0xffffu));
            gt[p.Mp] = __ushort_as_bfloat16((unsigned short)(pk >> 16));
          }
        }
      }
    }
    fence_proxy_async_all();
    __syncthreads();                                // the next step's A operand is complete
  }
}

// ------------------------------------------------------------------------------------------------ backward helpers
// dst[c, m] = bf16(src[m * ld + c]) for c < C, m < M; 0 for C <= c < Cp or M <= m < Mp.  64 x 64 tiles.
template <typename T>
__global__ void __launch_bounds__(256) pad_t_bf16_kernel(const T* __restrict__ src, int ld, int M, int C, int Cp, int Mp,
                                                        __nv_bfloat16* __restrict__ dst) {
  __shared__ float tile[64][65];
  const int m0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  for (int e = threadIdx.x; e < 64 * 64; e += 256) {
    const int mm = e >> 6, cc = e & 63, m = m0 + mm, c = c0 + cc;
    float v = 0.f;
    if (m < M && c < C) {
      if constexpr (sizeof(T) == 2) v = __bfloat162float(src[(size_t)m * ld + c]);
      else v = src[(size_t)m * ld + c];
    }
    tile[cc][mm] = v;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < 64 * 32; e += 256) {
    const int cc = e >> 5, mp = e & 31, c = c0 + cc, m = m0 + 2 * mp;
    if (c < Cp && m < Mp)
      *reinterpret_cast<uint32_t*>(dst + (size_t)c * Mp + m) = pack_bf16(tile[cc][2 * mp], tile[cc][2 * mp + 1]);
  }
}

// wxc[e, dir*4h + n] = bf16(kernel_dir[e, n]) for e < E, 0 for E <= e < Ep: the data gradient's K-major B operand
__global__ void pack_wx_cat_kernel(const float* __restrict__ k0, const float* __restrict__ k1, int E, int Ep, int ndir,
                                   __nv_bfloat16* __restrict__ wxc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = ndir * ET_G;
  if (i >= (long long)Ep * W) return;
  const int e = (int)(i / W), n = (int)(i - (long long)e * W);
  const int d = n / ET_G;
  const float v = e < E ? __ldg((d ? k1 : k0) + (size_t)e * ET_G + (n - d * ET_G)) : 0.f;
  wxc[i] = __float2bfloat16_rn(v);
}

// dx[m, k] = dxp[m, k] for k < E (dxp has Ep columns)
__global__ void compact_cols_kernel(const float* __restrict__ dxp, float* __restrict__ dx, long long M, int E, int Ep) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * E) return;
  const long long m = i / E;
  dx[i] = dxp[m * Ep + (i - m * E)];
}

// workspace of mac_lstm_bwd_tc: 1 KB-aligned slabs behind a 1 KB alignment slack
struct LstmBwdTcLayout {
  size_t dG, dGT, dGcat, xhT, dW, wpart, bpart, wxc, dxp, total;
  int ksplit;
};
inline LstmBwdTcLayout lstm_bwd_tc_layout(int B, int S, int E, int ndir) {
  auto al = [](size_t v) { return (v + 1023) & ~(size_t)1023; };
  const size_t M = (size_t)B * S, Mp = (size_t)et_pad_m((long long)M), Ep = (size_t)et_pad_e(E), In = Ep + ET_H;
  LstmBwdTcLayout l;
  l.ksplit = tc_pick_ksplit((int)Mp, (int)(In / TC_BM) * (ET_G / TC_BN));
  size_t o = 0;
  l.dG = o;    o += al((size_t)ndir * M * ET_G * 4);
  l.dGT = o;   o += al((size_t)ndir * ET_G * Mp * 2);
  l.dGcat = o; o += al(M * ndir * ET_G * 2);
  l.xhT = o;   o += al(In * Mp * 2);
  l.dW = o;    o += al(In * ET_G * 4);
  l.wpart = o; o += al((size_t)l.ksplit * In * ET_G * 4);
  l.bpart = o; o += al((size_t)B * ET_G * 4);
  l.wxc = o;   o += al(Ep * ndir * ET_G * 2);
  l.dxp = o;   o += al(M * Ep * 4);
  l.total = o + 1024;
  return l;
}

template <typename P>
inline int et_launch(void (*kern)(const P), const P& p, int ndir, int B, size_t smem, cudaStream_t stream) {
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(ET_CL, ndir, (B + ET_ROWS - 1) / ET_ROWS);
  cfg.blockDim = dim3(ET_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = ET_CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MAC_CUDA_TRY(cudaLaunchKernelEx(&cfg, kern, p));
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac

using namespace mac;

extern "C" int mac_embed_fwd_tc(const float* emb, const int32_t* idx, float keep, uint64_t seed, int site, int step,
                                float* out_raw, void* x_bf16, int B, int S, int V, int E, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!emb || !idx || !out_raw || !x_bf16 || B <= 0 || S <= 0 || V <= 0 || E <= 0 || (E & 3) || !(keep > 0.f && keep <= 1.f))
    return MAC_ERR_INVALID;
  if (!mac_aligned16(emb) || !mac_aligned16(out_raw) || !mac_aligned16(x_bf16)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  const int Ep = et_pad_e(E);
  const long long n4p = (long long)B * S * (Ep / 4);
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  embed_tc_kernel<<<(unsigned)((n4p + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(emb), idx, thr, scale, seed, site, step, reinterpret_cast<float4*>(out_raw),
      reinterpret_cast<uint2*>(x_bf16), n4p, E / 4, Ep / 4, V);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_pack_weight_bf16_kpad(const float* W, void* Wt_bf16, int K, int Kp, int n_out, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!W || !Wt_bf16 || K <= 0 || Kp < K || n_out <= 0) return MAC_ERR_INVALID;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  dim3 grid((n_out + 31) / 32, (Kp + 31) / 32), block(32, 8);
  pack_weight_kpad_kernel<<<grid, block, 0, stream>>>(W, reinterpret_cast<__nv_bfloat16*>(Wt_bf16), K, Kp, n_out);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_lstm_fwd_tc(const float* gx_fw, const float* gx_bw, const float* Wh_fw, const float* Wh_bw,
                               const int32_t* lengths, float forget_bias, float* out_seq, float* vecq, float* save_gates,
                               float* save_c, float* save_hprev, int B, int S, int h, int ndir, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!gx_fw || !Wh_fw || !lengths || !out_seq || B <= 0 || S <= 0 || h <= 0 || ndir < 1 || ndir > 2 ||
      (ndir == 2 && (!gx_bw || !Wh_bw)))
    return MAC_ERR_INVALID;
  if ((save_gates != nullptr) != (save_c != nullptr) || (save_gates != nullptr) != (save_hprev != nullptr))
    return MAC_ERR_INVALID;
  if ((long long)B * S * 4 * h >= (1LL << 31)) return MAC_ERR_INVALID;
  if (h != ET_H) return MAC_ERR_UNSUPPORTED;
  const void* al[] = {gx_fw, Wh_fw, out_seq, vecq, save_gates, save_c, save_hprev, ndir == 2 ? gx_bw : nullptr,
                      ndir == 2 ? Wh_bw : nullptr};
  for (const void* q : al)
    if (q && (reinterpret_cast<uintptr_t>(q) & 7)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  LstmTcFwdParams p{};
  p.gx[0] = gx_fw; p.gx[1] = gx_bw; p.Wh[0] = Wh_fw; p.Wh[1] = Wh_bw;
  p.lengths = lengths; p.forget_bias = forget_bias; p.out_seq = out_seq; p.vecq = vecq;
  p.save_gates = save_gates; p.save_c = save_c; p.save_hprev = save_hprev;
  p.B = B; p.S = S; p.ndir = ndir;
  return et_launch(lstm_fwd_tc_kernel, p, ndir, B, ETF_SMEM, stream);
}

extern "C" size_t mac_lstm_bwd_tc_workspace_bytes(int B, int S, int E, int h, int ndir) {
  if (B <= 0 || S <= 0 || E <= 0 || h != ET_H || ndir < 1 || ndir > 2) return 0;
  return lstm_bwd_tc_layout(B, S, E, ndir).total;
}

extern "C" int mac_lstm_bwd_tc(const void* x_bf16, const float* kernel_fw, const float* kernel_bw, const int32_t* lengths,
                               const float* save_gates, const float* save_c, const float* save_hprev, const float* d_out_seq,
                               const float* d_vecq, float* dkernel_fw, float* dkernel_bw, float* dbias_fw, float* dbias_bw,
                               float* dx, void* workspace, size_t workspace_bytes, int B, int S, int E, int h, int ndir,
                               mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_bf16 || !kernel_fw || !lengths || !save_gates || !save_c || !save_hprev || !d_out_seq || !dkernel_fw || !dbias_fw ||
      !dx || !workspace || B <= 0 || S <= 0 || E <= 0 || (E & 3) || h <= 0 || ndir < 1 || ndir > 2 ||
      (ndir == 2 && (!kernel_bw || !dkernel_bw || !dbias_bw)))
    return MAC_ERR_INVALID;
  if ((long long)B * S * 4 * h * ndir >= (1LL << 31)) return MAC_ERR_INVALID;
  if (h != ET_H) return MAC_ERR_UNSUPPORTED;
  const void* al[] = {x_bf16, kernel_fw, save_gates, save_c, save_hprev, d_out_seq, d_vecq, dkernel_fw, dbias_fw, dx,
                      ndir == 2 ? kernel_bw : nullptr, ndir == 2 ? dkernel_bw : nullptr, ndir == 2 ? dbias_bw : nullptr};
  for (const void* q : al)
    if (q && !mac_aligned16(q)) return MAC_ERR_ALIGN;
  const LstmBwdTcLayout l = lstm_bwd_tc_layout(B, S, E, ndir);
  if (workspace_bytes < l.total) return MAC_ERR_WORKSPACE;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  const int M = B * S, Mp = et_pad_m(M), Ep = et_pad_e(E), In = Ep + ET_H;
  char* base = tc_align1k(workspace);
  float* dG = reinterpret_cast<float*>(base + l.dG);
  __nv_bfloat16* dGT = reinterpret_cast<__nv_bfloat16*>(base + l.dGT);
  __nv_bfloat16* dGcat = reinterpret_cast<__nv_bfloat16*>(base + l.dGcat);
  __nv_bfloat16* xhT = reinterpret_cast<__nv_bfloat16*>(base + l.xhT);
  float* dW = reinterpret_cast<float*>(base + l.dW);
  float* wpart = reinterpret_cast<float*>(base + l.wpart);
  float* bpart = reinterpret_cast<float*>(base + l.bpart);
  __nv_bfloat16* wxc = reinterpret_cast<__nv_bfloat16*>(base + l.wxc);
  float* dxp = reinterpret_cast<float*>(base + l.dxp);
  const float* kern[2] = {kernel_fw, kernel_bw};
  float* dkern[2] = {dkernel_fw, dkernel_bw};
  float* dbias[2] = {dbias_fw, dbias_bw};

  // BPTT: gate gradients of every step, fp32 and in the two bf16 layouts of the GEMMs below
  for (int d = 0; d < ndir; ++d)      // columns M..Mp-1 of the K-major copy are the zero padding of the weight gradient's K
    if (Mp > M)
      MAC_CUDA_TRY(cudaMemset2DAsync(dGT + (size_t)d * ET_G * Mp + M, (size_t)Mp * 2, 0, (size_t)(Mp - M) * 2, ET_G, stream));
  LstmTcBwdParams p{};
  for (int d = 0; d < ndir; ++d) {
    p.Wh[d] = kern[d] + (size_t)E * ET_G;
    p.dG[d] = dG + (size_t)d * M * ET_G;
    p.dGT[d] = dGT + (size_t)d * ET_G * Mp;
  }
  p.lengths = lengths; p.save_gates = save_gates; p.save_c = save_c; p.d_out_seq = d_out_seq; p.d_vecq = d_vecq;
  p.dGcat = dGcat; p.B = B; p.S = S; p.ndir = ndir; p.Mp = Mp;
  int st = et_launch(lstm_bwd_tc_kernel, p, ndir, B, ETB_SMEM, stream);
  if (st != MAC_OK) return st;

  // dKernel += [X | h_prev]^T dG: one split-K wgrad over K = Mp per direction into [Ep + h, 4h], whose rows 0..E-1 and
  // Ep..Ep+h-1 are the kernel's rows 0..E-1 and E..E+h-1
  pad_t_bf16_kernel<__nv_bfloat16><<<dim3(Mp / 64, Ep / 64), 256, 0, stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(x_bf16), Ep, M, Ep, Ep, Mp, xhT);
  MAC_LAUNCH_CHECK();
  for (int d = 0; d < ndir; ++d) {
    pad_t_bf16_kernel<float><<<dim3(Mp / 64, ET_H / 64), 256, 0, stream>>>(save_hprev + (size_t)d * M * ET_H, ET_H, M, ET_H,
                                                                          ET_H, Mp, xhT + (size_t)Ep * Mp);
    MAC_LAUNCH_CHECK();
    MAC_CUDA_TRY(cudaMemsetAsync(dW, 0, (size_t)In * ET_G * 4, stream));
    st = tc_wgrad_splitk(xhT, dGT + (size_t)d * ET_G * Mp, dW, wpart, In, ET_G, Mp, stream);
    if (st != MAC_OK) return st;
    st = mac_axpy(dkern[d], dW, 1.f, (long long)E * ET_G, stream_);
    if (st != MAC_OK) return st;
    st = mac_axpy(dkern[d] + (size_t)E * ET_G, dW + (size_t)Ep * ET_G, 1.f, (long long)ET_H * ET_G, stream_);
    if (st != MAC_OK) return st;
    // dBias += column sums of dG (fp32): per sample over its S rows, then over the samples
    st = mac_colsum(dG + (size_t)d * M * ET_G, bpart, B, S, ET_G, 0, stream_);
    if (st != MAC_OK) return st;
    st = mac_colsum(bpart, dbias[d], 1, B, ET_G, 1, stream_);
    if (st != MAC_OK) return st;
  }

  // dX = [dG_fw | dG_bw] [Wx_fw | Wx_bw]^T  (K = ndir * 4h), then the first E of its Ep columns
  const long long nw = (long long)Ep * ndir * ET_G;
  pack_wx_cat_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, stream>>>(kernel_fw, kernel_bw, E, Ep, ndir, wxc);
  MAC_LAUNCH_CHECK();
  st = mac_linear_tc_fwd(dGcat, wxc, nullptr, MAC_ACT_NON, dxp, 0, M, ndir * ET_G, Ep, stream_);
  if (st != MAC_OK) return st;
  const long long nx = (long long)M * E;
  compact_cols_kernel<<<(unsigned)((nx + 255) / 256), 256, 0, stream>>>(dxp, dx, M, E, Ep);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}
