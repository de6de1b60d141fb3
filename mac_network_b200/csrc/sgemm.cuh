// fp32 FMA-pipe GEMM with fused A-operand prologues and epilogues: the <=1e-4 parity path of the
// d x d projections (ops.linear / ops.multiply, ops.py:50-59, 298-333) and of the read-unit chain.
//   C[M,N] = epilogue( Aview[M,K] @ W[K,N] )
// Aview is never materialised: concatenations (ops.py:65-78, 718), the broadcast multiply
// (ops.py:694-703) and dropout (ops.py:678) are applied while the tile is loaded.
// Optional split-K with an in-kernel, fixed-order ("last block reduces") combine so results are
// deterministic.
#pragma once
#include "common.cuh"
#include <stdlib.h>

namespace mac {

enum { A_SEGS = 0, A_ROWSCALE_CONCAT = 1, A_DROPOUT = 2,
       // transposed views for weight gradients dW[K_in, N] = X^T[K_in, rows] @ dY[rows, N]: A(m, k) = X[k][m]
       A_TRANS = 3, A_TRANS_ROWSCALE_CONCAT = 4, A_TRANS_DROPOUT = 5 };
enum { EPI_BIAS_ACT = 0, EPI_READ_LOGITS = 1, EPI_GATE = 2,
       EPI_MUL_ELUGRAD = 3,     // Y = acc * ELU'(aux) with aux = ELU(z) saved from forward: aux > 0 ? 1 : aux + 1
       EPI_ACCUM_DROPOUT = 4 }; // Y += acc * keep-mask(m, n) * scale   (gradient through tf.nn.dropout)

struct SgemmParams {
  // ---- A view
  int a_mode;
  const float* a[4];
  int ak[4];
  int lda[4];
  int nseg;
  const float* rowvec;   // A_ROWSCALE_CONCAT: y[B, K/2]; row m belongs to batch m / rows_per_batch
  int rows_per_batch;
  int rs_half;           // A_ROWSCALE_CONCAT: width of the scaled part (0 -> K/2; == K -> A = x*y, nothing concatenated)
  uint32_t a_thresh;     // A_DROPOUT
  float a_scale;
  uint64_t seed;
  int a_site;
  int step;
  // ---- B
  const float* W;
  int ldw;
  int M, N, K;
  // ---- epilogue
  int epi;
  const float* bias;     // [N] or NULL
  float bias_const;
  int act;
  float* Y;              // EPI_BIAS_ACT / EPI_GATE output; EPI_READ_LOGITS: optional I1 store (may be NULL)
  int ldy;
  int accumulate;        // EPI_BIAS_ACT: Y += result (parameter-gradient accumulation over the steps)
  float* Y2;             // EPI_BIAS_ACT: columns >= n_split go to Y2[m, n - n_split] (same ldy) when Y2 != NULL
  int n_split;
  const float* aux;      // EPI_MUL_ELUGRAD: saved activation [M, ldaux]; EPI_BIAS_ACT: optional pre-activation addend
  int ldaux;
  // EPI_READ_LOGITS: t = (acc+bias)*ctrl[b]; i2 = elu(t) (dropout) ; parts[m, blockIdx.x] = sum_n i2*wr[n]
  const float* ctrl;
  const float* wr;
  float* logit_parts;
  uint32_t e_thresh;
  float e_scale;
  int e_site;
  // EPI_GATE: z = sigmoid(acc+bias+bias_const); Y = gnew*z + gold*(1-z)
  const float* gnew;
  const float* gold;
  float* gate_z;
  // ---- split-K
  int splitk;
  float* partial;          // [splitk, M, N]
  unsigned int* counters;  // [tiles], zero on entry, zero on exit
};

__device__ __forceinline__ float4 sg_load_a(const SgemmParams& p, int m, int k) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (m >= p.M || k >= p.K) return v;
  if (p.a_mode == A_SEGS) {
    int off = 0;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      if (s < p.nseg) {
        if (k >= off && k < off + p.ak[s]) {
          v = __ldg(reinterpret_cast<const float4*>(p.a[s] + (size_t)m * p.lda[s] + (k - off)));
        }
        off += p.ak[s];
      }
    }
  } else if (p.a_mode == A_ROWSCALE_CONCAT) {
    const int half = p.rs_half ? p.rs_half : (p.K >> 1);
    if (k < half) {
      v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)m * p.lda[0] + k));
      const float4 y = __ldg(reinterpret_cast<const float4*>(p.rowvec + (size_t)(m / p.rows_per_batch) * half + k));
      v.x *= y.x; v.y *= y.y; v.z *= y.z; v.w *= y.w;
    } else {
      v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)m * p.lda[0] + (k - half)));
    }
  } else {  // A_DROPOUT
    v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)m * p.lda[0] + k));
    const uint64_t e = (uint64_t)m * (uint64_t)p.K + (uint64_t)k;
    const Philox4 r = philox4x32_10(p.seed, e >> 2, (uint32_t)p.a_site, (uint32_t)p.step);
    v.x = ((r.x >> 8) >= p.a_thresh) ? v.x * p.a_scale : 0.f;
    v.y = ((r.y >> 8) >= p.a_thresh) ? v.y * p.a_scale : 0.f;
    v.z = ((r.z >> 8) >= p.a_thresh) ? v.z * p.a_scale : 0.f;
    v.w = ((r.w >> 8) >= p.a_thresh) ? v.w * p.a_scale : 0.f;
  }
  return v;
}

// transposed view: four consecutive m (feature index) of row k of X
__device__ __forceinline__ float4 sg_load_at(const SgemmParams& p, int m, int k) {
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (m >= p.M || k >= p.K) return v;
  if (p.a_mode == A_TRANS) {
    v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)k * p.lda[0] + m));
  } else if (p.a_mode == A_TRANS_ROWSCALE_CONCAT) {
    const int half = p.M >> 1;
    if (m < half) {
      v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)k * p.lda[0] + m));
      const float4 y = __ldg(reinterpret_cast<const float4*>(p.rowvec + (size_t)(k / p.rows_per_batch) * half + m));
      v.x *= y.x; v.y *= y.y; v.z *= y.z; v.w *= y.w;
    } else {
      v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)k * p.lda[0] + (m - half)));
    }
  } else {  // A_TRANS_DROPOUT
    v = __ldg(reinterpret_cast<const float4*>(p.a[0] + (size_t)k * p.lda[0] + m));
    const uint64_t e = (uint64_t)k * (uint64_t)p.M + (uint64_t)m;
    const Philox4 r = philox4x32_10(p.seed, e >> 2, (uint32_t)p.a_site, (uint32_t)p.step);
    v.x = ((r.x >> 8) >= p.a_thresh) ? v.x * p.a_scale : 0.f;
    v.y = ((r.y >> 8) >= p.a_thresh) ? v.y * p.a_scale : 0.f;
    v.z = ((r.z >> 8) >= p.a_thresh) ? v.z * p.a_scale : 0.f;
    v.w = ((r.w >> 8) >= p.a_thresh) ? v.w * p.a_scale : 0.f;
  }
  return v;
}

#ifndef SGEMM_MIN_BLOCKS
#define SGEMM_MIN_BLOCKS 2      // forward: 128 registers, two CTAs per SM (+14 % on the [12544,1024]x[1024,512] projection)
#endif
template <int BM, int BN>
__global__ void __launch_bounds__(256, SGEMM_MIN_BLOCKS) sgemm_kernel(const SgemmParams p) {
  constexpr int BK = 16;
  constexpr int TM = BM / 16, TN = BN / 16;         // 8x8 (128x128) or 4x4 (64x64)
  constexpr int A_LD = BM + 4;
  constexpr int A_F4 = BM * BK / 4 / 256;           // float4 loads of A per thread
  constexpr int B_F4 = BK * BN / 4 / 256;
  static_assert(A_F4 >= 1 && B_F4 >= 1, "tile too small");
  __shared__ __align__(16) float As[2][BK][A_LD];
  __shared__ __align__(16) float Bs[2][BK][BN];
  __shared__ int s_last;

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

  // k range of this split
  const int kiters_total = (p.K + BK - 1) / BK;
  const int per = (kiters_total + p.splitk - 1) / p.splitk;
  const int it0 = blockIdx.z * per;
  const int it1 = min(kiters_total, it0 + per);

  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float4 ra[A_F4], rb[B_F4];
  auto gload = [&](int it) {
    const int k0 = it * BK;
#pragma unroll
    for (int i = 0; i < A_F4; ++i) {
      const int f = tid + i * 256;
      if (p.a_mode >= A_TRANS) {
        const int kr = f / (BM / 4), m4 = f % (BM / 4);
        ra[i] = sg_load_at(p, m0 + m4 * 4, k0 + kr);
      } else {
        const int row = f >> 2, kq = f & 3;
        ra[i] = sg_load_a(p, m0 + row, k0 + kq * 4);
      }
    }
#pragma unroll
    for (int i = 0; i < B_F4; ++i) {
      const int f = tid + i * 256;
      const int kr = f / (BN / 4), c4 = f % (BN / 4);
      const int k = k0 + kr, n = n0 + c4 * 4;
      rb[i] = (k < p.K && n < p.N) ? __ldg(reinterpret_cast<const float4*>(p.W + (size_t)k * p.ldw + n))
                                    : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < A_F4; ++i) {
      const int f = tid + i * 256;
      if (p.a_mode >= A_TRANS) {
        const int kr = f / (BM / 4), m4 = f % (BM / 4);
        *reinterpret_cast<float4*>(&As[buf][kr][m4 * 4]) = ra[i];
      } else {
        const int row = f >> 2, kq = f & 3;
        As[buf][kq * 4 + 0][row] = ra[i].x;
        As[buf][kq * 4 + 1][row] = ra[i].y;
        As[buf][kq * 4 + 2][row] = ra[i].z;
        As[buf][kq * 4 + 3][row] = ra[i].w;
      }
    }
#pragma unroll
    for (int i = 0; i < B_F4; ++i) {
      const int f = tid + i * 256;
      const int kr = f / (BN / 4), c4 = f % (BN / 4);
      *reinterpret_cast<float4*>(&Bs[buf][kr][c4 * 4]) = rb[i];
    }
  };

  if (it0 < it1) {
    gload(it0);
    sstore(0);
  }
  __syncthreads();
  for (int it = it0; it < it1; ++it) {
    const int buf = (it - it0) & 1;
    if (it + 1 < it1) gload(it + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[TM], b[TN];
#pragma unroll
      for (int i = 0; i < TM; i += 4) {
        const float4 t = *reinterpret_cast<const float4*>(&As[buf][k][(i / 4) * (BM / 2) + ty * 4]);
        a[i] = t.x; a[i + 1] = t.y; a[i + 2] = t.z; a[i + 3] = t.w;
      }
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const float4 t = *reinterpret_cast<const float4*>(&Bs[buf][k][(j / 4) * (BN / 2) + tx * 4]);
        b[j] = t.x; b[j + 1] = t.y; b[j + 2] = t.z; b[j + 3] = t.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (it + 1 < it1) sstore(buf ^ 1);
    __syncthreads();
  }

  // rows / cols owned by this thread: TM/4 groups of 4 rows at (g*BM/2 + ty*4), same for cols
  auto row_of = [&](int i) { return m0 + (i / 4) * (BM / 2) + ty * 4 + (i & 3); };
  auto col_of = [&](int j) { return n0 + (j / 4) * (BN / 2) + tx * 4 + (j & 3); };

  // ---- split-K combine (fixed order => deterministic)
  if (p.splitk > 1) {
    float* mine = p.partial + (size_t)blockIdx.z * p.M * p.N;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = row_of(i);
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const int n = col_of(j);
        if (n < p.N)
          *reinterpret_cast<float4*>(mine + (size_t)m * p.N + n) =
              make_float4(acc[i][j], acc[i][j + 1], acc[i][j + 2], acc[i][j + 3]);
      }
    }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      const unsigned int tile = blockIdx.y * gridDim.x + blockIdx.x;
      const unsigned int prev = atomicAdd(&p.counters[tile], 1u);
      s_last = (prev == (unsigned int)p.splitk - 1u);
      if (s_last) p.counters[tile] = 0u;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
    for (int z = 0; z < p.splitk; ++z) {
      const float* src = p.partial + (size_t)z * p.M * p.N;
#pragma unroll
      for (int i = 0; i < TM; ++i) {
        const int m = row_of(i);
        if (m >= p.M) continue;
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
          const int n = col_of(j);
          if (n < p.N) {
            const float4 t = __ldcg(reinterpret_cast<const float4*>(src + (size_t)m * p.N + n));
            acc[i][j] += t.x; acc[i][j + 1] += t.y; acc[i][j + 2] += t.z; acc[i][j + 3] += t.w;
          }
        }
      }
    }
  }

  // ---- epilogue
  if (p.epi == EPI_BIAS_ACT) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = row_of(i);
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const int n = col_of(j);
        if (n >= p.N) continue;
        float v[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          float t = acc[i][j + q] + p.bias_const;
          if (p.bias) t += __ldg(p.bias + n + q);
          if (p.aux) t += __ldg(p.aux + (size_t)m * p.ldaux + n + q);
          v[q] = apply_act(p.act, t);
        }
        float4* dst = (p.Y2 && n >= p.n_split) ? reinterpret_cast<float4*>(p.Y2 + (size_t)m * p.ldy + (n - p.n_split))
                                               : reinterpret_cast<float4*>(p.Y + (size_t)m * p.ldy + n);
        if (p.accumulate) {
          const float4 o = *dst;
          v[0] += o.x; v[1] += o.y; v[2] += o.z; v[3] += o.w;
        }
        *dst = make_float4(v[0], v[1], v[2], v[3]);
      }
    }
  } else if (p.epi == EPI_MUL_ELUGRAD) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = row_of(i);
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const int n = col_of(j);
        if (n >= p.N) continue;
        const float4 h = __ldg(reinterpret_cast<const float4*>(p.aux + (size_t)m * p.ldaux + n));
        *reinterpret_cast<float4*>(p.Y + (size_t)m * p.ldy + n) =
            make_float4(acc[i][j] * (h.x > 0.f ? 1.f : h.x + 1.f), acc[i][j + 1] * (h.y > 0.f ? 1.f : h.y + 1.f),
                        acc[i][j + 2] * (h.z > 0.f ? 1.f : h.z + 1.f), acc[i][j + 3] * (h.w > 0.f ? 1.f : h.w + 1.f));
      }
    }
  } else if (p.epi == EPI_ACCUM_DROPOUT) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = row_of(i);
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < TN; j += 4) {
        const int n = col_of(j);
        if (n >= p.N) continue;
        uint32_t bits[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
        if (p.e_thresh) {
          const uint64_t e = (uint64_t)m * (uint64_t)p.N + (uint64_t)n;
          const Philox4 r = philox4x32_10(p.seed, e >> 2, (uint32_t)p.e_site, (uint32_t)p.step);
          bits[0] = r.x; bits[1] = r.y; bits[2] = r.z; bits[3] = r.w;
        }
        float4* dst = reinterpret_cast<float4*>(p.Y + (size_t)m * p.ldy + n);
        float4 o = *dst;
        o.x += ((bits[0] >> 8) >= p.e_thresh) ? acc[i][j] * p.e_scale : 0.f;
        o.y += ((bits[1] >> 8) >= p.e_thresh) ? acc[i][j + 1] * p.e_scale : 0.f;
        o.z += ((bits[2] >> 8) >= p.e_thresh) ? acc[i][j + 2] * p.e_scale : 0.f;
        o.w += ((bits[3] >> 8) >= p.e_thresh) ? acc[i][j + 3] * p.e_scale : 0.f;
        *dst = o;
      }
    }
  } else if (p.epi == EPI_GATE) {
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = row_of(i);
      if (m >= p.M) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int n = col_of(j);
        if (n >= p.N) continue;
        float t = acc[i][j] + p.bias_const;
        if (p.bias) t += __ldg(p.bias + n);
        const float z = sigmoid_f(t);
        const size_t o = (size_t)m * p.ldy + n;
        if (p.gate_z) p.gate_z[o] = z;
        p.Y[o] = p.gnew[o] * z + p.gold[o] * (1.f - z);
      }
    }
  } else {  // EPI_READ_LOGITS
#pragma unroll
    for (int i = 0; i < TM; ++i) {
      const int m = row_of(i);
      float part = 0.f;
      if (m < p.M) {
        const float* c = p.ctrl + (size_t)(m / p.rows_per_batch) * p.N;
#pragma unroll
        for (int j = 0; j < TN; j += 4) {
          const int n = col_of(j);
          if (n >= p.N) continue;
          float i1[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) i1[q] = acc[i][j + q] + (p.bias ? __ldg(p.bias + n + q) : 0.f);
          if (p.Y) *reinterpret_cast<float4*>(p.Y + (size_t)m * p.ldy + n) = make_float4(i1[0], i1[1], i1[2], i1[3]);
          uint32_t bits[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
          if (p.e_thresh) {
            const uint64_t e = (uint64_t)m * (uint64_t)p.N + (uint64_t)n;
            const Philox4 r = philox4x32_10(p.seed, e >> 2, (uint32_t)p.e_site, (uint32_t)p.step);
            bits[0] = r.x; bits[1] = r.y; bits[2] = r.z; bits[3] = r.w;
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float t = elu_f(i1[q] * __ldg(c + n + q));
            t = ((bits[q] >> 8) >= p.e_thresh) ? t * p.e_scale : 0.f;
            part = fmaf(t, __ldg(p.wr + n + q), part);
          }
        }
      }
      // reduce over the 16 tx lanes that share this row (lanes of one warp: 2 ty x 16 tx)
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      if (tx == 0 && m < p.M) p.logit_parts[(size_t)m * gridDim.x + blockIdx.x] = part;
    }
  }
}

// host-side launch: picks the tile shape and a split-K factor that fills the SMs
inline size_t sgemm_workspace_bytes(int M, int N, int K) {
  // worst case: split so that each split has >= 2 k-iterations of 16; cap at 32 splits
  int splitk = K / 32;
  if (splitk > 32) splitk = 32;
  if (splitk < 1) splitk = 1;
  return (size_t)splitk * M * N * sizeof(float) + 256;
}

// 128x128 tiles only where they fill the machine: the batch-sized weight gradients (K = B = 64, M x N = 512 x 512 or
// 1024 x 512) get 16-32 tiles and at most 2 K slices out of them, 64x64 tiles give 64-128 tiles x 2 slices.
// (EPI_READ_LOGITS callers size their per-column-tile partial logits with sgemm_tile_n.)
inline bool sgemm_big_tiles(int M, int N, int K) {
  return (M >= 512) && (K >= 256 || ((M + 127) / 128) * ((N + 127) / 128) >= mac_num_sms());
}
inline int sgemm_tile_n(int M, int N, int K) { return sgemm_big_tiles(M, N, K) ? 128 : 64; }

inline bool skinny_ok(const SgemmParams& p);
inline int skinny_launch(const SgemmParams& p, cudaStream_t stream);

inline int sgemm_launch(SgemmParams p, unsigned int* counters, float* partial, size_t partial_bytes,
                        cudaStream_t stream, bool allow_splitk = true) {
  if (p.M <= 0 || p.N <= 0 || p.K <= 0) return MAC_ERR_INVALID;
  if ((p.N & 3) || ((p.K & 3) && p.a_mode < A_TRANS)) return MAC_ERR_INVALID;   // transposed views walk K row by row
  if (allow_splitk && skinny_ok(p) && !getenv("MAC_NO_SKINNY")) return skinny_launch(p, stream);   // M <= 64: cluster/DSMEM split-K kernel
  if (p.a_mode >= A_TRANS && (p.M & 3)) return MAC_ERR_INVALID;
  const bool big = sgemm_big_tiles(p.M, p.N, p.K);
  const int BM = big ? 128 : 64, BN = big ? 128 : 64;
  dim3 grid((p.N + BN - 1) / BN, (p.M + BM - 1) / BM, 1);
  if (p.epi == EPI_READ_LOGITS || counters == nullptr || partial == nullptr) allow_splitk = false;
  int splitk = 1;
  const int tiles = grid.x * grid.y;
  if (allow_splitk && tiles < mac_num_sms() && tiles <= 1024 && p.K >= 64) {
    splitk = (2 * mac_num_sms() + tiles - 1) / tiles;           // aim at ~2 CTAs per SM
    const int maxk = p.K / 32;                    // >= 2 k-iterations per split
    if (splitk > maxk) splitk = maxk;
    if (splitk > 32) splitk = 32;
    const int fit = (int)(partial_bytes / ((size_t)p.M * p.N * sizeof(float)));
    if (splitk > fit) splitk = fit;
    if (splitk < 1) splitk = 1;
  }
  p.splitk = splitk;
  p.partial = splitk > 1 ? partial : nullptr;
  p.counters = splitk > 1 ? counters : nullptr;
  grid.z = splitk;
  if (big)
    sgemm_kernel<128, 128><<<grid, 256, 0, stream>>>(p);
  else
    sgemm_kernel<64, 64><<<grid, 256, 0, stream>>>(p);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac
