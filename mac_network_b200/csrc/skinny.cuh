// Skinny fp32 GEMM for the latency-critical M <= 64 projections of the cell (projY, newMemory, gate, ctrlProj,
// qInput*: ops.linear at mac_cell.py:442-448, 322, 352, 363; ops.py:689):
//     Y[M<=64, N] = epilogue( Aview[M, K] @ W[K, N] )
// 33-100 MFLOP against 1-3 MB of weights: the problem is latency, not throughput.  Each CTA takes a 64 x 32 output
// tile and ONE K-slice (K / 8), loads its operands in a single round trip, multiplies from shared memory, and the 8
// CTAs of a thread-block cluster that share an output tile reduce their partial tiles over distributed shared
// memory (DSMEM) in a fixed order -- deterministic, one launch, no global scratch, no atomics.
#pragma once
#include <cooperative_groups.h>
#include "common.cuh"
#include "sgemm.cuh"

namespace mac {
namespace cg = cooperative_groups;

constexpr int SK_CLUSTER = 8;
constexpr int SK_BM = 64, SK_BN = 32, SK_THREADS = 128;

// pointer to four consecutive k of row m of the segmented A view (A_SEGS), or nullptr outside M
__device__ __forceinline__ const float* sk_ptr_a(const SgemmParams& p, int m, int k) {
  if (m >= p.M) return nullptr;
  int off = 0;
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    if (s < p.nseg) {
      if (k < off + p.ak[s]) return p.a[s] + (size_t)m * p.lda[s] + (k - off);
      off += p.ak[s];
    }
  }
  return nullptr;
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}

static __global__ void __launch_bounds__(SK_THREADS) skinny_gemm_kernel(const SgemmParams p, int ks) {
  extern __shared__ __align__(16) float sk_smem[];
  const int XP = ks + 4;                        // row pitch of the A slice (16-byte aligned rows)
  float* ws = sk_smem;                          // [ks][SK_BN]       W slice
  float* part = ws + (size_t)ks * SK_BN;        // [SK_BM][SK_BN]    this CTA's partial tile
  float* xs = part + SK_BM * SK_BN;             // [SK_BM][XP]       A slice, natural layout
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();   // K-slice index (cluster spans gridDim.x)
  const int tid = threadIdx.x;
  const int n0 = blockIdx.y * SK_BN;
  const int k0 = rank * ks;

  // ---- operand load: 16-byte cp.async (LDGSTS) straight into shared memory -- every request of the CTA is in flight
  //      at once, no register staging, one L2 round trip
  const int xc = ks / 4;
  for (int f = tid; f < SK_BM * xc; f += SK_THREADS) {
    const int row = f / xc, c = f % xc;
    const float* src = sk_ptr_a(p, row, k0 + c * 4);
    float* dst = xs + (size_t)row * XP + c * 4;
    if (src) cp_async16(dst, src);
    else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int f = tid; f < ks * (SK_BN / 4); f += SK_THREADS) {
    const int kr = f / (SK_BN / 4), c = f % (SK_BN / 4);
    const int n = n0 + c * 4;
    float* dst = ws + (size_t)kr * SK_BN + c * 4;
    if (n < p.N) cp_async16(dst, p.W + (size_t)(k0 + kr) * p.ldw + n);
    else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  // ---- 64 x 32 x ks product, 4 x 4 outputs per thread (2 LDS.128 per 16 FMAs: shared-memory bandwidth is the limit)
  const int rg = tid >> 3, cgp = tid & 7;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const float* xr = xs + (size_t)(rg * 4) * XP;
#pragma unroll 2
  for (int k = 0; k < ks; k += 4) {
    float4 a[4], w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = *reinterpret_cast<const float4*>(xr + (size_t)i * XP + k);
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) w[kk] = *reinterpret_cast<const float4*>(ws + (k + kk) * SK_BN + cgp * 4);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float av[4] = {a[i].x, a[i].y, a[i].z, a[i].w};
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        acc[i][0] = fmaf(av[kk], w[kk].x, acc[i][0]);
        acc[i][1] = fmaf(av[kk], w[kk].y, acc[i][1]);
        acc[i][2] = fmaf(av[kk], w[kk].z, acc[i][2]);
        acc[i][3] = fmaf(av[kk], w[kk].w, acc[i][3]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(part + (rg * 4 + i) * SK_BN + cgp * 4) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  cluster.sync();

  // ---- DSMEM reduction: CTA `rank` owns rows [8*rank, 8*rank+8) of the tile; fixed summation order
#pragma unroll
  for (int h = 0; h < (SK_BM / SK_CLUSTER) * SK_BN / SK_THREADS; ++h) {
    const int e = h * SK_THREADS + tid;
    const int rr = rank * (SK_BM / SK_CLUSTER) + e / SK_BN, c = e % SK_BN;
    float s = 0.f;
#pragma unroll
    for (int z = 0; z < SK_CLUSTER; ++z) s += cluster.map_shared_rank(part, z)[rr * SK_BN + c];
    const int m = rr, n = n0 + c;
    if (m < p.M && n < p.N) {
      float t = s + p.bias_const + (p.bias ? __ldg(p.bias + n) : 0.f);
      const size_t o = (size_t)m * p.ldy + n;
      if (p.epi == EPI_GATE) {
        const float z = sigmoid_f(t);
        if (p.gate_z) p.gate_z[o] = z;
        p.Y[o] = p.gnew[o] * z + p.gold[o] * (1.f - z);
      } else {
        t = apply_act(p.act, t);
        float* dst = (p.Y2 && n >= p.n_split) ? p.Y2 + (size_t)m * p.ldy + (n - p.n_split) : p.Y + o;
        *dst = p.accumulate ? *dst + t : t;
      }
    }
  }
  cluster.sync();      // keep every CTA's shared memory alive until all remote reads are done
}

// usable when M <= 64, K splits evenly into 8 slices of whole float4s, and the slice fits in shared memory
inline bool skinny_ok(const SgemmParams& p) {
  if (p.M > SK_BM || (p.epi != EPI_BIAS_ACT && p.epi != EPI_GATE) || p.a_mode != A_SEGS || p.aux) return false;
  if (p.K % (SK_CLUSTER * 4)) return false;
  const int ks = p.K / SK_CLUSTER;
  if (ks > 256) return false;
  return true;
}

inline int skinny_launch(const SgemmParams& p, cudaStream_t stream) {
  const int ks = p.K / SK_CLUSTER;
  const size_t smem = ((size_t)SK_BM * (ks + 4) + (size_t)ks * SK_BN + SK_BM * SK_BN) * sizeof(float);
  MAC_CUDA_TRY(cudaFuncSetAttribute(skinny_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(SK_CLUSTER, (p.N + SK_BN - 1) / SK_BN, 1);
  cfg.blockDim = dim3(SK_THREADS, 1, 1);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = SK_CLUSTER;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MAC_CUDA_TRY(cudaLaunchKernelEx(&cfg, skinny_gemm_kernel, p, ks));
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac
