// Layer-0 ingest of the image stem from channel-major features: [B, C, H, W] (fp32, bf16 or fp16, as the feature extractor or
// the feature file stored them) -> either the fp32 NHWC tensor Stem.forward takes, or directly the bf16 patch matrix of
// mac_im2col3x3 ([B*H*W, 9*C], tap-major, channel fastest, zero rows outside the image, no dropout), so that the bf16 stem never
// makes the NHWC copy.  The input is read from HBM once and the output written once.  The kernels are templates on the input
// element type IT; its one widening function ingest_f32 (exact for all three types) is the only place the type matters, so
// every input shares the slab copy, the transpose, the patch writes and the training mask.
//
// One CTA owns (sample, 64-channel slab).  The slab is one contiguous run of 64*H*W elements in NCHW, brought into shared
// memory by ONE 1-D bulk copy (cp.async.bulk + mbarrier; 16-byte aligned for any H*W because 64 elements are >= 128 bytes).
// A bulk copy cannot pad the rows it lands, and a channel-major slab read across channels at a fixed pixel strides by H*W
// words -- 196 at 14x14, four banks apart, an 8-way conflict for the 16-byte vectors the output wants.  So the slab is
// transposed inside shared memory first: lanes run along the pixels (conflict-free reads of the landed slab), each thread
// packs one 16-byte vector of consecutive channels and stores it to a pixel-major tile whose row stride is 64 channels + 16
// bytes (a quarter warp's eight 16-byte stores then cover all 32 banks).  The write-out reads that tile as 16-byte vectors
// (eight or sixteen consecutive lanes = one pixel's 128 or 256 contiguous bytes) and stores 128 contiguous bytes per pixel and
// tap (patch mode) or 256 per pixel (NHWC mode).
#pragma once
#include <cuda_fp16.h>
#include "common.cuh"
#include "tc_gemm.cuh"      // pack_bf16, pack_bf16_lo: the split-bf16 rounding of mac_im2col3x3_split

namespace mac {

constexpr int ING_CS = 64;          // channels per CTA
constexpr int ING_THREADS = 256;
constexpr size_t ING_STATIC_SMEM = 128;   // the mbarrier, padded to the dynamic tile's alignment (-Xptxas -v)

template <typename IT, bool PATCH>
struct IngestShape {
  static constexpr int OSZ = PATCH ? 2 : 4;                  // bytes per output element (bf16 patches / fp32 NHWC)
  static constexpr int V = 16 / OSZ;                         // channels per 16-byte vector
  static constexpr int G = ING_CS / V;                       // vectors per pixel
  static constexpr int TROW = ING_CS * OSZ + 16;             // padded row of the pixel-major tile, bytes
  __host__ __device__ static size_t in_bytes(int HW) { return (size_t)ING_CS * HW * sizeof(IT); }
  __host__ __device__ static size_t smem_bytes(int HW) { return in_bytes(HW) + (size_t)HW * TROW; }
};

// the widening of each input type to fp32: exact; for fp16 the conversion torch's Tensor.float() makes on the device, so a
// NaN keeps the payload it gets there
__device__ __forceinline__ float ingest_f32(float a) { return a; }
__device__ __forceinline__ float ingest_f32(__nv_bfloat16 a) { return __bfloat162float(a); }
__device__ __forceinline__ float ingest_f32(__half a) { return __half2float(a); }
// two channels of the bf16 patch matrix: the rounding of mac_im2col3x3(cols_bf16 = 1) of the widened values; bf16 in is a move
template <typename IT>
__device__ __forceinline__ uint32_t ingest_pair(IT a, IT b) {
  __nv_bfloat162 p = __floats2bfloat162_rn(ingest_f32(a), ingest_f32(b));
  return *reinterpret_cast<uint32_t*>(&p);
}
template <>
__device__ __forceinline__ uint32_t ingest_pair<__nv_bfloat16>(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

template <typename IT, bool PATCH>
__global__ void __launch_bounds__(ING_THREADS) ingest_nchw_kernel(const IT* __restrict__ x, void* __restrict__ out, int C,
                                                                  int H, int W) {
  using SH = IngestShape<IT, PATCH>;
  extern __shared__ __align__(128) unsigned char ing_smem[];
  __shared__ uint64_t bar;
  const int HW = H * W, tid = threadIdx.x, b = blockIdx.y, c0 = blockIdx.x * ING_CS;
  const IT* s_in = reinterpret_cast<const IT*>(ing_smem);                    // [64][HW] as it lies in NCHW
  unsigned char* s_t = ing_smem + SH::in_bytes(HW);                          // [HW][TROW bytes], pixel-major
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t bytes = (uint32_t)SH::in_bytes(HW);
    mbar_expect_tx(&bar, bytes);
    bulk_g2s(ing_smem, x + ((size_t)b * C + c0) * HW, bytes, &bar);
  }
  mbar_wait(&bar, 0);
  // transpose: one 16-byte vector of V consecutive channels per (vector g, pixel p); lanes along p
  for (int i = tid; i < SH::G * HW; i += ING_THREADS) {
    const int g = i / HW, p = i - g * HW;
    const IT* src = s_in + (size_t)(g * SH::V) * HW + p;
    uint4 q;
    if constexpr (PATCH) {
      q.x = ingest_pair(src[0], src[HW]);
      q.y = ingest_pair(src[2 * HW], src[3 * HW]);
      q.z = ingest_pair(src[4 * HW], src[5 * HW]);
      q.w = ingest_pair(src[6 * HW], src[7 * HW]);
    } else {
      q.x = __float_as_uint(ingest_f32(src[0]));
      q.y = __float_as_uint(ingest_f32(src[HW]));
      q.z = __float_as_uint(ingest_f32(src[2 * HW]));
      q.w = __float_as_uint(ingest_f32(src[3 * HW]));
    }
    *reinterpret_cast<uint4*>(s_t + (size_t)p * SH::TROW + g * 16) = q;
  }
  __syncthreads();
  if constexpr (PATCH) {
    // cols[(b,h,w), tap*C + c] = x[b, c, h + tap/3 - 1, w + tap%3 - 1], zero outside the image
    __nv_bfloat16* cols = reinterpret_cast<__nv_bfloat16*>(out);
    for (int i = tid; i < HW * 9 * SH::G; i += ING_THREADS) {
      const int g = i % SH::G, r = i / SH::G;
      const int tap = r % 9, pix = r / 9;
      const int h = pix / W, w = pix - h * W;
      const int hs = h + tap / 3 - 1, wsrc = w + tap % 3 - 1;
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W)
        v = *reinterpret_cast<const uint4*>(s_t + (size_t)(hs * W + wsrc) * SH::TROW + g * 16);
      *reinterpret_cast<uint4*>(cols + (((size_t)b * HW + pix) * 9 + tap) * C + c0 + g * SH::V) = v;
    }
  } else {
    float* y = reinterpret_cast<float*>(out);
    for (int i = tid; i < HW * SH::G; i += ING_THREADS) {
      const int g = i % SH::G, pix = i / SH::G;
      const uint4 v = *reinterpret_cast<const uint4*>(s_t + (size_t)pix * SH::TROW + g * 16);
      *reinterpret_cast<uint4*>(y + ((size_t)b * HW + pix) * C + c0 + g * SH::V) = v;
    }
  }
}

template <typename IT, bool PATCH>
static int ingest_nchw_launch(const void* x, void* out, int B, int C, int H, int W, cudaStream_t stream) {
  using SH = IngestShape<IT, PATCH>;
  const size_t smem = SH::smem_bytes(H * W);
  auto kern = ingest_nchw_kernel<IT, PATCH>;
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<dim3(C / ING_CS, B), ING_THREADS, smem, stream>>>(reinterpret_cast<const IT*>(x), out, C, H, W);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// shared memory one CTA needs; the entry point refuses shapes beyond one SM's 227 KB or the mbarrier's tx-count range
template <typename IT>
static inline size_t ingest_smem_bytes(int mode, int HW) {
  return mode ? IngestShape<IT, true>::smem_bytes(HW) : IngestShape<IT, false>::smem_bytes(HW);
}

// ------------------------------------------------------------------------------------------------ training ingest
// The training form of ingest_nchw_kernel: the same CTA (sample, 64-channel slab), the same one bulk copy, and two outputs
// from the one read -- the UNDROPPED fp32 NHWC tensor (the stem saves it as layer 0's input; the backward regenerates the
// mask from it) and layer 0's DROPPED-OUT patch matrix, bit for bit what mac_im2col3x3(cols_bf16 = 1) or
// mac_im2col3x3_split writes.  The mask is drawn once per source element while transposing, not once per tap: one
// philox4x32_10(seed, e >> 2, site, step) per (pixel, channel quad), e the NHWC flat index -- mac_im2col3x3's counter.
// Shared memory, per pixel: the slab (256 B fp32, 128 B fp16), the fp32 pixel-major tile (64 * 4 + 16 B) and the bf16 tile
// (64 * 2 + 16 B), and for the split form a second bf16 tile for the lo halves: 672 / 816 B for fp32 input (131.7 / 159.9 KB
// at 14x14), 544 / 688 B for fp16 (104.1 / 131.7 KB), one CTA per SM, so 512 threads keep more loads and stores in flight
// than ING_THREADS would.
constexpr int INGT_THREADS = 512;
constexpr int INGT_FROW = ING_CS * 4 + 16;     // fp32 tile row, bytes
constexpr int INGT_HROW = ING_CS * 2 + 16;     // bf16 tile row, bytes

template <typename IT, bool SPLIT>
struct IngestTrainShape {
  static constexpr int PIX = ING_CS * (int)sizeof(IT) + INGT_FROW + INGT_HROW * (SPLIT ? 2 : 1);     // shared bytes per pixel
  __host__ __device__ static size_t in_bytes(int HW) { return (size_t)ING_CS * HW * sizeof(IT); }
  __host__ __device__ static size_t smem_bytes(int HW) { return (size_t)HW * PIX; }
};

template <typename IT, bool SPLIT>
__global__ void __launch_bounds__(INGT_THREADS, 1) ingest_nchw_train_kernel(const IT* __restrict__ x,
                                                                            float* __restrict__ x_nhwc,
                                                                            __nv_bfloat16* __restrict__ cols, uint32_t thresh,
                                                                            float scale, uint64_t seed, int site, int step,
                                                                            int C, int H, int W) {
  extern __shared__ __align__(128) unsigned char ing_smem[];
  __shared__ uint64_t bar;
  const int HW = H * W, tid = threadIdx.x, b = blockIdx.y, c0 = blockIdx.x * ING_CS;
  using SH = IngestTrainShape<IT, SPLIT>;
  const IT* s_in = reinterpret_cast<const IT*>(ing_smem);                    // [64][HW] as it lies in NCHW
  unsigned char* s_f = ing_smem + SH::in_bytes(HW);                          // [HW][FROW], undropped fp32
  unsigned char* s_h = s_f + (size_t)HW * INGT_FROW;                         // [HW][HROW], bf16(dropped) or its hi half
  unsigned char* s_l = s_h + (size_t)HW * INGT_HROW;                         // [HW][HROW], the lo half (SPLIT)
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    const uint32_t bytes = (uint32_t)SH::in_bytes(HW);
    mbar_expect_tx(&bar, bytes);
    bulk_g2s(ing_smem, x + ((size_t)b * C + c0) * HW, bytes, &bar);
  }
  mbar_wait(&bar, 0);
  // transpose + mask: eight consecutive channels (two Philox quads) of one pixel per item; lanes along the pixels
  for (int i = tid; i < 8 * HW; i += INGT_THREADS) {
    const int g = i / HW, p = i - g * HW;
    const IT* src = s_in + (size_t)(g * 8) * HW + p;
    float v[8], d[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = d[j] = ingest_f32(src[j * HW]);
    if (thresh) {
      const uint64_t q = (((uint64_t)b * HW + p) * C + c0 + g * 8) >> 2;
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const Philox4 r = philox4x32_10(seed, q + k, (uint32_t)site, (uint32_t)step);
        // __fmul_rn: the product is rounded on its own, never contracted into the split form's lo subtraction
        d[4 * k + 0] = ((r.x >> 8) >= thresh) ? __fmul_rn(v[4 * k + 0], scale) : 0.f;
        d[4 * k + 1] = ((r.y >> 8) >= thresh) ? __fmul_rn(v[4 * k + 1], scale) : 0.f;
        d[4 * k + 2] = ((r.z >> 8) >= thresh) ? __fmul_rn(v[4 * k + 2], scale) : 0.f;
        d[4 * k + 3] = ((r.w >> 8) >= thresh) ? __fmul_rn(v[4 * k + 3], scale) : 0.f;
      }
    }
    float4* f = reinterpret_cast<float4*>(s_f + (size_t)p * INGT_FROW + g * 32);
    f[0] = make_float4(v[0], v[1], v[2], v[3]);
    f[1] = make_float4(v[4], v[5], v[6], v[7]);
    uint4 hi;
    hi.x = pack_bf16(d[0], d[1]); hi.y = pack_bf16(d[2], d[3]);
    hi.z = pack_bf16(d[4], d[5]); hi.w = pack_bf16(d[6], d[7]);
    *reinterpret_cast<uint4*>(s_h + (size_t)p * INGT_HROW + g * 16) = hi;
    if constexpr (SPLIT) {
      uint4 lo;
      lo.x = pack_bf16_lo(d[0], d[1], hi.x); lo.y = pack_bf16_lo(d[2], d[3], hi.y);
      lo.z = pack_bf16_lo(d[4], d[5], hi.z); lo.w = pack_bf16_lo(d[6], d[7], hi.w);
      *reinterpret_cast<uint4*>(s_l + (size_t)p * INGT_HROW + g * 16) = lo;
    }
  }
  __syncthreads();
  // NHWC: 256 contiguous bytes per pixel
  for (int i = tid; i < HW * 16; i += INGT_THREADS) {
    const int g = i & 15, pix = i >> 4;
    const uint4 v = *reinterpret_cast<const uint4*>(s_f + (size_t)pix * INGT_FROW + g * 16);
    *reinterpret_cast<uint4*>(x_nhwc + ((size_t)b * HW + pix) * C + c0 + g * 4) = v;
  }
  // patches: cols[(b,h,w), tap*C + c] (and, split, cols[(b,h,w), 9C + tap*C + c]); 128 contiguous bytes per pixel and tap
  constexpr int ROW = SPLIT ? 18 : 9;          // row length in units of C
  for (int i = tid; i < HW * 9 * 8; i += INGT_THREADS) {
    const int g = i & 7, r = i >> 3;
    const int tap = r % 9, pix = r / 9;
    const int h = pix / W, w = pix - h * W;
    const int hs = h + tap / 3 - 1, wsrc = w + tap % 3 - 1;
    uint4 hv = make_uint4(0u, 0u, 0u, 0u), lv = hv;
    if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W) {
      const size_t o = (size_t)(hs * W + wsrc) * INGT_HROW + g * 16;
      hv = *reinterpret_cast<const uint4*>(s_h + o);
      if constexpr (SPLIT) lv = *reinterpret_cast<const uint4*>(s_l + o);
    }
    __nv_bfloat16* row = cols + (((size_t)b * HW + pix) * ROW + tap) * C + c0 + g * 8;
    *reinterpret_cast<uint4*>(row) = hv;
    if constexpr (SPLIT) *reinterpret_cast<uint4*>(row + 9 * (size_t)C) = lv;
  }
}

template <typename IT, bool SPLIT>
static int ingest_nchw_train_launch(const void* x, float* x_nhwc, void* cols, uint32_t thresh, float scale, uint64_t seed,
                                    int site, int step, int B, int C, int H, int W, cudaStream_t stream) {
  const size_t smem = IngestTrainShape<IT, SPLIT>::smem_bytes(H * W);
  auto kern = ingest_nchw_train_kernel<IT, SPLIT>;
  MAC_CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<dim3(C / ING_CS, B), INGT_THREADS, smem, stream>>>(reinterpret_cast<const IT*>(x), x_nhwc, reinterpret_cast<__nv_bfloat16*>(cols), thresh, scale,
                                                            seed, site, step, C, H, W);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ knowledge-base gather
// Several questions about one image: the stem runs once per distinct image, kb_u [U, N*d] fp32, and each question's knowledge
// base is gathered from it, out[b] = kb_u[index[b]] (fp32, or bf16 rounded to nearest even as cast_bf16_kernel rounds).  A
// sample's N*d elements are contiguous in both, so the gather is a copy of B runs of N*d elements: blockIdx.x cuts a run
// into GATHER_V-element vectors (two 16-byte loads each), blockIdx.y (striding by gridDim.y past 65535) picks the sample.
// An index outside [0, U) writes a NaN row and reads nothing.
constexpr int GATHER_THREADS = 256;
constexpr int GATHER_V = 8;                 // elements per thread: 32 bytes read, 16 (bf16) or 32 (fp32) written

template <bool BF16>
__global__ void __launch_bounds__(GATHER_THREADS) kb_gather_kernel(const float4* __restrict__ kb_u,
                                                                   const int* __restrict__ index, void* __restrict__ out,
                                                                   int B, int U, int nvec) {
  const int j = blockIdx.x * GATHER_THREADS + threadIdx.x;          // vector within the sample's run
  if (j >= nvec) return;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const int u = __ldg(index + b);
    const size_t o = (size_t)b * nvec + j;
    float4 lo, hi;
    if (u >= 0 && u < U) {
      const float4* src = kb_u + ((size_t)u * nvec + j) * 2;
      lo = __ldg(src);
      hi = __ldg(src + 1);
    } else {
      lo = hi = make_float4(__int_as_float(0x7fc00000), __int_as_float(0x7fc00000), __int_as_float(0x7fc00000),
                            __int_as_float(0x7fc00000));
    }
    if constexpr (BF16) {
      __nv_bfloat162 p0 = __floats2bfloat162_rn(lo.x, lo.y), p1 = __floats2bfloat162_rn(lo.z, lo.w);
      __nv_bfloat162 p2 = __floats2bfloat162_rn(hi.x, hi.y), p3 = __floats2bfloat162_rn(hi.z, hi.w);
      uint4 v;
      v.x = *reinterpret_cast<uint32_t*>(&p0);
      v.y = *reinterpret_cast<uint32_t*>(&p1);
      v.z = *reinterpret_cast<uint32_t*>(&p2);
      v.w = *reinterpret_cast<uint32_t*>(&p3);
      reinterpret_cast<uint4*>(out)[o] = v;
    } else {
      float4* dst = reinterpret_cast<float4*>(out) + o * 2;
      dst[0] = lo;
      dst[1] = hi;
    }
  }
}

static int kb_gather_launch(const float* kb_u, const int* index, void* out, int out_bf16, int B, int U, int nvec,
                            cudaStream_t stream) {
  const dim3 grid((unsigned)((nvec + GATHER_THREADS - 1) / GATHER_THREADS), (unsigned)(B < 65535 ? B : 65535));
  const float4* src = reinterpret_cast<const float4*>(kb_u);
  if (out_bf16)
    kb_gather_kernel<true><<<grid, GATHER_THREADS, 0, stream>>>(src, index, out, B, U, nvec);
  else
    kb_gather_kernel<false><<<grid, GATHER_THREADS, 0, stream>>>(src, index, out, B, U, nvec);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ knowledge-base pool
// The device-resident cache of knowledge bases (serving.ModelPipeline(cache=C)): a pool of `capacity` rows of N*d elements,
// fp32 or bf16.  The insert writes the stem's output rows into it, pool[slot[u]] = kb_u[u] (bf16 rounded to nearest even as
// cast_bf16_kernel rounds); a slot outside [0, capacity) -- the stem's padding rows carry -1 -- writes nothing.  Same vectors
// and grid as the gather, with blockIdx.y picking the stem row u.  Two rows u with the same slot race: the caller's error.
template <bool BF16>
__global__ void __launch_bounds__(GATHER_THREADS) kb_pool_insert_kernel(const float4* __restrict__ kb_u,
                                                                        const int* __restrict__ slot, void* __restrict__ pool,
                                                                        int U, int capacity, int nvec) {
  const int j = blockIdx.x * GATHER_THREADS + threadIdx.x;          // vector within the sample's run
  if (j >= nvec) return;
  for (int u = blockIdx.y; u < U; u += gridDim.y) {
    const int r = __ldg(slot + u);
    if (r < 0 || r >= capacity) continue;
    const float4* src = kb_u + ((size_t)u * nvec + j) * 2;
    const float4 lo = __ldg(src), hi = __ldg(src + 1);
    const size_t o = (size_t)r * nvec + j;
    if constexpr (BF16) {
      __nv_bfloat162 p0 = __floats2bfloat162_rn(lo.x, lo.y), p1 = __floats2bfloat162_rn(lo.z, lo.w);
      __nv_bfloat162 p2 = __floats2bfloat162_rn(hi.x, hi.y), p3 = __floats2bfloat162_rn(hi.z, hi.w);
      uint4 v;
      v.x = *reinterpret_cast<uint32_t*>(&p0);
      v.y = *reinterpret_cast<uint32_t*>(&p1);
      v.z = *reinterpret_cast<uint32_t*>(&p2);
      v.w = *reinterpret_cast<uint32_t*>(&p3);
      reinterpret_cast<uint4*>(pool)[o] = v;
    } else {
      float4* dst = reinterpret_cast<float4*>(pool) + o * 2;
      dst[0] = lo;
      dst[1] = hi;
    }
  }
}

static int kb_pool_insert_launch(const float* kb_u, const int* slot, void* pool, int pool_bf16, int U, int capacity, int nvec,
                                 cudaStream_t stream) {
  const dim3 grid((unsigned)((nvec + GATHER_THREADS - 1) / GATHER_THREADS), (unsigned)(U < 65535 ? U : 65535));
  const float4* src = reinterpret_cast<const float4*>(kb_u);
  if (pool_bf16)
    kb_pool_insert_kernel<true><<<grid, GATHER_THREADS, 0, stream>>>(src, slot, pool, U, capacity, nvec);
  else
    kb_pool_insert_kernel<false><<<grid, GATHER_THREADS, 0, stream>>>(src, slot, pool, U, capacity, nvec);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// The gather from the bf16 pool: out[b] = kb_u[index[b]], bf16 to bf16, a copy.  One 16-byte vector (eight elements) per
// thread and question; an index outside [0, U) writes a row of bf16 quiet NaNs (0x7fc0) and reads nothing.
__global__ void __launch_bounds__(GATHER_THREADS) kb_gather_bf16_kernel(const uint4* __restrict__ kb_u,
                                                                        const int* __restrict__ index,
                                                                        uint4* __restrict__ out, int B, int U, int nvec) {
  const int j = blockIdx.x * GATHER_THREADS + threadIdx.x;          // vector within the sample's run
  if (j >= nvec) return;
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    const int u = __ldg(index + b);
    const uint4 v = (u >= 0 && u < U) ? __ldg(kb_u + (size_t)u * nvec + j)
                                      : make_uint4(0x7fc07fc0u, 0x7fc07fc0u, 0x7fc07fc0u, 0x7fc07fc0u);
    out[(size_t)b * nvec + j] = v;
  }
}

static int kb_gather_bf16_launch(const void* kb_u, const int* index, void* out, int B, int U, int nvec, cudaStream_t stream) {
  const dim3 grid((unsigned)((nvec + GATHER_THREADS - 1) / GATHER_THREADS), (unsigned)(B < 65535 ? B : 65535));
  kb_gather_bf16_kernel<<<grid, GATHER_THREADS, 0, stream>>>(reinterpret_cast<const uint4*>(kb_u), index,
                                                             reinterpret_cast<uint4*>(out), B, U, nvec);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ knowledge-base gather: backward
// The gradient of the gather: d_kb_u[u] = sum over b ascending with index[b] == u of d_out[b], in fp32, starting from the first
// matching row itself (a lone term is copied, -0.0 included) and adding the later ones in ascending b; an image no question
// uses gets zeros, an index outside [0, U) contributes nothing.  The order is fixed, so the result is that sequential float32
// sum bit for bit, with no atomics.  Same vectors as the gather: blockIdx.x cuts a sample's run of N*d elements into GATHER_V
// -element vectors, blockIdx.y (striding by gridDim.y past 65535) picks the image.  Every thread of a block scans the same
// index entries, staged through shared memory GATHER_BWD_CHUNK at a time (any B), so the branch on a match is uniform.  Each
// question row is read by the one block column of its image: B*N*d*4 bytes read, U*N*d*4 written.
constexpr int GATHER_BWD_CHUNK = 1024;

__global__ void __launch_bounds__(GATHER_THREADS) kb_gather_bwd_kernel(const float4* __restrict__ d_out,
                                                                       const int* __restrict__ index,
                                                                       float4* __restrict__ d_kb_u, int B, int U, int nvec) {
  __shared__ int s_idx[GATHER_BWD_CHUNK];
  const int j = blockIdx.x * GATHER_THREADS + threadIdx.x;          // vector within the sample's run
  const bool live = j < nvec;                                        // the others still stage the index
  for (int u = blockIdx.y; u < U; u += gridDim.y) {
    float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
    bool first = true;
    for (int b0 = 0; b0 < B; b0 += GATHER_BWD_CHUNK) {
      const int n = min(GATHER_BWD_CHUNK, B - b0);
      __syncthreads();                                               // the previous chunk has been scanned
      for (int i = threadIdx.x; i < n; i += GATHER_THREADS) s_idx[i] = __ldg(index + b0 + i);
      __syncthreads();
      if (!live) continue;
      for (int i = 0; i < n; ++i) {
        if (s_idx[i] != u) continue;
        const float4* src = d_out + ((size_t)(b0 + i) * nvec + j) * 2;
        const float4 a = __ldg(src), c = __ldg(src + 1);
        if (first) {
          lo = a;
          hi = c;
          first = false;
        } else {
          lo.x += a.x; lo.y += a.y; lo.z += a.z; lo.w += a.w;
          hi.x += c.x; hi.y += c.y; hi.z += c.z; hi.w += c.w;
        }
      }
    }
    if (live) {
      float4* dst = d_kb_u + ((size_t)u * nvec + j) * 2;
      dst[0] = lo;
      dst[1] = hi;
    }
  }
}

static int kb_gather_bwd_launch(const float* d_out, const int* index, float* d_kb_u, int B, int U, int nvec,
                                cudaStream_t stream) {
  const dim3 grid((unsigned)((nvec + GATHER_THREADS - 1) / GATHER_THREADS), (unsigned)(U < 65535 ? U : 65535));
  kb_gather_bwd_kernel<<<grid, GATHER_THREADS, 0, stream>>>(reinterpret_cast<const float4*>(d_out), index,
                                                            reinterpret_cast<float4*>(d_kb_u), B, U, nvec);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

}  // namespace mac
