// C-ABI entry points of the three MAC units (fp32 projection path) and the elementwise helpers.
#include "common.cuh"
#include "sgemm.cuh"
#include "skinny.cuh"
#include "tc_gemm.cuh"
#include "read_step.cuh"
#include "read_inv.cuh"
#include "read_step_fp8.cuh"
#include "tc_gemm_fp8.cuh"
#include "skinny_tc.cuh"
#include "encoder_tc.cuh"
#include "linear_tc.cuh"
#include "ingest.cuh"

using namespace mac;

namespace mac {
constexpr size_t WS_HEADER = 4096;   // split-K tile counters live here; zero on entry and on exit of every call

__global__ void bcast_mul_kernel(const float4* __restrict__ x, const float4* __restrict__ v, float mb,
                                 float4* __restrict__ out, long long total4, int N, int d4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const long long row = i / d4;
  const int k4 = (int)(i - row * d4);
  const float4 a = x[i];
  const float4 y = __ldg(v + (row / N) * d4 + k4);
  out[i] = make_float4((a.x + mb) * (y.x + mb), (a.y + mb) * (y.y + mb), (a.z + mb) * (y.z + mb), (a.w + mb) * (y.w + mb));
}

__global__ void activation_kernel(const float* __restrict__ x, int act, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = apply_act(act, x[i]);
}

__global__ void dropout_kernel(const float* __restrict__ x, uint32_t thresh, float scale, uint64_t seed, int site,
                               int step, float* __restrict__ out, float* __restrict__ u_out, long long n) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long base = i4 * 4;
  if (base >= n) return;
  const Philox4 r = philox4x32_10(seed, (uint64_t)i4, (uint32_t)site, (uint32_t)step);
  const uint32_t bits[4] = {r.x >> 8, r.y >> 8, r.z >> 8, r.w >> 8};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    if (base + q < n) {
      if (u_out) u_out[base + q] = (float)bits[q] * (1.0f / 16777216.0f);
      if (out) out[base + q] = (bits[q] >= thresh) ? x[base + q] * scale : 0.f;
    }
  }
}

__global__ void cast_bf16_kernel(const float4* __restrict__ x, uint2* __restrict__ out, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = x[i];
  __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
  uint2 o;
  o.x = *reinterpret_cast<uint32_t*>(&lo);
  o.y = *reinterpret_cast<uint32_t*>(&hi);
  out[i] = o;
}
}  // namespace mac

// ------------------------------------------------------------------------------------------------ misc
#include <atomic>
static std::atomic<long long> g_launches{0};
extern "C" void mac_b200_count_launch_(void) { g_launches.fetch_add(1, std::memory_order_relaxed); }
extern "C" long long mac_b200_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
extern "C" int mac_b200_abi_version(void) { return MAC_B200_ABI_VERSION; }

extern "C" const char* mac_b200_strerror(int status) {
  switch (status) {
    case MAC_OK: return "ok";
    case MAC_ERR_INVALID: return "invalid argument (size or null pointer)";
    case MAC_ERR_ALIGN: return "pointer or stride not 16-byte aligned";
    case MAC_ERR_UNSUPPORTED: return "flag/shape combination outside the fused path";
    case MAC_ERR_WORKSPACE: return "workspace too small";
    case MAC_ERR_ARCH: return "device is not sm_90 or the tensor-map driver entry point is missing";
    default: return status > 0 ? cudaGetErrorString((cudaError_t)status) : "unknown mac_b200 status";
  }
}

extern "C" int mac_b200_device_ok(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  int major = 0, minor = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return 0;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return 0;
  return major == 9 && minor == 0 ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ linear
extern "C" size_t mac_linear_workspace_bytes(int M, int K, int n_out) {
  return WS_HEADER + sgemm_workspace_bytes(M, n_out, K);
}

extern "C" int mac_linear_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* W,
                              const float* b, float bias_const, int act, float* y, int ldy, int M, int n_out,
                              void* workspace, size_t workspace_bytes, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !ldx || nseg < 1 || nseg > 4 || !W || !y || M <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  SgemmParams p{};
  p.a_mode = A_SEGS;
  p.nseg = nseg;
  int K = 0;
  for (int i = 0; i < nseg; ++i) {
    if (!x_segs[i] || k_segs[i] <= 0 || (k_segs[i] & 3) || (ldx[i] & 3)) return MAC_ERR_INVALID;
    if (!mac_aligned16(x_segs[i])) return MAC_ERR_ALIGN;
    p.a[i] = x_segs[i];
    p.ak[i] = k_segs[i];
    p.lda[i] = ldx[i];
    K += k_segs[i];
  }
  if (!mac_aligned16(W) || !mac_aligned16(y) || (ldy & 3) || (n_out & 3)) return MAC_ERR_ALIGN;
  p.W = W; p.ldw = n_out; p.M = M; p.N = n_out; p.K = K;
  p.epi = EPI_BIAS_ACT; p.bias = b; p.bias_const = bias_const; p.act = act; p.Y = y; p.ldy = ldy;
  char* ws = reinterpret_cast<char*>(workspace);
  const bool have_ws = ws != nullptr && workspace_bytes > WS_HEADER;
  return sgemm_launch(p, have_ws ? reinterpret_cast<unsigned int*>(ws) : nullptr,
                      have_ws ? reinterpret_cast<float*>(ws + WS_HEADER) : nullptr,
                      have_ws ? workspace_bytes - WS_HEADER : 0, stream);
}

// ------------------------------------------------------------------------------------------------ read unit
#include "read_fwd.cuh"

// ------------------------------------------------------------------------------------------------ write unit
extern "C" size_t mac_write_workspace_bytes(int B, int d) {
  return WS_HEADER + (size_t)B * d * 4 + 256 + sgemm_workspace_bytes(B, 2 * d, 3 * d);
}

// plain write unit + the next step's memory projection in one GEMM (inference; see mac_b200.h)
extern "C" int mac_write_fwd_next_y(const float* memory, const float* info, const float* Wf, const float* bf,
                                    float* new_memory, float* y_next, void* workspace, size_t workspace_bytes, int B,
                                    int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!memory || !info || !Wf || !new_memory || !y_next || !workspace || B <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  if (workspace_bytes < mac_write_workspace_bytes(B, d)) return MAC_ERR_WORKSPACE;
  char* ws = reinterpret_cast<char*>(workspace);
  const size_t o_sk = WS_HEADER + (((size_t)B * d * 4 + 255) & ~(size_t)255);
  SgemmParams p{};
  p.a_mode = A_SEGS; p.nseg = 2;
  p.a[0] = memory; p.ak[0] = d; p.lda[0] = d;
  p.a[1] = info; p.ak[1] = d; p.lda[1] = d;
  p.W = Wf; p.ldw = 2 * d; p.M = B; p.N = 2 * d; p.K = 2 * d;
  p.epi = EPI_BIAS_ACT; p.bias = bf; p.act = MAC_ACT_NON;
  p.Y = new_memory; p.ldy = d; p.Y2 = y_next; p.n_split = d;
  return sgemm_launch(p, reinterpret_cast<unsigned int*>(ws), reinterpret_cast<float*>(ws + o_sk),
                      workspace_bytes - o_sk, stream);
}

extern "C" int mac_write_fwd(const float* memory, const float* info, const float* self_smry, const float* control,
                             const float* Ww, const float* bw, const float* Wg, const float* bg, float gate_bias,
                             float* new_memory, float* gate_out, void* workspace, size_t workspace_bytes, int B, int d,
                             mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!memory || !info || !Ww || !new_memory || !workspace || B <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  if (Wg && !control) return MAC_ERR_INVALID;
  if (workspace_bytes < mac_write_workspace_bytes(B, d)) return MAC_ERR_WORKSPACE;
  char* ws = reinterpret_cast<char*>(workspace);
  float* tmp = reinterpret_cast<float*>(ws + WS_HEADER);
  const size_t o_sk = WS_HEADER + (((size_t)B * d * 4 + 255) & ~(size_t)255);
  // m' = [memory, info(, self_smry)] @ Ww + bw   (mac_cell.py:339-352), concat never materialised
  SgemmParams p{};
  p.a_mode = A_SEGS;
  p.a[0] = memory; p.ak[0] = d; p.lda[0] = d;
  p.a[1] = info; p.ak[1] = d; p.lda[1] = d;
  p.nseg = 2;
  if (self_smry) { p.a[2] = self_smry; p.ak[2] = d; p.lda[2] = d; p.nseg = 3; }
  p.W = Ww; p.ldw = d; p.M = B; p.N = d; p.K = p.nseg * d;
  p.epi = EPI_BIAS_ACT; p.bias = bw; p.act = MAC_ACT_NON;
  p.Y = Wg ? tmp : new_memory; p.ldy = d;
  {
    int st = sgemm_launch(p, reinterpret_cast<unsigned int*>(ws), reinterpret_cast<float*>(ws + o_sk),
                          workspace_bytes - o_sk, stream);
    if (st != MAC_OK) return st;
  }
  if (Wg) {
    // z = sigmoid(control @ Wg + bg + gate_bias); m' = m'*z + memory*(1-z)   (mac_cell.py:358-367)
    SgemmParams g{};
    g.a_mode = A_SEGS; g.nseg = 1; g.a[0] = control; g.ak[0] = d; g.lda[0] = d;
    g.W = Wg; g.ldw = d; g.M = B; g.N = d; g.K = d;
    g.epi = EPI_GATE; g.bias = bg; g.bias_const = gate_bias; g.Y = new_memory; g.ldy = d;
    g.gnew = tmp; g.gold = memory; g.gate_z = gate_out;
    int st = sgemm_launch(g, reinterpret_cast<unsigned int*>(ws), reinterpret_cast<float*>(ws + o_sk),
                          workspace_bytes - o_sk, stream);
    if (st != MAC_OK) return st;
  }
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ elementwise
extern "C" int mac_bcast_mul(const float* x, const float* v, float mul_bias, float* out, int B, int N, int d,
                             mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !v || !out || B <= 0 || N <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  if (!mac_aligned16(x) || !mac_aligned16(v) || !mac_aligned16(out)) return MAC_ERR_ALIGN;
  const long long total4 = (long long)B * N * d / 4;
  bcast_mul_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(v), mul_bias, reinterpret_cast<float4*>(out),
      total4, N, d / 4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_activation(const float* x, int act, float* out, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !out || n <= 0) return MAC_ERR_INVALID;
  activation_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(x, act, out, n);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_dropout_fwd(const float* x, float keep, uint64_t seed, int site, int step, float* out, long long n,
                               mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !out || n <= 0 || !(keep > 0.f && keep <= 1.f)) return MAC_ERR_INVALID;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  dropout_kernel<<<(unsigned)(((n + 3) / 4 + 255) / 256), 256, 0, stream>>>(x, thr, scale, seed, site, step, out,
                                                                            nullptr, n);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_dropout_uniform(uint64_t seed, int site, int step, float* u, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!u || n <= 0) return MAC_ERR_INVALID;
  dropout_kernel<<<(unsigned)(((n + 3) / 4 + 255) / 256), 256, 0, stream>>>(nullptr, 0u, 1.f, seed, site, step, nullptr,
                                                                            u, n);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_cast_bf16(const float* x, void* out_bf16, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !out_bf16 || n <= 0 || (n & 3)) return MAC_ERR_INVALID;
  if (!mac_aligned16(x) || (reinterpret_cast<uintptr_t>(out_bf16) & 7)) return MAC_ERR_ALIGN;
  cast_bf16_kernel<<<(unsigned)((n / 4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(x),
                                                                       reinterpret_cast<uint2*>(out_bf16), n / 4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ tensor-core helpers
extern "C" int mac_pack_weight_bf16(const float* W, void* Wt_bf16, int K, int N, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!W || !Wt_bf16 || K <= 0 || N <= 0) return MAC_ERR_INVALID;
  dim3 grid((N + 31) / 32, (K + 31) / 32), block(32, 8);
  pack_weight_bf16_kernel<<<grid, block, 0, stream>>>(W, reinterpret_cast<__nv_bfloat16*>(Wt_bf16), K, N);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_pack_weight_fp8(const float* W, void* Wt_e4m3, float* col_scale, int K, int N, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!W || !Wt_e4m3 || !col_scale || K <= 0 || N <= 0) return MAC_ERR_INVALID;
  pack_weight_fp8_kernel<<<(N + 31) / 32, dim3(32, 8), 0, stream>>>(W, reinterpret_cast<uint8_t*>(Wt_e4m3), col_scale, K, N);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// internal (not in the ABI header): split-K weight gradient for backward.cu, which does not include the tensor-core templates
extern "C" int mac_tc_wgrad_splitk_(const void* xT, const void* gT, float* dW, float* partial, int in_dim, int out_dim, int K,
                                    mac_stream_t stream_) {
  return tc_wgrad_splitk(xT, gT, dW, partial, in_dim, out_dim, K, reinterpret_cast<cudaStream_t>(stream_));
}
extern "C" size_t mac_tc_wgrad_partial_bytes_(int in_dim, int out_dim) { return tc_wgrad_partial_bytes(in_dim, out_dim); }

extern "C" int mac_pack_t_bf16_(int mode, const float* X, void* Xt, void* Xrm, int K, int N, const float* rowvec,
                                int rows_per_batch, uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                mac_stream_t stream_) {
  PackTArgs a;
  a.rowvec = rowvec; a.rows_per_batch = rows_per_batch; a.thresh = thresh; a.scale = scale; a.seed = seed; a.site = site;
  a.step = step;
  return pack_t_bf16_launch(mode, X, Xt, Xrm, K, N, a, reinterpret_cast<cudaStream_t>(stream_));
}

// internal: the split-bf16 ("tc32") pieces of mac_read_bwd_tc32 (backward.cu)
extern "C" int mac_pack_t_split_(int mode, const float* X, void* Xt, void* Xrm, int K, int N, int segs, const float* rowvec,
                                 int rows_per_batch, uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                 mac_stream_t stream_) {
  PackTArgs a;
  a.rowvec = rowvec; a.rows_per_batch = rows_per_batch; a.thresh = thresh; a.scale = scale; a.seed = seed; a.site = site;
  a.step = step;
  return pack_t_split_launch(mode, X, Xt, Xrm, K, N, segs, a, reinterpret_cast<cudaStream_t>(stream_));
}
extern "C" int mac_tc3_wgrad_splitk_(const void* xT2, const void* gT3, float* dW, float* partial, int in_dim, int out_dim,
                                     int kp, mac_stream_t stream_) {
  return tc3_wgrad_splitk(xT2, gT3, dW, partial, in_dim, out_dim, kp, reinterpret_cast<cudaStream_t>(stream_));
}
// W [R, C] fp32 -> [R, 3C] = [hi | hi | lo] per row (split3_rows_kernel)
extern "C" int mac_split3_rows_(const float* W, void* W3, int R, int C, mac_stream_t stream_) {
  if (!W || !W3 || R <= 0 || C <= 0 || (C & 3)) return MAC_ERR_INVALID;
  const long long n4 = (long long)R * C / 4;
  split3_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const float4*>(W), reinterpret_cast<uint2*>(W3), C, n4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}
// y[M, n_out] = A @ W with A' = [A_hi | A_lo] [M, 2K] and W' [n_out, 3K]: mac_linear_tc32_fwd without bias or activation
extern "C" int mac_tc3_linear_(const void* a_split, const void* wt3, float* y, int M, int K, int n_out, mac_stream_t stream_) {
  return mac_linear_tc32_fwd(a_split, wt3, nullptr, MAC_ACT_NON, y, M, K, n_out, stream_);
}

extern "C" int mac_linear_tc32_fwd(const void* a_split, const void* wt3, const float* b, int act, float* y, int M, int K,
                                   int n_out, mac_stream_t stream_) {
  if (!a_split || !wt3 || !y || M <= 0 || K <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  if ((K % TC_BK) || (n_out % TC_BN) || act < MAC_ACT_NON || act > MAC_ACT_RELU) return MAC_ERR_UNSUPPORTED;
  if ((M + TC_BM - 1) / TC_BM > 65535) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(a_split) || !mac_aligned16(wt3) || (reinterpret_cast<uintptr_t>(y) & 7)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  TcGemmParams p{};
  p.M = M; p.N = n_out; p.act = act; p.bias = b; p.ldo = n_out; p.rows_per_batch = 1;
  p.epi = TC_EPI_F32; p.outf = y;
  p.promote = 1;            // the stem's K = 9 C: two-level accumulation keeps the long contraction at fp32 accuracy
  return tc3_gemm(a_split, K, wt3, p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int mac_widen_bf16(const void* const* src_bf16, float* const* dst, int nslab, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src_bf16 || !dst || nslab < 1 || nslab > 3 || n <= 0 || (n & 7)) return MAC_ERR_INVALID;
  for (int i = 0; i < nslab; ++i) {
    if (!src_bf16[i] || !dst[i]) return MAC_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(src_bf16[i]) | reinterpret_cast<uintptr_t>(dst[i])) & 15) return MAC_ERR_ALIGN;
  }
  return widen3_bf16_launch(src_bf16, dst, nslab, n, stream);
}

extern "C" int mac_pack_weight_split3(const float* W, void* Wt3_bf16, int K, int N, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!W || !Wt3_bf16 || K <= 0 || N <= 0) return MAC_ERR_INVALID;
  dim3 grid((N + 31) / 32, (K + 31) / 32), block(32, 8);
  pack_weight_split3_kernel<<<grid, block, 0, stream>>>(W, reinterpret_cast<__nv_bfloat16*>(Wt3_bf16), K, N);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_linear_tc_fwd(const void* x_bf16, const void* wt_bf16, const float* b, int act, void* y, int y_is_bf16,
                                 int M, int K, int n_out, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_bf16 || !wt_bf16 || !y || M <= 0) return MAC_ERR_INVALID;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  TcGemmParams p{};
  p.M = M; p.N = n_out; p.act = act; p.bias = b; p.ldo = n_out; p.rows_per_batch = 1;
  if (y_is_bf16) {
    if (!b) return MAC_ERR_INVALID;
    p.epi = TC_EPI_ACT; p.out0 = reinterpret_cast<__nv_bfloat16*>(y);
  } else {
    p.epi = TC_EPI_F32; p.outf = reinterpret_cast<float*>(y);
  }
  return tc_gemm_launch(x_bf16, K, nullptr, 0, wt_bf16, p, stream);
}

// y = act(x @ W + y) in place (TC_EPI_F32_ADD): the second product of a sum of two GEMMs, the first written by
// mac_linear_tc_fwd / mac_linear_tc32_fwd with act NON and fp32 out
extern "C" int mac_linear_tc_fwd_acc(const void* x_bf16, const void* wt_bf16, int act, float* y, int M, int K, int n_out,
                                     mac_stream_t stream_) {
  if (!x_bf16 || !wt_bf16 || !y || M <= 0 || K <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  if ((K % TC_BK) || (n_out % TC_BN) || (act != MAC_ACT_NON && act != MAC_ACT_ELU && act != MAC_ACT_RELU))
    return MAC_ERR_UNSUPPORTED;
  if ((M + TC_BM - 1) / TC_BM > 65535) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(x_bf16) || !mac_aligned16(wt_bf16) || !mac_aligned16(y)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  TcGemmParams p{};
  p.M = M; p.N = n_out; p.act = act; p.ldo = n_out; p.rows_per_batch = 1;
  p.epi = TC_EPI_F32_ADD; p.outf = y; p.addf = y; p.ldaf = n_out;
  return tc_gemm_launch(x_bf16, K, nullptr, 0, wt_bf16, p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int mac_linear_tc32_fwd_acc(const void* a_split, const void* wt3, int act, float* y, int M, int K, int n_out,
                                       mac_stream_t stream_) {
  if (!a_split || !wt3 || !y || M <= 0 || K <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  if ((K % TC_BK) || (n_out % TC_BN) || (act != MAC_ACT_NON && act != MAC_ACT_ELU && act != MAC_ACT_RELU))
    return MAC_ERR_UNSUPPORTED;
  if ((M + TC_BM - 1) / TC_BM > 65535) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(a_split) || !mac_aligned16(wt3) || !mac_aligned16(y)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  TcGemmParams p{};
  p.M = M; p.N = n_out; p.act = act; p.ldo = n_out; p.rows_per_batch = 1;
  p.epi = TC_EPI_F32_ADD; p.outf = y; p.addf = y; p.ldaf = n_out;
  p.promote = 1;            // as mac_linear_tc32_fwd
  return tc3_gemm(a_split, K, wt3, p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int mac_pack_weight_bf16_split(const float* W, void* hi_bf16, void* lo_bf16, int K, int N, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!W || !hi_bf16 || !lo_bf16 || K <= 0 || N <= 0) return MAC_ERR_INVALID;
  dim3 grid((N + 31) / 32, (K + 31) / 32), block(32, 8);
  pack_weight_bf16_split_kernel<<<grid, block, 0, stream>>>(W, reinterpret_cast<__nv_bfloat16*>(hi_bf16),
                                                            reinterpret_cast<__nv_bfloat16*>(lo_bf16), K, N);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_linear_tc_small_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg,
                                       const void* wt_hi, const void* wt_lo, const float* b, float bias_const, int act,
                                       float* y, int ldy, float* y2, int n_split, const float* gate_new,
                                       const float* gate_old, float* gate_z, int M, int n_out, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !ldx || nseg < 1 || nseg > 4 || !wt_hi || !y || M <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  if ((gate_new != nullptr) != (gate_old != nullptr)) return MAC_ERR_INVALID;
  SkinnyTcParams p{};
  p.nseg = nseg;
  for (int i = 0; i < nseg; ++i) {
    p.a[i] = x_segs[i];
    p.ak[i] = k_segs[i];
    p.lda[i] = ldx[i];
    p.K += k_segs[i];
  }
  p.M = M; p.N = n_out; p.bias = b; p.bias_const = bias_const; p.act = act;
  p.Y = y; p.ldy = ldy; p.Y2 = y2; p.n_split = n_split;
  p.gnew = gate_new; p.gold = gate_old; p.gate_z = gate_z;
  const int st = skinny_tc_check(p, wt_hi, wt_lo);
  if (st != MAC_OK) return st;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  return skinny_tc_launch(p, wt_hi, wt_lo, stream);
}

// ------------------------------------------------------------------------------------------------ general (unfused) path
// Primitives that let the host compose the cell for flag combinations outside the fused read/write kernels
// (SURVEY.md section 8(a) "P2": controlConcatWords/Proj, read*AttType in {BL, ADD}, readCtrlConcatKB, readSmryKBProj,
// writeInputs in {MEM, INFO, SUM}, ...).  Not performance-tuned; same arithmetic order as the reference ops.
namespace mac {
// out[r] = sum over segments of x_s[r,:] . w[koff_s:...] + b      (ops.linear with outDim == 1, ops.py:316-317)
__global__ void __launch_bounds__(256) rowdot_kernel(const float* x0, const float* x1, const float* x2, int k0, int k1,
                                                    int k2, int ld0, int ld1, int ld2, const float* __restrict__ w,
                                                    float b, float* __restrict__ out, long long R) {
  const long long r = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  float acc = 0.f;
  for (int k = lane; k < k0; k += 32) acc = fmaf(x0[r * ld0 + k], __ldg(w + k), acc);
  if (x1) for (int k = lane; k < k1; k += 32) acc = fmaf(x1[r * ld1 + k], __ldg(w + k0 + k), acc);
  if (x2) for (int k = lane; k < k2; k += 32) acc = fmaf(x2[r * ld2 + k], __ldg(w + k0 + k1 + k), acc);
  acc = warp_sum(acc);
  if (lane == 0) out[r] = acc + b;
}

// att[b,:] = softmax(logits[b,:] - 1e30*[m >= len[b]]);  out[b,:] = sum_m att[b,m] * feats[b,m,:]
// grid (ceil(d/128), B), 128 threads; feats row (b,m) at feats + b*bstride + m*rstride
__global__ void __launch_bounds__(128) attend_kernel(const float* __restrict__ logits, const int32_t* __restrict__ lengths,
                                                    const float* __restrict__ feats, long long bstride, long long rstride,
                                                    float* __restrict__ att, float* __restrict__ out, int M, int d) {
  extern __shared__ float s_a[];
  __shared__ float s_red[4];
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int len = lengths ? min(max(lengths[b], 0), M) : M;
  float mx = -INFINITY;
  for (int m = tid; m < M; m += 128) {
    const float l = logits[(size_t)b * M + m] + (m < len ? 0.f : -1e30f);
    s_a[m] = l;
    mx = fmaxf(mx, l);
  }
  mx = warp_max(mx);
  if (lane == 0) s_red[warp] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(s_red[0], s_red[1]), fmaxf(s_red[2], s_red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int m = tid; m < M; m += 128) {
    const float e = expf(s_a[m] - mx);
    s_a[m] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) s_red[warp] = sum;
  __syncthreads();
  const float inv = 1.f / (s_red[0] + s_red[1] + s_red[2] + s_red[3]);
  for (int m = tid; m < M; m += 128) {
    const float a = s_a[m] * inv;
    s_a[m] = a;
    if (blockIdx.x == 0) att[(size_t)b * M + m] = a;
  }
  __syncthreads();
  const int k = blockIdx.x * 128 + tid;
  if (k < d) {
    const float* f = feats + (size_t)b * bstride + k;
    float acc = 0.f;
    for (int m = 0; m < M; ++m) acc = fmaf(s_a[m], f[(size_t)m * rstride], acc);
    out[(size_t)b * d + k] = acc;
  }
}

// ops.mul interaction modes on a broadcast operand (ops.py:694-713): mode 0 MUL (x+mb)*(v+mb); 1 BL x*v + bias[k];
// 2 ADD tanh(x+v)
__global__ void bcast_op_kernel(const float* __restrict__ x, const float* __restrict__ v, int mode, float mb,
                                const float* __restrict__ bias, float* __restrict__ out, long long total, int N, int d) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long row = i / d;
  const int k = (int)(i - row * d);
  const float a = x[i], y = v[(row / N) * d + k];
  out[i] = mode == 0 ? (a + mb) * (y + mb) : mode == 1 ? a * y + (bias ? bias[k] : 0.f) : tanhf(a + y);
}
}  // namespace mac

extern "C" int mac_rowdot_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* w,
                              float b, float* out, long long R, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !ldx || nseg < 1 || nseg > 3 || !w || !out || R <= 0) return MAC_ERR_INVALID;
  const float* x[3] = {nullptr, nullptr, nullptr};
  int k[3] = {0, 0, 0}, ld[3] = {0, 0, 0};
  for (int i = 0; i < nseg; ++i) { x[i] = x_segs[i]; k[i] = k_segs[i]; ld[i] = ldx[i]; }
  rowdot_kernel<<<(unsigned)((R + 7) / 8), 256, 0, stream>>>(x[0], x[1], x[2], k[0], k[1], k[2], ld[0], ld[1], ld[2], w, b,
                                                            out, R);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_attend_fwd(const float* logits, const int32_t* lengths, const float* feats, long long feat_bstride,
                              long long feat_rstride, float* att, float* out, int B, int M, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!logits || !feats || !att || !out || B <= 0 || M <= 0 || d <= 0) return MAC_ERR_INVALID;
  if ((size_t)M * 4 > 160 * 1024) return MAC_ERR_UNSUPPORTED;
  MAC_CUDA_TRY(cudaFuncSetAttribute(attend_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, M * 4 + 16));
  attend_kernel<<<dim3((d + 127) / 128, B), 128, (size_t)M * 4 + 16, stream>>>(logits, lengths, feats, feat_bstride,
                                                                             feat_rstride, att, out, M, d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_bcast_op(const float* x, const float* v, int mode, float mul_bias, const float* bias, float* out,
                            int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !v || !out || B <= 0 || N <= 0 || d <= 0 || mode < 0 || mode > 2) return MAC_ERR_INVALID;
  const long long total = (long long)B * N * d;
  bcast_op_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, v, mode, mul_bias, bias, out, total, N, d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ answer loss
// losses[b] = logsumexp(logits[b,:]) - logits[b, label[b]]   (tf.nn.sparse_softmax_cross_entropy_with_logits, model.py:595)
// dlogits[b,:] = (softmax(logits[b,:]) - onehot(label[b])) * scale       one warp per row
namespace mac {
__global__ void __launch_bounds__(256) softmax_xent_kernel(const float* __restrict__ logits, const int32_t* __restrict__ labels,
                                                          float* __restrict__ losses, float* __restrict__ dlogits,
                                                          float scale, int B, int A) {
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const float* row = logits + (size_t)b * A;
  float mx = -INFINITY;
  for (int a = lane; a < A; a += 32) mx = fmaxf(mx, row[a]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int a = lane; a < A; a += 32) sum += expf(row[a] - mx);
  sum = warp_sum(sum);
  const int lab = labels[b];
  const bool lab_ok = lab >= 0 && lab < A;       // an out-of-range label must not read outside the row: NaN loss, no one-hot
  if (lane == 0) losses[b] = lab_ok ? mx + logf(sum) - row[lab] : __int_as_float(0x7fc00000);
  const float inv = 1.f / sum;
  for (int a = lane; a < A; a += 32) dlogits[(size_t)b * A + a] = (expf(row[a] - mx) * inv - (a == lab ? 1.f : 0.f)) * scale;
}
}  // namespace mac

extern "C" int mac_softmax_xent(const float* logits, const int32_t* labels, float* losses, float* dlogits, float scale,
                                int B, int A, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!logits || !labels || !losses || !dlogits || B <= 0 || A <= 0) return MAC_ERR_INVALID;
  softmax_xent_kernel<<<(B + 7) / 8, 256, 0, stream>>>(logits, labels, losses, dlogits, scale, B, A);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ answers without labels
// Per row: softmax probabilities (max-subtracted, fp32) and the k largest logits with their answer ids, ties to the lower id
// (torch.argmax / tf.argmax order, model.py:603-612).  One warp per row; round r picks the largest element that sorts after
// round r-1's pick in (logit descending, id ascending) order, so nothing is marked and the row is only read.
namespace mac {
__global__ void __launch_bounds__(256) answer_topk_kernel(const float* __restrict__ logits, int B, int A, int k,
                                                         int32_t* __restrict__ ids, float* __restrict__ probs) {
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  const float* row = logits + (size_t)b * A;
  float mx = -INFINITY;
  for (int a = lane; a < A; a += 32) mx = fmaxf(mx, row[a]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int a = lane; a < A; a += 32) sum += expf(row[a] - mx);
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
  float pv = INFINITY;
  int pi = -1;
  for (int r = 0; r < k; ++r) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;                                     // no candidate yet (a row of NaNs never finds one: id -1)
    for (int a = lane; a < A; a += 32) {
      const float v = row[a];
      const bool after_prev = v < pv || (v == pv && a > pi);
      if (after_prev && (bi == 0x7fffffff || v > bv)) { bv = v; bi = a; }      // ascending a: the first of equals stays
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != 0x7fffffff && (bi == 0x7fffffff || ov > bv || (ov == bv && oi < bi))) { bv = ov; bi = oi; }
    }
    if (lane == 0) {
      ids[(size_t)b * k + r] = bi == 0x7fffffff ? -1 : bi;
      probs[(size_t)b * k + r] = bi == 0x7fffffff ? __int_as_float(0x7fc00000) : expf(bv - mx) * inv;
    }
    pv = bv;
    pi = bi;
  }
}
}  // namespace mac

extern "C" int mac_answer_topk(const float* logits, int B, int A, int k, int32_t* ids, float* probs, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!logits || !ids || !probs || B <= 0 || A <= 0) return MAC_ERR_INVALID;
  if (k < 1 || k > 8 || k > A) return MAC_ERR_INVALID;
  answer_topk_kernel<<<(B + 7) / 8, 256, 0, stream>>>(logits, B, A, k, ids, probs);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ stem: im2col
// cols[(b,h,w), (kh*3+kw)*C + c] = dropout(x)[b, h+kh-1, w+kw-1, c]  (zero outside the image: SAME padding, ops.py:395)
// The keep-mask is a function of the SOURCE element's flat index, so every copy of a pixel carries the same mask
// (tf.nn.dropout is applied to the layer input before the convolution, ops.py:393).
namespace mac {
template <typename OT>
__global__ void im2col3x3_kernel(const float* __restrict__ x, OT* __restrict__ cols, uint32_t thresh, float scale,
                                 uint64_t seed, int site, int step, int B, int H, int W, int C) {
  const int c4n = C / 4;
  const long long total = (long long)B * H * W * 9 * c4n;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c4 = (int)(i % c4n);
  long long r = i / c4n;
  const int tap = (int)(r % 9);
  r /= 9;
  const int w = (int)(r % W);
  r /= W;
  const int h = (int)(r % H), b = (int)(r / H);
  const int hs = h + tap / 3 - 1, wsrc = w + tap % 3 - 1;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W) {
    const long long e = (((long long)b * H + hs) * W + wsrc) * C + c4 * 4;
    v = __ldg(reinterpret_cast<const float4*>(x + e));
    if (thresh) {
      const Philox4 p = philox4x32_10(seed, (uint64_t)e >> 2, (uint32_t)site, (uint32_t)step);
      v.x = ((p.x >> 8) >= thresh) ? v.x * scale : 0.f;
      v.y = ((p.y >> 8) >= thresh) ? v.y * scale : 0.f;
      v.z = ((p.z >> 8) >= thresh) ? v.z * scale : 0.f;
      v.w = ((p.w >> 8) >= thresh) ? v.w * scale : 0.f;
    }
  }
  const long long o = ((((long long)b * H + h) * W + w) * 9 + tap) * C + c4 * 4;
  if constexpr (sizeof(OT) == 2) {
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 q;
    q.x = *reinterpret_cast<uint32_t*>(&lo);
    q.y = *reinterpret_cast<uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(cols + o) = q;
  } else {
    *reinterpret_cast<float4*>(cols + o) = v;
  }
}
}  // namespace mac

extern "C" int mac_im2col3x3(const float* x, void* cols, int cols_bf16, float keep, uint64_t seed, int site, int step,
                             int B, int H, int W, int C, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !cols || B <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 3) || !(keep > 0.f && keep <= 1.f)) return MAC_ERR_INVALID;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const long long total = (long long)B * H * W * 9 * (C / 4);
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (cols_bf16)
    im2col3x3_kernel<__nv_bfloat16><<<grid, 256, 0, stream>>>(x, reinterpret_cast<__nv_bfloat16*>(cols), thr, scale, seed,
                                                             site, step, B, H, W, C);
  else
    im2col3x3_kernel<float><<<grid, 256, 0, stream>>>(x, reinterpret_cast<float*>(cols), thr, scale, seed, site, step, B, H,
                                                     W, C);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ stem: ingest from NCHW
// The checks and the launch of one input type: every refusal precedes any CUDA call.
template <typename IT>
static int ingest_nchw_checked(const void* x_nchw, void* out, int mode, int B, int C, int H, int W, cudaStream_t stream) {
  if (!x_nchw || !out || B <= 0 || C <= 0 || H <= 0 || W <= 0) return MAC_ERR_INVALID;
  if (!mac_aligned16(x_nchw) || !mac_aligned16(out)) return MAC_ERR_ALIGN;
  if ((C % ING_CS) || (mode != MAC_INGEST_NHWC_F32 && mode != MAC_INGEST_PATCH_BF16)) return MAC_ERR_UNSUPPORTED;
  // one slab, its transposed tile and the kernel's static shared memory in one SM's 227 KB, the slab inside the mbarrier's
  // tx-count range; gridDim.y
  if ((long long)H * W > 4096 || ingest_smem_bytes<IT>(mode, H * W) + ING_STATIC_SMEM > 227 * 1024 || B > 65535)
    return MAC_ERR_UNSUPPORTED;
  return mode == MAC_INGEST_PATCH_BF16 ? ingest_nchw_launch<IT, true>(x_nchw, out, B, C, H, W, stream)
                                       : ingest_nchw_launch<IT, false>(x_nchw, out, B, C, H, W, stream);
}

extern "C" int mac_ingest_nchw(const void* x_nchw, int x_bf16, void* out, int mode, int B, int C, int H, int W,
                               mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  return x_bf16 ? ingest_nchw_checked<__nv_bfloat16>(x_nchw, out, mode, B, C, H, W, stream)
                : ingest_nchw_checked<float>(x_nchw, out, mode, B, C, H, W, stream);
}

extern "C" int mac_ingest_nchw_f16(const void* x_f16, void* out, int mode, int B, int C, int H, int W, mac_stream_t stream_) {
  return ingest_nchw_checked<__half>(x_f16, out, mode, B, C, H, W, reinterpret_cast<cudaStream_t>(stream_));
}

template <typename IT>
static int ingest_nchw_train_checked(const void* x_nchw, float* x_nhwc, void* cols, int cols_form, float keep, uint64_t seed,
                                     int site, int step, int B, int C, int H, int W, cudaStream_t stream) {
  if (!x_nchw || !x_nhwc || !cols || B <= 0 || C <= 0 || H <= 0 || W <= 0 || !(keep > 0.f && keep <= 1.f))
    return MAC_ERR_INVALID;
  if (!mac_aligned16(x_nchw) || !mac_aligned16(x_nhwc) || !mac_aligned16(cols)) return MAC_ERR_ALIGN;
  if ((C % ING_CS) || (cols_form != MAC_INGEST_COLS_BF16 && cols_form != MAC_INGEST_COLS_SPLIT) || B > 65535)
    return MAC_ERR_UNSUPPORTED;
  // the slab and its tiles with the kernel's static shared memory in one SM's 227 KB (H*W <= 345 / 284 for fp32 input,
  // 427 / 337 for fp16)
  const bool split = cols_form == MAC_INGEST_COLS_SPLIT;
  if ((long long)H * W > 4096 ||
      (split ? IngestTrainShape<IT, true>::smem_bytes(H * W) : IngestTrainShape<IT, false>::smem_bytes(H * W)) +
              ING_STATIC_SMEM > 227 * 1024)
    return MAC_ERR_UNSUPPORTED;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  return split ? ingest_nchw_train_launch<IT, true>(x_nchw, x_nhwc, cols, thr, scale, seed, site, step, B, C, H, W, stream)
               : ingest_nchw_train_launch<IT, false>(x_nchw, x_nhwc, cols, thr, scale, seed, site, step, B, C, H, W, stream);
}

extern "C" int mac_ingest_nchw_train(const float* x_nchw, float* x_nhwc, void* cols, int cols_form, float keep, uint64_t seed,
                                     int site, int step, int B, int C, int H, int W, mac_stream_t stream_) {
  return ingest_nchw_train_checked<float>(x_nchw, x_nhwc, cols, cols_form, keep, seed, site, step, B, C, H, W,
                                          reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int mac_ingest_nchw_train_f16(const void* x_f16, float* x_nhwc, void* cols, int cols_form, float keep,
                                         uint64_t seed, int site, int step, int B, int C, int H, int W, mac_stream_t stream_) {
  return ingest_nchw_train_checked<__half>(x_f16, x_nhwc, cols, cols_form, keep, seed, site, step, B, C, H, W,
                                           reinterpret_cast<cudaStream_t>(stream_));
}

// ------------------------------------------------------------------------------------------------ knowledge-base gather
extern "C" int mac_kb_gather(const float* kb_u, const int* index, void* out, int out_bf16, int B, int U, int N, int d,
                             mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!kb_u || !index || !out || B <= 0 || U <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  // one sample's run of N*d elements in GATHER_V-element vectors, counted in an int
  if ((out_bf16 != 0 && out_bf16 != 1) || (d % GATHER_V) || (long long)N * d / GATHER_V > 0x7fffffffLL)
    return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(kb_u) || !mac_aligned16(index) || !mac_aligned16(out)) return MAC_ERR_ALIGN;
  return kb_gather_launch(kb_u, index, out, out_bf16, B, U, (int)((long long)N * d / GATHER_V), stream);
}

extern "C" int mac_kb_pool_insert(const float* kb_u, const int* slot, void* pool, int pool_bf16, int U, int capacity, int N,
                                  int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!kb_u || !slot || !pool || U <= 0 || capacity <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  if ((pool_bf16 != 0 && pool_bf16 != 1) || (d % GATHER_V) || (long long)N * d / GATHER_V > 0x7fffffffLL)
    return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(kb_u) || !mac_aligned16(slot) || !mac_aligned16(pool)) return MAC_ERR_ALIGN;
  return kb_pool_insert_launch(kb_u, slot, pool, pool_bf16, U, capacity, (int)((long long)N * d / GATHER_V), stream);
}

extern "C" int mac_kb_gather_bf16(const void* kb_u, const int* index, void* out, int B, int U, int N, int d,
                                  mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!kb_u || !index || !out || B <= 0 || U <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  if ((d % GATHER_V) || (long long)N * d / GATHER_V > 0x7fffffffLL) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(kb_u) || !mac_aligned16(index) || !mac_aligned16(out)) return MAC_ERR_ALIGN;
  return kb_gather_bf16_launch(kb_u, index, out, B, U, (int)((long long)N * d / GATHER_V), stream);
}

extern "C" int mac_kb_gather_bwd(const float* d_out, const int* index, float* d_kb_u, int B, int U, int N, int d,
                                 mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!d_out || !index || !d_kb_u || B <= 0 || U <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  if ((d % GATHER_V) || (long long)N * d / GATHER_V > 0x7fffffffLL) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(d_out) || !mac_aligned16(index) || !mac_aligned16(d_kb_u)) return MAC_ERR_ALIGN;
  return kb_gather_bwd_launch(d_out, index, d_kb_u, B, U, (int)((long long)N * d / GATHER_V), stream);
}

// ------------------------------------------------------------------------------------------------ stem: split-bf16 patches
// The patch matrix of mac_im2col3x3 as the A operand of tc3_gemm: cols2[m, k] = bf16(v), cols2[m, 9C + k] = bf16(v - hi) with
// v the fp32 value mac_im2col3x3 writes at cols[m, k] (same Philox draw: the quad index of the SOURCE element).  Eight
// channels per thread: two 16-byte loads, one 16-byte store per half.
namespace mac {
__global__ void __launch_bounds__(256) im2col3x3_split_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ cols2,
                                                             uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                                             int B, int H, int W, int C) {
  const int c8n = C / 8;
  const long long total = (long long)B * H * W * 9 * c8n;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % c8n);
  long long r = i / c8n;
  const int tap = (int)(r % 9);
  const long long m = r / 9;
  const int w = (int)(m % W);
  r = m / W;
  const int h = (int)(r % H), b = (int)(r / H);
  const int hs = h + tap / 3 - 1, wsrc = w + tap % 3 - 1;
  float4 v[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W) {
    const long long e = (((long long)b * H + hs) * W + wsrc) * C + c8 * 8;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      v[q] = __ldg(reinterpret_cast<const float4*>(x + e) + q);
      if (thresh) {
        const Philox4 p = philox4x32_10(seed, ((uint64_t)e >> 2) + q, (uint32_t)site, (uint32_t)step);
        v[q].x = ((p.x >> 8) >= thresh) ? v[q].x * scale : 0.f;
        v[q].y = ((p.y >> 8) >= thresh) ? v[q].y * scale : 0.f;
        v[q].z = ((p.z >> 8) >= thresh) ? v[q].z * scale : 0.f;
        v[q].w = ((p.w >> 8) >= thresh) ? v[q].w * scale : 0.f;
      }
    }
  }
  uint4 hi, lo;
  hi.x = pack_bf16(v[0].x, v[0].y); hi.y = pack_bf16(v[0].z, v[0].w);
  hi.z = pack_bf16(v[1].x, v[1].y); hi.w = pack_bf16(v[1].z, v[1].w);
  lo.x = pack_bf16_lo(v[0].x, v[0].y, hi.x); lo.y = pack_bf16_lo(v[0].z, v[0].w, hi.y);
  lo.z = pack_bf16_lo(v[1].x, v[1].y, hi.z); lo.w = pack_bf16_lo(v[1].z, v[1].w, hi.w);
  __nv_bfloat16* row = cols2 + (m * 18 + tap) * C + c8 * 8;
  *reinterpret_cast<uint4*>(row) = hi;
  *reinterpret_cast<uint4*>(row + 9 * C) = lo;
}
}  // namespace mac

extern "C" int mac_im2col3x3_split(const float* x, void* cols2, float keep, uint64_t seed, int site, int step, int B, int H,
                                   int W, int C, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !cols2 || B <= 0 || H <= 0 || W <= 0 || C <= 0 || !(keep > 0.f && keep <= 1.f)) return MAC_ERR_INVALID;
  if ((long long)B * H * W > (1LL << 30)) return MAC_ERR_INVALID;
  if (C % TC_BK) return MAC_ERR_UNSUPPORTED;                 // 9C = whole k-blocks of mac_linear_tc32_fwd
  if (!mac_aligned16(x) || !mac_aligned16(cols2)) return MAC_ERR_ALIGN;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const long long total = (long long)B * H * W * 9 * (C / 8);
  im2col3x3_split_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(x, reinterpret_cast<__nv_bfloat16*>(cols2), thr,
                                                                             scale, seed, site, step, B, H, W, C);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ stem: e4m3 inference
// (tc_gemm_fp8.cuh)
extern "C" size_t mac_im2col3x3_fp8_workspace_bytes(int B, int H, int W, int C) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0) return 0;
  return im2col3x3_fp8_workspace_bytes((long long)B * H * W);
}

extern "C" int mac_im2col3x3_fp8(const float* x, void* cols_e4m3, float* row_scale, void* workspace, size_t workspace_bytes,
                                 int B, int H, int W, int C, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !cols_e4m3 || !row_scale || !workspace) return MAC_ERR_INVALID;
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || (long long)B * H * W > (1LL << 30)) return MAC_ERR_INVALID;
  if (C % 128) return MAC_ERR_UNSUPPORTED;                  // 9C = whole 128-byte k-blocks of mac_linear_fp8_fwd
  if (!mac_aligned16(x) || !mac_aligned16(cols_e4m3) || !mac_aligned16(workspace)) return MAC_ERR_ALIGN;
  if (workspace_bytes < mac_im2col3x3_fp8_workspace_bytes(B, H, W, C)) return MAC_ERR_WORKSPACE;
  return im2col3x3_fp8_launch(x, cols_e4m3, row_scale, workspace, B, H, W, C, stream);
}

extern "C" int mac_linear_fp8_fwd(const void* x_e4m3, const float* x_scale, const void* wt_e4m3, const float* w_scale,
                                  const float* b, int act, float* y, int M, int K, int n_out, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_e4m3 || !x_scale || !wt_e4m3 || !w_scale || !y || M <= 0 || K <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  if ((K % F8_BK) || (n_out % TC_BN) || !linear_fp8_act_supported(act)) return MAC_ERR_UNSUPPORTED;
  if ((M + TC_BM - 1) / TC_BM > 65535) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(x_e4m3) || !mac_aligned16(wt_e4m3) || !mac_aligned16(w_scale) || !mac_aligned16(y)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  return linear_fp8_launch(x_e4m3, x_scale, wt_e4m3, w_scale, b, act, y, M, K, n_out, stream);
}

// ------------------------------------------------------------------------------------------------ stem: col2im (backward)
// dx[b,h,w,c] = keep-mask(b,h,w,c)/keep * sum_{kh,kw} dcols[(b, h-kh+1, w-kw+1), (kh*3+kw)*C + c]   (taps whose output
// position falls outside the image contribute nothing).  Gather form: each thread owns four channels of one input pixel and
// adds its <= 9 copies in a fixed order, so the gradient is deterministic and needs no atomics.
namespace mac {
__global__ void col2im3x3_kernel(const float* __restrict__ dcols, float* __restrict__ dx, uint32_t thresh, float scale,
                                 uint64_t seed, int site, int step, int B, int H, int W, int C) {
  const int c4n = C / 4;
  const long long total = (long long)B * H * W * c4n;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c4 = (int)(i % c4n);
  long long r = i / c4n;
  const int w = (int)(r % W);
  r /= W;
  const int h = (int)(r % H), b = (int)(r / H);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const int ho = h - (tap / 3 - 1), wo = w - (tap % 3 - 1);      // the output pixel whose tap `tap` read (h, w)
    if (ho >= 0 && ho < H && wo >= 0 && wo < W) {
      const long long o = ((((long long)b * H + ho) * W + wo) * 9 + tap) * C + c4 * 4;
      const float4 v = __ldg(reinterpret_cast<const float4*>(dcols + o));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  const long long e = (((long long)b * H + h) * W + w) * C + c4 * 4;
  if (thresh) {
    const Philox4 p = philox4x32_10(seed, (uint64_t)e >> 2, (uint32_t)site, (uint32_t)step);
    acc.x = ((p.x >> 8) >= thresh) ? acc.x * scale : 0.f;
    acc.y = ((p.y >> 8) >= thresh) ? acc.y * scale : 0.f;
    acc.z = ((p.z >> 8) >= thresh) ? acc.z * scale : 0.f;
    acc.w = ((p.w >> 8) >= thresh) ? acc.w * scale : 0.f;
  }
  *reinterpret_cast<float4*>(dx + e) = acc;
}
}  // namespace mac

extern "C" int mac_col2im3x3(const float* dcols, float* dx, float keep, uint64_t seed, int site, int step, int B, int H,
                             int W, int C, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dcols || !dx || B <= 0 || H <= 0 || W <= 0 || C <= 0 || (C & 3) || !(keep > 0.f && keep <= 1.f)) return MAC_ERR_INVALID;
  if (!mac_aligned16(dcols) || !mac_aligned16(dx)) return MAC_ERR_ALIGN;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const long long total = (long long)B * H * W * (C / 4);
  col2im3x3_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dcols, dx, thr, scale, seed, site, step, B, H, W, C);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ stem: any k x k, stride s
// tf.nn.conv2d's SAME geometry (ops.py:397): Ho = ceil(H / s), pad_total = max((Ho - 1) s + k - H, 0), pad_top =
// pad_total / 2 (the odd row goes to the bottom), and the same for the width.  Output pixel (ho, wo) reads input
// (ho s - pad_top + kh, wo s - pad_left + kw) for tap kh k + kw.  At k = 3, s = 1 this is the 3x3 kernels' geometry; those
// stay (they are fused with the NCHW ingest), and these serve every other layer.
namespace mac {
struct ConvGeom {
  int B, H, W, C, k, s, Ho, Wo, pt, pl;
};
inline ConvGeom conv_geom(int B, int H, int W, int C, int k, int s) {
  ConvGeom g{B, H, W, C, k, s, (H + s - 1) / s, (W + s - 1) / s, 0, 0};
  g.pt = std::max((g.Ho - 1) * s + k - H, 0) / 2;
  g.pl = std::max((g.Wo - 1) * s + k - W, 0) / 2;
  return g;
}
constexpr int CONV_MAX_K = 16, CONV_MAX_S = 16;

// The refusals every general stem entry point shares, before any launch: sizes, k, s, keep, and the 2^30-row bound.
inline int conv_geom_check(int B, int H, int W, int C, int k, int s, float keep) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || k <= 0 || s <= 0 || !(keep > 0.f && keep <= 1.f)) return MAC_ERR_INVALID;
  if (k > CONV_MAX_K || s > CONV_MAX_S) return MAC_ERR_UNSUPPORTED;
  const ConvGeom g = conv_geom(B, H, W, C, k, s);
  if ((long long)B * H * W > (1LL << 30) || (long long)B * g.Ho * g.Wo > (1LL << 30)) return MAC_ERR_INVALID;
  return MAC_OK;
}

__device__ __forceinline__ void dropout_quad(float4& v, uint64_t seed, long long e, int site, int step, uint32_t thresh,
                                             float scale) {
  const Philox4 p = philox4x32_10(seed, (uint64_t)e >> 2, (uint32_t)site, (uint32_t)step);
  v.x = ((p.x >> 8) >= thresh) ? v.x * scale : 0.f;
  v.y = ((p.y >> 8) >= thresh) ? v.y * scale : 0.f;
  v.z = ((p.z >> 8) >= thresh) ? v.z * scale : 0.f;
  v.w = ((p.w >> 8) >= thresh) ? v.w * scale : 0.f;
}

// cols[m, tap C + c] (FORM fp32 / bf16) or cols[m, [hi | lo]] (FORM split, each k^2 C wide) of the dropped-out input; the
// Philox draw is the SOURCE element's quad, so every copy of a pixel shares its mask and a pixel no tap reads is never drawn.
// V channels per thread: one 16-byte store per thread and half (V = 4 fp32, V = 8 bf16 and split; V = 4 bf16 when C % 8).
template <int V, int FORM>
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, void* __restrict__ cols_, uint32_t thresh,
                                                     float scale, uint64_t seed, int site, int step, ConvGeom g) {
  const int cvn = g.C / V, taps = g.k * g.k;
  const long long total = (long long)g.B * g.Ho * g.Wo * taps * cvn;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int cv = (int)(i % cvn);
  long long r = i / cvn;
  const int tap = (int)(r % taps);
  const long long m = r / taps;
  const int wo = (int)(m % g.Wo);
  r = m / g.Wo;
  const int ho = (int)(r % g.Ho), b = (int)(r / g.Ho);
  const int hs = ho * g.s - g.pt + tap / g.k, wsrc = wo * g.s - g.pl + tap % g.k;
  float4 v[V / 4];
#pragma unroll
  for (int q = 0; q < V / 4; ++q) v[q] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (hs >= 0 && hs < g.H && wsrc >= 0 && wsrc < g.W) {
    const long long e = (((long long)b * g.H + hs) * g.W + wsrc) * g.C + cv * V;
#pragma unroll
    for (int q = 0; q < V / 4; ++q) {
      v[q] = __ldg(reinterpret_cast<const float4*>(x + e) + q);
      if (thresh) dropout_quad(v[q], seed, e + 4 * q, site, step, thresh, scale);
    }
  }
  const long long K = (long long)taps * g.C;
  if constexpr (FORM == 0) {
    *reinterpret_cast<float4*>(reinterpret_cast<float*>(cols_) + m * K + (long long)tap * g.C + cv * V) = v[0];
  } else if constexpr (FORM == 1) {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(cols_) + m * K + (long long)tap * g.C + cv * V;
    if constexpr (V == 8) {
      *reinterpret_cast<uint4*>(o) = make_uint4(pack_bf16(v[0].x, v[0].y), pack_bf16(v[0].z, v[0].w),
                                                pack_bf16(v[1].x, v[1].y), pack_bf16(v[1].z, v[1].w));
    } else {
      *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16(v[0].x, v[0].y), pack_bf16(v[0].z, v[0].w));
    }
  } else {
    uint4 hi, lo;
    hi.x = pack_bf16(v[0].x, v[0].y); hi.y = pack_bf16(v[0].z, v[0].w);
    hi.z = pack_bf16(v[1].x, v[1].y); hi.w = pack_bf16(v[1].z, v[1].w);
    lo.x = pack_bf16_lo(v[0].x, v[0].y, hi.x); lo.y = pack_bf16_lo(v[0].z, v[0].w, hi.y);
    lo.z = pack_bf16_lo(v[1].x, v[1].y, hi.z); lo.w = pack_bf16_lo(v[1].z, v[1].w, hi.w);
    __nv_bfloat16* row = reinterpret_cast<__nv_bfloat16*>(cols_) + m * 2 * K + (long long)tap * g.C + cv * V;
    *reinterpret_cast<uint4*>(row) = hi;
    *reinterpret_cast<uint4*>(row + K) = lo;
  }
}

// dx[b,h,w,c] = keep-mask/keep * sum over taps (kh, kw) ascending of dcols[(b, ho, wo), tap C + c] for every output pixel
// (ho, wo) whose tap read (h, w).  Gather per input pixel in a fixed order: deterministic, no atomics.
__global__ void __launch_bounds__(256) col2im_kernel(const float* __restrict__ dcols, float* __restrict__ dx, uint32_t thresh,
                                                     float scale, uint64_t seed, int site, int step, ConvGeom g) {
  const int c4n = g.C / 4;
  const long long total = (long long)g.B * g.H * g.W * c4n;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c4 = (int)(i % c4n);
  long long r = i / c4n;
  const int w = (int)(r % g.W);
  r /= g.W;
  const int h = (int)(r % g.H), b = (int)(r / g.H);
  const long long K = (long long)g.k * g.k * g.C;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int kh = 0; kh < g.k; ++kh) {
    const int th = h + g.pt - kh;                               // = ho * s for the output row that read (h, w) with this kh
    if (th < 0 || th % g.s || th / g.s >= g.Ho) continue;
    for (int kw = 0; kw < g.k; ++kw) {
      const int tw = w + g.pl - kw;
      if (tw < 0 || tw % g.s || tw / g.s >= g.Wo) continue;
      const long long o = (((long long)b * g.Ho + th / g.s) * g.Wo + tw / g.s) * K + (long long)(kh * g.k + kw) * g.C + c4 * 4;
      const float4 v = __ldg(reinterpret_cast<const float4*>(dcols + o));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  }
  const long long e = (((long long)b * g.H + h) * g.W + w) * g.C + c4 * 4;
  if (thresh) dropout_quad(acc, seed, e, site, step, thresh, scale);
  *reinterpret_cast<float4*>(dx + e) = acc;
}
}  // namespace mac

extern "C" int mac_im2col(const float* x, void* cols, int form, float keep, uint64_t seed, int site, int step, int B, int H,
                          int W, int C, int k, int s, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !cols) return MAC_ERR_INVALID;
  const int st = conv_geom_check(B, H, W, C, k, s, keep);
  if (st != MAC_OK) return st;
  if (form != MAC_COLS_F32 && form != MAC_COLS_BF16 && form != MAC_COLS_SPLIT) return MAC_ERR_UNSUPPORTED;
  if (C % 4 || (form == MAC_COLS_SPLIT && C % TC_BK)) return MAC_ERR_UNSUPPORTED;   // float4 reads; split: whole k-blocks
  if (!mac_aligned16(x) || !mac_aligned16(cols)) return MAC_ERR_ALIGN;
  const ConvGeom g = conv_geom(B, H, W, C, k, s);
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const int V = form == MAC_COLS_F32 || (form == MAC_COLS_BF16 && C % 8) ? 4 : 8;
  const long long total = (long long)B * g.Ho * g.Wo * k * k * (C / V);
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (form == MAC_COLS_F32)
    im2col_kernel<4, 0><<<grid, 256, 0, stream>>>(x, cols, thr, scale, seed, site, step, g);
  else if (form == MAC_COLS_SPLIT)
    im2col_kernel<8, 2><<<grid, 256, 0, stream>>>(x, cols, thr, scale, seed, site, step, g);
  else if (V == 8)
    im2col_kernel<8, 1><<<grid, 256, 0, stream>>>(x, cols, thr, scale, seed, site, step, g);
  else
    im2col_kernel<4, 1><<<grid, 256, 0, stream>>>(x, cols, thr, scale, seed, site, step, g);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_col2im(const float* dcols, float* dx, float keep, uint64_t seed, int site, int step, int B, int H, int W,
                          int C, int k, int s, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dcols || !dx) return MAC_ERR_INVALID;
  const int st = conv_geom_check(B, H, W, C, k, s, keep);
  if (st != MAC_OK) return st;
  if (C % 4) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(dcols) || !mac_aligned16(dx)) return MAC_ERR_ALIGN;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const long long total = (long long)B * H * W * (C / 4);
  col2im_kernel<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(dcols, dx, thr, scale, seed, site, step,
                                                                      conv_geom(B, H, W, C, k, s));
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ stem: location features
// --locationAware (ops.py:448-559, mod CNCT): layer 0 reads concat(x, g) with the constant grid g [H, W, l].  Its patch matrix
// splits into the image patches P (mac_im2col / mac_im2col3x3, unchanged) and the location patches Q [M, Kq], tap-major and
// channel fastest as P, Kq = k^2 l rounded up to 128 (one wgmma tile of tc_wgrad_splitk), the columns k^2 l..Kq-1 zero.  The
// dropout of the location channels is a Philox stream of its own (site): the draw of Q[m, tap l + j] is component e & 3
// of philox4x32_10(seed, e >> 2, site, step) with e = ((b H + hs) W + ws) l + j the NHWC flat index of the [B, H, W, l]
// location tensor at the source pixel (hs, ws), so every tap copy of an element shares its draw.
namespace mac {
inline int loc_width(int l, int k) { return (k * k * l + 127) / 128 * 128; }

__device__ __forceinline__ float loc_value(const float* __restrict__ grid, const ConvGeom& g, int Kl, long long m, int col,
                                           uint32_t thresh, float scale, uint64_t seed, int site, int step) {
  if (m >= (long long)g.B * g.Ho * g.Wo || col >= Kl) return 0.f;
  const int tap = col / g.C, j = col - tap * g.C;
  const int wo = (int)(m % g.Wo);
  const long long r = m / g.Wo;
  const int ho = (int)(r % g.Ho), b = (int)(r / g.Ho);
  const int hs = ho * g.s - g.pt + tap / g.k, ws = wo * g.s - g.pl + tap % g.k;
  if (hs < 0 || hs >= g.H || ws < 0 || ws >= g.W) return 0.f;
  float v = __ldg(grid + ((long long)hs * g.W + ws) * g.C + j);
  if (thresh) {
    const long long e = (((long long)b * g.H + hs) * g.W + ws) * g.C + j;
    const Philox4 p = philox4x32_10(seed, (uint64_t)e >> 2, (uint32_t)site, (uint32_t)step);
    const uint32_t u = (e & 3) == 0 ? p.x : (e & 3) == 1 ? p.y : (e & 3) == 2 ? p.z : p.w;
    v = (u >> 8) >= thresh ? v * scale : 0.f;
  }
  return v;
}

// One element per thread (Q is small: k^2 l columns against the image's k^2 C).  TRANS = false: Q [M, Kq] in fp32 (FORM 0),
// bf16 (1) or [hi | lo] [M, 2 Kq] (2).  TRANS = true: Q^T [Kq, Mp] (FORM 1) or [Kq, 2 Mp] = [hi | lo] (FORM 2), the weight
// gradient's operand, zero in columns M..Mp-1.  g.C is l.
template <int FORM, bool TRANS>
__global__ void __launch_bounds__(256) loc_cols_kernel(const float* __restrict__ grid, void* __restrict__ out, uint32_t thresh,
                                                       float scale, uint64_t seed, int site, int step, ConvGeom g, int Kq,
                                                       int Mp) {
  const long long rows = TRANS ? (long long)Kq : (long long)g.B * g.Ho * g.Wo, cols = TRANS ? (long long)Mp : (long long)Kq;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const long long r = i / cols, c = i - r * cols;
  const long long m = TRANS ? c : r;
  const int col = (int)(TRANS ? r : c);
  const float v = loc_value(grid, g, g.k * g.k * g.C, m, col, thresh, scale, seed, site, step);
  if constexpr (FORM == 0) {
    reinterpret_cast<float*>(out)[i] = v;
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(out);
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    if constexpr (FORM == 1) {
      o[i] = hi;
    } else {
      const long long at = r * 2 * cols + c;
      o[at] = hi;
      o[at + cols] = __float2bfloat16_rn(v - __bfloat162float(hi));
    }
  }
}

// The refusals of every location entry point after its own pointer checks: l, B, H, W, k, s, keep and the row bounds.
inline int loc_check(int B, int H, int W, int l, int k, int s, float keep) {
  if (l <= 0) return MAC_ERR_INVALID;
  const int st = conv_geom_check(B, H, W, l, k, s, keep);
  if (st != MAC_OK) return st;
  if (l > 65536) return MAC_ERR_UNSUPPORTED;
  const ConvGeom g = conv_geom(B, H, W, l, k, s);
  const long long Mp = ((long long)B * g.Ho * g.Wo + 63) & ~63LL;
  if (Mp * loc_width(l, k) >= (1LL << 39)) return MAC_ERR_UNSUPPORTED;     // one thread per element, 256 per block
  return MAC_OK;
}

inline void loc_cols_launch(const float* grid, void* out, int form, bool trans, float keep, uint64_t seed, int site, int step,
                            const ConvGeom& g, cudaStream_t stream) {
  const int Kq = loc_width(g.C, g.k);
  const long long M = (long long)g.B * g.Ho * g.Wo;
  const int Mp = (int)((M + 63) & ~63LL);
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const long long n = (trans ? (long long)Mp : M) * Kq;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (trans && form == MAC_COLS_SPLIT)
    loc_cols_kernel<2, true><<<blocks, 256, 0, stream>>>(grid, out, thr, scale, seed, site, step, g, Kq, Mp);
  else if (trans)
    loc_cols_kernel<1, true><<<blocks, 256, 0, stream>>>(grid, out, thr, scale, seed, site, step, g, Kq, Mp);
  else if (form == MAC_COLS_F32)
    loc_cols_kernel<0, false><<<blocks, 256, 0, stream>>>(grid, out, thr, scale, seed, site, step, g, Kq, Mp);
  else if (form == MAC_COLS_BF16)
    loc_cols_kernel<1, false><<<blocks, 256, 0, stream>>>(grid, out, thr, scale, seed, site, step, g, Kq, Mp);
  else
    loc_cols_kernel<2, false><<<blocks, 256, 0, stream>>>(grid, out, thr, scale, seed, site, step, g, Kq, Mp);
}
}  // namespace mac

extern "C" int mac_loc_cols_width(int l, int k) { return l <= 0 || k <= 0 || k > CONV_MAX_K ? 0 : loc_width(l, k); }

extern "C" int mac_loc_cols(const float* grid, void* cols, int form, float keep, uint64_t seed, int site, int step, int B, int H,
                            int W, int l, int k, int s, mac_stream_t stream_) {
  if (!grid || !cols) return MAC_ERR_INVALID;
  const int st = loc_check(B, H, W, l, k, s, keep);
  if (st != MAC_OK) return st;
  if (form != MAC_COLS_F32 && form != MAC_COLS_BF16 && form != MAC_COLS_SPLIT) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(grid) || !mac_aligned16(cols)) return MAC_ERR_ALIGN;
  loc_cols_launch(grid, cols, form, false, keep, seed, site, step, conv_geom(B, H, W, l, k, s),
                  reinterpret_cast<cudaStream_t>(stream_));
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_loc_cols_t(const float* grid, void* colsT, int split, float keep, uint64_t seed, int site, int step, int B,
                              int H, int W, int l, int k, int s, mac_stream_t stream_) {
  if (!grid || !colsT) return MAC_ERR_INVALID;
  const int st = loc_check(B, H, W, l, k, s, keep);
  if (st != MAC_OK) return st;
  if (split != 0 && split != 1) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(grid) || !mac_aligned16(colsT)) return MAC_ERR_ALIGN;
  loc_cols_launch(grid, colsT, split ? MAC_COLS_SPLIT : MAC_COLS_BF16, true, keep, seed, site, step,
                  conv_geom(B, H, W, l, k, s), reinterpret_cast<cudaStream_t>(stream_));
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ stem: backward on wgmma
// One 3x3 convolution layer's backward with its two GEMMs on tensor cores (fp32 accumulation, fp32 element-wise work),
// M = B*H*W rows, Mp = M rounded up to the 64-row k-block of the weight gradient.  mac_conv3x3_bwd_tc (bf16 operands):
//   dZ = dy * act'(y)                      -> bf16 dZ [M, Cout] (dgrad A operand), bf16 dZ^T [Cout, Mp], fp32 column partials
//   colsT = bf16(dropout(x)) patches^T     -> [9C, Mp], the forward's keep-mask (mac_im2col3x3's Philox numbering)
//   dKernel [9C, Cout] += colsT @ dZ       (tc_wgrad_splitk, K = Mp; the HWIO kernel viewed as [9C, Cout] is its output)
//   dBias += column sums of dZ             (fixed order: per-64-row-tile partials, then mac_colsum)
//   dcols [M, 9C] = dZ @ Kernel^T          (mac_linear_tc_fwd with bf16(Kernel) in its own [9C, Cout] layout as the
//                                           K-major B operand);  dx = col2im(dcols) * mask / keep   (mac_col2im3x3)
// mac_conv3x3_bwd_tc32 (SPLIT: split-bf16 operands, see tc3_gemm) is the same schedule on hi | lo operands:
//   dZ -> [dZ_hi | dZ_lo] [M, 2 Cout] (only when dx is wanted) and [dZ_hi^T | dZ_hi^T | dZ_lo^T] [Cout, 3 Mp];
//   colsT -> [cols_hi^T | cols_lo^T] [9C, 2 Mp];  dKernel by tc3_wgrad_splitk (one split-K launch over K = 3 Mp);
//   dcols = mac_linear_tc32_fwd([dZ_hi | dZ_lo], split3_rows(Kernel) [9C, 3 Cout]).
// Columns M..Mp-1 of every transposed segment are written as zeros on every call: the workspace is not assumed zero.
namespace mac {
template <bool SPLIT>
__global__ void __launch_bounds__(256) conv_dz_pack_kernel(const float* __restrict__ y, const float* __restrict__ dy, int act,
                                                          __nv_bfloat16* __restrict__ dz, __nv_bfloat16* __restrict__ dzT,
                                                          float* __restrict__ bpart, int M, int Mp, int N) {
  __shared__ float tile[64][65];                              // [col][row]
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tq = threadIdx.x & 15, tr = threadIdx.x >> 4;     // 16 column quads x 16 rows per pass
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int mm = tr + 16 * p, m = m0 + mm, n = n0 + tq * 4;
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) {
      const size_t o = (size_t)m * N + n;
      const float4 v = __ldg(reinterpret_cast<const float4*>(y + o));
      const float4 d = __ldg(reinterpret_cast<const float4*>(dy + o));
      g.x = d.x * act_grad_from_output(act, v.x);
      g.y = d.y * act_grad_from_output(act, v.y);
      g.z = d.z * act_grad_from_output(act, v.z);
      g.w = d.w * act_grad_from_output(act, v.w);
      if constexpr (!SPLIT) {
        *reinterpret_cast<uint2*>(dz + o) = make_uint2(pack_bf16(g.x, g.y), pack_bf16(g.z, g.w));
      } else if (dz) {                                        // [hi | lo] rows: the data gradient's A operand
        const uint32_t h01 = pack_bf16(g.x, g.y), h23 = pack_bf16(g.z, g.w);
        __nv_bfloat16* row = dz + (size_t)m * 2 * N + n;
        *reinterpret_cast<uint2*>(row) = make_uint2(h01, h23);
        *reinterpret_cast<uint2*>(row + N) = make_uint2(pack_bf16_lo(g.x, g.y, h01), pack_bf16_lo(g.z, g.w, h23));
      }
    }
    tile[tq * 4 + 0][mm] = g.x;
    tile[tq * 4 + 1][mm] = g.y;
    tile[tq * 4 + 2][mm] = g.z;
    tile[tq * 4 + 3][mm] = g.w;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < 64; r += 8) {
    const float a = tile[r][2 * lane], b = tile[r][2 * lane + 1];
    if constexpr (!SPLIT) {
      *reinterpret_cast<uint32_t*>(dzT + (size_t)(n0 + r) * Mp + m0 + 2 * lane) = pack_bf16(a, b);
    } else {                                                  // [hi | hi | lo], each Mp wide
      const uint32_t hw = pack_bf16(a, b);
      __nv_bfloat16* row = dzT + (size_t)(n0 + r) * 3 * Mp + m0 + 2 * lane;
      *reinterpret_cast<uint32_t*>(row) = hw;
      *reinterpret_cast<uint32_t*>(row + Mp) = hw;
      *reinterpret_cast<uint32_t*>(row + 2 * Mp) = pack_bf16_lo(a, b, hw);
    }
    const float s = warp_sum(a + b);
    if (lane == 0) bpart[(size_t)blockIdx.y * N + n0 + r] = s;
  }
}

// colsT[tap*C + c, m] = bf16(dropout(x))[pixel m shifted by tap, c], zero outside the image and for m >= M; with SPLIT the
// row is [hi | lo], each Mp wide.  One 64 (k) x 64 (pixel) tile per block; C % 64 == 0, so a tile lies within one tap.
// 256-byte channel reads, 128-byte row writes.
template <bool SPLIT>
__global__ void __launch_bounds__(256) im2col3x3_t_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ colsT,
                                                         uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                                         int B, int H, int W, int C, int Mp) {
  __shared__ float tile[64][65];                              // [channel][pixel]
  const int k0 = blockIdx.y * 64, m0 = blockIdx.x * 64;
  const int tap = k0 / C, c0 = k0 - tap * C;
  const int dh = tap / 3 - 1, dw = tap % 3 - 1;
  const int M = B * H * W;
  const int tq = threadIdx.x & 15, tr = threadIdx.x >> 4;     // 16 channel quads x 16 pixels per pass
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int mm = tr + 16 * p, m = m0 + mm;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) {
      const int w = m % W, r = m / W;
      const int h = r % H, b = r / H;
      const int hs = h + dh, wsrc = w + dw;
      if (hs >= 0 && hs < H && wsrc >= 0 && wsrc < W) {
        const long long e = (((long long)b * H + hs) * W + wsrc) * C + c0 + tq * 4;
        v = __ldg(reinterpret_cast<const float4*>(x + e));
        if (thresh) {
          const Philox4 q = philox4x32_10(seed, (uint64_t)e >> 2, (uint32_t)site, (uint32_t)step);
          v.x = ((q.x >> 8) >= thresh) ? v.x * scale : 0.f;
          v.y = ((q.y >> 8) >= thresh) ? v.y * scale : 0.f;
          v.z = ((q.z >> 8) >= thresh) ? v.z * scale : 0.f;
          v.w = ((q.w >> 8) >= thresh) ? v.w * scale : 0.f;
        }
      }
    }
    tile[tq * 4 + 0][mm] = v.x;
    tile[tq * 4 + 1][mm] = v.y;
    tile[tq * 4 + 2][mm] = v.z;
    tile[tq * 4 + 3][mm] = v.w;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < 64; r += 8) {
    if constexpr (!SPLIT) {
      *reinterpret_cast<uint32_t*>(colsT + (size_t)(k0 + r) * Mp + m0 + 2 * lane) =
          pack_bf16(tile[r][2 * lane], tile[r][2 * lane + 1]);
    } else {
      const float a = tile[r][2 * lane], b = tile[r][2 * lane + 1];
      const uint32_t hw = pack_bf16(a, b);
      __nv_bfloat16* row = colsT + (size_t)(k0 + r) * 2 * Mp + m0 + 2 * lane;
      *reinterpret_cast<uint32_t*>(row) = hw;
      *reinterpret_cast<uint32_t*>(row + Mp) = pack_bf16_lo(a, b, hw);
    }
  }
}

// im2col3x3_t_kernel for any ConvGeom: colsT[tap C + c, m] = bf16(dropout(x))[the pixel output m's tap reads, c], zero
// outside the image and for m >= M (the padding columns are written on every call).  C % 64 == 0.
template <bool SPLIT>
__global__ void __launch_bounds__(256) im2col_t_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ colsT,
                                                       uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                                       ConvGeom g, int Mp) {
  __shared__ float tile[64][65];                              // [channel][pixel]
  const int k0 = blockIdx.y * 64, m0 = blockIdx.x * 64;
  const int tap = k0 / g.C, c0 = k0 - tap * g.C;
  const int dh = tap / g.k - g.pt, dw = tap % g.k - g.pl;
  const int M = g.B * g.Ho * g.Wo;
  const int tq = threadIdx.x & 15, tr = threadIdx.x >> 4;     // 16 channel quads x 16 pixels per pass
#pragma unroll
  for (int p = 0; p < 4; ++p) {
    const int mm = tr + 16 * p, m = m0 + mm;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (m < M) {
      const int wo = m % g.Wo, r = m / g.Wo;
      const int ho = r % g.Ho, b = r / g.Ho;
      const int hs = ho * g.s + dh, wsrc = wo * g.s + dw;
      if (hs >= 0 && hs < g.H && wsrc >= 0 && wsrc < g.W) {
        const long long e = (((long long)b * g.H + hs) * g.W + wsrc) * g.C + c0 + tq * 4;
        v = __ldg(reinterpret_cast<const float4*>(x + e));
        if (thresh) dropout_quad(v, seed, e, site, step, thresh, scale);
      }
    }
    tile[tq * 4 + 0][mm] = v.x;
    tile[tq * 4 + 1][mm] = v.y;
    tile[tq * 4 + 2][mm] = v.z;
    tile[tq * 4 + 3][mm] = v.w;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int r = warp; r < 64; r += 8) {
    const float a = tile[r][2 * lane], b = tile[r][2 * lane + 1];
    const uint32_t hw = pack_bf16(a, b);
    if constexpr (!SPLIT) {
      *reinterpret_cast<uint32_t*>(colsT + (size_t)(k0 + r) * Mp + m0 + 2 * lane) = hw;
    } else {
      __nv_bfloat16* row = colsT + (size_t)(k0 + r) * 2 * Mp + m0 + 2 * lane;
      *reinterpret_cast<uint32_t*>(row) = hw;
      *reinterpret_cast<uint32_t*>(row + Mp) = pack_bf16_lo(a, b, hw);
    }
  }
}

// im2col_t_kernel's launch: one 64-row tile (within one tap: C % 64 == 0) per gridDim.y index, at most 65535 of them
inline bool im2col_t_grid_ok(int k, int C) { return (long long)k * k * C / 64 <= 65535; }
// conv_dz_pack_kernel's launch: one 64-row block of dZ per gridDim.y index, Mp / 64 <= 65535 (M <= 4 194 240)
inline bool conv_dz_grid_ok(const ConvGeom& g) { return ((long long)g.B * g.Ho * g.Wo + 63) / 64 <= 65535; }

// workspace of mac_conv3x3_bwd_tc / _tc32: 1 KB-aligned slabs behind a 1 KB alignment slack.  `split`: the bf16 operands
// carry 2 (dz rows, colsT) or 3 (dzT, kernel) segments, and the weight gradient contracts over 3 Mp.
struct ConvBwdLayout {
  size_t dz, dzT, colsT, bpart, wpart, k16, dcols, qT, qpart, total;
};
// `l` > 0: the location-aware layer 0 (mac_conv_bwd_loc_tc / _tc32) also holds Q^T [Kq, Mp] (split: [Kq, 2 Mp]) and the
// split-K partials of dW_loc, after every slab of the location-free layout
inline ConvBwdLayout conv_bwd_layout(const ConvGeom& g, int Cout, bool with_dx, bool split, int l_ = 0) {
  auto al = [](size_t v) { return (v + 1023) & ~(size_t)1023; };
  const size_t M = (size_t)g.B * g.Ho * g.Wo, Mp = (M + 63) & ~(size_t)63, K = (size_t)g.k * g.k * g.C;
  const size_t s2 = split ? 2 : 1, s3 = split ? 3 : 1;
  // the split-K partials for the slice count the weight gradient will use on this device (tc_wgrad_splitk / tc3_wgrad_splitk)
  const int S = tc_pick_ksplit((int)(s3 * Mp), (int)(K / TC_BM) * (Cout / TC_BN));
  ConvBwdLayout l;
  size_t o = 0;
  l.dz = o;    o += (split && !with_dx) ? 0 : al(M * Cout * 2 * s2);
  l.dzT = o;   o += al((size_t)Cout * Mp * 2 * s3);
  l.colsT = o; o += al(K * Mp * 2 * s2);
  l.bpart = o; o += al(Mp / 64 * Cout * 4);
  l.wpart = o; o += al((size_t)S * K * Cout * 4);
  l.k16 = l.dcols = o;
  if (with_dx) {
    o += al(K * Cout * 2 * s3);
    l.dcols = o; o += al(M * K * 4);
  }
  l.qT = l.qpart = o;
  if (l_ > 0) {
    const size_t Kq = (size_t)loc_width(l_, g.k);
    const int Sq = tc_pick_ksplit((int)(s3 * Mp), (int)(Kq / TC_BM) * (Cout / TC_BN));
    o += al(Kq * Mp * 2 * s2);
    l.qpart = o; o += al((size_t)Sq * Kq * Cout * 4);
  }
  l.total = o + 1024;
  return l;
}

// The location half of a location-aware layer 0: grid [H, W, l], its dropout site, and dW_loc [Kq, Cout] (+=).
struct ConvBwdLoc {
  const float* grid;
  int l, site;
  float* dwloc;
};

// k = 3, s = 1 runs the 3x3 kernels (im2col3x3_t_kernel, mac_col2im3x3), every other geometry the general ones.  With `loc`,
// the same schedule then adds dW_loc += Q^T dZ from the same dZ^T.
static int conv_bwd_wgmma(bool split, const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                          uint64_t seed, int site, int step, float* dkernel, float* dbias, float* dx, void* workspace,
                          size_t workspace_bytes, int B, int H, int W, int C, int Cout, int k, int s, mac_stream_t stream_,
                          const ConvBwdLoc* loc = nullptr) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !y || !dy || !kernel || !dkernel || !dbias || !workspace) return MAC_ERR_INVALID;
  if (loc && (!loc->grid || !loc->dwloc)) return MAC_ERR_INVALID;
  if (Cout <= 0) return MAC_ERR_INVALID;
  const int gst = conv_geom_check(B, H, W, C, k, s, keep);
  if (gst != MAC_OK) return gst;
  if (loc) {
    const int lst = loc_check(B, H, W, loc->l, k, s, keep);
    if (lst != MAC_OK) return lst;
  }
  if ((C % 128) || (Cout % 128)) return MAC_ERR_UNSUPPORTED;     // wgmma tiles: k^2 C and Cout are GEMM N / M extents
  const ConvGeom g = conv_geom(B, H, W, C, k, s);
  if (!im2col_t_grid_ok(k, C) || !conv_dz_grid_ok(g)) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(x) || !mac_aligned16(y) || !mac_aligned16(dy) || !mac_aligned16(kernel) || !mac_aligned16(dkernel) ||
      (dx && !mac_aligned16(dx)) || (loc && (!mac_aligned16(loc->grid) || !mac_aligned16(loc->dwloc))))
    return MAC_ERR_ALIGN;
  const bool k3s1 = k == 3 && s == 1;
  const ConvBwdLayout l = conv_bwd_layout(g, Cout, dx != nullptr, split, loc ? loc->l : 0);
  if (workspace_bytes < l.total) return MAC_ERR_WORKSPACE;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  const int M = B * g.Ho * g.Wo, Mp = (M + 63) & ~63, K = k * k * C;
  char* base = tc_align1k(workspace);
  __nv_bfloat16* dz = reinterpret_cast<__nv_bfloat16*>(base + l.dz);
  __nv_bfloat16* dzT = reinterpret_cast<__nv_bfloat16*>(base + l.dzT);
  __nv_bfloat16* colsT = reinterpret_cast<__nv_bfloat16*>(base + l.colsT);
  float* bpart = reinterpret_cast<float*>(base + l.bpart);
  float* wpart = reinterpret_cast<float*>(base + l.wpart);
  const dim3 gz(Cout / 64, Mp / 64), gc(Mp / 64, K / 64);
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  if (split) {
    conv_dz_pack_kernel<true><<<gz, 256, 0, stream>>>(y, dy, act, dx ? dz : nullptr, dzT, bpart, M, Mp, Cout);
    MAC_LAUNCH_CHECK();
    if (k3s1)
      im2col3x3_t_kernel<true><<<gc, 256, 0, stream>>>(x, colsT, thr, scale, seed, site, step, B, H, W, C, Mp);
    else
      im2col_t_kernel<true><<<gc, 256, 0, stream>>>(x, colsT, thr, scale, seed, site, step, g, Mp);
  } else {
    conv_dz_pack_kernel<false><<<gz, 256, 0, stream>>>(y, dy, act, dz, dzT, bpart, M, Mp, Cout);
    MAC_LAUNCH_CHECK();
    if (k3s1)
      im2col3x3_t_kernel<false><<<gc, 256, 0, stream>>>(x, colsT, thr, scale, seed, site, step, B, H, W, C, Mp);
    else
      im2col_t_kernel<false><<<gc, 256, 0, stream>>>(x, colsT, thr, scale, seed, site, step, g, Mp);
  }
  MAC_LAUNCH_CHECK();
  int st = mac_colsum(bpart, dbias, 1, Mp / 64, Cout, 1, stream_);
  if (st != MAC_OK) return st;
  st = split ? tc3_wgrad_splitk(colsT, dzT, dkernel, wpart, K, Cout, Mp, stream)
             : tc_wgrad_splitk(colsT, dzT, dkernel, wpart, K, Cout, Mp, stream);
  if (st != MAC_OK) return st;
  if (loc) {                                                    // dW_loc += Q^T dZ on the same dZ^T
    void* qT = base + l.qT;
    float* qpart = reinterpret_cast<float*>(base + l.qpart);
    const int Kq = loc_width(loc->l, k);
    loc_cols_launch(loc->grid, qT, split ? MAC_COLS_SPLIT : MAC_COLS_BF16, true, keep, seed, loc->site, step,
                    conv_geom(B, H, W, loc->l, k, s), stream);
    MAC_LAUNCH_CHECK();
    st = split ? tc3_wgrad_splitk(qT, dzT, loc->dwloc, qpart, Kq, Cout, Mp, stream)
               : tc_wgrad_splitk(qT, dzT, loc->dwloc, qpart, Kq, Cout, Mp, stream);
    if (st != MAC_OK) return st;
  }
  if (!dx) return MAC_OK;
  void* k16 = base + l.k16;                                     // the kernel in its own [9C, Cout] layout: K-major B operand
  float* dcols = reinterpret_cast<float*>(base + l.dcols);
  if (split) {
    st = mac_split3_rows_(kernel, k16, K, Cout, stream_);
    if (st != MAC_OK) return st;
    st = mac_linear_tc32_fwd(dz, k16, nullptr, MAC_ACT_NON, dcols, M, Cout, K, stream_);
  } else {
    st = mac_cast_bf16(kernel, k16, (long long)K * Cout, stream_);
    if (st != MAC_OK) return st;
    st = mac_linear_tc_fwd(dz, k16, nullptr, MAC_ACT_NON, dcols, 0, M, Cout, K, stream_);
  }
  if (st != MAC_OK) return st;
  return k3s1 ? mac_col2im3x3(dcols, dx, keep, seed, site, step, B, H, W, C, stream_)
              : mac_col2im(dcols, dx, keep, seed, site, step, B, H, W, C, k, s, stream_);
}
}  // namespace mac

extern "C" int mac_im2col_t(const float* x, void* colsT, int split, float keep, uint64_t seed, int site, int step, int B, int H,
                            int W, int C, int k, int s, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !colsT) return MAC_ERR_INVALID;
  const int st = conv_geom_check(B, H, W, C, k, s, keep);
  if (st != MAC_OK) return st;
  if ((split != 0 && split != 1) || C % 64 || !im2col_t_grid_ok(k, C)) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(x) || !mac_aligned16(colsT)) return MAC_ERR_ALIGN;
  const ConvGeom g = conv_geom(B, H, W, C, k, s);
  const int M = B * g.Ho * g.Wo, Mp = (M + 63) & ~63;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  const dim3 gc(Mp / 64, k * k * C / 64);
  if (split)
    im2col_t_kernel<true><<<gc, 256, 0, stream>>>(x, reinterpret_cast<__nv_bfloat16*>(colsT), thr, scale, seed, site, step, g,
                                                  Mp);
  else
    im2col_t_kernel<false><<<gc, 256, 0, stream>>>(x, reinterpret_cast<__nv_bfloat16*>(colsT), thr, scale, seed, site, step, g,
                                                   Mp);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" size_t mac_conv_bwd_tc_workspace_bytes(int B, int H, int W, int C, int Cout, int k, int s, int with_dx) {
  if (Cout <= 0 || conv_geom_check(B, H, W, C, k, s, 1.f) != MAC_OK || !im2col_t_grid_ok(k, C) ||
      !conv_dz_grid_ok(conv_geom(B, H, W, C, k, s)))
    return 0;
  return conv_bwd_layout(conv_geom(B, H, W, C, k, s), Cout, with_dx != 0, false).total;
}

extern "C" int mac_conv_bwd_tc(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                               uint64_t seed, int site, int step, float* dkernel, float* dbias, float* dx, void* workspace,
                               size_t workspace_bytes, int B, int H, int W, int C, int Cout, int k, int s, mac_stream_t stream_) {
  return conv_bwd_wgmma(false, x, y, dy, kernel, act, keep, seed, site, step, dkernel, dbias, dx, workspace, workspace_bytes,
                        B, H, W, C, Cout, k, s, stream_);
}

extern "C" size_t mac_conv_bwd_tc32_workspace_bytes(int B, int H, int W, int C, int Cout, int k, int s, int with_dx) {
  if (Cout <= 0 || conv_geom_check(B, H, W, C, k, s, 1.f) != MAC_OK || !im2col_t_grid_ok(k, C) ||
      !conv_dz_grid_ok(conv_geom(B, H, W, C, k, s)))
    return 0;
  return conv_bwd_layout(conv_geom(B, H, W, C, k, s), Cout, with_dx != 0, true).total;
}

extern "C" int mac_conv_bwd_tc32(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                                 uint64_t seed, int site, int step, float* dkernel, float* dbias, float* dx, void* workspace,
                                 size_t workspace_bytes, int B, int H, int W, int C, int Cout, int k, int s,
                                 mac_stream_t stream_) {
  return conv_bwd_wgmma(true, x, y, dy, kernel, act, keep, seed, site, step, dkernel, dbias, dx, workspace, workspace_bytes,
                        B, H, W, C, Cout, k, s, stream_);
}

extern "C" size_t mac_conv3x3_bwd_tc_workspace_bytes(int B, int H, int W, int C, int Cout, int with_dx) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || !conv_dz_grid_ok(conv_geom(B, H, W, C, 3, 1))) return 0;
  return conv_bwd_layout(conv_geom(B, H, W, C, 3, 1), Cout, with_dx != 0, false).total;
}

extern "C" int mac_conv3x3_bwd_tc(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                                  uint64_t seed, int site, int step, float* dkernel, float* dbias, float* dx, void* workspace,
                                  size_t workspace_bytes, int B, int H, int W, int C, int Cout, mac_stream_t stream_) {
  return conv_bwd_wgmma(false, x, y, dy, kernel, act, keep, seed, site, step, dkernel, dbias, dx, workspace, workspace_bytes,
                        B, H, W, C, Cout, 3, 1, stream_);
}

extern "C" size_t mac_conv3x3_bwd_tc32_workspace_bytes(int B, int H, int W, int C, int Cout, int with_dx) {
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || Cout <= 0 || !conv_dz_grid_ok(conv_geom(B, H, W, C, 3, 1))) return 0;
  return conv_bwd_layout(conv_geom(B, H, W, C, 3, 1), Cout, with_dx != 0, true).total;
}

extern "C" int mac_conv3x3_bwd_tc32(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                                    uint64_t seed, int site, int step, float* dkernel, float* dbias, float* dx, void* workspace,
                                    size_t workspace_bytes, int B, int H, int W, int C, int Cout, mac_stream_t stream_) {
  return conv_bwd_wgmma(true, x, y, dy, kernel, act, keep, seed, site, step, dkernel, dbias, dx, workspace, workspace_bytes,
                        B, H, W, C, Cout, 3, 1, stream_);
}

// The location-aware layer 0 (--locationAware): mac_conv_bwd_tc / _tc32 of the image half (kernel and dkernel are the image
// rows [k^2 C, Cout]), then dW_loc [Kq, Cout] += Q^T dZ.  The location channels take no data gradient.
extern "C" size_t mac_conv_bwd_loc_tc_workspace_bytes(int B, int H, int W, int C, int Cout, int l, int k, int s, int with_dx) {
  if (Cout <= 0 || conv_geom_check(B, H, W, C, k, s, 1.f) != MAC_OK || !im2col_t_grid_ok(k, C) ||
      !conv_dz_grid_ok(conv_geom(B, H, W, C, k, s)) ||
      loc_check(B, H, W, l, k, s, 1.f) != MAC_OK)
    return 0;
  return conv_bwd_layout(conv_geom(B, H, W, C, k, s), Cout, with_dx != 0, false, l).total;
}

extern "C" int mac_conv_bwd_loc_tc(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                                   uint64_t seed, int site, int step, const float* grid, int l, int loc_site, float* dkernel,
                                   float* dwloc, float* dbias, float* dx, void* workspace, size_t workspace_bytes, int B,
                                   int H, int W, int C, int Cout, int k, int s, mac_stream_t stream_) {
  const ConvBwdLoc loc{grid, l, loc_site, dwloc};
  return conv_bwd_wgmma(false, x, y, dy, kernel, act, keep, seed, site, step, dkernel, dbias, dx, workspace, workspace_bytes,
                        B, H, W, C, Cout, k, s, stream_, &loc);
}

extern "C" size_t mac_conv_bwd_loc_tc32_workspace_bytes(int B, int H, int W, int C, int Cout, int l, int k, int s,
                                                        int with_dx) {
  if (Cout <= 0 || conv_geom_check(B, H, W, C, k, s, 1.f) != MAC_OK || !im2col_t_grid_ok(k, C) ||
      !conv_dz_grid_ok(conv_geom(B, H, W, C, k, s)) ||
      loc_check(B, H, W, l, k, s, 1.f) != MAC_OK)
    return 0;
  return conv_bwd_layout(conv_geom(B, H, W, C, k, s), Cout, with_dx != 0, true, l).total;
}

extern "C" int mac_conv_bwd_loc_tc32(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep,
                                     uint64_t seed, int site, int step, const float* grid, int l, int loc_site, float* dkernel,
                                     float* dwloc, float* dbias, float* dx, void* workspace, size_t workspace_bytes, int B,
                                     int H, int W, int C, int Cout, int k, int s, mac_stream_t stream_) {
  const ConvBwdLoc loc{grid, l, loc_site, dwloc};
  return conv_bwd_wgmma(true, x, y, dy, kernel, act, keep, seed, site, step, dkernel, dbias, dx, workspace, workspace_bytes,
                        B, H, W, C, Cout, k, s, stream_, &loc);
}
