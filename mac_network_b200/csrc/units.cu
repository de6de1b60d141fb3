// C-ABI entry points of the three MAC units (fp32 projection path) and the elementwise helpers.
#include "common.cuh"
#include "sgemm.cuh"
#include "skinny.cuh"
#include "tc_gemm.cuh"
#include "read_step.cuh"
#include "skinny_tc.cuh"

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
// workspace layout: [header 4 KB | md [B,d] | y [B,d] | P [BN,d] | H [BN,d] | logit parts [BN, <=32] | split-K]
static size_t read_ws_layout(int B, int N, int d, size_t* off_md, size_t* off_y, size_t* off_P, size_t* off_H,
                             size_t* off_parts, size_t* off_splitk) {
  size_t o = WS_HEADER;
  auto take = [&](size_t bytes) { size_t r = o; o += (bytes + 255) & ~(size_t)255; return r; };
  *off_md = take((size_t)B * d * 4);
  *off_y = take((size_t)B * d * 4);
  *off_P = take((size_t)B * N * d * 4);
  *off_H = take((size_t)B * N * d * 4);
  *off_parts = take((size_t)B * N * 32 * 4);
  *off_splitk = o;
  o += sgemm_workspace_bytes(B, d, d);
  return o;
}

extern "C" size_t mac_read_workspace_bytes(int B, int N, int d, int prec) {
  size_t a, b, c, e, f, g;
  size_t fp32 = read_ws_layout(B, N, d, &a, &b, &c, &e, &f, &g);
  if (prec == MAC_PREC_BF16) return fp32 + tc_read_extra_workspace_bytes(B, N, d);
  if (prec == MAC_PREC_TC32) return fp32 + tc3_extra_workspace_bytes(B, N, d);
  return fp32;
}

// ---- step-invariant part of the eval-mode read unit (see tc_read_invariant in tc_gemm.cuh): inv = [P | Q]
static size_t read_inv_fp32_bytes(int B, int N, int d) { return (size_t)2 * B * N * d * 4 + 256; }

extern "C" size_t mac_read_invariant_bytes(int B, int N, int d, int prec) {
  if (prec == MAC_PREC_TC32) return tc3_invariant_bytes(B, N, d);
  return prec == MAC_PREC_BF16 ? tc_read_invariant_bytes(B, N, d) : read_inv_fp32_bytes(B, N, d);
}

extern "C" int mac_read_invariant(const float* kb, const void* kb_bf16, const mac_read_weights* w, int prec, void* inv,
                                  size_t inv_bytes, int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  // the bf16 path reads only kb_bf16: the fp32 knowledge base may be absent (host-cast front end)
  if ((!kb && !(prec == MAC_PREC_BF16 && kb_bf16)) || !w || !inv || B <= 0 || N <= 0 || d <= 0 || (d & 3))
    return MAC_ERR_INVALID;
  if ((kb && !mac_aligned16(kb)) || !mac_aligned16(inv)) return MAC_ERR_ALIGN;
  if (inv_bytes < mac_read_invariant_bytes(B, N, d, prec)) return MAC_ERR_WORKSPACE;
  if (prec == MAC_PREC_BF16) return tc_read_invariant(kb_bf16, w, inv, inv_bytes, B, N, d, stream);
  if (prec == MAC_PREC_TC32) return tc3_read_invariant(kb, w, inv, inv_bytes, B, N, d, stream);
  const int M = B * N;
  float* P = reinterpret_cast<float*>(inv);
  float* Q = P + (size_t)M * d;
  SgemmParams p{};
  // P = KB @ Wx + bx   (ops.py:688)
  p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = kb; p.ak[0] = d; p.lda[0] = d;
  p.W = w->Wx; p.ldw = d; p.M = M; p.N = d; p.K = d;
  p.epi = EPI_BIAS_ACT; p.bias = w->bx; p.act = MAC_ACT_NON; p.Y = P; p.ldy = d;
  int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
  if (st != MAC_OK) return st;
  // Q = P @ Wm[d:2d, :] + bm   (the un-scaled half of the concat, mac_cell.py:236-238)
  p.a[0] = P; p.W = w->Wm + (size_t)d * d; p.bias = w->bm; p.Y = Q;
  return sgemm_launch(p, nullptr, nullptr, 0, stream, false);
}

static int read_fwd_impl(const float* kb, const void* kb_bf16, const void* inv, const float* y_pre,
                         const float* memory_in, const float* control, const mac_read_weights* w, float keep_read,
                         uint64_t seed, int step, int prec, float* info, float* att, float* save, void* workspace,
                         size_t workspace_bytes, int B, int N, int d, mac_stream_t stream_);

// MAC_READ_FUSED=0 keeps the four-launch form of the inference read step (scale, two GEMMs, attention) for comparison
static bool read_step_enabled() {
  static const bool on = !(getenv("MAC_READ_FUSED") && atoi(getenv("MAC_READ_FUSED")) == 0);
  return on;
}

extern "C" int mac_read_step_fused(const void* inv, const void* kb_bf16, const float* y, const float* control,
                                   const mac_read_weights* w, float* info, float* att, int B, int N, int d,
                                   mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!inv || !kb_bf16 || !y || !control || !w || !info || !att || B <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  if (!mac_aligned16(inv) || !mac_aligned16(kb_bf16) || !mac_aligned16(y) || !mac_aligned16(control)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  return read_step_launch(inv, kb_bf16, y, control, w, att, info, B, N, d, stream);
}
extern "C" int mac_step_fused(const void* inv, const void* kb_bf16, const float* mem_prev, const float* info_prev,
                              const float* control, const mac_read_weights* w, const void* Ww_t_bf16, const float* bw,
                              const void* Wy_t_bf16, float* mem_out, float* info, float* att, int B, int N, int d,
                              mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!inv || !kb_bf16 || !mem_prev || !control || !w || !Wy_t_bf16 || !info || !att || B <= 0 || N <= 0 || d <= 0)
    return MAC_ERR_INVALID;
  if (!mac_aligned16(inv) || !mac_aligned16(kb_bf16) || !mac_aligned16(control)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  WholeStepArgs ws{mem_prev, info_prev, Ww_t_bf16, bw, Wy_t_bf16, mem_out};
  return read_step_launch(inv, kb_bf16, nullptr, control, w, att, info, B, N, d, stream, &ws);
}
extern "C" int mac_step_fused_supported(int B, int N, int d) { return whole_step_supported(B, N, d) ? 1 : 0; }

extern "C" int mac_read_step_fused_supported(int B, int N, int d) { return read_step_supported(B, N, d) ? 1 : 0; }

extern "C" int mac_read_fwd(const float* kb, const void* kb_bf16, const float* memory_in, const float* control,
                            const mac_read_weights* w, float keep_read, uint64_t seed, int step, int prec, float* info,
                            float* att, float* save, void* workspace, size_t workspace_bytes, int B, int N, int d,
                            mac_stream_t stream_) {
  return read_fwd_impl(kb, kb_bf16, nullptr, nullptr, memory_in, control, w, keep_read, seed, step, prec, info, att,
                       save, workspace, workspace_bytes, B, N, d, stream_);
}

extern "C" int mac_read_fwd_inv(const float* kb, const void* kb_bf16, const void* inv, const float* y_pre,
                                const float* memory_in, const float* control, const mac_read_weights* w, int prec,
                                float* info, float* att, void* workspace, size_t workspace_bytes, int B, int N, int d,
                                mac_stream_t stream_) {
  if (!inv || !mac_aligned16(inv) || (y_pre && !mac_aligned16(y_pre))) return MAC_ERR_INVALID;
  return read_fwd_impl(kb, kb_bf16, inv, y_pre, memory_in, control, w, 1.f, 0, 0, prec, info, att, nullptr, workspace,
                       workspace_bytes, B, N, d, stream_);
}

static int read_fwd_impl(const float* kb, const void* kb_bf16, const void* inv, const float* y_pre,
                         const float* memory_in, const float* control, const mac_read_weights* w, float keep_read,
                         uint64_t seed, int step, int prec, float* info, float* att, float* save, void* workspace,
                         size_t workspace_bytes, int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const bool kb_opt = inv && prec == MAC_PREC_BF16 && kb_bf16;     // eval bf16 path: only the bf16 copy is read
  if ((!kb && !kb_opt) || !memory_in || !control || !w || !info || !att || !workspace) return MAC_ERR_INVALID;
  if (B <= 0 || N <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  if (!(keep_read > 0.f && keep_read <= 1.f)) return MAC_ERR_INVALID;
  if ((kb && !mac_aligned16(kb)) || !mac_aligned16(memory_in) || !mac_aligned16(control) || !mac_aligned16(workspace))
    return MAC_ERR_ALIGN;
  if (workspace_bytes < mac_read_workspace_bytes(B, N, d, prec)) return MAC_ERR_WORKSPACE;
  size_t o_md, o_y, o_P, o_H, o_parts, o_sk;
  const size_t fp32_total = read_ws_layout(B, N, d, &o_md, &o_y, &o_P, &o_H, &o_parts, &o_sk);
  char* ws = reinterpret_cast<char*>(workspace);
  float* md = reinterpret_cast<float*>(ws + o_md);
  const int M = B * N;
  // saved activations for backward live in the caller's `save` when given: [P | H | I1 | y]
  float* P = save ? save : reinterpret_cast<float*>(ws + o_P);
  float* H = save ? save + (size_t)M * d : reinterpret_cast<float*>(ws + o_H);
  float* I1 = save ? save + (size_t)2 * M * d : nullptr;
  float* y = save ? save + (size_t)3 * M * d : reinterpret_cast<float*>(ws + o_y);
  float* parts = reinterpret_cast<float*>(ws + o_parts);
  const bool drop = keep_read < 1.f;
  const uint32_t thr = drop ? keep_threshold(keep_read) : 0u;
  const float scale = drop ? 1.f / keep_read : 1.f;

  // md = dropout(memory_in, keep_read)   (ops.py:679)
  const float* mem = memory_in;
  if (drop) {
    const long long n = (long long)B * d;
    dropout_kernel<<<(unsigned)(((n + 3) / 4 + 255) / 256), 256, 0, stream>>>(memory_in, thr, scale, seed,
                                                                            MAC_SITE_READ_MEM, step, md, nullptr, n);
    MAC_LAUNCH_CHECK();
    mem = md;
  }
  // y = md @ Wy + by   (ops.py:689) -- unless the caller already has it (mac_write_fwd_next_y of the previous step)
  if (y_pre) {
    y = const_cast<float*>(y_pre);
  } else {
    SgemmParams p{};
    p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = mem; p.ak[0] = d; p.lda[0] = d;
    p.W = w->Wy; p.ldw = d; p.M = B; p.N = d; p.K = d;
    p.epi = EPI_BIAS_ACT; p.bias = w->by; p.act = MAC_ACT_NON; p.Y = y; p.ldy = d;
    int st = sgemm_launch(p, reinterpret_cast<unsigned int*>(ws), reinterpret_cast<float*>(ws + o_sk),
                          fp32_total - o_sk, stream);
    if (st != MAC_OK) return st;
  }
  int nparts = 0;
  if (inv && prec == MAC_PREC_BF16 && kb_bf16 && read_step_supported(B, N, d) && read_step_enabled()) {
    // the whole step (P*y, both projections, logits, softmax, weighted sum) as ONE kernel: read_step.cuh
    return read_step_launch(inv, kb_bf16, y, control, w, att, info, B, N, d, stream);
  }
  if (prec == MAC_PREC_TC32) {
    if (!inv) return MAC_ERR_UNSUPPORTED;          // split-bf16 products: inference form only
    int st = tc3_read_chain_inv(inv, y, control, w, parts, &nparts, ws + fp32_total, workspace_bytes - fp32_total, B, N, d,
                                stream);
    if (st != MAC_OK) return st;
  } else if (inv && prec == MAC_PREC_BF16) {
    int st = tc_read_chain_inv(inv, y, control, w, parts, &nparts, ws + fp32_total, workspace_bytes - fp32_total, B, N,
                               d, stream);
    if (st != MAC_OK) return st;
  } else if (inv) {
    const float* Pi = reinterpret_cast<const float*>(inv);
    const float* Qi = Pi + (size_t)M * d;
    // H = ELU((P*y) @ Wm[0:d, :] + Q)   (bm is inside Q)
    {
      SgemmParams p{};
      p.a_mode = A_ROWSCALE_CONCAT; p.rs_half = d; p.nseg = 1; p.a[0] = Pi; p.lda[0] = d; p.rowvec = y; p.rows_per_batch = N;
      p.W = w->Wm; p.ldw = d; p.M = M; p.N = d; p.K = d;
      p.epi = EPI_BIAS_ACT; p.bias = nullptr; p.aux = Qi; p.ldaux = d; p.act = MAC_ACT_ELU; p.Y = H; p.ldy = d;
      int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
      if (st != MAC_OK) return st;
    }
    {
      SgemmParams p{};
      p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = H; p.ak[0] = d; p.lda[0] = d;
      p.W = w->Wm2; p.ldw = d; p.M = M; p.N = d; p.K = d; p.rows_per_batch = N;
      p.epi = EPI_READ_LOGITS; p.bias = w->bm2; p.Y = nullptr; p.ldy = d;
      p.ctrl = control; p.wr = w->wr; p.logit_parts = parts; p.e_thresh = 0u; p.e_scale = 1.f;
      int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
      if (st != MAC_OK) return st;
      nparts = (d + sgemm_tile_n(M, d, d) - 1) / sgemm_tile_n(M, d, d);
    }
  } else if (prec == MAC_PREC_BF16) {
    int st = tc_read_chain(kb, kb_bf16, y, control, w, thr, scale, seed, step, P, H, I1, parts, &nparts,
                           ws + fp32_total, workspace_bytes - fp32_total, B, N, d, save != nullptr, stream);
    if (st != MAC_OK) return st;
  } else {
    // P = dropout(KB) @ Wx + bx   (ops.py:678, 688)
    {
      SgemmParams p{};
      p.a_mode = drop ? A_DROPOUT : A_SEGS; p.nseg = 1; p.a[0] = kb; p.ak[0] = d; p.lda[0] = d;
      p.a_thresh = thr; p.a_scale = scale; p.seed = seed; p.a_site = MAC_SITE_READ_KB; p.step = step;
      p.W = w->Wx; p.ldw = d; p.M = M; p.N = d; p.K = d;
      p.epi = EPI_BIAS_ACT; p.bias = w->bx; p.act = MAC_ACT_NON; p.Y = P; p.ldy = d;
      int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
      if (st != MAC_OK) return st;
    }
    // H = ELU([P*y, P] @ Wm + bm)   (ops.py:694-719, mac_cell.py:236-238)
    {
      SgemmParams p{};
      p.a_mode = A_ROWSCALE_CONCAT; p.nseg = 1; p.a[0] = P; p.lda[0] = d; p.rowvec = y; p.rows_per_batch = N;
      p.W = w->Wm; p.ldw = d; p.M = M; p.N = d; p.K = 2 * d;
      p.epi = EPI_BIAS_ACT; p.bias = w->bm; p.act = MAC_ACT_ELU; p.Y = H; p.ldy = d;
      int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
      if (st != MAC_OK) return st;
    }
    // I1 = H @ Wm2 + bm2 ; I2 = ELU(I1 * control) ; logits = dropout(I2) . wr   (ops.py:325-328, mac_cell.py:248-266)
    {
      SgemmParams p{};
      p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = H; p.ak[0] = d; p.lda[0] = d;
      p.W = w->Wm2; p.ldw = d; p.M = M; p.N = d; p.K = d; p.rows_per_batch = N;
      p.epi = EPI_READ_LOGITS; p.bias = w->bm2; p.Y = I1; p.ldy = d;
      p.ctrl = control; p.wr = w->wr; p.logit_parts = parts;
      p.e_thresh = thr; p.e_scale = scale; p.e_site = MAC_SITE_READ_INTER; p.seed = seed; p.step = step;
      int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
      if (st != MAC_OK) return st;
      nparts = (d + sgemm_tile_n(M, d, d) - 1) / sgemm_tile_n(M, d, d);
    }
  }
  if (nparts > 32) return MAC_ERR_UNSUPPORTED;
  // att = softmax(logits); info = sum_n att * KB   (original, un-dropped KB: mac_cell.py:271-275)
  if (prec == MAC_PREC_BF16 && kb_bf16 != nullptr)
    return mac_kb_attend_fwd(parts, nparts, w->br, kb_bf16, 1, att, info, B, N, d, stream_);
  return mac_kb_attend_fwd(parts, nparts, w->br, kb, 0, att, info, B, N, d, stream_);
}

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

extern "C" int mac_widen_bf16(const void* const* src_bf16, float* const* dst, int nslab, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!src_bf16 || !dst || nslab < 1 || nslab > 3 || n <= 0 || (n & 7)) return MAC_ERR_INVALID;
  const uint4* s[3] = {nullptr, nullptr, nullptr};
  float4* d[3] = {nullptr, nullptr, nullptr};
  for (int i = 0; i < nslab; ++i) {
    if (!src_bf16[i] || !dst[i]) return MAC_ERR_INVALID;
    if ((reinterpret_cast<uintptr_t>(src_bf16[i]) | reinterpret_cast<uintptr_t>(dst[i])) & 15) return MAC_ERR_ALIGN;
    s[i] = reinterpret_cast<const uint4*>(src_bf16[i]);
    d[i] = reinterpret_cast<float4*>(dst[i]);
  }
  const long long n8 = n / 8;
  const unsigned gx = (unsigned)std::min<long long>((n8 + 255) / 256, (long long)mac_num_sms() * 16);
  widen3_bf16_kernel<<<dim3(gx, nslab), 256, 0, stream>>>(s[0], s[1], s[2], d[0], d[1], d[2], n8);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
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
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
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
