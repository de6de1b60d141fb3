// ops.linear (ops.py:298-333) on [B*N, .] rows with bf16 operands on wgmma tensor cores and fp32 accumulation: the composed
// read unit of MACCell(prec="bf16") (the flag sets outside the fused read kernel) and its backward on the tape (tape.py).
//
//   forward   y[M, n_out] = act(concat(x_0 .. x_{nseg-1}) @ W + b + bias_const)          (mac_linear_tc_seg_fwd)
//             seg_cast_bf16_kernel writes bf16(concat(x_s)) as ONE K-major A operand [M, K] (16-byte loads and stores,
//             round to nearest even); then one tc_gemm launch with the fp32 epilogue (TC_EPI_F32: bias, bias_const, act, ldy).
//   backward  (mac_linear_bwd_tc; mac_linear_bwd's conventions)
//             pack_t_bf16 of dy        -> bf16 dy^T [n_out, Mp] (zero columns M..Mp-1) and bf16 dy [M, n_out]
//             dW_s += x_s^T dy         pack_t_bf16 of x_s -> bf16 x_s^T [k_s, Mp] (zero columns M..Mp-1), tc_wgrad_splitk, K = Mp
//             dx_s (+)= dy W_s^T       tc_gemm of bf16 dy against bf16(W_s) in its own [k_s, n_out] layout (the K-major B
//                                      operand), fp32 epilogue storing or adding at ld_dx
//             db += colsum(dy)         per-64-row partial sums, then their sum: fixed order
//   Mp = M rounded up to the 64-wide k-block.  The zero columns are rewritten on every call (the workspace is not assumed
//   zero), so any M >= 1 works.  Every k_s and n_out must be a multiple of 128 (the 128 x 128 output tiles of tc_gemm; each
//   segment is the M or N extent of one of the backward products).  Every check precedes the first launch.
#pragma once
#include "common.cuh"
#include "tc_gemm.cuh"

namespace mac {

struct SegCastArgs {
  const float* x[4];
  int koff[4];          // first column of segment s in the concatenation
  int ldx[4];
  int nseg;
};

// A[m, koff_s + c] = bf16(x_s[m, c]): 8 columns per thread (two 16-byte loads, one 16-byte store).  Segment widths are
// multiples of 128, so no group of 8 straddles two segments.
__global__ void __launch_bounds__(256) seg_cast_bf16_kernel(const SegCastArgs a, uint4* __restrict__ out, int K, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const int K8 = K / 8;
  const long long m = i / K8;
  const int c = (int)(i - m * K8) * 8;
  const int s = (a.nseg > 3 && c >= a.koff[3]) ? 3 : (a.nseg > 2 && c >= a.koff[2]) ? 2 : (a.nseg > 1 && c >= a.koff[1]) ? 1 : 0;
  const float* base = s == 0 ? a.x[0] : s == 1 ? a.x[1] : s == 2 ? a.x[2] : a.x[3];
  const int ld = s == 0 ? a.ldx[0] : s == 1 ? a.ldx[1] : s == 2 ? a.ldx[2] : a.ldx[3];
  const int k0 = s == 0 ? a.koff[0] : s == 1 ? a.koff[1] : s == 2 ? a.koff[2] : a.koff[3];
  const float4* src = reinterpret_cast<const float4*>(base + m * ld + (c - k0));
  const float4 v0 = __ldg(src), v1 = __ldg(src + 1);
  out[i] = make_uint4(pack_bf16(v0.x, v0.y), pack_bf16(v0.z, v0.w), pack_bf16(v1.x, v1.y), pack_bf16(v1.z, v1.w));
}

inline size_t lt_align(size_t v) { return (v + 1023) & ~(size_t)1023; }

// workspace of mac_linear_bwd_tc: 1 KB-aligned slabs behind a 1 KB alignment slack
struct LinBwdLayout {
  size_t g16, gT, xT, w16, bpart, wpart, total;
};
inline LinBwdLayout lin_bwd_layout(int M, const int* k_segs, int nseg, int n_out) {
  const size_t Mp = ((size_t)M + 63) & ~(size_t)63;
  size_t K = 0, kmax = 0, wp = 0;
  for (int s = 0; s < nseg; ++s) {
    const size_t k = (size_t)k_segs[s];
    K += k;
    kmax = k > kmax ? k : kmax;
    // the split-K partials for the slice count tc_wgrad_splitk picks on this device
    const size_t S = (size_t)tc_pick_ksplit((int)Mp, (int)(k / TC_BM) * (n_out / TC_BN));
    wp = S * k * n_out * 4 > wp ? S * k * n_out * 4 : wp;
  }
  LinBwdLayout l;
  size_t o = 0;
  l.g16 = o;   o += lt_align((size_t)M * n_out * 2);
  l.gT = o;    o += lt_align((size_t)n_out * Mp * 2);
  l.xT = o;    o += lt_align(kmax * Mp * 2);
  l.w16 = o;   o += lt_align(K * n_out * 2);
  l.bpart = o; o += lt_align(Mp / 64 * (size_t)n_out * 4);
  l.wpart = o; o += lt_align(wp);
  l.total = o + 1024;
  return l;
}

}  // namespace mac

using namespace mac;

extern "C" size_t mac_linear_tc_seg_workspace_bytes(int M, int K) {
  if (M <= 0 || K <= 0) return 0;
  return lt_align((size_t)M * K * 2) + 1024;
}

extern "C" int mac_linear_tc_seg_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const void* wt_bf16,
                                     const float* b, float bias_const, int act, float* y, int ldy, int M, int n_out,
                                     void* workspace, size_t workspace_bytes, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !ldx || nseg < 1 || nseg > 4 || !wt_bf16 || !y || !workspace || M <= 0 || n_out <= 0)
    return MAC_ERR_INVALID;
  if (act < MAC_ACT_NON || act > MAC_ACT_RELU || ldy < n_out) return MAC_ERR_INVALID;
  SegCastArgs a{};
  a.nseg = nseg;
  int K = 0;
  for (int s = 0; s < nseg; ++s) {
    if (!x_segs[s] || k_segs[s] <= 0 || ldx[s] < k_segs[s]) return MAC_ERR_INVALID;
    if (k_segs[s] % TC_BN) return MAC_ERR_UNSUPPORTED;
    if (!mac_aligned16(x_segs[s]) || (ldx[s] & 3)) return MAC_ERR_ALIGN;
    a.x[s] = x_segs[s]; a.koff[s] = K; a.ldx[s] = ldx[s];
    K += k_segs[s];
  }
  if ((n_out % TC_BN) || (M + TC_BM - 1) / TC_BM > 65535) return MAC_ERR_UNSUPPORTED;
  if (!mac_aligned16(wt_bf16) || !mac_aligned16(y) || (ldy & 3)) return MAC_ERR_ALIGN;
  if (workspace_bytes < mac_linear_tc_seg_workspace_bytes(M, K)) return MAC_ERR_WORKSPACE;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  void* A = tc_align1k(workspace);
  const long long n8 = (long long)M * K / 8;
  seg_cast_bf16_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, stream>>>(a, reinterpret_cast<uint4*>(A), K, n8);
  MAC_LAUNCH_CHECK();
  TcGemmParams p{};
  p.M = M; p.N = n_out; p.epi = TC_EPI_F32; p.act = act; p.bias = b; p.bias_const = bias_const; p.outf = y; p.ldo = ldy;
  p.rows_per_batch = 1;
  return tc_gemm_launch(A, K, nullptr, 0, wt_bf16, p, stream);
}

extern "C" size_t mac_linear_bwd_tc_workspace_bytes(int M, const int* k_segs, int nseg, int n_out) {
  if (M <= 0 || !k_segs || nseg < 1 || nseg > 4 || n_out <= 0) return 0;
  for (int s = 0; s < nseg; ++s)
    if (k_segs[s] <= 0) return 0;
  return lin_bwd_layout(M, k_segs, nseg, n_out).total;
}

extern "C" int mac_linear_bwd_tc(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* W,
                                 const float* dy, int ldy, float* const* dx_segs, const int* ld_dx, const int* dx_accum,
                                 float* dW, float* db, int M, int n_out, void* workspace, size_t workspace_bytes,
                                 mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !ldx || !dy || !workspace || nseg < 1 || nseg > 4 || M <= 0 || n_out <= 0 || ldy < n_out)
    return MAC_ERR_INVALID;
  bool any_dx = false;
  int K = 0;
  for (int s = 0; s < nseg; ++s) {
    const bool dx = dx_segs && dx_segs[s];
    any_dx = any_dx || dx;
    if (k_segs[s] <= 0 || (dW && (!x_segs[s] || ldx[s] < k_segs[s])) || (dx && (!ld_dx || ld_dx[s] < k_segs[s])))
      return MAC_ERR_INVALID;
    if (k_segs[s] % TC_BN) return MAC_ERR_UNSUPPORTED;
    if (dW && (!mac_aligned16(x_segs[s]) || (ldx[s] & 3))) return MAC_ERR_ALIGN;
    if (dx && (!mac_aligned16(dx_segs[s]) || (ld_dx[s] & 3))) return MAC_ERR_ALIGN;
    K += k_segs[s];
  }
  if (any_dx && !W) return MAC_ERR_INVALID;
  if ((n_out % TC_BN) || (M + TC_BM - 1) / TC_BM > 65535) return MAC_ERR_UNSUPPORTED;
  if (db && ldy != n_out) return MAC_ERR_UNSUPPORTED;                     // the column sums read dy as [M, n_out]
  if (!mac_aligned16(dy) || (ldy & 3) || (W && !mac_aligned16(W)) || (dW && !mac_aligned16(dW))) return MAC_ERR_ALIGN;
  const LinBwdLayout l = lin_bwd_layout(M, k_segs, nseg, n_out);
  if (workspace_bytes < l.total) return MAC_ERR_WORKSPACE;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  const int Mp = (M + 63) & ~63;
  char* base = tc_align1k(workspace);
  __nv_bfloat16* g16 = reinterpret_cast<__nv_bfloat16*>(base + l.g16);
  __nv_bfloat16* gT = reinterpret_cast<__nv_bfloat16*>(base + l.gT);
  __nv_bfloat16* xT = reinterpret_cast<__nv_bfloat16*>(base + l.xT);
  __nv_bfloat16* w16 = reinterpret_cast<__nv_bfloat16*>(base + l.w16);
  float* bpart = reinterpret_cast<float*>(base + l.bpart);
  float* wpart = reinterpret_cast<float*>(base + l.wpart);
  int st;
  if (dW || any_dx) {
    // bf16(dy)^T [n_out, Mp] for the weight gradients, bf16(dy) [M, n_out] for the data gradients: one read of dy
    st = pack_t_bf16_launch(0, dy, gT, any_dx ? g16 : nullptr, M, n_out, PackTArgs{}, stream, ldy, Mp);
    if (st != MAC_OK) return st;
  }
  if (any_dx) {
    st = mac_cast_bf16(W, w16, (long long)K * n_out, stream_);
    if (st != MAC_OK) return st;
  }
  int koff = 0;
  for (int s = 0; s < nseg; ++s) {
    const int k = k_segs[s];
    if (dW) {
      st = pack_t_bf16_launch(0, x_segs[s], xT, nullptr, M, k, PackTArgs{}, stream, ldx[s], Mp);
      if (st != MAC_OK) return st;
      st = tc_wgrad_splitk(xT, gT, dW + (size_t)koff * n_out, wpart, k, n_out, Mp, stream);
      if (st != MAC_OK) return st;
    }
    if (dx_segs && dx_segs[s]) {
      TcGemmParams p{};
      p.M = M; p.N = k; p.epi = TC_EPI_F32; p.act = MAC_ACT_NON; p.outf = dx_segs[s]; p.ldo = ld_dx[s];
      p.accum = dx_accum ? dx_accum[s] : 0; p.rows_per_batch = 1;
      st = tc_gemm_launch(g16, n_out, nullptr, 0, w16 + (size_t)koff * n_out, p, stream);
      if (st != MAC_OK) return st;
    }
    koff += k;
  }
  if (db) {
    // fixed order: column sums of each 64-row block (the last one may be short), then the sum of those, added to db
    const int q = M / 64, r = M - q * 64;
    if (q > 0) {
      st = mac_colsum(dy, bpart, q, 64, n_out, 0, stream_);
      if (st != MAC_OK) return st;
    }
    if (r > 0) {
      st = mac_colsum(dy + (size_t)q * 64 * n_out, bpart + (size_t)q * n_out, 1, r, n_out, 0, stream_);
      if (st != MAC_OK) return st;
    }
    st = mac_colsum(bpart, db, 1, Mp / 64, n_out, 1, stream_);
    if (st != MAC_OK) return st;
  }
  return MAC_OK;
}
