// The read unit's forward (mac_cell.py:209-277, see mac_read_fwd in mac_b200.h) in each of its forms, and the C entry points
// that pick one: mac_read_fwd, mac_read_fwd_inv, mac_read_invariant, mac_read_step_fused and their size queries.
//
//   FP32_TRAIN, BF16_TRAIN, TC32_TRAIN   mac_read_fwd with MAC_PREC_FP32 / BF16 / TC32: P, H, I1 + logits on the FMA pipe,
//                                        on tc_gemm, or as split-bf16 products (tc3_gemm)
//   FP32_INV, BF16_INV, TC32_INV         mac_read_fwd_inv: H from the hoisted P and Q (mac_read_invariant), I1 + logits
//   BF16_STEP, FP8_STEP                  mac_read_fwd_inv with MAC_PREC_BF16 / FP8, kb_bf16 and read_step_supported(B, N, d):
//                                        the fused read step (read_step.cuh, read_step_fp8.cuh); FP8 has no other form
// Every form first computes md = dropout(memory_in) and y = md @ Wy + by (unless the caller gives y); all but the fused
// steps (which end in it) finish with kb_attend on the partial logits.
//
// Every call is classified (read_form), checked against everything its form reads and every limit of the kernels it
// launches (read_fwd_check, read_inv_check), and only then dispatched: a refusal never follows a launch or a write, and the
// form functions check nothing themselves.  Included by units.cu only.
#pragma once

namespace mac {

enum ReadForm { RF_NONE, RF_FP32_TRAIN, RF_FP32_INV, RF_BF16_TRAIN, RF_BF16_STEP, RF_BF16_INV, RF_TC32_TRAIN, RF_TC32_INV,
                RF_FP8_STEP };

// `inv`: the form of mac_read_fwd_inv (and which step-invariant part mac_read_invariant computes); RF_NONE: no form
inline ReadForm read_form(int prec, bool inv, bool kb_bf16, bool step_shape) {
  switch (prec) {
    case MAC_PREC_BF16: return !inv ? RF_BF16_TRAIN : kb_bf16 && step_shape ? RF_BF16_STEP : RF_BF16_INV;
    case MAC_PREC_TC32: return inv ? RF_TC32_INV : RF_TC32_TRAIN;
    case MAC_PREC_FP8: return inv && kb_bf16 && step_shape ? RF_FP8_STEP : RF_NONE;   // the inference read step only
    default: return inv ? RF_FP32_INV : RF_FP32_TRAIN;
  }
}

// partial logits per knowledge-base row: one per column tile of the logits GEMM, one for the fused steps
inline int read_nparts(ReadForm f, int M, int d) {
  if (f == RF_FP32_TRAIN || f == RF_FP32_INV) return (d + sgemm_tile_n(M, d, d) - 1) / sgemm_tile_n(M, d, d);
  if (f == RF_BF16_STEP || f == RF_FP8_STEP) return 1;
  return d / TC_BN;
}

inline size_t align1k(size_t b) { return (b + 1023) & ~(size_t)1023; }
inline char* at(uintptr_t a) { return reinterpret_cast<char*>(a); }

// ------------------------------------------------------------------------------------------------ layouts
// The read workspace of every precision, first in fp32:
//   [header 4 KB (split-K counters) | md [B,d] | y [B,d] | P [BN,d] | H [BN,d] | logit parts [BN, <=32] | split-K]
// then, behind it and 1 KB aligned:
//   MAC_PREC_BF16  five bf16 [BN, d] slabs: P, P*y, H, I1, dropout(KB)
//   MAC_PREC_TC32  two bf16 [BN, 2d] slabs: 0 = (P*y) as hi | lo (inference) or the fp32 P without `save` (training),
//                  1 = H as hi | lo
// ws may be NULL when only `bytes` is wanted.
struct ReadWs {
  float *md, *y, *P, *H, *parts, *splitk;
  size_t splitk_bytes;
  char* tc;          // the first slab behind the fp32 part
  size_t slab;       // bytes from one slab to the next
  size_t bytes;      // mac_read_workspace_bytes
};
inline ReadWs read_ws_layout(int prec, void* ws, int B, int N, int d) {
  const size_t M = (size_t)B * N;
  const uintptr_t base = reinterpret_cast<uintptr_t>(ws);
  size_t o = WS_HEADER;
  auto take = [&](size_t bytes) { const size_t r = o; o += (bytes + 255) & ~(size_t)255; return (float*)at(base + r); };
  ReadWs L;
  L.md = take((size_t)B * d * 4);
  L.y = take((size_t)B * d * 4);
  L.P = take(M * d * 4);
  L.H = take(M * d * 4);
  L.parts = take(M * 32 * 4);
  L.splitk = (float*)at(base + o);
  L.splitk_bytes = sgemm_workspace_bytes(B, d, d);
  const size_t fp32 = o + L.splitk_bytes;
  L.tc = at((base + fp32 + 1023) & ~(uintptr_t)1023);
  L.slab = align1k(M * d * 2 * (prec == MAC_PREC_TC32 ? 2 : 1));
  L.bytes = fp32 + (prec == MAC_PREC_BF16 ? 5 * L.slab + 1024 : prec == MAC_PREC_TC32 ? 2 * L.slab + 1024 : 0);
  return L;
}

// `inv` of every precision, the step-invariant P = KB @ Wx + bx and Q = P @ Wm[d:2d, :] + bm:
//   MAC_PREC_FP32  [P | Q] fp32 [BN, d]
//   MAC_PREC_TC32  [P | Q] fp32, then 1 KB aligned a bf16 [BN, 2d] hi | lo scratch for the splits of KB and P
//   MAC_PREC_BF16  1 KB aligned: [P | Q] bf16 slabs, then the fused read step's logits, one per row [BN]
//   MAC_PREC_FP8   1 KB aligned: P8 e4m3 [BN, d] | sP [BN] | Q bf16 | logits [BN] | P bf16, each slab 1 KB aligned
// inv may be NULL when only `bytes` is wanted.
struct ReadInv {
  void *P, *Q, *split;
  float *logits, *sP;
  uint8_t* P8;
  size_t bytes;      // mac_read_invariant_bytes
};
inline ReadInv read_inv_layout(int prec, const void* inv, int B, int N, int d) {
  const size_t M = (size_t)B * N, f32 = M * d * 4, b16 = align1k(M * d * 2);
  const uintptr_t p = reinterpret_cast<uintptr_t>(inv), a = (p + 1023) & ~(uintptr_t)1023;
  ReadInv L{};
  if (prec == MAC_PREC_BF16) {
    L.P = at(a); L.Q = at(a + b16); L.logits = (float*)at(a + 2 * b16);
    L.bytes = 2 * b16 + M * 4 + 1024;
  } else if (prec == MAC_PREC_FP8) {
    const size_t o_sP = align1k(M * d), o_Q = o_sP + align1k(M * 4), o_lg = o_Q + b16, o_P = o_lg + align1k(M * 4);
    L.P8 = (uint8_t*)at(a); L.sP = (float*)at(a + o_sP); L.Q = at(a + o_Q); L.logits = (float*)at(a + o_lg); L.P = at(a + o_P);
    L.bytes = o_P + b16 + 1024;
  } else {
    L.P = at(p); L.Q = at(p + f32);
    L.split = at((p + 2 * f32 + 1023) & ~(uintptr_t)1023);
    L.bytes = prec == MAC_PREC_TC32 ? 2 * f32 + align1k(M * 2 * d * 2) + 2048 : 2 * f32 + 256;
  }
  return L;
}

// ------------------------------------------------------------------------------------------------ helper kernels
// training mode: bf16 copy of dropout(KB) for this step (ops.py:678), same Philox stream as the fp32 path
__global__ void dropout_cast_bf16_kernel(const float4* __restrict__ x, uint2* __restrict__ out, uint32_t thresh,
                                         float scale, uint64_t seed, int site, int step, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = x[i];
  const Philox4 r = philox4x32_10(seed, (uint64_t)i, (uint32_t)site, (uint32_t)step);
  const float a = ((r.x >> 8) >= thresh) ? v.x * scale : 0.f, b = ((r.y >> 8) >= thresh) ? v.y * scale : 0.f;
  const float c = ((r.z >> 8) >= thresh) ? v.z * scale : 0.f, d = ((r.w >> 8) >= thresh) ? v.w * scale : 0.f;
  out[i] = make_uint2(pack_bf16(a, b), pack_bf16(c, d));
}

// PY[m, :] = P[m, :] * y[m / rows_per_batch, :]   (8 bf16 per thread)
__global__ void scale_rows_bf16_kernel(const uint4* __restrict__ P, const float* __restrict__ y, uint4* __restrict__ out,
                                       int rows_per_batch, int d, long long n8) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const long long e = i * 8;
  const int c = (int)(e % d);
  const long long b = (e / d) / rows_per_batch;
  const uint4 v = P[i];
  const float4 y0 = __ldg(reinterpret_cast<const float4*>(y + b * d + c));
  const float4 y1 = __ldg(reinterpret_cast<const float4*>(y + b * d + c + 4));
  auto lo = [](uint32_t w) { return __uint_as_float(w << 16); };
  auto hi = [](uint32_t w) { return __uint_as_float(w & 0xffff0000u); };
  out[i] = make_uint4(pack_bf16(lo(v.x) * y0.x, hi(v.x) * y0.y), pack_bf16(lo(v.y) * y0.z, hi(v.y) * y0.w),
                      pack_bf16(lo(v.z) * y1.x, hi(v.z) * y1.y), pack_bf16(lo(v.w) * y1.z, hi(v.w) * y1.w));
}

// The split-bf16 ("tc32", see tc3_gemm in tc_gemm.cuh) operands of the read unit's products:
// out[m, c] = hi(x[m, c] * y[m / rows_per_batch, c]), out[m, d + c] = lo(...)     (y == NULL: plain split); 4 columns / thread
__global__ void split_rows_kernel(const float4* __restrict__ x, const float* __restrict__ y, uint2* __restrict__ out,
                                  int rows_per_batch, int d, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int d4 = d / 4;
  const long long m = i / d4;
  const int c4 = (int)(i - m * d4);
  float4 v = x[i];
  if (y) {
    const float4 s = __ldg(reinterpret_cast<const float4*>(y + (m / rows_per_batch) * d) + c4);
    v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
  }
  const uint32_t h01 = pack_bf16(v.x, v.y), h23 = pack_bf16(v.z, v.w);
  const uint32_t l01 = pack_bf16(v.x - __uint_as_float(h01 << 16), v.y - __uint_as_float(h01 & 0xffff0000u));
  const uint32_t l23 = pack_bf16(v.z - __uint_as_float(h23 << 16), v.w - __uint_as_float(h23 & 0xffff0000u));
  uint2* row = out + m * (2 * d4);
  row[c4] = make_uint2(h01, h23);
  row[d4 + c4] = make_uint2(l01, l23);
}
inline int split_rows_launch(const float* x, const float* y, void* out, int rows_per_batch, int d, long long M,
                             cudaStream_t stream) {
  const long long n4 = M * d / 4;
  split_rows_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(x), y,
                                                                      reinterpret_cast<uint2*>(out), rows_per_batch, d, n4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// The training form's splits (read_tc32_train):
struct SplitRowsArgs {
  const float* y = nullptr;    // row scale y[m / rows_per_batch, c] (NULL: none)
  int rows_per_batch = 1;
  int both = 0;                // also write the unscaled x at columns d .. 2d of each half ([x*y | x] per half)
  uint32_t thresh = 0;         // dropout(x) with the forward's Philox stream (0: none): one draw per aligned column quad of
  float scale = 1.f;           //   element index m*d + c (mac_dropout_fwd's, dropout_cast_bf16_kernel's numbering)
  uint64_t seed = 0;
  int site = 0, step = 0;
};
// out[m, c] = hi(v), out[m, H + c] = lo(v) with v = dropout(x)[m, c] (* y[m / rows_per_batch, c]) and H = d (both: H = 2d,
// and the unscaled x goes to columns d + c and H + d + c); 4 columns / thread
__global__ void split_rows_train_kernel(const float4* __restrict__ x, uint2* __restrict__ out, int d, long long n4,
                                        const SplitRowsArgs a) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const int d4 = d / 4;
  const long long m = i / d4;
  const int c4 = (int)(i - m * d4);
  float4 v = x[i];
  if (a.thresh) {
    const Philox4 r = philox4x32_10(a.seed, (uint64_t)i, (uint32_t)a.site, (uint32_t)a.step);
    v.x = ((r.x >> 8) >= a.thresh) ? v.x * a.scale : 0.f;
    v.y = ((r.y >> 8) >= a.thresh) ? v.y * a.scale : 0.f;
    v.z = ((r.z >> 8) >= a.thresh) ? v.z * a.scale : 0.f;
    v.w = ((r.w >> 8) >= a.thresh) ? v.w * a.scale : 0.f;
  }
  const int half4 = a.both ? 2 * d4 : d4;
  uint2* row = out + m * (2 * half4);
  auto put = [&](float4 u, int col4) {
    const uint32_t h01 = pack_bf16(u.x, u.y), h23 = pack_bf16(u.z, u.w);
    const uint32_t l01 = pack_bf16(u.x - __uint_as_float(h01 << 16), u.y - __uint_as_float(h01 & 0xffff0000u));
    const uint32_t l23 = pack_bf16(u.z - __uint_as_float(h23 << 16), u.w - __uint_as_float(h23 & 0xffff0000u));
    row[col4] = make_uint2(h01, h23);
    row[half4 + col4] = make_uint2(l01, l23);
  };
  if (a.both) put(v, d4 + c4);
  if (a.y) {
    const float4 s = __ldg(reinterpret_cast<const float4*>(a.y + (m / a.rows_per_batch) * d) + c4);
    v.x *= s.x; v.y *= s.y; v.z *= s.z; v.w *= s.w;
  }
  put(v, c4);
}
inline int split_rows_train_launch(const float* x, void* out, int d, long long M, const SplitRowsArgs& a,
                                   cudaStream_t stream) {
  const long long n4 = M * d / 4;
  split_rows_train_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(reinterpret_cast<const float4*>(x),
                                                                            reinterpret_cast<uint2*>(out), d, n4, a);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ forms
// What one mac_read_fwd / mac_read_fwd_inv call was given, with y (this step's memory projection) and the dropout threshold
// and scale filled in by read_fwd_run once y is there.
struct ReadCall {
  const float* kb; const void* kb_bf16; const void* inv; const float* y_pre; const float* memory_in; const float* control;
  const mac_read_weights* w;
  float keep; uint64_t seed; int step; int prec;
  float *info, *att, *save;
  void* ws; size_t ws_bytes;
  int B, N, d;
  cudaStream_t stream;
  const float* y; uint32_t thr; float scale;
};

// Each form below writes the partial logits to L.parts (the fused steps run to the end) and returns MAC_OK or a CUDA error.
// read_fwd_check has checked, for all of them, every pointer the form reads and its alignment, the workspace size, d % 4,
// at most 32 partial logits per row, d % 128 for the tensor-core forms and read_step_supported for the fused steps.

// P = dropout(KB) @ Wx + bx ; H = ELU([P*y, P] @ Wm + bm) ; I1 = H @ Wm2 + bm2 with the logits epilogue, on the FMA pipe;
// P, H, I1 into `save` when given
static int read_fp32_train(const ReadCall& c, const ReadWs& L) {
  const int M = c.B * c.N, d = c.d;
  float* P = c.save ? c.save : L.P;
  float* H = c.save ? c.save + (size_t)M * d : L.H;
  float* I1 = c.save ? c.save + (size_t)2 * M * d : nullptr;
  // P = dropout(KB) @ Wx + bx   (ops.py:678, 688)
  SgemmParams p{};
  p.a_mode = c.thr ? A_DROPOUT : A_SEGS; p.nseg = 1; p.a[0] = c.kb; p.ak[0] = d; p.lda[0] = d;
  p.a_thresh = c.thr; p.a_scale = c.scale; p.seed = c.seed; p.a_site = MAC_SITE_READ_KB; p.step = c.step;
  p.W = c.w->Wx; p.ldw = d; p.M = M; p.N = d; p.K = d;
  p.epi = EPI_BIAS_ACT; p.bias = c.w->bx; p.act = MAC_ACT_NON; p.Y = P; p.ldy = d;
  int st = sgemm_launch(p, nullptr, nullptr, 0, c.stream, false);
  if (st != MAC_OK) return st;
  // H = ELU([P*y, P] @ Wm + bm)   (ops.py:694-719, mac_cell.py:236-238)
  SgemmParams h{};
  h.a_mode = A_ROWSCALE_CONCAT; h.nseg = 1; h.a[0] = P; h.lda[0] = d; h.rowvec = c.y; h.rows_per_batch = c.N;
  h.W = c.w->Wm; h.ldw = d; h.M = M; h.N = d; h.K = 2 * d;
  h.epi = EPI_BIAS_ACT; h.bias = c.w->bm; h.act = MAC_ACT_ELU; h.Y = H; h.ldy = d;
  st = sgemm_launch(h, nullptr, nullptr, 0, c.stream, false);
  if (st != MAC_OK) return st;
  // I1 = H @ Wm2 + bm2 ; I2 = ELU(I1 * control) ; logits = dropout(I2) . wr   (ops.py:325-328, mac_cell.py:248-266)
  SgemmParams g{};
  g.a_mode = A_SEGS; g.nseg = 1; g.a[0] = H; g.ak[0] = d; g.lda[0] = d;
  g.W = c.w->Wm2; g.ldw = d; g.M = M; g.N = d; g.K = d; g.rows_per_batch = c.N;
  g.epi = EPI_READ_LOGITS; g.bias = c.w->bm2; g.Y = I1; g.ldy = d;
  g.ctrl = c.control; g.wr = c.w->wr; g.logit_parts = L.parts;
  g.e_thresh = c.thr; g.e_scale = c.scale; g.e_site = MAC_SITE_READ_INTER; g.seed = c.seed; g.step = c.step;
  return sgemm_launch(g, nullptr, nullptr, 0, c.stream, false);
}

// H = ELU((P*y) @ Wm[0:d, :] + Q) (bm is inside Q), then the logits as in read_fp32_train
static int read_fp32_inv(const ReadCall& c, const ReadWs& L) {
  const int M = c.B * c.N, d = c.d;
  const ReadInv I = read_inv_layout(MAC_PREC_FP32, c.inv, c.B, c.N, d);
  SgemmParams h{};
  h.a_mode = A_ROWSCALE_CONCAT; h.rs_half = d; h.nseg = 1; h.a[0] = (const float*)I.P; h.lda[0] = d; h.rowvec = c.y;
  h.rows_per_batch = c.N; h.W = c.w->Wm; h.ldw = d; h.M = M; h.N = d; h.K = d;
  h.epi = EPI_BIAS_ACT; h.bias = nullptr; h.aux = (const float*)I.Q; h.ldaux = d; h.act = MAC_ACT_ELU; h.Y = L.H; h.ldy = d;
  int st = sgemm_launch(h, nullptr, nullptr, 0, c.stream, false);
  if (st != MAC_OK) return st;
  SgemmParams g{};
  g.a_mode = A_SEGS; g.nseg = 1; g.a[0] = L.H; g.ak[0] = d; g.lda[0] = d;
  g.W = c.w->Wm2; g.ldw = d; g.M = M; g.N = d; g.K = d; g.rows_per_batch = c.N;
  g.epi = EPI_READ_LOGITS; g.bias = c.w->bm2; g.Y = nullptr; g.ldy = d;
  g.ctrl = c.control; g.wr = c.w->wr; g.logit_parts = L.parts; g.e_thresh = 0u; g.e_scale = 1.f;
  return sgemm_launch(g, nullptr, nullptr, 0, c.stream, false);
}

// The three projections on tensor cores: P and P*y, H = ELU([P*y, P] @ Wm + bm), I1 (kept for backward with `save`) with
// the logits epilogue, all bf16 in the workspace slabs; read_fwd_run widens P, H and I1 into `save`
static int read_bf16_train(const ReadCall& c, const ReadWs& L) {
  const int M = c.B * c.N, d = c.d;
  __nv_bfloat16 *P = (__nv_bfloat16*)L.tc, *PY = (__nv_bfloat16*)(L.tc + L.slab), *H = (__nv_bfloat16*)(L.tc + 2 * L.slab);
  const void* kb16 = c.kb_bf16;
  if (c.thr != 0) {
    // A operand of the first projection = dropout(KB) (ops.py:678): TMA cannot mask in flight, so make this step's copy
    void* kbd = L.tc + 4 * L.slab;
    const long long n4 = (long long)M * d / 4;
    dropout_cast_bf16_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, c.stream>>>(
        reinterpret_cast<const float4*>(c.kb), reinterpret_cast<uint2*>(kbd), c.thr, c.scale, c.seed, MAC_SITE_READ_KB, c.step,
        n4);
    MAC_LAUNCH_CHECK();
    kb16 = kbd;
  }
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = c.N; p.ldo = d; p.seed = c.seed; p.step = c.step;
  // P = KB @ Wx + bx ; also P*y
  p.epi = TC_EPI_P; p.bias = c.w->bx; p.out0 = P; p.out1 = PY; p.y = c.y;
  int st = tc_gemm_launch(kb16, d, nullptr, 0, c.w->Wx_bf16, p, c.stream);
  if (st != MAC_OK) return st;
  // H = ELU([P*y, P] @ Wm + bm)
  p.epi = TC_EPI_ACT; p.act = MAC_ACT_ELU; p.bias = c.w->bm; p.out0 = H; p.out1 = nullptr;
  st = tc_gemm_launch(PY, d, P, d, c.w->Wm_bf16, p, c.stream);
  if (st != MAC_OK) return st;
  // logits parts = sum_n ELU((H @ Wm2 + bm2) * control) * wr
  p.epi = TC_EPI_LOGITS; p.bias = c.w->bm2; p.out0 = c.save ? (__nv_bfloat16*)(L.tc + 3 * L.slab) : nullptr;
  p.ctrl = c.control; p.wr = c.w->wr; p.parts = L.parts;
  p.e_thresh = c.thr; p.e_scale = c.scale; p.e_site = MAC_SITE_READ_INTER;
  return tc_gemm_launch(H, d, nullptr, 0, c.w->Wm2_bf16, p, c.stream);
}

// Eval-mode read (readDropout == 1): dropout(KB) == KB at every step and the read weights are shared over the steps
// (mac_cell.py:209-277 is called with the same variables for each of the netLength cells), so P and Q (see read_inv_layout)
// do not depend on the step.  mac_read_invariant computes them once per forward, and each step runs
//   PY = P * y_b ;  H = ELU(PY @ Wm[0:d, :] + Q) ;  logits = ... (unchanged)
// i.e. 2 x d instead of 4 x d MACs per knowledge-base element and step.
static int read_bf16_inv(const ReadCall& c, const ReadWs& L) {
  const int M = c.B * c.N, d = c.d;
  const ReadInv I = read_inv_layout(MAC_PREC_BF16, c.inv, c.B, c.N, d);
  __nv_bfloat16 *PY = (__nv_bfloat16*)(L.tc + L.slab), *H = (__nv_bfloat16*)(L.tc + 2 * L.slab);
  const long long n8 = (long long)M * d / 8;
  scale_rows_bf16_kernel<<<(unsigned)((n8 + 255) / 256), 256, 0, c.stream>>>(
      reinterpret_cast<const uint4*>(I.P), c.y, reinterpret_cast<uint4*>(PY), c.N, d, n8);
  MAC_LAUNCH_CHECK();
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = c.N; p.ldo = d;
  // H = ELU(PY @ Wm[0:d] + Q)      (bm is inside Q)
  p.epi = TC_EPI_ADDACT; p.act = MAC_ACT_ELU; p.bias = nullptr; p.out0 = H; p.add = (const __nv_bfloat16*)I.Q;
  int st = tc_gemm_launch(PY, d, nullptr, 0, c.w->Wm_bf16, p, c.stream, 2 * d);
  if (st != MAC_OK) return st;
  p.epi = TC_EPI_LOGITS; p.act = MAC_ACT_NON; p.bias = c.w->bm2; p.out0 = nullptr; p.add = nullptr;
  p.ctrl = c.control; p.wr = c.w->wr; p.parts = L.parts;
  return tc_gemm_launch(H, d, nullptr, 0, c.w->Wm2_bf16, p, c.stream);
}

// Split-bf16 training form: P = dropout(KB) @ Wx + bx, H = ELU([P*y | P] @ Wm + bm) as ONE split product over K = 2d
// (A' = [(P*y)_hi | P_hi | (P*y)_lo | P_lo], W' = split3 of the whole Wm), I1 = H @ Wm2 + bm2, all in fp32 into `save` (P into
// slab 0 and H, I1 not stored without it).  The fp32 layout's P and H regions (contiguous, [M, 4d] bf16 together) hold
// dropout(KB) as hi | lo in their first half, then A' of the H product; slab 1 holds H as hi | lo.
static int read_tc32_train(const ReadCall& c, const ReadWs& L) {
  const int M = c.B * c.N, d = c.d;
  float* P = c.save ? c.save : (float*)L.tc;
  void* s2 = L.P;
  void* Hs = L.tc + L.slab;
  SplitRowsArgs sa;
  sa.thresh = c.thr; sa.scale = c.scale; sa.seed = c.seed; sa.site = MAC_SITE_READ_KB; sa.step = c.step;
  int st = split_rows_train_launch(c.kb, s2, d, M, sa, c.stream);                  // dropout(KB) as hi | lo   (ops.py:678)
  if (st != MAC_OK) return st;
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = c.N; p.ldo = d; p.seed = c.seed; p.step = c.step;
  p.epi = TC_EPI_F32; p.act = MAC_ACT_NON; p.bias = c.w->bx; p.outf = P;
  st = tc3_gemm(s2, d, c.w->Wx_s3, p, c.stream);                              // P = dropout(KB) @ Wx + bx  (ops.py:688)
  if (st != MAC_OK) return st;
  SplitRowsArgs sb;
  sb.y = c.y; sb.rows_per_batch = c.N; sb.both = 1;
  st = split_rows_train_launch(P, s2, d, M, sb, c.stream);                        // [(P*y)_hi | P_hi | (P*y)_lo | P_lo]
  if (st != MAC_OK) return st;
  p.epi = TC_EPI_ACT_SPLIT; p.act = MAC_ACT_ELU; p.bias = c.w->bm; p.outf = c.save ? c.save + (size_t)M * d : nullptr;
  p.out0 = (__nv_bfloat16*)Hs; p.ldo = 2 * d;
  st = tc3_gemm(s2, 2 * d, c.w->Wm_s3, p, c.stream);                          // H = ELU([P*y | P] @ Wm + bm)  (mac_cell.py:236-238)
  if (st != MAC_OK) return st;
  p.epi = TC_EPI_LOGITS; p.act = MAC_ACT_NON; p.bias = c.w->bm2; p.outf = c.save ? c.save + (size_t)2 * M * d : nullptr;
  p.out0 = nullptr; p.ldo = d; p.ctrl = c.control; p.wr = c.w->wr; p.parts = L.parts;
  p.e_thresh = c.thr; p.e_scale = c.scale; p.e_site = MAC_SITE_READ_INTER;
  return tc3_gemm(Hs, d, c.w->Wm2_s3, p, c.stream);                           // I1, logits partial sums  (mac_cell.py:248-266)
}

// Split-bf16 inference form: (P*y) split, H = ELU((P*y) @ Wm[0:d] + Q) as hi | lo, then the logits
static int read_tc32_inv(const ReadCall& c, const ReadWs& L) {
  const int M = c.B * c.N, d = c.d;
  const ReadInv I = read_inv_layout(MAC_PREC_TC32, c.inv, c.B, c.N, d);
  void* PYs = L.tc;
  __nv_bfloat16* Hs = (__nv_bfloat16*)(L.tc + L.slab);
  int st = split_rows_launch((const float*)I.P, c.y, PYs, c.N, d, M, c.stream);   // (P * y_b) as hi | lo       (ops.py:694-703)
  if (st != MAC_OK) return st;
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = c.N;
  p.epi = TC_EPI_ACT_SPLIT; p.act = MAC_ACT_ELU; p.bias = nullptr; p.addf = (const float*)I.Q; p.ldaf = d; p.out0 = Hs;
  p.ldo = 2 * d;
  st = tc3_gemm(PYs, d, c.w->Wma_s3, p, c.stream);                            // H = ELU((P*y) @ Wm[0:d] + Q) as hi | lo
  if (st != MAC_OK) return st;
  p.epi = TC_EPI_LOGITS; p.act = MAC_ACT_NON; p.bias = c.w->bm2; p.addf = nullptr; p.out0 = nullptr; p.ldo = d;
  p.ctrl = c.control; p.wr = c.w->wr; p.parts = L.parts;
  return tc3_gemm(Hs, d, c.w->Wm2_s3, p, c.stream);                           // logits partial sums         (mac_cell.py:248-266)
}

// ------------------------------------------------------------------------------------------------ step-invariant parts
// mac_read_invariant's forms; read_inv_check has checked every pointer each reads, its alignment, inv_bytes, d % 4, and
// d % 128 (tensor-core forms) or read_step_supported (MAC_PREC_FP8).
static int read_fp32_invariant(const float* kb, const mac_read_weights* w, const ReadInv& I, int B, int N, int d,
                               cudaStream_t stream) {
  SgemmParams p{};
  // P = KB @ Wx + bx   (ops.py:688)
  p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = kb; p.ak[0] = d; p.lda[0] = d;
  p.W = w->Wx; p.ldw = d; p.M = B * N; p.N = d; p.K = d;
  p.epi = EPI_BIAS_ACT; p.bias = w->bx; p.act = MAC_ACT_NON; p.Y = (float*)I.P; p.ldy = d;
  int st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
  if (st != MAC_OK) return st;
  // Q = P @ Wm[d:2d, :] + bm   (the un-scaled half of the concat, mac_cell.py:236-238)
  p.a[0] = (const float*)I.P; p.W = w->Wm + (size_t)d * d; p.bias = w->bm; p.Y = (float*)I.Q;
  return sgemm_launch(p, nullptr, nullptr, 0, stream, false);
}

// P and Q in bf16 (MAC_PREC_BF16, and the P and Q that MAC_PREC_FP8 quantises)
static int read_bf16_invariant(const void* kb_bf16, const mac_read_weights* w, const ReadInv& I, int B, int N, int d,
                               cudaStream_t stream) {
  TcGemmParams p{};
  p.M = B * N; p.N = d; p.rows_per_batch = N; p.ldo = d;
  p.epi = TC_EPI_ACT; p.act = MAC_ACT_NON; p.bias = w->bx; p.out0 = (__nv_bfloat16*)I.P;
  int st = tc_gemm_launch(kb_bf16, d, nullptr, 0, w->Wx_bf16, p, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bm; p.out0 = (__nv_bfloat16*)I.Q;
  return tc_gemm_launch(I.P, d, nullptr, 0, reinterpret_cast<const __nv_bfloat16*>(w->Wm_bf16) + d, p, stream, 2 * d);
}

static int read_tc32_invariant(const float* kb, const mac_read_weights* w, const ReadInv& I, int B, int N, int d,
                               cudaStream_t stream) {
  const int M = B * N;
  TcGemmParams p{};
  p.M = M; p.N = d; p.rows_per_batch = N; p.ldo = d; p.epi = TC_EPI_F32; p.act = MAC_ACT_NON;
  int st = split_rows_launch(kb, nullptr, I.split, N, d, M, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bx; p.outf = (float*)I.P;
  st = tc3_gemm(I.split, d, w->Wx_s3, p, stream);                        // P = KB @ Wx + bx            (ops.py:688)
  if (st != MAC_OK) return st;
  st = split_rows_launch((const float*)I.P, nullptr, I.split, N, d, M, stream);
  if (st != MAC_OK) return st;
  p.bias = w->bm; p.outf = (float*)I.Q;
  return tc3_gemm(I.split, d, w->Wmb_s3, p, stream);                     // Q = P @ Wm[d:2d] + bm       (mac_cell.py:236-238)
}

// P and Q exactly as read_bf16_invariant computes them, then P8 and sP from P
static int read_fp8_invariant(const void* kb_bf16, const mac_read_weights* w, const ReadInv& I, int B, int N, int d,
                              cudaStream_t stream) {
  const int st = read_bf16_invariant(kb_bf16, w, I, B, N, d, stream);
  if (st != MAC_OK) return st;
  const int M = B * N;
  quant_rows_e4m3_kernel<<<(M + 7) / 8, 256, 0, stream>>>((const __nv_bfloat16*)I.P, I.P8, I.sP, M);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ checks
// What every form checks first: that it exists (MAC_ERR_UNSUPPORTED), d % 128 for the tensor-core forms (UNSUPPORTED; it
// also covers kb_attend's d % 64 on a bf16 knowledge base), and the operands it reads through TMA (weight packs, knowledge
// base), each present (INVALID) and 16-byte aligned (ALIGN).  `inv`: the operands of mac_read_invariant's part of the form.
static int read_check_form(ReadForm f, bool inv, const float* kb, const void* kb_bf16, const mac_read_weights* w, int d) {
  const bool tc = f == RF_BF16_TRAIN || f == RF_BF16_INV || f == RF_TC32_TRAIN || f == RF_TC32_INV;
  if (f == RF_NONE || (tc && d % 128)) return MAC_ERR_UNSUPPORTED;
  if (!w) return MAC_ERR_INVALID;
  struct { const void* p[4]; int n; } t = {{}, 0};
  const bool bf16_kb = f == RF_BF16_TRAIN || f == RF_BF16_STEP || f == RF_BF16_INV || f == RF_FP8_STEP;
  if (f == RF_BF16_TRAIN) t = {{kb_bf16, w->Wx_bf16, w->Wm_bf16, w->Wm2_bf16}, 4};
  else if (bf16_kb && inv) t = {{kb_bf16, w->Wx_bf16, w->Wm_bf16}, 3};
  else if (f == RF_FP8_STEP) t = {{w->Wm_fp8, w->Wm2_fp8}, 2};
  else if (bf16_kb) t = {{w->Wm_bf16, w->Wm2_bf16}, 2};
  else if (f == RF_TC32_TRAIN) t = {{w->Wx_s3, w->Wm_s3, w->Wm2_s3}, 3};
  else if (f == RF_TC32_INV && inv) t = {{kb, w->Wx_s3, w->Wmb_s3}, 3};
  else if (f == RF_TC32_INV) t = {{w->Wma_s3, w->Wm2_s3}, 2};
  for (int i = 0; i < t.n; ++i)
    if (!t.p[i]) return MAC_ERR_INVALID;
  for (int i = 0; i < t.n; ++i)
    if (!mac_aligned16(t.p[i])) return MAC_ERR_ALIGN;
  // a bf16 knowledge base given to these forms is read (by kb_attend at least) even where it is optional
  return bf16_kb && kb_bf16 && !mac_aligned16(kb_bf16) ? MAC_ERR_ALIGN : MAC_OK;
}

static int read_fwd_check(ReadForm f, const ReadCall& c) {
  const int st = read_check_form(f, false, c.kb, c.kb_bf16, c.w, c.d);
  if (st != MAC_OK) return st;
  if (f == RF_FP8_STEP && (!c.w->Wm_fp8_scale || !c.w->Wm2_fp8_scale)) return MAC_ERR_INVALID;
  // the bf16 and fp8 inference forms read only kb_bf16: the fp32 knowledge base may be absent (host-cast front end)
  const bool kb_opt = c.inv && c.kb_bf16 && (c.prec == MAC_PREC_BF16 || c.prec == MAC_PREC_FP8);
  if ((!c.kb && !kb_opt) || !c.memory_in || !c.control || !c.info || !c.att || !c.ws) return MAC_ERR_INVALID;
  if (c.B <= 0 || c.N <= 0 || c.d <= 0 || (c.d & 3) || !(c.keep > 0.f && c.keep <= 1.f)) return MAC_ERR_INVALID;
  if ((c.kb && !mac_aligned16(c.kb)) || !mac_aligned16(c.memory_in) || !mac_aligned16(c.control) || !mac_aligned16(c.ws))
    return MAC_ERR_ALIGN;
  if (f == RF_BF16_TRAIN && c.save && !mac_aligned16(c.save)) return MAC_ERR_ALIGN;    // widened into with 16-byte stores
  if (c.ws_bytes < read_ws_layout(c.prec, nullptr, c.B, c.N, c.d).bytes) return MAC_ERR_WORKSPACE;
  // the logits GEMM leaves one partial logit per column tile in a [B*N, 32] region
  return read_nparts(f, c.B * c.N, c.d) > 32 ? MAC_ERR_UNSUPPORTED : MAC_OK;
}

static int read_inv_check(ReadForm f, const float* kb, const void* kb_bf16, const mac_read_weights* w, int prec,
                          const void* inv, size_t inv_bytes, int B, int N, int d) {
  const int st = read_check_form(f, true, kb, kb_bf16, w, d);
  if (st != MAC_OK) return st;
  const bool kb_opt = (prec == MAC_PREC_BF16 || prec == MAC_PREC_FP8) && kb_bf16;
  if ((!kb && !kb_opt) || !inv || B <= 0 || N <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  if ((kb && !mac_aligned16(kb)) || !mac_aligned16(inv)) return MAC_ERR_ALIGN;
  return inv_bytes < read_inv_layout(prec, nullptr, B, N, d).bytes ? MAC_ERR_WORKSPACE : MAC_OK;
}

// ------------------------------------------------------------------------------------------------ dispatch
static int read_fwd_run(ReadForm f, ReadCall c) {
  const ReadWs L = read_ws_layout(c.prec, c.ws, c.B, c.N, c.d);
  const int B = c.B, N = c.N, d = c.d, M = B * N;
  const bool drop = c.keep < 1.f;
  c.thr = drop ? keep_threshold(c.keep) : 0u;
  c.scale = drop ? 1.f / c.keep : 1.f;
  // md = dropout(memory_in, keep_read)   (ops.py:679)
  const float* mem = c.memory_in;
  if (drop) {
    const long long n = (long long)B * d;
    dropout_kernel<<<(unsigned)(((n + 3) / 4 + 255) / 256), 256, 0, c.stream>>>(c.memory_in, c.thr, c.scale, c.seed,
                                                                              MAC_SITE_READ_MEM, c.step, L.md, nullptr, n);
    MAC_LAUNCH_CHECK();
    mem = L.md;
  }
  // y = md @ Wy + by   (ops.py:689), into `save` behind P, H, I1 -- unless the caller already has it (mac_write_fwd_next_y)
  c.y = c.y_pre;
  if (!c.y_pre) {
    float* y = c.save ? c.save + (size_t)3 * M * d : L.y;
    SgemmParams p{};
    p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = mem; p.ak[0] = d; p.lda[0] = d;
    p.W = c.w->Wy; p.ldw = d; p.M = B; p.N = d; p.K = d;
    p.epi = EPI_BIAS_ACT; p.bias = c.w->by; p.act = MAC_ACT_NON; p.Y = y; p.ldy = d;
    const int st = sgemm_launch(p, reinterpret_cast<unsigned int*>(c.ws), L.splitk, L.splitk_bytes, c.stream);
    if (st != MAC_OK) return st;
    c.y = y;
  }
  int st = MAC_OK;
  switch (f) {
    case RF_BF16_STEP: {
      const ReadInv I = read_inv_layout(MAC_PREC_BF16, c.inv, B, N, d);
      return read_step_launch(I.P, I.Q, I.logits, c.kb_bf16, c.y, c.control, c.w, c.att, c.info, B, N, d, c.stream);
    }
    case RF_FP8_STEP: {
      const ReadInv I = read_inv_layout(MAC_PREC_FP8, c.inv, B, N, d);
      return read_step_fp8_launch(I.P8, I.sP, I.Q, I.logits, c.kb_bf16, c.y, c.control, c.w, c.att, c.info, B, N, d, c.stream);
    }
    case RF_FP32_TRAIN: st = read_fp32_train(c, L); break;
    case RF_FP32_INV: st = read_fp32_inv(c, L); break;
    case RF_BF16_TRAIN: st = read_bf16_train(c, L); break;
    case RF_BF16_INV: st = read_bf16_inv(c, L); break;
    case RF_TC32_TRAIN: st = read_tc32_train(c, L); break;
    default: st = read_tc32_inv(c, L); break;
  }
  if (st != MAC_OK) return st;
  // att = softmax(logits); info = sum_n att * KB   (original, un-dropped KB: mac_cell.py:271-275)
  const bool kb16 = c.prec == MAC_PREC_BF16 && c.kb_bf16;
  st = mac_kb_attend_fwd(L.parts, read_nparts(f, M, d), c.w->br, kb16 ? c.kb_bf16 : c.kb, kb16, c.att, c.info, B, N, d,
                         c.stream);
  if (st != MAC_OK || f != RF_BF16_TRAIN || !c.save) return st;
  // `save` is fp32 for every precision: widen the chain's bf16 P, H and I1
  const void* src[3] = {L.tc, L.tc + 2 * L.slab, L.tc + 3 * L.slab};
  float* dst[3] = {c.save, c.save + (size_t)M * d, c.save + (size_t)2 * M * d};
  return widen3_bf16_launch(src, dst, 3, (long long)M * d, c.stream);
}

}  // namespace mac

// ------------------------------------------------------------------------------------------------ entry points
extern "C" size_t mac_read_workspace_bytes(int B, int N, int d, int prec) {
  return read_ws_layout(prec, nullptr, B, N, d).bytes;
}
extern "C" size_t mac_read_invariant_bytes(int B, int N, int d, int prec) {
  return read_inv_layout(prec, nullptr, B, N, d).bytes;
}

extern "C" int mac_read_invariant(const float* kb, const void* kb_bf16, const mac_read_weights* w, int prec, void* inv,
                                  size_t inv_bytes, int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const ReadForm f = read_form(prec, true, kb_bf16 != nullptr, read_step_supported(B, N, d));
  const int st = read_inv_check(f, kb, kb_bf16, w, prec, inv, inv_bytes, B, N, d);
  if (st != MAC_OK) return st;
  const ReadInv I = read_inv_layout(prec, inv, B, N, d);
  switch (f) {
    case RF_BF16_STEP: case RF_BF16_INV: return read_bf16_invariant(kb_bf16, w, I, B, N, d, stream);
    case RF_TC32_INV: return read_tc32_invariant(kb, w, I, B, N, d, stream);
    case RF_FP8_STEP: return read_fp8_invariant(kb_bf16, w, I, B, N, d, stream);
    default: return read_fp32_invariant(kb, w, I, B, N, d, stream);
  }
}

extern "C" int mac_read_fwd(const float* kb, const void* kb_bf16, const float* memory_in, const float* control,
                            const mac_read_weights* w, float keep_read, uint64_t seed, int step, int prec, float* info,
                            float* att, float* save, void* workspace, size_t workspace_bytes, int B, int N, int d,
                            mac_stream_t stream_) {
  const ReadCall c{kb, kb_bf16, nullptr, nullptr, memory_in, control, w, keep_read, seed, step, prec, info, att, save,
                   workspace, workspace_bytes, B, N, d, reinterpret_cast<cudaStream_t>(stream_), nullptr, 0u, 1.f};
  const ReadForm f = read_form(prec, false, kb_bf16 != nullptr, read_step_supported(B, N, d));
  const int st = read_fwd_check(f, c);
  return st != MAC_OK ? st : read_fwd_run(f, c);
}

extern "C" int mac_read_fwd_inv(const float* kb, const void* kb_bf16, const void* inv, const float* y_pre,
                                const float* memory_in, const float* control, const mac_read_weights* w, int prec,
                                float* info, float* att, void* workspace, size_t workspace_bytes, int B, int N, int d,
                                mac_stream_t stream_) {
  if (!inv || !mac_aligned16(inv) || (y_pre && !mac_aligned16(y_pre))) return MAC_ERR_INVALID;
  const ReadCall c{kb, kb_bf16, inv, y_pre, memory_in, control, w, 1.f, 0, 0, prec, info, att, nullptr,
                   workspace, workspace_bytes, B, N, d, reinterpret_cast<cudaStream_t>(stream_), nullptr, 0u, 1.f};
  const ReadForm f = read_form(prec, true, kb_bf16 != nullptr, read_step_supported(B, N, d));
  const int st = read_fwd_check(f, c);
  return st != MAC_OK ? st : read_fwd_run(f, c);
}

extern "C" int mac_read_step_fused(const void* inv, const void* kb_bf16, const float* y, const float* control,
                                   const mac_read_weights* w, float* info, float* att, int B, int N, int d,
                                   mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!inv || !kb_bf16 || !y || !control || !w || !info || !att || B <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  if (!mac_aligned16(inv) || !mac_aligned16(kb_bf16) || !mac_aligned16(y) || !mac_aligned16(control)) return MAC_ERR_ALIGN;
  if (!mac_b200_device_ok()) return MAC_ERR_ARCH;
  if (!read_step_supported(B, N, d)) return MAC_ERR_UNSUPPORTED;
  if (!w->Wm_bf16 || !w->Wm2_bf16) return MAC_ERR_INVALID;
  const ReadInv I = read_inv_layout(MAC_PREC_BF16, inv, B, N, d);
  return read_step_launch(I.P, I.Q, I.logits, kb_bf16, y, control, w, att, info, B, N, d, stream);
}
extern "C" int mac_read_step_fused_supported(int B, int N, int d) { return read_step_supported(B, N, d) ? 1 : 0; }
