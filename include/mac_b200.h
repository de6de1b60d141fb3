/*
 * mac_b200.h -- C ABI of the GPU-native MAC reasoning cell (libmac_b200.so, sm_90a).
 *
 * Drop-in boundary for the hot path of stanfordnlp/mac-network: the three units of
 * `MACCell` (reference `mac_cell.py`) plus the slice of `ops.py` they call.  The reference
 * has no FFI of its own (it is a TensorFlow-1 graph; the only runtime boundary is
 * `sess.run`, `model.py:746`), so the entry points below are what a binding for this path
 * would bind: one call per reference function, same argument meaning, same order of
 * arithmetic.  INTEGRATION.md shows the Python (ctypes) stub that puts them behind the
 * reference's `MACCell.control/read/write/__call__`.
 *
 * Conventions (SURVEY.md section 8(b)):
 *   - all pointers are DEVICE pointers owned by the caller, row-major, feature dim fastest,
 *     16-byte aligned; float32 unless stated; `lengths` is int32.
 *   - sizes: B batch, S question length, N knowledge-base cells (H*W), d = memDim = ctrlDim =
 *     attDim.  d % 64 == 0 is required by the tensor-core path, d % 4 == 0 by the fp32 path.
 *   - no allocation inside: scratch comes from `workspace` (size from the matching
 *     `*_workspace_bytes`).  Every call is asynchronous on `stream` (a cudaStream_t).
 *   - return value: 0 ok; <0 one of MAC_ERR_*; >0 a cudaError_t.  No exceptions, no global
 *     state except a lazily created per-device attribute cache; re-entrant across streams
 *     as long as workspaces are not shared.
 *   - the inputs (knowledge base, words, question vector) are never written.
 */
#ifndef MAC_B200_H_
#define MAC_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MAC_B200_ABI_VERSION 1

typedef void* mac_stream_t; /* cudaStream_t */

enum {
  MAC_OK = 0,
  MAC_ERR_INVALID = -1,     /* bad size / null pointer */
  MAC_ERR_ALIGN = -2,       /* pointer or leading dimension not 16-byte aligned */
  MAC_ERR_UNSUPPORTED = -3, /* flag combination outside the fused path */
  MAC_ERR_WORKSPACE = -4,   /* workspace too small */
  MAC_ERR_ARCH = -5         /* not an sm_90 device / tensor-map driver entry point missing */
};

/* ops.activations (ops.py:181-187) with the config.relu switch (ops.py:161-179) resolved by the caller */
enum { MAC_ACT_NON = 0, MAC_ACT_TANH = 1, MAC_ACT_SIGMOID = 2, MAC_ACT_ELU = 3, MAC_ACT_RELU = 4 };

/* arithmetic of the d x d projections */
enum {
  MAC_PREC_FP32 = 0, /* fp32 FMA pipe, fp32 accumulate: the <=1e-4 parity configuration */
  MAC_PREC_BF16 = 1, /* bf16 operands on wgmma tensor cores, fp32 accumulate: the headline configuration */
  MAC_PREC_TC32 = 2, /* split-bf16 on wgmma (x = hi + lo, three of the four partial products, fp32 accumulate): a tensor-core
                        path inside the 1e-4 parity bar.  Inference form: mac_read_invariant / mac_read_fwd_inv.  Training
                        form: mac_read_fwd without `inv` (any keep_read, `save` = [P | H | I1 | y] in fp32 as MAC_PREC_FP32
                        writes it; needs the Wx_s3, Wm_s3 and Wm2_s3 packs) and its backward mac_read_bwd_tc32.  fp32
                        knowledge base; d % 128 == 0 (else MAC_ERR_UNSUPPORTED before any launch); everything outside the
                        three [B*N, .] projections as in MAC_PREC_FP32 */
  MAC_PREC_FP8 = 3   /* e4m3 operands on wgmma for the two per-step products of the read step, fp32 accumulate, per-row /
                        per-column fp32 scales (csrc/read_step_fp8.cuh).  Inference form only (mac_read_invariant /
                        mac_read_fwd_inv), the shapes of mac_read_step_fused_supported, bf16 knowledge base; P and Q as in
                        MAC_PREC_BF16.  About ten times the bf16 error: opt-in, never a default */
};

int mac_b200_abi_version(void);
const char* mac_b200_strerror(int status);
/* 1 if the current device is compute capability 9.0 (wgmma/TMA available) */
int mac_b200_device_ok(void);
/* number of kernels this library has launched (or recorded into a stream capture) in this process */
long long mac_b200_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * ops.linear (ops.py:298-333) / ops.multiply (ops.py:50-59)
 *   y[M,n_out] = act( concat_k(x_0 .. x_{nseg-1})[M, sum k_i] @ W[sum k_i, n_out] + b[n_out] + bias_const )
 * The concat of the reference (ops.py:65-78, mac_cell.py:339-347) is never materialised: the
 * segments are separate pointers with their own leading dimension `ldx[i]` (elements).
 * `b` may be NULL.  The reference's nested "<name>_2" layer (ops.py:325-328) is a second call.
 * --------------------------------------------------------------------------------------------- */
int mac_linear_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg,
                   const float* W, const float* b, float bias_const, int act,
                   float* y, int ldy, int M, int n_out,
                   void* workspace, size_t workspace_bytes, mac_stream_t stream);
size_t mac_linear_workspace_bytes(int M, int K, int n_out);

/* ------------------------------------------------------------------------------------------------
 * Control unit, attention part (mac_cell.py:155-181 with controlConcatWords/controlProj off):
 *   logits[t,b,s] = sum_k cc[t,b,k] * in_words[b,s,k] * w_logit[k] + b_logit          (155, 169)
 *   att[t,b,:]    = softmax_s( logits - 1e30 * [s >= lengths[b]] )                     (175, ops.py:243-247)
 *   out[t,b,:]    = sum_s att[t,b,s] * out_words[b,s,:]                                (181, ops.py:149-150)
 * `nsteps` independent query vectors share one pass over the words (with controlFeedPrev off the
 * whole control chain is memory-independent, so all netLength steps go in one launch).
 * The same kernel is the write unit's self-attention (mac_cell.py:324-330): in_words = history of
 * controls, out_words = history of memories, S = i+1, lengths = NULL, cc = projected control.
 * Strides are in elements: cc[t,b,:] at cc + t*cc_tstride + b*cc_bstride; word row (b,s) at
 * words + b*bstride + s*rstride (rstride == d: one bulk copy per batch row; step-major history buffers
 * use rstride = B*d, bstride = d).  att is [nsteps,B,S] and out [nsteps,B,d], both contiguous.
 * --------------------------------------------------------------------------------------------- */
int mac_control_attend_fwd(const float* cc, long long cc_tstride, long long cc_bstride,
                           const float* in_words, long long in_bstride, long long in_rstride,
                           const float* out_words, long long out_bstride, long long out_rstride,
                           const int32_t* lengths, const float* w_logit, float b_logit,
                           float* att, float* out, int nsteps, int B, int S, int d, mac_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Read unit (mac_cell.py:209-277) on the shipped-config path
 *   (readProjInputs, readMemConcatKB, readMemConcatProj, readMemProj, readCtrl, MUL/MUL, ELU/ELU):
 *   md = dropout(memory_in, keep_read)                      (ops.py:678-679; memory_in already carries the
 *                                                            variational mask, mac_cell.py:214-217)
 *   P  = dropout(KB, keep_read) @ Wx + bx                   (ops.py:688)      [B*N, d]
 *   y  = md @ Wy + by                                       (ops.py:689)      [B, d]
 *   H  = ELU([P * y, P] @ Wm + bm)                          (ops.py:700-719, mac_cell.py:236-238)
 *   I1 = H @ Wm2 + bm2                                      (ops.py:325-328)
 *   I2 = ELU(I1 * control)                                  (mac_cell.py:248-250, 262)
 *   kl = dropout(I2, keep_read) . wr + br                   (mac_cell.py:266, ops.py:312-317)
 *   att = softmax_n(kl);  info = sum_n att * KB             (ops.py:143, 149-150; original KB, mac_cell.py:271-275)
 * Training: keep_read < 1 draws Philox4x32-10 masks from (seed, step) (see mac_dropout_uniform);
 * `save` (may be NULL, 16-byte aligned) receives P, H, I1 ([B*N,d] each, in that order) and y ([B,d]) for backward, in
 * fp32 for every precision: MAC_PREC_BF16 computes P, H and I1 in bf16 and widens them into `save` (one more launch).
 * MAC_PREC_FP32 takes every d % 4 == 0 up to d <= 2048 when B*N < 512 and d <= 4096 otherwise (at most 32 partial logits
 * per row, one per 64- or 128-column tile).  MAC_PREC_BF16 and MAC_PREC_TC32 take d % 128 == 0 up to d <= 4096 and need
 * the packs they read (see mac_read_weights; MAC_PREC_BF16 also kb_bf16).
 * mac_read_fwd, mac_read_fwd_inv and mac_read_invariant return every MAC_ERR_* before any launch and before any write:
 * a refused call leaves info, att, save, inv and the workspace as they were.
 * --------------------------------------------------------------------------------------------- */
typedef struct mac_read_weights {
  const float* Wx;  const float* bx;   /* read/mulmemInter/linearLayerprojX            [d,d],[d]  */
  const float* Wy;  const float* by;   /* read/mulmemInter/linearLayerprojY            [d,d],[d]  */
  const float* Wm;  const float* bm;   /* read/linearLayermemKbProj                    [2d,d],[d] */
  const float* Wm2; const float* bm2;  /* read/linearLayermemKbProj/linearLayermemKbProj_2 [d,d],[d] */
  const float* wr;  float br;          /* read/inter2att/inter2logits/linearLayerlogits [d], []   */
  /* bf16 [out,in] copies of Wx, Wm, Wm2 (mac_pack_weight_bf16); NULL for MAC_PREC_FP32 */
  const void* Wx_bf16; const void* Wm_bf16; const void* Wm2_bf16;
  /* MAC_PREC_TC32 only: split-bf16 copies [out, 3*in] = [hi | hi | lo] (mac_pack_weight_split3) of Wx, Wm[0:d], Wm[d:2d], Wm2 */
  const void* Wx_s3; const void* Wma_s3; const void* Wmb_s3; const void* Wm2_s3;
  /* MAC_PREC_FP8 only (read under no other precision): e4m3 [out, in] copies of Wm[0:d] and Wm2 with their per-output-column
   * fp32 scales [d] (mac_pack_weight_fp8) */
  const void* Wm_fp8; const float* Wm_fp8_scale; const void* Wm2_fp8; const float* Wm2_fp8_scale;
  /* MAC_PREC_TC32 training form only (mac_read_fwd without `inv`): split-bf16 copy [d, 6d] of the whole Wm [2d, d]
   * (mac_pack_weight_split3 with K = 2d), the B operand of H = ELU([P*y | P] @ Wm + bm) as one product over K = 2d */
  const void* Wm_s3;
} mac_read_weights;

int mac_read_fwd(const float* kb, const void* kb_bf16, const float* memory_in, const float* control,
                 const mac_read_weights* w, float keep_read, uint64_t seed, int step, int prec,
                 float* info, float* att, float* save,
                 void* workspace, size_t workspace_bytes, int B, int N, int d, mac_stream_t stream);
size_t mac_read_workspace_bytes(int B, int N, int d, int prec);

/* Inference form of the read unit.  With readDropout == 1 (eval: mac_cell.py:209-277 runs with keep = 1.0) the
 * dropout on the knowledge base is the identity and the read weights are the same variables at every one of the
 * netLength steps, so two of the three big projections do not depend on the step:
 *   P = KB @ Wx + bx                 (ops.py:688)
 *   Q = P @ Wm[d:2d, :] + bm         (the un-scaled half of the [P*y, P] concat, mac_cell.py:236-238)
 * mac_read_invariant computes `inv` = [P | Q] once per forward (fp32 for MAC_PREC_FP32, bf16 for MAC_PREC_BF16; for
 * MAC_PREC_FP8 `inv` = [P8 | sP | Q | logit scratch | P]: P8 = e4m3(P / sP) with sP = max|P row| / 448 per row, Q and P bf16,
 * from kb_bf16 and the bf16 packs Wx_bf16 / Wm_bf16);
 * mac_read_fwd_inv is mac_read_fwd(keep_read = 1, save = NULL) with H = ELU((P*y) @ Wm[0:d, :] + Q): the same
 * function with 2d instead of 4d multiply-adds per knowledge-base element and step.  With MAC_PREC_FP8 it runs
 * read_step_fp8_kernel + kb_attend (see MAC_PREC_FP8); an unsupported shape or a missing kb_bf16 / inv returns
 * MAC_ERR_UNSUPPORTED before any launch, and so does mac_read_fwd with MAC_PREC_FP8. */
size_t mac_read_invariant_bytes(int B, int N, int d, int prec);
int mac_read_invariant(const float* kb, const void* kb_bf16, const mac_read_weights* w, int prec, void* inv,
                       size_t inv_bytes, int B, int N, int d, mac_stream_t stream);
int mac_read_fwd_inv(const float* kb, const void* kb_bf16, const void* inv, const float* y_pre,
                     const float* memory_in, const float* control, const mac_read_weights* w, int prec,
                     float* info, float* att, void* workspace, size_t workspace_bytes, int B, int N, int d,
                     mac_stream_t stream);
/* y_pre (may be NULL): y = memory_in @ Wy + by [B, d] when the caller already has it, see mac_write_fwd_next_y. */
/* mac_read_fwd with MAC_PREC_TC32 (the training form): dropout(KB) is split into [hi | lo] with the fp32 path's Philox
 * numbering; P = KBd @ Wx + bx (Wx_s3), H = ELU([P*y | P] @ Wm + bm) as ONE product over K = 2d (Wm_s3, the split3 pack of
 * the whole [2d, d] Wm) and I1 = H @ Wm2 + bm2 (Wm2_s3, the read-inter dropout in the logits epilogue) are split-bf16 products;
 * P, H and I1 are stored in fp32 as their epilogues computed them, then kb_attend on the fp32 knowledge base.  Any B*N.  The
 * workspace query is unchanged: the split operands reuse the fp32 layout's P and H regions and the tc32 slabs behind it. */

/* One inference read step (csrc/read_step.cuh): given inv = [P | Q] from mac_read_invariant (bf16), the bf16 knowledge base,
 * y = memory @ Wy + by [B, d] (ops.py:689) and the control state [B, d], computes
 *   H = ELU((P*y) @ Wm[0:d] + Q);  logits = ELU((H @ Wm2 + bm2) * control) . wr + br;  att = softmax_n(logits);
 *   info = sum_n att * KB                                     (mac_cell.py:230-275 at readDropout == 1)
 * as one wgmma kernel over 64-row tiles of the knowledge base (P*y, H and I2 stay on the SM; one logit per row) and the
 * kb_attend launch (softmax + weighted sum).  The logits go to the scratch that mac_read_invariant_bytes reserves behind
 * [P | Q] in `inv`, one float per row (so `inv` is read AND written by this call: one call at a time per `inv`).
 * Returns MAC_ERR_UNSUPPORTED unless mac_read_step_fused_supported(B, N, d) (d == 512, N <= 256, B < 2^22).
 * mac_read_fwd_inv with MAC_PREC_BF16 and kb_bf16 dispatches to it whenever the shape is supported, and runs other
 * shapes as four launches (scale, two GEMMs, kb_attend). */
int mac_read_step_fused(const void* inv, const void* kb_bf16, const float* y, const float* control,
                        const mac_read_weights* w, float* info, float* att, int B, int N, int d, mac_stream_t stream);
int mac_read_step_fused_supported(int B, int N, int d);

/* The HBM-bound tail of the read unit on its own (ops.py:143, 149-150):
 *   att[b,:] = softmax_n( sum_p logit_parts[(b*N+n)*nparts + p] + br );  info[b,:] = sum_n att[b,n] * KB[b,n,:]
 * kb_is_bf16 != 0: `kb` points at bf16 data.  Needs d % 4 == 0 for an fp32 and d % 64 == 0 for a bf16 knowledge base. */
int mac_kb_attend_fwd(const float* logit_parts, int nparts, float br, const void* kb, int kb_is_bf16,
                      float* att, float* info, int B, int N, int d, mac_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Write unit (mac_cell.py:305-375) for writeInputs=BOTH, writeMemProj, optional self-attention
 * summary and gate:
 *   m' = [memory, info(, self_smry)] @ Ww + bw                       (339-352)
 *   z  = sigmoid(control @ Wg + bg + gate_bias); m' = m'*z + memory*(1-z)   (358-367)   if Wg != NULL
 * gate_out (may be NULL) receives z (attentions["gate"], mac_cell.py:365).
 * --------------------------------------------------------------------------------------------- */
int mac_write_fwd(const float* memory, const float* info, const float* self_smry, const float* control,
                  const float* Ww, const float* bw, const float* Wg, const float* bg, float gate_bias,
                  float* new_memory, float* gate_out,
                  void* workspace, size_t workspace_bytes, int B, int d, mac_stream_t stream);
size_t mac_write_workspace_bytes(int B, int d);

/* Inference, plain write unit (writeInputs=BOTH, writeMemProj; no self-attention, no gate, no activation): the new
 * memory and the NEXT step's read-unit memory projection are both linear in [memory, info] (no dropout in between
 * when memoryDropout == readDropout == 1), so one GEMM against the folded weight gives both:
 *   new_memory = [memory, info] @ Wf[:, 0:d]  + bf[0:d]         Wf[:, 0:d]  = Ww          (mac_cell.py:339-352)
 *   y_next     = [memory, info] @ Wf[:, d:2d] + bf[d:2d]        Wf[:, d:2d] = Ww @ Wy, bf[d:2d] = bw @ Wy + by
 *                                                                (= new_memory @ Wy + by, ops.py:689)
 * Wf is [2d, 2d] row-major, built by the caller once per parameter update. */
int mac_write_fwd_next_y(const float* memory, const float* info, const float* Wf, const float* bf,
                         float* new_memory, float* y_next, void* workspace, size_t workspace_bytes, int B, int d,
                         mac_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Elementwise helpers used by the Python-composed (non-fused) flag combinations and by state init.
 * --------------------------------------------------------------------------------------------- */
/* out[b,n,:] = (x[b,n,:] + mul_bias) * (v[b,:] + mul_bias)     ops.mul MUL (ops.py:694-703); x may equal out */
int mac_bcast_mul(const float* x, const float* v, float mul_bias, float* out, int B, int N, int d, mac_stream_t stream);
/* out = act(x) elementwise */
int mac_activation(const float* x, int act, float* out, long long n, mac_stream_t stream);
/* fp32 <- bf16 widening of up to three equally long slabs in ONE launch (n elements each, n % 8 == 0, 16-byte aligned): the
 * activations the tensor-core training forward leaves in bf16, read in fp32 by the backward kernels */
int mac_widen_bf16(const void* const* src_bf16, float* const* dst, int nslab, long long n, mac_stream_t stream);
/* ---- general (unfused) path: primitives for the flag combinations outside mac_read_fwd / mac_write_fwd ---- */
/* out[r] = sum_s x_s[r,:] . w[k-range of s] + b      (ops.linear with outDim == 1 on concatenated inputs, ops.py:316-317) */
int mac_rowdot_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* w, float b,
                   float* out, long long R, mac_stream_t stream);
/* att = softmax(logits - 1e30*[m >= len]) (lengths may be NULL); out[b,:] = sum_m att[b,m] * feats[b,m,:]   (ops.py:143-150, 243-247) */
int mac_attend_fwd(const float* logits, const int32_t* lengths, const float* feats, long long feat_bstride,
                   long long feat_rstride, float* att, float* out, int B, int M, int d, mac_stream_t stream);
/* ops.mul interaction on a broadcast operand (ops.py:694-713): mode 0 MUL (x+mb)*(v+mb); 1 BL x*v + bias[k]; 2 ADD tanh(x+v) */
int mac_bcast_op(const float* x, const float* v, int mode, float mul_bias, const float* bias, float* out,
                 int B, int N, int d, mac_stream_t stream);
/* variational / plain dropout: out = x / keep * [u >= 1-keep]  with u from mac_dropout_uniform(seed, site, step) */
int mac_dropout_fwd(const float* x, float keep, uint64_t seed, int site, int step, float* out, long long n,
                    mac_stream_t stream);
/* the uniforms the kernels draw, materialised (tests feed them to the oracle): u[i] in [0,1), 24 bits */
int mac_dropout_uniform(uint64_t seed, int site, int step, float* u, long long n, mac_stream_t stream);
/* fp32 -> bf16 (round-to-nearest-even), plain row-major; used once per forward for KB and per weight update */
int mac_cast_bf16(const float* x, void* out_bf16, long long n, mac_stream_t stream);

/* HOST-side twin of mac_cast_bf16 for the host-buffer front end (mac_network_b200/serving.py): src and dst are host
 * pointers; round-to-nearest-even, bit-identical to the device cast for finite inputs; `nthreads` worker threads of a
 * persistent pool inside the library (<= 1: the calling thread).  Lets the bf16 path copy 2 instead of 4 bytes per
 * knowledge-base element over PCIe. */
int mac_host_cast_bf16(const float* src, void* dst_bf16, long long n, int nthreads);
/* asynchronous form: _begin posts the job to the pool and returns (one job in flight; a second _begin first waits for
 * the previous job), _end blocks until the posted job is done.  The caller keeps src/dst alive in between. */
int mac_host_cast_bf16_begin(const float* src, void* dst_bf16, long long n, int nthreads);
int mac_host_cast_bf16_end(void);

/* HOST: CRC-32C (Castagnoli) of n bytes continuing from `crc` (0 to start): the checksum TensorFlow's checkpoint format stores
 * per tensor and per index block (mac_network_b200/tf_bundle.py reads / writes real `weights{epoch}.ckpt` files, main.py:163-201). */
uint32_t mac_host_crc32c(const void* data, long long n, uint32_t crc);

/* ------------------------------------------------------------------------------------------------
 * Tensor-core (MAC_PREC_BF16) helpers.
 * mac_pack_weight_bf16: fp32 W[K, n_out] (the reference's [in, out] layout, ops.py:304) -> bf16 Wt[n_out, K], the
 *   K-major B operand wgmma consumes; call once per weight update.
 * mac_linear_tc_fwd: y[M,n_out] = act(x[M,K] @ W + b) with x bf16 row-major and W given as the packed Wt;
 *   fp32 accumulation; output fp32, or bf16 when y_is_bf16 (the form the read-unit chain uses; act in
 *   {NON, ELU}, b required).  Requires K % 64 == 0 and n_out % 128 == 0.
 * --------------------------------------------------------------------------------------------- */
int mac_pack_weight_bf16(const float* W, void* Wt_bf16, int K, int n_out, mac_stream_t stream);
/* fp32 W[K, n_out] -> bf16 Wt3[n_out, 3K] = [hi | hi | lo] (hi = bf16(W), lo = bf16(W - hi)): the B operand of the split-bf16
 * products of MAC_PREC_TC32 (see tc3_gemm in csrc/tc_gemm.cuh).  A row block of a taller weight is passed as W + k0*n_out. */
int mac_pack_weight_split3(const float* W, void* Wt3_bf16, int K, int n_out, mac_stream_t stream);
/* fp32 W[K, n_out] -> e4m3 Wt[n_out, K] = e4m3(W / s_c) (round to nearest even, saturating) with the per-output-column scale
 * col_scale[c] = s_c = max_k |W[k, c]| / 448 (0 for an all-zero column, which packs to zeros): the B operand of the
 * MAC_PREC_FP8 read step.  A row block of a taller weight is passed as W (its first K rows). */
int mac_pack_weight_fp8(const float* W, void* Wt_e4m3, float* col_scale, int K, int n_out, mac_stream_t stream);
int mac_linear_tc_fwd(const void* x_bf16, const void* wt_bf16, const float* b, int act, void* y, int y_is_bf16,
                      int M, int K, int n_out, mac_stream_t stream);

/* The cell's M <= 128 projections on tensor cores (csrc/skinny_tc.cuh) -- ops.linear at mac_cell.py:442-448 (qInput,
 * qInput{i}), 322 (ctrlProj), 352 (newMemory), 363 (gate) and ops.py:689 (projY), the calls whose M is the batch:
 *   y[M, n_out] = epilogue( concat_k(x_0 .. x_{nseg-1})[M, K] @ W + b + bias_const ),  M <= 128, fp32 in / fp32 out.
 * mac_pack_weight_bf16_split: fp32 W[K, n_out] -> bf16 hi and lo halves, both [n_out, K] (K-major), W ~= hi + lo.
 * With wt_lo != NULL the product is three wgmma passes (x_hi W_hi + x_lo W_hi + x_hi W_lo, the activations split in the
 * kernel) accumulated in fp32 registers: fp32-class accuracy (~1e-5) on the tensor pipe, so the recurrent state
 * does not pass through bf16.  wt_lo == NULL: one plain bf16 pass.
 * Epilogue: act in MAC_ACT_*; y2 != NULL sends columns >= n_split to y2[m, n - n_split] (the folded write unit, see
 * mac_write_fwd_next_y); gate_new != NULL selects the write gate z = sigmoid(t), y = gate_new*z + gate_old*(1-z), z stored
 * to gate_z when given (mac_cell.py:358-367).  Needs k_segs[i] % 64 == 0, n_out % 32 == 0, else MAC_ERR_UNSUPPORTED. */
int mac_pack_weight_bf16_split(const float* W, void* hi_bf16, void* lo_bf16, int K, int n_out, mac_stream_t stream);
int mac_linear_tc_small_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg,
                            const void* wt_hi, const void* wt_lo, const float* b, float bias_const, int act,
                            float* y, int ldy, float* y2, int n_split, const float* gate_new, const float* gate_old,
                            float* gate_z, int M, int n_out, mac_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Backward (fp32 path).  The reference differentiates the graph with TF autodiff (model.py:626-636); each forward
 * entry point above has a counterpart here (math: SURVEY.md Appendix E).  "+=" outputs accumulate (zero them once per
 * backward pass).  `*_part` outputs are per-sample partial sums [B, d] (or [B]) to be reduced over B with mac_colsum
 * at the end of the pass -- every reduction has a fixed order, so gradients are deterministic.
 * --------------------------------------------------------------------------------------------- */
/* y = concat(x_s) @ W + b:  dx_s (+)= dy @ W[k-range of s, :]^T (Wt = W^T [n_out, K] row-major); dW += x^T dy; db += colsum(dy) */
int mac_linear_bwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* Wt,
                   const float* dy, int ldy, float* const* dx_segs, const int* ld_dx, const int* dx_accum,
                   float* dW, float* db, int M, int n_out, void* workspace, size_t workspace_bytes, mac_stream_t stream);
/* backward of mac_control_attend_fwd (control unit attention and write-unit self-attention); d_in_words/d_out_words += (they
 * may be the same buffer), dq = gradient w.r.t. cc (optionally accumulated), dw_part [B,d] +=, db_part [B] += */
int mac_control_attend_bwd(const float* cc, long long cc_tstride, long long cc_bstride,
                           const float* in_words, long long in_bstride, long long in_rstride,
                           const float* out_words, long long out_bstride, long long out_rstride,
                           const float* w_logit, const float* att, const float* g_out, long long g_tstride, long long g_bstride,
                           float* d_in_words, float* d_out_words, float* dq, long long dq_tstride, long long dq_bstride,
                           int dq_accumulate, float* dw_part, float* db_part, int nsteps, int B, int S, int d, mac_stream_t stream);
/* backward of mac_kb_attend_fwd: dkl [B,N] = softmax-backward of the logits; dkb [B,N,d] += att (x) dinfo (dkb may be NULL) */
int mac_kb_attend_bwd(const float* kb, const float* att, const float* dinfo, float* dka_scratch, float* dkl,
                      float* dkb, float* dbr_part, int B, int N, int d, mac_stream_t stream);
/* Backward of mac_read_fwd's training forms; `save` is what the forward wrote.  Three forms with the same outputs and
 * accumulation conventions: dkb (may be NULL: not computed) +=, dmem_in =, dcontrol +=, dWx, dWy, dWm, dWm2 += [in, out],
 * dby += [d], the bias and wr gradients as per-sample partials dbx_part, dbm_part, dbm2_part, dwr_part [B, d] +=,
 * dbr_part [B] += (may be NULL); dWy and dby may be NULL (not computed).  Every one returns all its MAC_ERR_* before any
 * launch and any write, so a refused call leaves the outputs and the workspace as they were:
 *   MAC_ERR_INVALID      a required pointer NULL (kb, memory_in, control, w, w->wr, att, save, dinfo, dmem_in, dcontrol,
 *                        Wy_t, dbx_part, dbm_part, dbm2_part, dwr_part, workspace, the form's weights below); B, N or d <= 0;
 *                        d % 4 != 0; keep_read outside (0, 1]
 *   MAC_ERR_UNSUPPORTED  the form's shape limits below
 *   MAC_ERR_ALIGN        kb, memory_in, control, w->wr, save, dinfo, dmem_in, Wy_t, workspace, the form's weights, or a
 *                        given dkb, dWx, dWy, dWm, dWm2 not 16-byte aligned
 *   MAC_ERR_WORKSPACE    workspace_bytes below the form's *_workspace_bytes
 *   MAC_ERR_ARCH         (tensor-core forms) not an sm_90 device
 * mac_read_bwd (MAC_PREC_FP32): the FMA pipe.  Weights: the transposed Wm_t, Wm2_t, and Wx_t when dkb is given; dWx, dWm
 * and dWm2 may be NULL (not computed). */
int mac_read_bwd(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                 const float* Wx_t, const float* Wy_t, const float* Wm_t, const float* Wm2_t,
                 const float* att, const float* save, const float* dinfo, float keep_read, uint64_t seed, int step,
                 float* dkb, float* dmem_in, float* dcontrol, float* dWx, float* dbx_part, float* dWy, float* dby,
                 float* dWm, float* dbm_part, float* dWm2, float* dbm2_part, float* dwr_part, float* dbr_part,
                 void* workspace, size_t workspace_bytes, int B, int N, int d, mac_stream_t stream);
size_t mac_read_bwd_workspace_bytes(int B, int N, int d);
/* mac_read_bwd with its six [B*N, .] products on wgmma tensor cores (bf16 operands, fp32 accumulation; all element-wise
 * work in fp32): dgrad = mac_linear_tc_fwd(bf16(dY), bf16(W) in its own [in,out] layout), wgrad = mac_linear_tc_fwd(bf16(X)^T,
 * bf16(dY)^T) with K = B*N, fed by mac_cast_bf16 / mac_pack_weight_bf16.  Same arguments and accumulation conventions as
 * mac_read_bwd (the transposed fp32 weights are not needed except Wy_t).  Weights: w->Wm, w->Wm2, and w->Wx when dkb is
 * given; dWx, dWm, dWm2 are required.  Needs d % 128 == 0 and (B*N) % 64 == 0, else MAC_ERR_UNSUPPORTED. */
int mac_read_bwd_tc(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                    const float* Wy_t, const float* att, const float* save, const float* dinfo, float keep_read,
                    uint64_t seed, int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx, float* dbx_part,
                    float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2, float* dbm2_part, float* dwr_part,
                    float* dbr_part, void* workspace, size_t workspace_bytes, int B, int N, int d, mac_stream_t stream);
size_t mac_read_bwd_tc_workspace_bytes(int B, int N, int d);
/* Backward of the MAC_PREC_TC32 training forward: mac_read_bwd_tc's arguments and accumulation conventions, with its six
 * [B*N, .] products as split-bf16 products (x = hi + lo, three of the four partial products, fp32 accumulation), so the
 * gradients keep the forward's fp32-class accuracy.  Data gradients: [G_hi | G_lo] against [W_hi | W_hi | W_lo] per row of W
 * in its own [in, out] layout, packed into the workspace on every call.  Weight gradients: ONE split-K launch over the
 * contraction B*N rounded up to 64 (zero columns written on every call), slices summed in a fixed order: reruns are
 * bit-identical.  Weights and required gradients as mac_read_bwd_tc.  Any B*N; needs d % 128 == 0, else
 * MAC_ERR_UNSUPPORTED. */
int mac_read_bwd_tc32(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                      const float* Wy_t, const float* att, const float* save, const float* dinfo, float keep_read,
                      uint64_t seed, int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx, float* dbx_part,
                      float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2, float* dbm2_part, float* dwr_part,
                      float* dbr_part, void* workspace, size_t workspace_bytes, int B, int N, int d, mac_stream_t stream);
size_t mac_read_bwd_tc32_workspace_bytes(int B, int N, int d);
/* ops.linear on tensor cores for the [B*N, .] products of the composed read unit (csrc/linear_tc.cuh; MACCell(prec="bf16")
 * with read-unit flags outside mac_read_fwd): bf16 operands (round to nearest even), fp32 accumulation, fp32 in / fp32 out.
 * mac_linear_tc_seg_fwd: mac_linear_fwd's y[M, n_out] = act(concat(x_0 .. x_{nseg-1}) @ W + b + bias_const) with W given as
 *   the packed bf16 Wt [n_out, K] (mac_pack_weight_bf16); b may be NULL; act any MAC_ACT_*.  The segments are cast into one
 *   bf16 [M, K] operand in the workspace (mac_linear_tc_seg_workspace_bytes(M, K), K = sum k_segs).
 * mac_linear_bwd_tc: mac_linear_bwd's arguments and accumulation conventions, except that W is the fp32 weight [K, n_out] in
 *   its own layout (not its transpose): dx_s (+)= bf16(dy) @ bf16(W_s)^T (dx_accum[s]); dW [K, n_out] += bf16(x)^T @ bf16(dy)
 *   (split-K over M rounded up to 64); db [n_out] += colsum(dy) in a fixed order (needs ldy == n_out).  Reruns are
 *   bit-identical.  Workspace: mac_linear_bwd_tc_workspace_bytes(M, k_segs, nseg, n_out), need not be zeroed.
 * Both need every k_segs[i] and n_out to be multiples of 128 (any M >= 1), else MAC_ERR_UNSUPPORTED; all checks precede any
 * launch. */
int mac_linear_tc_seg_fwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const void* wt_bf16,
                          const float* b, float bias_const, int act, float* y, int ldy, int M, int n_out,
                          void* workspace, size_t workspace_bytes, mac_stream_t stream);
size_t mac_linear_tc_seg_workspace_bytes(int M, int K);
int mac_linear_bwd_tc(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* W,
                      const float* dy, int ldy, float* const* dx_segs, const int* ld_dx, const int* dx_accum,
                      float* dW, float* db, int M, int n_out, void* workspace, size_t workspace_bytes, mac_stream_t stream);
size_t mac_linear_bwd_tc_workspace_bytes(int M, const int* k_segs, int nseg, int n_out);
/* write gate (mac_cell.py:358-367): dmnew = g*z; dmprev += g*(1-z); dpre = g*(mnew-mprev)*z*(1-z) */
int mac_gate_bwd(const float* g, const float* z, const float* mnew, const float* mprev, float* dmnew, float* dmprev,
                 float* dpre, long long n, mac_stream_t stream);
/* backward of mac_bcast_op (ops.mul on a broadcast operand, ops.py:694-713), g = dL/dout [B,N,d]; dx [B,N,d] +=, dv [B,d] +=,
 * dbias_part [B,d] += (mode 1 only); any of the three may be NULL.  `out` (the forward result) is read by mode 2 only. */
int mac_bcast_op_bwd(const float* x, const float* v, const float* out, const float* g, int mode, float mul_bias, float* dx,
                     float* dv, float* dbias_part, int B, int N, int d, mac_stream_t stream);
/* backward of mac_rowdot_fwd (ops.linear with outDim == 1, ops.py:316-317), g = dL/dout [R]: dx_s [R,k_s] += g (x) w_s
 * (entries / the array may be NULL), dw [sum k] +=, db [1] += (may be NULL).  Deterministic: per-64-row partial sums in the
 * workspace (mac_rowdot_bwd_workspace_bytes), reduced in block order. */
int mac_rowdot_bwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* w, const float* g,
                   float* const* dx_segs, const int* ld_dx, float* dw, float* db, void* workspace, size_t workspace_bytes,
                   long long R, mac_stream_t stream);
size_t mac_rowdot_bwd_workspace_bytes(long long R, int k_total);
/* Batch normalisation of the new memory (mac_cell.py:369-373: tf.contrib.layers.batch_norm(newMemory, decay, center, scale,
 * is_training, updates_collections=None), epsilon 0.001; rank-2 input = TF's fused path).  x, y [B,d] (y may alias x).
 * training != 0: batch mean / biased variance normalise, and moving_mean / moving_var move IN PLACE by (1 - decay) towards the
 * batch mean / the Bessel-corrected batch variance; training == 0: the stored statistics normalise.  gamma / beta may be NULL
 * (scale / center off).  save_mean, save_invstd [d] are what mac_batchnorm_bwd needs. */
int mac_batchnorm_fwd(const float* x, const float* gamma, const float* beta, float* moving_mean, float* moving_var, float decay,
                      float eps, int training, float* y, float* save_mean, float* save_invstd, int B, int d,
                      mac_stream_t stream);
/* dx [B,d] += , dgamma [d] +=, dbeta [d] += (each may be NULL); training as in the forward (eval: the statistics are constants) */
int mac_batchnorm_bwd(const float* x, const float* gamma, const float* save_mean, const float* save_invstd, const float* dy,
                      int training, float* dx, float* dgamma, float* dbeta, int B, int d, mac_stream_t stream);
/* dx = dy * act'(.) given the saved activation OUTPUT y */
int mac_activation_bwd(const float* y, const float* dy, int act, float* dx, long long n, mac_stream_t stream);
/* out[b,k] (+)= sum_n x[b,n,k] */
int mac_colsum(const float* x, float* out, int B, int N, int d, int accumulate, mac_stream_t stream);
/* dst += alpha * src */
int mac_axpy(float* dst, const float* src, float alpha, long long n, mac_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Training step on a flat fp32 bucket (the buffer NCCL all-reduces in data-parallel training):
 *   g' = grads * grad_scale;  norm = ||g'||;  g'' = g' * max_norm / max(norm, max_norm)   (tf.clip_by_global_norm, model.py:645-650)
 *   Adam with TF's bias-corrected step size (model.py:618);  ema = decay*ema + (1-decay)*p   (model.py:658-667; ema may be NULL)
 * norm_out[0] = global norm, norm_out[1] = clip factor (device memory, no host sync).  step >= 1.
 * --------------------------------------------------------------------------------------------- */
int mac_clip_adam_ema_step(float* params, const float* grads, float* adam_m, float* adam_v, float* ema, long long n,
                           float grad_scale, float max_norm, float lr, float beta1, float beta2, float eps, int step,
                           float ema_decay, float* norm_out, void* workspace, size_t workspace_bytes, mac_stream_t stream);
size_t mac_optimizer_workspace_bytes(void);

/* ------------------------------------------------------------------------------------------------
 * Answer loss of the output unit ("next" row, model.py:593-596): mean sparse softmax cross entropy.
 *   losses[b] = logsumexp(logits[b,:]) - logits[b, labels[b]];  dlogits = (softmax - onehot) * scale
 *   A label outside [0, A) gives losses[b] = NaN (like TF's GPU kernel) and no one-hot term; nothing is read out of bounds.
 * --------------------------------------------------------------------------------------------- */
int mac_softmax_xent(const float* logits, const int32_t* labels, float* losses, float* dlogits, float scale,
                     int B, int A, mac_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Image stem ("next" row, model.py:165-204, ops.py:380-438): convolution as GEMM.
 * mac_im2col3x3: cols[(b,h,w), (kh*3+kw)*C + c] = dropout(x)[b, h+kh-1, w+kw-1, c] for NHWC x, zero outside (SAME padding);
 * the [9*C, Cout] reshape of the HWIO kernel is the GEMM weight.  cols is fp32, or bf16 when cols_bf16 != 0.
 * --------------------------------------------------------------------------------------------- */
int mac_im2col3x3(const float* x, void* cols, int cols_bf16, float keep, uint64_t seed, int site, int step,
                  int B, int H, int W, int C, mac_stream_t stream);
/* Inference stem layer in e4m3 (csrc/tc_gemm_fp8.cuh; Stem(prec="fp8")), no dropout.  All scales fp32; e4m3 rounds to nearest
 * even and saturates at +-448.
 * mac_im2col3x3_fp8: the patch matrix of mac_im2col3x3 (same tap-major, channel-fastest layout) as e4m3 cols_e4m3 [M, 9C],
 *   M = B*H*W, with one scale per row: amax_m = max |x| over the in-image pixels of output pixel m's 3x3 window,
 *   row_scale[m] = amax_m / 448, cols_e4m3[m, k] = e4m3(patch[m, k] * (448 / amax_m)); a window that is all zero gives
 *   row_scale 0 and zero bytes.  Needs C % 128 == 0 (else MAC_ERR_UNSUPPORTED) and a workspace of
 *   mac_im2col3x3_fp8_workspace_bytes (one float per input pixel, need not be zeroed).
 * mac_linear_fp8_fwd: y[M, n_out] = act((x_e4m3[M, K] @ wt_e4m3[n_out, K]^T) * x_scale[m] * w_scale[n] + b[n]), fp32 y; wt /
 *   w_scale from mac_pack_weight_fp8.  wgmma m64n128k32 e4m3, every 128-element k-block accumulated in its own registers
 *   and added into an fp32 master accumulator.  act in {NON, ELU, RELU}; b may be NULL; K % 128 == 0 and n_out % 128 == 0,
 *   else MAC_ERR_UNSUPPORTED.  M need not be a multiple of 128.  All checks precede any launch. */
int mac_im2col3x3_fp8(const float* x, void* cols_e4m3, float* row_scale, void* workspace, size_t workspace_bytes,
                      int B, int H, int W, int C, mac_stream_t stream);
size_t mac_im2col3x3_fp8_workspace_bytes(int B, int H, int W, int C);
int mac_linear_fp8_fwd(const void* x_e4m3, const float* x_scale, const void* wt_e4m3, const float* w_scale, const float* b,
                       int act, float* y, int M, int K, int n_out, mac_stream_t stream);
/* backward of mac_im2col3x3 (fp32): dx[b,h,w,c] = keep-mask/keep * sum of the <= 9 entries of dcols that copied x[b,h,w,c]
 * (gather form, fixed order: deterministic).  The weight / bias gradients of the convolution are mac_linear_bwd on cols. */
int mac_col2im3x3(const float* dcols, float* dx, float keep, uint64_t seed, int site, int step, int B, int H, int W, int C,
                  mac_stream_t stream);
/* Backward of one stem layer y = act(conv3x3(dropout(x), kernel) + bias) with both GEMMs on wgmma tensor cores (bf16 operands,
 * fp32 accumulation; the activation derivative, the bias sums and col2im stay fp32).  x [B,H,W,C] is the layer input BEFORE
 * dropout, y [B*H*W, Cout] the output after the activation (as the forward saved them), dy the gradient w.r.t. y, kernel the
 * HWIO fp32 variable.  dkernel [3,3,C,Cout] += and dbias [Cout] += (fixed-order reductions: deterministic); dx [B,H,W,C] =
 * (NULL skips the data gradient and its GEMM).  keep / seed / site / step are the forward's mac_im2col3x3 arguments, so the
 * keep-mask is the forward's.  Needs C % 128 == 0 and Cout % 128 == 0, else MAC_ERR_UNSUPPORTED; the workspace
 * (mac_conv3x3_bwd_tc_workspace_bytes with with_dx = (dx != NULL)) need not be zeroed.  All checks precede any launch. */
int mac_conv3x3_bwd_tc(const float* x, const float* y, const float* dy, const float* kernel, int act, float keep, uint64_t seed,
                       int site, int step, float* dkernel, float* dbias, float* dx, void* workspace, size_t workspace_bytes,
                       int B, int H, int W, int C, int Cout, mac_stream_t stream);
size_t mac_conv3x3_bwd_tc_workspace_bytes(int B, int H, int W, int C, int Cout, int with_dx);

/* ------------------------------------------------------------------------------------------------
 * Question input unit ("next" row, model.py:208-220, 279-307; ops.py:859-905): embedding lookup + bi-LSTM encoder.
 * mac_embed_fwd: out[b,s,:] = dropout( idx[b,s] == 0 ? 0 : emb[idx[b,s]-1, :] )  (the reference prepends a zero padding
 *   row to the variable `qEmbeddings/emb` [V,E], model.py:217-218; ids outside 0..V read as zero); out_raw (may be NULL)
 *   receives the undropped words (`questionWords`).  E % 4 == 0.
 * mac_embed_bwd: d_emb[v,:] += sum_{(b,s): idx == v+1} d_out[b,s,:] * keep-mask / keep, positions in a fixed order.
 * mac_lstm_fwd: tf.nn.(bidirectional_)dynamic_rnn over BasicLSTMCell (gate order i,j,f,o; TF kernel [E+h, 4h]) with
 *   sequence_length = lengths.  The caller supplies the hoisted input projection gx_dir [B*S, 4h] = X @ kernel[0:E] + bias
 *   (mac_linear_fwd) and Wh_dir = kernel + E*4h (the recurrent rows).  Direction 1 walks t = len-1 .. 0 (reverse_sequence).
 *   out_seq [B,S,ndir*h] = [fw | bw] outputs, zero for t >= len; vecq [B,ndir*h] (may be NULL) = the final h of each
 *   direction (ops.py:893-898).  save_gates [ndir,B*S,4h], save_c / save_hprev [ndir,B*S,h] (all or none NULL) keep what
 *   the backward needs, indexed by time; save_hprev is zero for t >= len.  Issues S launches (one per step, both directions)
 *   on `stream`.
 * mac_lstm_bwd: BPTT.  dG_dir [B*S, 4h] receives the gradient w.r.t. the pre-activation gates; parameter and input
 *   gradients are then GEMMs over all steps: mac_linear_bwd(x_segs = [dropout(X), save_hprev_dir], dy = dG_dir).
 * --------------------------------------------------------------------------------------------- */
int mac_embed_fwd(const float* emb, const int32_t* idx, float keep, uint64_t seed, int site, int step, float* out_raw,
                  float* out, int B, int S, int V, int E, mac_stream_t stream);
int mac_embed_bwd(const float* d_out, const int32_t* idx, float keep, uint64_t seed, int site, int step, float* d_emb,
                  int B, int S, int V, int E, mac_stream_t stream);
size_t mac_lstm_workspace_bytes(int B, int h, int ndir);
int mac_lstm_fwd(const float* gx_fw, const float* gx_bw, const float* Wh_fw, const float* Wh_bw, const int32_t* lengths,
                 float forget_bias, float* out_seq, float* vecq, float* save_gates, float* save_c, float* save_hprev,
                 void* workspace, size_t workspace_bytes, int B, int S, int h, int ndir, mac_stream_t stream);
int mac_lstm_bwd(const float* Wh_fw, const float* Wh_bw, const int32_t* lengths, const float* save_gates,
                 const float* save_c, const float* d_out_seq, const float* d_vecq, float* dG_fw, float* dG_bw,
                 void* workspace, size_t workspace_bytes, int B, int S, int h, int ndir, mac_stream_t stream);
/* The question encoder on wgmma tensor cores (csrc/encoder_tc.cuh; QuestionEncoder(prec="bf16")): bf16 matrix-product
 * operands, fp32 accumulation; the cell state, gate non-linearities, outputs, saved tensors and element-wise backward steps
 * are fp32.  Ep = E rounded up to a multiple of 128; the bf16 operands carry zero columns E..Ep-1.  h must be 256
 * (MAC_ERR_UNSUPPORTED otherwise).  All checks precede any launch.
 * mac_embed_fwd_tc: mac_embed_fwd's out_raw (required) and x_bf16 [B*S, Ep] = bf16(dropout(words)) with the same keep-mask.
 * mac_pack_weight_bf16_kpad: fp32 W[K, n_out] -> bf16 Wt[n_out, Kp] with zero columns K..Kp-1 (Kp >= K); with W = kernel[0:E]
 *   and Kp = Ep it is the B operand of gx_dir = mac_linear_tc_fwd(x_bf16, Wt, bias_dir, NON, gx_dir, 0, B*S, Ep, 4h).
 * mac_lstm_fwd_tc: mac_lstm_fwd's recurrence and outputs (same saved-tensor layout) in ONE launch: per (direction, 64 batch
 *   rows) a cluster of 8 CTAs keeps the bf16 recurrent weights in shared memory and runs the recurrent product of every
 *   step on wgmma with bf16(h) as its operand.  Wh_dir is the fp32 kernel + E*4h.  Rows t >= len of out_seq and of the
 *   saved tensors are written as zeros.  No workspace.
 * mac_lstm_bwd_tc: the whole backward of the recurrence and the input projection: BPTT in one cluster launch, then
 *   dkernel_dir [E+h, 4h] += [X | h_prev]^T dG (x_bf16 as mac_embed_fwd_tc wrote it, h_prev = bf16(save_hprev)),
 *   dbias_dir [4h] += column sums of the fp32 gate gradients (fixed order), dx [B*S, E] = sum_dir dG_dir kernel_dir[0:E]^T
 *   (the gradient w.r.t. dropout(X): feed it to mac_embed_bwd).  kernel_dir is the fp32 TF kernel [E+h, 4h].  The
 *   workspace (mac_lstm_bwd_tc_workspace_bytes; 0 for an unsupported shape) need not be zeroed. */
int mac_embed_fwd_tc(const float* emb, const int32_t* idx, float keep, uint64_t seed, int site, int step, float* out_raw,
                     void* x_bf16, int B, int S, int V, int E, mac_stream_t stream);
int mac_pack_weight_bf16_kpad(const float* W, void* Wt_bf16, int K, int Kp, int n_out, mac_stream_t stream);
int mac_lstm_fwd_tc(const float* gx_fw, const float* gx_bw, const float* Wh_fw, const float* Wh_bw, const int32_t* lengths,
                    float forget_bias, float* out_seq, float* vecq, float* save_gates, float* save_c, float* save_hprev,
                    int B, int S, int h, int ndir, mac_stream_t stream);
int mac_lstm_bwd_tc(const void* x_bf16, const float* kernel_fw, const float* kernel_bw, const int32_t* lengths,
                    const float* save_gates, const float* save_c, const float* save_hprev, const float* d_out_seq,
                    const float* d_vecq, float* dkernel_fw, float* dkernel_bw, float* dbias_fw, float* dbias_bw, float* dx,
                    void* workspace, size_t workspace_bytes, int B, int S, int E, int h, int ndir, mac_stream_t stream);
size_t mac_lstm_bwd_tc_workspace_bytes(int B, int S, int E, int h, int ndir);

/* dropout sites (the `site` word of the Philox counter) */
enum { MAC_SITE_MEM_VAR = 0, MAC_SITE_READ_KB = 1, MAC_SITE_READ_MEM = 2, MAC_SITE_READ_INTER = 3,
       MAC_SITE_WRITE_INFO = 4, MAC_SITE_MEM_PLAIN = 5 };

#ifdef __cplusplus
}
#endif
#endif /* MAC_B200_H_ */
