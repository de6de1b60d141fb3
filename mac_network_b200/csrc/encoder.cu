// Question input unit of the reference model (SURVEY.md section 8(f) rank 3): word-embedding lookup + input dropout
// (model.py:208-220, ops.py:877) and the bidirectional BasicLSTMCell encoder run under
// tf.nn.bidirectional_dynamic_rnn(sequence_length = questionLengths) (ops.py:859-905, model.py:279-307).
//
// GPU formulation.  The input half of the LSTM kernel does not depend on the recurrence, so
//     gx[dir] = dropout(X)[B*S, E] @ kernel[dir][0:E, :] + bias[dir]
// is ONE GEMM per direction over all time steps (mac_linear_fwd).  What is left per step is the recurrent half
//     gates(b, :) = gx[dir][b, t, :] + h_prev[dir][b, :] @ kernel[dir][E:E+h, :]
// a [B, h] x [h, 4h] product with the cell update fused behind it.  lstm_step_kernel runs both directions of one step in
// one launch: CTA (unit chunk, dir, row chunk) stages its [h x 32] slice of the recurrent weights and the h_prev rows in
// shared memory, every thread owns the FOUR gates of one hidden unit for two batch rows, so the gate non-linearities, the
// cell update, the sequence-length masking (zero output + state carried through, as dynamic_rnn does) and the backward
// direction's per-row time index (reverse_sequence) are its epilogue.  The S launches of a forward are issued by ONE C call
// (mac_lstm_fwd) and captured in the caller's CUDA graph.
//
// Backward (BPTT) mirrors it: lstm_step_bwd_kernel computes dh = dgates(step s+1) @ Wh^T for its unit chunk as the prologue
// and the gate derivatives of step s as the epilogue; the parameter and input gradients of all steps are then two GEMMs per
// direction over the [B*S, 4h] gate-gradient matrix (mac_linear_bwd on the segments [dropout(X), h_prev]).
#include <cooperative_groups.h>
#include "common.cuh"

namespace mac {
namespace cg = cooperative_groups;

constexpr int LS_HC = 8;        // hidden units per CTA (x 4 gates = 32 weight columns)
constexpr int LS_ROWS = 64;     // batch rows per CTA
constexpr int LS_THREADS = 256; // thread (jj = tid & 7, bg = tid >> 3) owns unit j0 + jj for rows bg and bg + 32

// ------------------------------------------------------------------------------------------------ embedding
__global__ void embed_kernel(const float4* __restrict__ emb, const int32_t* __restrict__ idx, uint32_t thresh, float scale,
                             uint64_t seed, int site, int step, float4* __restrict__ raw, float4* __restrict__ out,
                             long long n4, int E4, int V) {
  const long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i4 >= n4) return;
  const long long row = i4 / E4;
  const int k4 = (int)(i4 - row * E4);
  const int id = idx[row];
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);           // id == 0: the padding row (model.py:217)
  if (id > 0 && id <= V) v = __ldg(emb + (size_t)(id - 1) * E4 + k4);
  if (raw) raw[i4] = v;
  if (thresh) {
    const Philox4 r = philox4x32_10(seed, (uint64_t)i4, (uint32_t)site, (uint32_t)step);
    v.x = ((r.x >> 8) >= thresh) ? v.x * scale : 0.f;
    v.y = ((r.y >> 8) >= thresh) ? v.y * scale : 0.f;
    v.z = ((r.z >> 8) >= thresh) ? v.z * scale : 0.f;
    v.w = ((r.w >> 8) >= thresh) ? v.w * scale : 0.f;
  }
  out[i4] = v;
}

// d_emb[v, :] += sum over positions with idx == v + 1 of d_x[pos, :] * mask(pos, :) * scale, in position order
// (one CTA per vocabulary row: a fixed summation order, so the gradient is deterministic without atomics)
__global__ void embed_bwd_kernel(const float4* __restrict__ dx, const int32_t* __restrict__ idx, uint32_t thresh, float scale,
                                 uint64_t seed, int site, int step, float4* __restrict__ demb, long long npos, int E4) {
  const int v = blockIdx.x;
  for (int k4 = threadIdx.x; k4 < E4; k4 += blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (long long pos = 0; pos < npos; ++pos) {
      if (idx[pos] != v + 1) continue;                  // uniform over the CTA: no divergence
      const long long i4 = pos * E4 + k4;
      float4 g = __ldg(dx + i4);
      if (thresh) {
        const Philox4 r = philox4x32_10(seed, (uint64_t)i4, (uint32_t)site, (uint32_t)step);
        g.x = ((r.x >> 8) >= thresh) ? g.x * scale : 0.f;
        g.y = ((r.y >> 8) >= thresh) ? g.y * scale : 0.f;
        g.z = ((r.z >> 8) >= thresh) ? g.z * scale : 0.f;
        g.w = ((r.w >> 8) >= thresh) ? g.w * scale : 0.f;
      }
      acc.x += g.x; acc.y += g.y; acc.z += g.z; acc.w += g.w;
    }
    float4 o = demb[(size_t)v * E4 + k4];
    o.x += acc.x; o.y += acc.y; o.z += acc.z; o.w += acc.w;
    demb[(size_t)v * E4 + k4] = o;
  }
}

// ------------------------------------------------------------------------------------------------ LSTM step, forward
struct LstmFwdParams {
  const float* gx[2];        // [B*S, 4h]: dropout(X) @ kernel[0:E] + bias
  const float* Wh[2];        // [h, 4h]: rows E.. of the TF kernel
  float* c;                  // [ndir, B, h], updated in place
  const float* h_prev;       // [ndir, B, h]
  float* h_next;             // [ndir, B, h]
  const int32_t* lengths;    // [B]
  float forget_bias;
  float* out_seq;            // [B, S, ndir*h]   (pre-zeroed: rows t >= length stay 0)
  float* vecq;               // [B, ndir*h] final h of both directions, written at s == S-1 (may be NULL)
  float* save_gates;         // [ndir, B*S, 4h] activated i, j, f, o by TIME index (may be NULL)
  float* save_c;             // [ndir, B*S, h] new cell state by TIME index
  float* save_hprev;         // [ndir, B*S, h] the h the step consumed, by TIME index
  int s, B, S, h, ndir;
};

__global__ void __launch_bounds__(LS_THREADS) lstm_step_kernel(const LstmFwdParams p) {
  extern __shared__ __align__(16) float ls_smem[];
  const int h = p.h, G = 4 * h, hp = h + 4;
  const int dir = blockIdx.y, j0 = blockIdx.x * LS_HC, b_base = blockIdx.z * LS_ROWS;
  float* hs = ls_smem;                   // [LS_ROWS][h + 4]
  float* ws = ls_smem + LS_ROWS * hp;    // [h][LS_HC][4]: (k, unit, gate), gate fastest -> one LDS.128 per (k, unit)
  const int tid = threadIdx.x;
  const float* __restrict__ Wh = dir ? p.Wh[1] : p.Wh[0];
  for (int e = tid; e < h * 8; e += LS_THREADS) {
    const int k = e >> 3, g = (e >> 1) & 3, half = e & 1;
    const float4 v = __ldg(reinterpret_cast<const float4*>(Wh + (size_t)k * G + g * h + j0 + half * 4));
    float* dst = ws + (k * LS_HC + half * 4) * 4 + g;
    dst[0] = v.x; dst[4] = v.y; dst[8] = v.z; dst[12] = v.w;
  }
  const int rows = min(LS_ROWS, p.B - b_base);
  const float* __restrict__ hprev = p.h_prev + ((size_t)dir * p.B + b_base) * h;
  const int h4 = h >> 2;
  for (int e = tid; e < LS_ROWS * h4; e += LS_THREADS) {
    const int r = e / h4, k4 = e - r * h4;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < rows) v = __ldg(reinterpret_cast<const float4*>(hprev + (size_t)r * h) + k4);
    *reinterpret_cast<float4*>(hs + r * hp + k4 * 4) = v;
  }
  __syncthreads();
  const int jj = tid & 7, bg = tid >> 3;
  float acc[2][4];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int g = 0; g < 4; ++g) acc[r][g] = 0.f;
  const float* h0 = hs + bg * hp;
  const float* h1 = hs + (bg + 32) * hp;
  for (int k = 0; k < h; k += 4) {
    const float4 a = *reinterpret_cast<const float4*>(h0 + k);
    const float4 b = *reinterpret_cast<const float4*>(h1 + k);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 w = *reinterpret_cast<const float4*>(ws + ((k + q) * LS_HC + jj) * 4);
      acc[0][0] = fmaf(av[q], w.x, acc[0][0]); acc[0][1] = fmaf(av[q], w.y, acc[0][1]);
      acc[0][2] = fmaf(av[q], w.z, acc[0][2]); acc[0][3] = fmaf(av[q], w.w, acc[0][3]);
      acc[1][0] = fmaf(bv[q], w.x, acc[1][0]); acc[1][1] = fmaf(bv[q], w.y, acc[1][1]);
      acc[1][2] = fmaf(bv[q], w.z, acc[1][2]); acc[1][3] = fmaf(bv[q], w.w, acc[1][3]);
    }
  }
  const int col = j0 + jj;
  const int W2 = p.ndir * h;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int lr = bg + 32 * r, b = b_base + lr;
    if (b >= p.B) continue;
    const int len = seq_len(p.lengths, b, p.S);
    const bool live = p.s < len;
    const float hold = hs[lr * hp + col];
    const size_t sidx = ((size_t)dir * p.B + b) * h + col;
    float hnew = hold;                                  // dynamic_rnn: state carried through past the sequence end
    if (live) {
      const int t = dir ? (len - 1 - p.s) : p.s;        // reverse_sequence: the backward cell walks t = len-1 .. 0
      const size_t row = (size_t)b * p.S + t;
      const float* gx = (dir ? p.gx[1] : p.gx[0]) + row * G + col;
      const float gi = sigmoid_f(acc[r][0] + gx[0]);
      const float gj = tanhf(acc[r][1] + gx[h]);
      const float gf = sigmoid_f(acc[r][2] + gx[2 * h] + p.forget_bias);
      const float go = sigmoid_f(acc[r][3] + gx[3 * h]);
      const float cn = p.c[sidx] * gf + gi * gj;
      hnew = tanhf(cn) * go;
      p.c[sidx] = cn;
      p.out_seq[row * W2 + dir * h + col] = hnew;
      if (p.save_gates) {
        float* sg = p.save_gates + ((size_t)dir * p.B * p.S + row) * G + col;
        sg[0] = gi; sg[h] = gj; sg[2 * h] = gf; sg[3 * h] = go;
        p.save_c[((size_t)dir * p.B * p.S + row) * h + col] = cn;
        p.save_hprev[((size_t)dir * p.B * p.S + row) * h + col] = hold;
      }
    }
    p.h_next[sidx] = hnew;
    if (p.vecq && p.s == p.S - 1) p.vecq[(size_t)b * W2 + dir * h + col] = hnew;
  }
}

// ------------------------------------------------------------------------------------------------ LSTM, persistent form
// The whole recurrence of one (direction, 8 batch rows) in ONE launch by a thread-block cluster of 8 CTAs (h == 256).
// CTA `rank` owns hidden units [32*rank, 32*rank + 32): its [256 x 128] slice of the recurrent weights is loaded into shared
// memory ONCE (128 KB) and stays there for all S steps; the cell state lives in a register of the thread that owns
// (row, unit); what the CTAs exchange per step is h: each CTA stages its [8 x 32] block and copies it with 16-byte stores
// into the next-step h buffer of the seven other CTAs over distributed shared memory, then one cluster barrier (which is
// also the release/acquire point for those remote stores).  Double-buffered h: a CTA can only run ahead into step s+1 after
// every CTA has passed the barrier of step s, i.e. after all reads of the buffer it is about to overwrite.
// Thread mapping: warp w owns units 4w..4w+3, lane = (unit & 3) + 4*row  ->  per k the warp reads 64 B of weights (broadcast
// over the 8 rows) and 8 x 16 B of h (conflict-free with the +4 row pad): 5 shared-memory wavefronts per 16 FMAs per thread.
constexpr int LP_CL = 8, LP_RB = 8, LP_THREADS = 256, LP_HU = 32, LP_H = LP_CL * LP_HU;

static __global__ void __launch_bounds__(LP_THREADS) lstm_seq_kernel(const LstmFwdParams p) {
  extern __shared__ __align__(16) float lp_smem[];
  constexpr int h = LP_H, G = 4 * LP_H, hp = LP_H + 4;
  float* wsl = lp_smem;                          // [h][LP_HU][4]   (k, unit, gate)
  float* hbuf = lp_smem + h * LP_HU * 4;         // [2][LP_RB][hp]
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();    // cluster spans gridDim.x
  const int dir = blockIdx.y, b_base = blockIdx.z * LP_RB;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int ul = warp * 4 + (lane & 3), row = lane >> 2;
  const int gu = rank * LP_HU + ul;              // hidden unit this thread owns
  const int b = b_base + row;
  const float* __restrict__ Wh = dir ? p.Wh[1] : p.Wh[0];
  for (int e = tid; e < h * 32; e += LP_THREADS) {
    const int q = e & 7, g = (e >> 3) & 3, k = e >> 5;
    const float4 v = __ldg(reinterpret_cast<const float4*>(Wh + (size_t)k * G + g * h + rank * LP_HU + q * 4));
    float* dst = wsl + (k * LP_HU + q * 4) * 4 + g;
    dst[0] = v.x; dst[4] = v.y; dst[8] = v.z; dst[12] = v.w;
  }
  for (int e = tid; e < 2 * LP_RB * hp; e += LP_THREADS) hbuf[e] = 0.f;     // cell.zero_state
  cluster.sync();                                // every CTA's buffers are zeroed before any remote store can land
  const bool valid = b < p.B;
  const int len = valid ? seq_len(p.lengths, b, p.S) : 0;
  const int W2 = p.ndir * h;
  const float* __restrict__ gxd = dir ? p.gx[1] : p.gx[0];
  const size_t dbase = (size_t)dir * p.B * p.S;
  float c = 0.f, hcur = 0.f;
  for (int s = 0; s < p.S; ++s) {
    const float* hb = hbuf + (s & 1) * (LP_RB * hp) + row * hp;
    const bool live = s < len;
    const int t = dir ? (len - 1 - s) : s;
    const size_t rowi = live ? ((size_t)b * p.S + t) : 0;
    float g0 = 0.f, g1 = 0.f, g2 = 0.f, g3 = 0.f;
    if (live) {                                  // issued before the product so the L2 latency hides under it
      const float* gx = gxd + rowi * G + gu;
      g0 = __ldg(gx); g1 = __ldg(gx + h); g2 = __ldg(gx + 2 * h); g3 = __ldg(gx + 3 * h);
    }
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
    for (int k = 0; k < h; k += 4) {
      const float4 x = *reinterpret_cast<const float4*>(hb + k);
      const float4 w0 = *reinterpret_cast<const float4*>(wsl + ((k + 0) * LP_HU + ul) * 4);
      const float4 w1 = *reinterpret_cast<const float4*>(wsl + ((k + 1) * LP_HU + ul) * 4);
      const float4 w2 = *reinterpret_cast<const float4*>(wsl + ((k + 2) * LP_HU + ul) * 4);
      const float4 w3 = *reinterpret_cast<const float4*>(wsl + ((k + 3) * LP_HU + ul) * 4);
      a0 = fmaf(x.x, w0.x, a0); a1 = fmaf(x.x, w0.y, a1); a2 = fmaf(x.x, w0.z, a2); a3 = fmaf(x.x, w0.w, a3);
      a0 = fmaf(x.y, w1.x, a0); a1 = fmaf(x.y, w1.y, a1); a2 = fmaf(x.y, w1.z, a2); a3 = fmaf(x.y, w1.w, a3);
      a0 = fmaf(x.z, w2.x, a0); a1 = fmaf(x.z, w2.y, a1); a2 = fmaf(x.z, w2.z, a2); a3 = fmaf(x.z, w2.w, a3);
      a0 = fmaf(x.w, w3.x, a0); a1 = fmaf(x.w, w3.y, a1); a2 = fmaf(x.w, w3.z, a2); a3 = fmaf(x.w, w3.w, a3);
    }
    float hnew = hcur;                           // dynamic_rnn: state carried through past the sequence end
    if (live) {
      const float gi = sigmoid_f(a0 + g0), gj = tanhf(a1 + g1);
      const float gf = sigmoid_f(a2 + g2 + p.forget_bias), go = sigmoid_f(a3 + g3);
      c = c * gf + gi * gj;
      hnew = tanhf(c) * go;
      p.out_seq[rowi * W2 + dir * h + gu] = hnew;
      if (p.save_gates) {
        float* sg = p.save_gates + (dbase + rowi) * G + gu;
        sg[0] = gi; sg[h] = gj; sg[2 * h] = gf; sg[3 * h] = go;
        p.save_c[(dbase + rowi) * h + gu] = c;
        p.save_hprev[(dbase + rowi) * h + gu] = hcur;
      }
    }
    hcur = hnew;
    // exchange: stage the CTA's [8 x 32] block in its own next buffer, then 16-byte copies into the 7 peers
    float* nb = hbuf + ((s + 1) & 1) * (LP_RB * hp);
    nb[row * hp + gu] = hnew;
    __syncthreads();
    for (int e = tid; e < (LP_CL - 1) * LP_RB * (LP_HU / 4); e += LP_THREADS) {
      const int q = e & 7, r = (e >> 3) & 7, z = e >> 6;                     // float4 q of row r -> peer z (skipping self)
      const int peer = z + (z >= rank ? 1 : 0);
      float* src = nb + r * hp + rank * LP_HU + q * 4;
      *reinterpret_cast<float4*>(cluster.map_shared_rank(src, peer)) = *reinterpret_cast<const float4*>(src);
    }
    cluster.sync();
  }
  if (valid && p.vecq) p.vecq[(size_t)b * W2 + dir * h + gu] = hcur;
}

// ------------------------------------------------------------------------------------------------ LSTM step, backward
struct LstmBwdParams {
  float* dG[2];              // [B*S, 4h] gradient w.r.t. the pre-activation gates by TIME index (pre-zeroed)
  const float* Wh[2];        // [h, 4h]
  const float* save_gates;   // [ndir, B*S, 4h]
  const float* save_c;       // [ndir, B*S, h]
  const float* d_out_seq;    // [B, S, ndir*h]
  const float* d_vecq;       // [B, ndir*h] (may be NULL = 0)
  float* dcc;                // [ndir, B, h] running gradient w.r.t. the cell state (pre-zeroed), in place
  const int32_t* lengths;
  int s, B, S, h, ndir;
};

constexpr int LB_KC = 256;    // gate-gradient columns staged per chunk

__global__ void __launch_bounds__(LS_THREADS) lstm_step_bwd_kernel(const LstmBwdParams p) {
  extern __shared__ __align__(16) float ls_smem[];
  const int h = p.h, G = 4 * h, gp = G + 4, kp = LB_KC + 4;
  const int dir = blockIdx.y, j0 = blockIdx.x * LS_HC, b_base = blockIdx.z * LS_ROWS;
  float* wt = ls_smem;                 // [LS_HC][4h + 4]: rows j0.. of Wh (= columns of Wh^T)
  float* dg = ls_smem + LS_HC * gp;    // [LS_ROWS][LB_KC + 4]
  const int tid = threadIdx.x;
  const int jj = tid & 7, bg = tid >> 3;
  float acc[2] = {0.f, 0.f};
  const bool any_next = (p.s + 1 < p.S);
  if (any_next) {
    const float* __restrict__ Wh = dir ? p.Wh[1] : p.Wh[0];
    const int G4 = G >> 2;
    for (int e = tid; e < LS_HC * G4; e += LS_THREADS) {
      const int r = e / G4, k4 = e - r * G4;
      *reinterpret_cast<float4*>(wt + r * gp + k4 * 4) =
          __ldg(reinterpret_cast<const float4*>(Wh + (size_t)(j0 + r) * G) + k4);
    }
    const float* __restrict__ dGd = dir ? p.dG[1] : p.dG[0];
    for (int kc = 0; kc < G; kc += LB_KC) {
      __syncthreads();                 // previous chunk consumed (and wt visible on the first pass)
      for (int e = tid; e < LS_ROWS * (LB_KC / 4); e += LS_THREADS) {
        const int r = e / (LB_KC / 4), k4 = e - r * (LB_KC / 4);
        const int b = b_base + r;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (b < p.B && kc + k4 * 4 < G) {
          const int len = seq_len(p.lengths, b, p.S);
          if (p.s + 1 < len) {         // the row was live at step s+1: its gate gradients sit at that step's time index
            const int t1 = dir ? (len - 2 - p.s) : (p.s + 1);
            v = *(reinterpret_cast<const float4*>(dGd + ((size_t)b * p.S + t1) * G + kc) + k4);
          }
        }
        *reinterpret_cast<float4*>(dg + r * kp + k4 * 4) = v;
      }
      __syncthreads();
      const float* d0 = dg + bg * kp;
      const float* d1 = dg + (bg + 32) * kp;
      const float* w = wt + jj * gp + kc;
      const int kmax = min(LB_KC, G - kc);
      for (int k = 0; k < kmax; k += 4) {
        const float4 a = *reinterpret_cast<const float4*>(d0 + k);
        const float4 b = *reinterpret_cast<const float4*>(d1 + k);
        const float4 ww = *reinterpret_cast<const float4*>(w + k);
        acc[0] = fmaf(a.x, ww.x, acc[0]); acc[0] = fmaf(a.y, ww.y, acc[0]);
        acc[0] = fmaf(a.z, ww.z, acc[0]); acc[0] = fmaf(a.w, ww.w, acc[0]);
        acc[1] = fmaf(b.x, ww.x, acc[1]); acc[1] = fmaf(b.y, ww.y, acc[1]);
        acc[1] = fmaf(b.z, ww.z, acc[1]); acc[1] = fmaf(b.w, ww.w, acc[1]);
      }
    }
  }
  const int col = j0 + jj;
  const int W2 = p.ndir * h;
  const size_t BS = (size_t)p.B * p.S;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int b = b_base + bg + 32 * r;
    if (b >= p.B) continue;
    const int len = seq_len(p.lengths, b, p.S);
    if (p.s >= len) continue;          // past the end: state was carried through, nothing to differentiate
    const int t = dir ? (len - 1 - p.s) : p.s;
    const size_t row = (size_t)b * p.S + t;
    float dh = p.d_out_seq[row * W2 + dir * h + col];
    if (p.s + 1 < len) dh += acc[r];
    else if (p.d_vecq) dh += p.d_vecq[(size_t)b * W2 + dir * h + col];   // last live step: its h is the final state
    const float* sg = p.save_gates + ((size_t)dir * BS + row) * G + col;
    const float gi = sg[0], gj = sg[h], gf = sg[2 * h], go = sg[3 * h];
    const float cn = p.save_c[((size_t)dir * BS + row) * h + col];
    float cprev = 0.f;
    if (p.s > 0) {
      const int tp = dir ? (t + 1) : (t - 1);
      cprev = p.save_c[((size_t)dir * BS + (size_t)b * p.S + tp) * h + col];
    }
    const float tc = tanhf(cn);
    const size_t sidx = ((size_t)dir * p.B + b) * h + col;
    const float dc = p.dcc[sidx] + dh * go * (1.f - tc * tc);
    float* out = (dir ? p.dG[1] : p.dG[0]) + row * G + col;
    out[0] = dc * gj * gi * (1.f - gi);
    out[h] = dc * gi * (1.f - gj * gj);
    out[2 * h] = dc * cprev * gf * (1.f - gf);
    out[3 * h] = dh * tc * go * (1.f - go);
    p.dcc[sidx] = dc * gf;
  }
}

}  // namespace mac

using namespace mac;

extern "C" int mac_embed_fwd(const float* emb, const int32_t* idx, float keep, uint64_t seed, int site, int step,
                             float* out_raw, float* out, int B, int S, int V, int E, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!emb || !idx || !out || B <= 0 || S <= 0 || V <= 0 || E <= 0 || (E & 3) || !(keep > 0.f && keep <= 1.f))
    return MAC_ERR_INVALID;
  if (!mac_aligned16(emb) || !mac_aligned16(out) || (out_raw && !mac_aligned16(out_raw))) return MAC_ERR_ALIGN;
  const long long n4 = (long long)B * S * (E / 4);
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  embed_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(emb), idx, thr, scale, seed, site, step, reinterpret_cast<float4*>(out_raw),
      reinterpret_cast<float4*>(out), n4, E / 4, V);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_embed_bwd(const float* d_out, const int32_t* idx, float keep, uint64_t seed, int site, int step,
                             float* d_emb, int B, int S, int V, int E, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!d_out || !idx || !d_emb || B <= 0 || S <= 0 || V <= 0 || E <= 0 || (E & 3) || !(keep > 0.f && keep <= 1.f))
    return MAC_ERR_INVALID;
  if (!mac_aligned16(d_out) || !mac_aligned16(d_emb)) return MAC_ERR_ALIGN;
  const uint32_t thr = keep < 1.f ? keep_threshold(keep) : 0u;
  const float scale = keep < 1.f ? 1.f / keep : 1.f;
  embed_bwd_kernel<<<V, 128, 0, stream>>>(reinterpret_cast<const float4*>(d_out), idx, thr, scale, seed, site, step,
                                          reinterpret_cast<float4*>(d_emb), (long long)B * S, E / 4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

static size_t lstm_state_bytes(int B, int h, int ndir) { return (size_t)ndir * B * h * sizeof(float); }

extern "C" size_t mac_lstm_workspace_bytes(int B, int h, int ndir) {
  return 3 * ((lstm_state_bytes(B, h, ndir) + 255) & ~(size_t)255);    // c, h ping, h pong
}

extern "C" int mac_lstm_fwd(const float* gx_fw, const float* gx_bw, const float* Wh_fw, const float* Wh_bw,
                            const int32_t* lengths, float forget_bias, float* out_seq, float* vecq, float* save_gates,
                            float* save_c, float* save_hprev, void* workspace, size_t workspace_bytes, int B, int S, int h,
                            int ndir, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!gx_fw || !Wh_fw || !lengths || !out_seq || !workspace || B <= 0 || S <= 0 || h <= 0 || (h % LS_HC) ||
      ndir < 1 || ndir > 2 || (ndir == 2 && (!gx_bw || !Wh_bw)))
    return MAC_ERR_INVALID;
  if (save_gates && (!save_c || !save_hprev)) return MAC_ERR_INVALID;
  if (!mac_aligned16(gx_fw) || !mac_aligned16(Wh_fw) || (ndir == 2 && (!mac_aligned16(gx_bw) || !mac_aligned16(Wh_bw))) ||
      !mac_aligned16(workspace))
    return MAC_ERR_ALIGN;
  if (workspace_bytes < mac_lstm_workspace_bytes(B, h, ndir)) return MAC_ERR_WORKSPACE;
  const size_t smem = ((size_t)LS_ROWS * (h + 4) + (size_t)h * LS_HC * 4) * sizeof(float);
  if (smem > 227u * 1024u) return MAC_ERR_UNSUPPORTED;
  const size_t sb = (lstm_state_bytes(B, h, ndir) + 255) & ~(size_t)255;
  char* ws = reinterpret_cast<char*>(workspace);
  MAC_CUDA_TRY(cudaMemsetAsync(out_seq, 0, (size_t)B * S * ndir * h * sizeof(float), stream));
  // the backward's weight-gradient GEMM multiplies every row of save_hprev, those of t >= len by zero gate gradients: they
  // must be finite, and whatever the caller's buffer held (NaN included) would otherwise reach the gradient
  if (save_hprev) MAC_CUDA_TRY(cudaMemsetAsync(save_hprev, 0, (size_t)ndir * B * S * h * sizeof(float), stream));
  LstmFwdParams p{};
  p.gx[0] = gx_fw; p.gx[1] = gx_bw; p.Wh[0] = Wh_fw; p.Wh[1] = Wh_bw;
  p.lengths = lengths; p.forget_bias = forget_bias; p.out_seq = out_seq; p.vecq = vecq;
  p.save_gates = save_gates; p.save_c = save_c; p.save_hprev = save_hprev;
  p.B = B; p.S = S; p.h = h; p.ndir = ndir;
  // h == 256 (encDim 512, the reference default): the whole recurrence in one cluster launch (703 vs 805 us for the encoder
  // forward at B=64, S=40, profiles/r1/lstm_bench_r1.jsonl); every other h runs the per-step kernels below.
  if (h == LP_H) {
    const size_t psmem = ((size_t)LP_H * LP_HU * 4 + (size_t)2 * LP_RB * (LP_H + 4)) * sizeof(float);
    MAC_CUDA_TRY(cudaFuncSetAttribute(lstm_seq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psmem));
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(LP_CL, ndir, (B + LP_RB - 1) / LP_RB);
    cfg.blockDim = dim3(LP_THREADS, 1, 1);
    cfg.dynamicSmemBytes = psmem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = LP_CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    MAC_CUDA_TRY(cudaLaunchKernelEx(&cfg, lstm_seq_kernel, p));
    MAC_LAUNCH_CHECK();
    return MAC_OK;
  }
  MAC_CUDA_TRY(cudaFuncSetAttribute(lstm_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  MAC_CUDA_TRY(cudaMemsetAsync(ws, 0, 2 * sb, stream));                                  // c = h = 0 (cell.zero_state)
  p.c = reinterpret_cast<float*>(ws);
  float* hbuf[2] = {reinterpret_cast<float*>(ws + sb), reinterpret_cast<float*>(ws + 2 * sb)};
  const dim3 grid(h / LS_HC, ndir, (B + LS_ROWS - 1) / LS_ROWS);
  for (int s = 0; s < S; ++s) {
    p.s = s;
    p.h_prev = hbuf[s & 1];
    p.h_next = hbuf[(s + 1) & 1];
    lstm_step_kernel<<<grid, LS_THREADS, smem, stream>>>(p);
    MAC_LAUNCH_CHECK();
  }
  return MAC_OK;
}

extern "C" int mac_lstm_bwd(const float* Wh_fw, const float* Wh_bw, const int32_t* lengths, const float* save_gates,
                            const float* save_c, const float* d_out_seq, const float* d_vecq, float* dG_fw, float* dG_bw,
                            void* workspace, size_t workspace_bytes, int B, int S, int h, int ndir, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!Wh_fw || !lengths || !save_gates || !save_c || !d_out_seq || !dG_fw || !workspace || B <= 0 || S <= 0 || h <= 0 ||
      (h % LS_HC) || ndir < 1 || ndir > 2 || (ndir == 2 && (!Wh_bw || !dG_bw)))
    return MAC_ERR_INVALID;
  if (!mac_aligned16(Wh_fw) || !mac_aligned16(dG_fw) || (ndir == 2 && (!mac_aligned16(Wh_bw) || !mac_aligned16(dG_bw))))
    return MAC_ERR_ALIGN;
  if (workspace_bytes < mac_lstm_workspace_bytes(B, h, ndir)) return MAC_ERR_WORKSPACE;
  const size_t smem = ((size_t)LS_HC * (4 * h + 4) + (size_t)LS_ROWS * (LB_KC + 4)) * sizeof(float);
  if (smem > 227u * 1024u) return MAC_ERR_UNSUPPORTED;
  MAC_CUDA_TRY(cudaFuncSetAttribute(lstm_step_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const size_t sb = (lstm_state_bytes(B, h, ndir) + 255) & ~(size_t)255;
  MAC_CUDA_TRY(cudaMemsetAsync(workspace, 0, sb, stream));                               // dcc = 0
  const size_t gbytes = (size_t)B * S * 4 * h * sizeof(float);
  MAC_CUDA_TRY(cudaMemsetAsync(dG_fw, 0, gbytes, stream));
  if (ndir == 2) MAC_CUDA_TRY(cudaMemsetAsync(dG_bw, 0, gbytes, stream));
  LstmBwdParams p{};
  p.dG[0] = dG_fw; p.dG[1] = dG_bw; p.Wh[0] = Wh_fw; p.Wh[1] = Wh_bw;
  p.save_gates = save_gates; p.save_c = save_c; p.d_out_seq = d_out_seq; p.d_vecq = d_vecq;
  p.dcc = reinterpret_cast<float*>(workspace); p.lengths = lengths;
  p.B = B; p.S = S; p.h = h; p.ndir = ndir;
  const dim3 grid(h / LS_HC, ndir, (B + LS_ROWS - 1) / LS_ROWS);
  for (int s = S - 1; s >= 0; --s) {
    p.s = s;
    lstm_step_bwd_kernel<<<grid, LS_THREADS, smem, stream>>>(p);
    MAC_LAUNCH_CHECK();
  }
  return MAC_OK;
}
