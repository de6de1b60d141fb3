// Backward of the MAC cell (fp32 path).  The reference obtains it from TF autodiff (`optimizer.compute_gradients`,
// model.py:626-636); here each forward entry point of mac_b200.h has a hand-written counterpart.  Math: SURVEY.md
// Appendix E.  Reductions are per-sample partial sums (one CTA owns a (sample, column-slice)), reduced over the batch
// at the end of the backward pass, so gradients are deterministic (no atomics anywhere).
#include "common.cuh"
#define SGEMM_MIN_BLOCKS 1      // the transposed-A / split-K weight-gradient GEMMs are faster with the full register budget
#include "sgemm.cuh"
#include "skinny.cuh"

using namespace mac;

namespace mac {
constexpr size_t BW_HEADER = 4096;

// ------------------------------------------------------------------------------------------------ small helpers
__global__ void axpy_kernel(float* __restrict__ dst, const float* __restrict__ src, float alpha, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += alpha * src[i];
}

// dst += dropout(src): the gradient through tf.nn.dropout added onto an accumulator in one pass (same Philox numbering as
// mac_dropout_fwd: one draw per aligned quad of elements)
__global__ void axpy_dropout_kernel(float4* __restrict__ dst, const float4* __restrict__ src, uint32_t thresh, float scale,
                                    uint64_t seed, int site, int step, long long n4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 v = src[i];
  float4 o = dst[i];
  const Philox4 r = philox4x32_10(seed, (uint64_t)i, (uint32_t)site, (uint32_t)step);
  if ((r.x >> 8) >= thresh) o.x = fmaf(v.x, scale, o.x);
  if ((r.y >> 8) >= thresh) o.y = fmaf(v.y, scale, o.y);
  if ((r.z >> 8) >= thresh) o.z = fmaf(v.z, scale, o.z);
  if ((r.w >> 8) >= thresh) o.w = fmaf(v.w, scale, o.w);
  dst[i] = o;
}

// dZ = g * ELU'(H) (through the saved output H: H > 0 ? 1 : H + 1) and dbm_part[b,:] += sum_n dZ[b,n,:] in one pass.
// grid (ceil(d/128), B), 256 threads: 32 column quads x 8 row groups (the map of read_bwd_logits_kernel), d % 4 == 0.
__global__ void __launch_bounds__(256) elu_bwd_colsum_kernel(const float* __restrict__ H, const float* __restrict__ g,
                                                            float* __restrict__ dZ, float* __restrict__ dsum_part, int N,
                                                            int d) {
  __shared__ float s_red[8][128];
  const int q = threadIdx.x & 31, rg = threadIdx.x >> 5, b = blockIdx.y;
  const int k = blockIdx.x * 128 + q * 4;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (k < d) {
    for (int n = rg; n < N; n += 8) {
      const size_t o = ((size_t)b * N + n) * d + k;
      const float4 h = *reinterpret_cast<const float4*>(H + o);
      const float4 gi = *reinterpret_cast<const float4*>(g + o);
      float4 z;
      z.x = gi.x * (h.x > 0.f ? 1.f : h.x + 1.f);
      z.y = gi.y * (h.y > 0.f ? 1.f : h.y + 1.f);
      z.z = gi.z * (h.z > 0.f ? 1.f : h.z + 1.f);
      z.w = gi.w * (h.w > 0.f ? 1.f : h.w + 1.f);
      *reinterpret_cast<float4*>(dZ + o) = z;
      s[0] += z.x; s[1] += z.y; s[2] += z.z; s[3] += z.w;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) s_red[rg][q * 4 + j] = s[j];
  __syncthreads();
  if (threadIdx.x < 128) {
    const int kk = blockIdx.x * 128 + threadIdx.x;
    if (kk < d) {
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) a += s_red[i][threadIdx.x];
      dsum_part[(size_t)b * d + kk] += a;
    }
  }
}

// dx = dy * act'(.) expressed through the saved OUTPUT y
__global__ void act_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, int act,
                               float* __restrict__ dx, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  dx[i] = dy[i] * act_grad_from_output(act, y[i]);
}

// out[b, k] (+)= sum_n x[b, n, k]     grid (ceil(d/128), B), 256 threads = 32 column quads x 8 row groups (fixed-order reduce)
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, float* __restrict__ out, int N, int d,
                                                    int accumulate) {
  __shared__ float s_red[8][128];
  const int q = threadIdx.x & 31, rg = threadIdx.x >> 5, b = blockIdx.y;
  const int k = blockIdx.x * 128 + q * 4;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  if (k < d) {
    const float* p = x + (size_t)b * N * d + k;
    if (((d & 3) == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0)) {
      for (int n = rg; n < N; n += 8) {
        const float4 v = *reinterpret_cast<const float4*>(p + (size_t)n * d);
        s[0] += v.x;
        s[1] += v.y;
        s[2] += v.z;
        s[3] += v.w;
      }
    } else {                                   // any width (classifier outputs, outDim == 1): scalar loads
      for (int n = rg; n < N; n += 8)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (k + j < d) s[j] += p[(size_t)n * d + j];
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) s_red[rg][q * 4 + j] = s[j];
  __syncthreads();
  if (threadIdx.x < 128) {
    const int kk = blockIdx.x * 128 + threadIdx.x;
    if (kk < d) {
      float a = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) a += s_red[g][threadIdx.x];
      float* o = out + (size_t)b * d + kk;
      *o = accumulate ? *o + a : a;
    }
  }
}

// write gate backward (mac_cell.py:358-367): m = m'*z + mprev*(1-z), z = sigmoid(pre)
//   dm' = g*z ; dmprev += g*(1-z) ; dpre = g*(m' - mprev)*z*(1-z)
__global__ void gate_bwd_kernel(const float* __restrict__ g, const float* __restrict__ z, const float* __restrict__ mnew,
                                const float* __restrict__ mprev, float* __restrict__ dmnew, float* __restrict__ dmprev,
                                float* __restrict__ dpre, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i], zi = z[i];
  dmnew[i] = gi * zi;
  dmprev[i] += gi * (1.f - zi);
  dpre[i] = gi * (mnew[i] - mprev[i]) * zi * (1.f - zi);
}

// ------------------------------------------------------------------------------------------------ attention backward
// Backward of mac_control_attend_fwd for ONE batch row per CTA, all `nsteps` query vectors in turn:
//   d_out_words[s,:] += att_s * g ; datt_s = out_words[s,:] . g ; dlogit = att * (datt - sum att*datt)
//   d_in_words[s,k] += dlogit_s * q_k * w_k ; dq_k = w_k * sum_s dlogit_s * in[s,k]
//   dw_part[b,k] += q_k * sum_s dlogit_s * in[s,k] ; db_part[b] += sum_s dlogit_s
constexpr int AB_THREADS = 256;
__global__ void __launch_bounds__(AB_THREADS) control_attend_bwd_kernel(
    const float* __restrict__ cc, long long cc_t, long long cc_b, const float* __restrict__ in_words, long long in_b,
    long long in_r, const float* __restrict__ out_words, long long out_b, long long out_r,
    const float* __restrict__ w_logit, const float* __restrict__ att, const float* __restrict__ g_out, long long g_t,
    long long g_b, float* d_in, float* d_out /* may alias d_in */, float* __restrict__ dq, long long dq_t,
    long long dq_b, int dq_accum, float* __restrict__ dw_part, float* __restrict__ db_part, int nsteps, int B, int S,
    int d) {
  extern __shared__ __align__(16) float ab_smem[];
  float* s_datt = ab_smem;            // [S]
  float* s_dl = s_datt + S;           // [S]
  float* s_att = s_dl + S;            // [S]
  __shared__ float s_red[AB_THREADS / 32];
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int NW = AB_THREADS / 32;
  const float* inw = in_words + (size_t)b * in_b;
  const float* outw = out_words + (size_t)b * out_b;
  float* din = d_in + (size_t)b * in_b;
  float* dout = d_out + (size_t)b * out_b;
  for (int t = 0; t < nsteps; ++t) {
    const float* q = cc + (size_t)t * cc_t + (size_t)b * cc_b;
    const float* g = g_out + (size_t)t * g_t + (size_t)b * g_b;
    const float* a = att + ((size_t)t * B + b) * S;
    for (int s = tid; s < S; s += AB_THREADS) s_att[s] = a[s];
    __syncthreads();
    // datt_s = out_words[s,:] . g     (warp per word row)
    for (int s = warp; s < S; s += NW) {
      const float* row = outw + (size_t)s * out_r;
      float acc = 0.f;
      for (int k = lane; k < d; k += 32) acc = fmaf(row[k], g[k], acc);
      acc = warp_sum(acc);
      if (lane == 0) s_datt[s] = acc;
    }
    __syncthreads();
    float part = 0.f;
    for (int s = tid; s < S; s += AB_THREADS) part += s_att[s] * s_datt[s];
    part = warp_sum(part);
    if (lane == 0) s_red[warp] = part;
    __syncthreads();
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < NW; ++i) dot += s_red[i];
    __syncthreads();
    float dlsum = 0.f;
    for (int s = tid; s < S; s += AB_THREADS) {
      const float dl = s_att[s] * (s_datt[s] - dot);
      s_dl[s] = dl;
      dlsum += dl;
    }
    dlsum = warp_sum(dlsum);
    if (lane == 0) s_red[warp] = dlsum;
    __syncthreads();
    if (tid == 0) {
      float tsum = 0.f;
#pragma unroll
      for (int i = 0; i < NW; ++i) tsum += s_red[i];
      db_part[b] += tsum;
    }
    // column-wise pass: thread per feature k
    for (int k = tid; k < d; k += AB_THREADS) {
      const float qk = q[k], wk = __ldg(w_logit + k), gk = g[k];
      float sx = 0.f;   // sum_s dlogit_s * in[s,k]
      for (int s = 0; s < S; ++s) {
        const float dl = s_dl[s];
        const float x = inw[(size_t)s * in_r + k];
        sx = fmaf(dl, x, sx);
        // the two word gradients may alias (control unit: in_words == out_words): update sequentially
        dout[(size_t)s * out_r + k] += s_att[s] * gk;
        din[(size_t)s * in_r + k] += dl * qk * wk;
      }
      float* o = dq + (size_t)t * dq_t + (size_t)b * dq_b + k;
      *o = dq_accum ? *o + wk * sx : wk * sx;
      dw_part[(size_t)b * d + k] += qk * sx;
    }
    __syncthreads();
  }
}

// dka[b,n] = KB[b,n,:] . dinfo[b,:]        grid (ceil(N/8), B), 256 threads = 8 warps, warp per KB row
__global__ void __launch_bounds__(256) kb_dot_kernel(const float* __restrict__ kb, const float* __restrict__ dinfo,
                                                    float* __restrict__ dka, int N, int d) {
  const int b = blockIdx.y, n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  const float4* row = reinterpret_cast<const float4*>(kb + ((size_t)b * N + n) * d);
  const float4* g = reinterpret_cast<const float4*>(dinfo + (size_t)b * d);
  float acc = 0.f;
  for (int k = lane; k < d / 4; k += 32) {
    const float4 x = __ldg(row + k), y = __ldg(g + k);
    acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) dka[(size_t)b * N + n] = acc;
}

// softmax backward over the KB + rank-1 KB gradient:  dkl = ka*(dka - sum ka*dka);  dkb[b,n,:] += ka[n]*dinfo[b,:]
// grid (ceil(N/32), B), 256 threads
__global__ void __launch_bounds__(256) kb_attend_bwd_kernel(const float* __restrict__ att, const float* __restrict__ dka,
                                                           const float* __restrict__ dinfo, float* __restrict__ dkl,
                                                           float* __restrict__ dkb, float* __restrict__ dbr_part, int N,
                                                           int d) {
  __shared__ float s_red[8];
  __shared__ float s_dot;
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* a = att + (size_t)b * N;
  const float* dk = dka + (size_t)b * N;
  float part = 0.f;
  for (int n = tid; n < N; n += 256) part += a[n] * dk[n];
  part = warp_sum(part);
  if (lane == 0) s_red[warp] = part;
  __syncthreads();
  if (tid == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += s_red[i];
    s_dot = t;
  }
  __syncthreads();
  const float dot = s_dot;
  const int n0 = blockIdx.x * 32;
  // dkl[n] = ka[n] * (dka[n] - sum_m ka[m] dka[m]) cancels catastrophically in fp32 when the attention is peaked (ka[n] -> 1:
  // dka[n] - dot is the difference of two nearly equal numbers, and that n carries most of the gradient).  The same value as a
  // sum of weighted differences, ka[n] * sum_m ka[m] * (dka[n] - dka[m]), has no such cancellation; O(N^2) per sample is
  // nothing at N = 196.  8 lanes per n (tid / 8 -> n, tid % 8 -> slice of m), reduced with shuffles.
  {
    const int n = n0 + (tid >> 3), part_i = tid & 7;
    float acc = 0.f;
    if (n < N) {
      const float dn = dk[n];
      for (int m = part_i; m < N; m += 8) acc = fmaf(a[m], dn - dk[m], acc);
    }
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    acc += __shfl_xor_sync(0xffffffffu, acc, 4);
    if (n < N && part_i == 0) dkl[(size_t)b * N + n] = a[n] * acc;
  }
  if (blockIdx.x == 0 && dbr_part) {
    // sum_n dkl = sum ka*dka - dot*sum ka = dot - dot*1 = 0 up to round-off; computed explicitly for fidelity
    float s = 0.f;
    for (int n = tid; n < N; n += 256) s += a[n] * (dk[n] - dot);
    s = warp_sum(s);
    __syncthreads();
    if (lane == 0) s_red[warp] = s;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) t += s_red[i];
      dbr_part[b] += t;
    }
  }
  if (dkb) {
    const float4* g4 = reinterpret_cast<const float4*>(dinfo + (size_t)b * d);
    for (int r = 0; r < 32 && n0 + r < N; ++r) {
      const float an = a[n0 + r];
      float4* row = reinterpret_cast<float4*>(dkb + ((size_t)b * N + n0 + r) * d);
      for (int k = tid; k < d / 4; k += 256) {
        float4 o = row[k];
        const float4 g = __ldg(g4 + k);
        o.x = fmaf(an, g.x, o.x); o.y = fmaf(an, g.y, o.y); o.z = fmaf(an, g.z, o.z); o.w = fmaf(an, g.w, o.w);
        row[k] = o;
      }
    }
  }
}

// Backward through the logits epilogue of the read unit (mac_cell.py:248-266):
//   T = I1*c ; I2 = ELU(T) ; I2d = I2*mask*scale ; kl = I2d.wr + br
//   dI2 = dkl*wr*mask*scale ; dT = dI2*ELU'(T) ; dI1 = dT*c ; dc[b,:] += sum_n dT*I1 ; dwr_part[b,:] += sum_n dkl*I2d
//   dbm2_part[b,:] += sum_n dI1
// grid (ceil(d/128), B), 256 threads: thread = (column quad q = tid % 32: 4 consecutive columns, row group rg = tid / 32 of 8).
// One Philox draw serves the quad's four elements (round 1: one thread per column recomputed the draw four times and walked the
// N rows serially: 131 us per launch, 11.7 % of a tensor-core training step); the eight row groups are reduced in shared memory
// in a fixed order, so the per-sample sums stay deterministic.
__global__ void __launch_bounds__(256) read_bwd_logits_kernel(
    const float* __restrict__ I1, const float* __restrict__ ctrl, const float* __restrict__ wr,
    const float* __restrict__ dkl, uint32_t thresh, float scale, uint64_t seed, int step, float* __restrict__ dI1,
    float* __restrict__ dc, float* __restrict__ dwr_part, float* __restrict__ dbm2_part, int N, int d) {
  __shared__ float s_red[3][8][128];
  const int q = threadIdx.x & 31, rg = threadIdx.x >> 5, b = blockIdx.y;
  const int k = blockIdx.x * 128 + q * 4;
  const bool ok = k < d;                       // d % 4 == 0: a quad is inside or outside as a whole
  float sdc[4] = {0.f, 0.f, 0.f, 0.f}, sdw[4] = {0.f, 0.f, 0.f, 0.f}, sdb[4] = {0.f, 0.f, 0.f, 0.f};
  if (ok) {
    const float4 c4 = *reinterpret_cast<const float4*>(ctrl + (size_t)b * d + k);
    const float4 w4 = __ldg(reinterpret_cast<const float4*>(wr + k));
    const float c[4] = {c4.x, c4.y, c4.z, c4.w}, w[4] = {w4.x, w4.y, w4.z, w4.w};
    for (int n = rg; n < N; n += 8) {
      const size_t row = (size_t)b * N + n;
      const float4 i4 = *reinterpret_cast<const float4*>(I1 + row * d + k);
      const float i1[4] = {i4.x, i4.y, i4.z, i4.w};
      float m[4] = {1.f, 1.f, 1.f, 1.f};
      if (thresh) {
        const uint64_t e = row * (uint64_t)d + (uint64_t)k;
        const Philox4 r = philox4x32_10(seed, e >> 2, MAC_SITE_READ_INTER, (uint32_t)step);
        m[0] = ((r.x >> 8) >= thresh) ? scale : 0.f;
        m[1] = ((r.y >> 8) >= thresh) ? scale : 0.f;
        m[2] = ((r.z >> 8) >= thresh) ? scale : 0.f;
        m[3] = ((r.w >> 8) >= thresh) ? scale : 0.f;
      }
      const float g = dkl[row];
      float o[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float t = i1[j] * c[j];
        const float i2 = elu_f(t);
        const float dT = g * w[j] * m[j] * (t > 0.f ? 1.f : i2 + 1.f);
        o[j] = dT * c[j];
        sdc[j] = fmaf(dT, i1[j], sdc[j]);
        sdw[j] = fmaf(g, i2 * m[j], sdw[j]);
        sdb[j] += o[j];
      }
      *reinterpret_cast<float4*>(dI1 + row * d + k) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s_red[0][rg][q * 4 + j] = sdc[j];
    s_red[1][rg][q * 4 + j] = sdw[j];
    s_red[2][rg][q * 4 + j] = sdb[j];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int kk = blockIdx.x * 128 + threadIdx.x;
    if (kk < d) {
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        a0 += s_red[0][g][threadIdx.x];
        a1 += s_red[1][g][threadIdx.x];
        a2 += s_red[2][g][threadIdx.x];
      }
      dc[(size_t)b * d + kk] += a0;
      dwr_part[(size_t)b * d + kk] += a1;
      dbm2_part[(size_t)b * d + kk] += a2;
    }
  }
}

// dP = dI0[:, :d]*y + dI0[:, d:] ; dy[b,:] = sum_n dI0[:, :d]*P ; dbx_part[b,:] += sum_n dP     (ops.py:694-719)
// Same thread map as read_bwd_logits_kernel: 32 column quads x 8 row groups, 16-byte accesses, fixed-order reduction.
__global__ void __launch_bounds__(256) read_bwd_p_kernel(const float* __restrict__ dI0, const float* __restrict__ P,
                                                        const float* __restrict__ y, float* __restrict__ dP,
                                                        float* __restrict__ dy, float* __restrict__ dbx_part, int N,
                                                        int d) {
  __shared__ float s_red[2][8][128];
  const int q = threadIdx.x & 31, rg = threadIdx.x >> 5, b = blockIdx.y;
  const int k = blockIdx.x * 128 + q * 4;
  float sdy[4] = {0.f, 0.f, 0.f, 0.f}, sdb[4] = {0.f, 0.f, 0.f, 0.f};
  if (k < d) {
    const float4 y4 = *reinterpret_cast<const float4*>(y + (size_t)b * d + k);
    for (int n = rg; n < N; n += 8) {
      const size_t row = (size_t)b * N + n;
      const float4 top = *reinterpret_cast<const float4*>(dI0 + row * 2 * d + k);
      const float4 bot = *reinterpret_cast<const float4*>(dI0 + row * 2 * d + d + k);
      const float4 p4 = *reinterpret_cast<const float4*>(P + row * d + k);
      float4 o;
      o.x = fmaf(top.x, y4.x, bot.x);
      o.y = fmaf(top.y, y4.y, bot.y);
      o.z = fmaf(top.z, y4.z, bot.z);
      o.w = fmaf(top.w, y4.w, bot.w);
      *reinterpret_cast<float4*>(dP + row * d + k) = o;
      sdy[0] = fmaf(top.x, p4.x, sdy[0]);
      sdy[1] = fmaf(top.y, p4.y, sdy[1]);
      sdy[2] = fmaf(top.z, p4.z, sdy[2]);
      sdy[3] = fmaf(top.w, p4.w, sdy[3]);
      sdb[0] += o.x;
      sdb[1] += o.y;
      sdb[2] += o.z;
      sdb[3] += o.w;
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    s_red[0][rg][q * 4 + j] = sdy[j];
    s_red[1][rg][q * 4 + j] = sdb[j];
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int kk = blockIdx.x * 128 + threadIdx.x;
    if (kk < d) {
      float a0 = 0.f, a1 = 0.f;
#pragma unroll
      for (int g = 0; g < 8; ++g) {
        a0 += s_red[0][g][threadIdx.x];
        a1 += s_red[1][g][threadIdx.x];
      }
      dy[(size_t)b * d + kk] = a0;
      dbx_part[(size_t)b * d + kk] += a1;
    }
  }
}

// Backward of mac_bcast_op (ops.mul interaction on a broadcast operand, ops.py:694-713).  g = dL/dout [B,N,d]:
//   mode 0 MUL: dx += g*(v+mb) ; dv[b,:] += sum_n g*(x+mb)
//   mode 1 BL : dx += g*v      ; dv[b,:] += sum_n g*x ; dbias_part[b,:] += sum_n g
//   mode 2 ADD: t = g*(1-out^2): dx += t ; dv[b,:] += sum_n t
// grid (ceil(d/128), B), 256 threads = 128 columns x 2 row groups; the two groups are added in a fixed order.
__global__ void __launch_bounds__(256) bcast_op_bwd_kernel(const float* __restrict__ x, const float* __restrict__ v,
                                                          const float* __restrict__ out, const float* __restrict__ g,
                                                          int mode, float mb, float* __restrict__ dx,
                                                          float* __restrict__ dv, float* __restrict__ dbias_part, int N,
                                                          int d) {
  __shared__ float s_red[2][128];
  const int col = threadIdx.x & 127, rg = threadIdx.x >> 7, b = blockIdx.y;
  const int k = blockIdx.x * 128 + col;
  float sv = 0.f, sb = 0.f;
  if (k < d) {
    const float vk = v[(size_t)b * d + k];
    for (int n = rg; n < N; n += 2) {
      const size_t i = ((size_t)b * N + n) * d + k;
      const float gi = g[i];
      float gx, gv;
      if (mode == 0) {
        gx = gi * (vk + mb);
        gv = gi * (x[i] + mb);
      } else if (mode == 1) {
        gx = gi * vk;
        gv = gi * x[i];
        sb += gi;
      } else {
        const float o = out[i];
        gx = gv = gi * (1.f - o * o);
      }
      if (dx) dx[i] += gx;
      sv += gv;
    }
  }
  if (rg == 1) {
    s_red[0][col] = sv;
    s_red[1][col] = sb;
  }
  __syncthreads();
  if (rg == 0 && k < d) {
    if (dv) dv[(size_t)b * d + k] += sv + s_red[0][col];
    if (dbias_part && mode == 1) dbias_part[(size_t)b * d + k] += sb + s_red[1][col];
  }
}

// Backward of mac_rowdot_fwd (ops.linear with outDim == 1, ops.py:316-317): out[r] = sum_s x_s[r,:].w_s + b, g = dL/dout [R]
//   dx_s[r,:] += g[r]*w_s ;  part[blk, kk] = sum_{r in block blk} g[r]*x[r, kk]   (kk = Ktot: the bias column, x = 1)
// grid (ceil((Ktot+1)/128), ceil(R/RD_ROWS)), 128 threads (one column each, coalesced over kk).
constexpr int RD_ROWS = 64;
__global__ void __launch_bounds__(128) rowdot_bwd_kernel(const float* x0, const float* x1, const float* x2, int k0, int k1,
                                                        int k2, int ld0, int ld1, int ld2, const float* __restrict__ w,
                                                        const float* __restrict__ g, float* dx0, float* dx1, float* dx2,
                                                        int ldd0, int ldd1, int ldd2, float* __restrict__ part,
                                                        long long R) {
  const int Ktot = k0 + k1 + k2;
  const int kk = blockIdx.x * 128 + threadIdx.x;
  if (kk > Ktot) return;
  const long long r0 = (long long)blockIdx.y * RD_ROWS, r1 = min(R, r0 + RD_ROWS);
  const float* x = nullptr;
  float* dx = nullptr;
  int ld = 0, ldd = 0, kl = kk;
  if (kk < k0) { x = x0; dx = dx0; ld = ld0; ldd = ldd0; }
  else if (kk < k0 + k1) { x = x1; dx = dx1; ld = ld1; ldd = ldd1; kl = kk - k0; }
  else if (kk < Ktot) { x = x2; dx = dx2; ld = ld2; ldd = ldd2; kl = kk - k0 - k1; }
  const float wk = kk < Ktot ? __ldg(w + kk) : 0.f;
  float s = 0.f;
  for (long long r = r0; r < r1; ++r) {
    const float gr = g[r];
    if (x) {
      s = fmaf(gr, x[r * ld + kl], s);
      if (dx) dx[r * ldd + kl] += gr * wk;
    } else {
      s += gr;
    }
  }
  part[(size_t)blockIdx.y * (Ktot + 1) + kk] = s;
}

// dw[kk] += sum_blk part[blk, kk] (kk < Ktot) ; db[0] += sum_blk part[blk, Ktot]     fixed order over the blocks
__global__ void rowdot_bwd_reduce_kernel(const float* __restrict__ part, int nblk, int Ktot, float* __restrict__ dw,
                                         float* __restrict__ db) {
  const int kk = blockIdx.x * blockDim.x + threadIdx.x;
  if (kk > Ktot) return;
  float s = 0.f;
  for (int i = 0; i < nblk; ++i) s += part[(size_t)i * (Ktot + 1) + kk];
  if (kk < Ktot) {
    if (dw) dw[kk] += s;
  } else if (db) {
    db[0] += s;
  }
}

// Batch normalisation of the new memory (mac_cell.py:369-373: tf.contrib.layers.batch_norm, rank-2 input -> TF's fused path).
// x, y [B, d]; one thread per column (B is the batch: tens to hundreds of rows), rows are d floats apart -> coalesced over k.
//   training: mean / biased variance of the batch normalise; the stored statistics move by (1 - decay) towards the batch mean
//             and the Bessel-corrected batch variance (what FusedBatchNorm hands to assign_moving_average), in place;
//   eval:     the stored statistics normalise.
// save_mean / save_invstd [d] keep what the backward needs.  y may alias x.
__global__ void batchnorm_fwd_kernel(const float* x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                     float* __restrict__ moving_mean, float* __restrict__ moving_var, float decay, float eps,
                                     int training, float* y, float* __restrict__ save_mean, float* __restrict__ save_invstd,
                                     int B, int d) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= d) return;
  float mean, var;
  if (training) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += x[(size_t)b * d + k];
    mean = s / (float)B;
    float q = 0.f;
    for (int b = 0; b < B; ++b) {
      const float c = x[(size_t)b * d + k] - mean;
      q = fmaf(c, c, q);
    }
    var = q / (float)B;
    const float unbiased = var * ((float)B / (float)max(B - 1, 1));
    moving_mean[k] -= (moving_mean[k] - mean) * (1.f - decay);
    moving_var[k] -= (moving_var[k] - unbiased) * (1.f - decay);
  } else {
    mean = moving_mean[k];
    var = moving_var[k];
  }
  const float invstd = 1.f / sqrtf(var + eps);
  const float g = gamma ? gamma[k] : 1.f, bt = beta ? beta[k] : 0.f;
  for (int b = 0; b < B; ++b) {
    const size_t i = (size_t)b * d + k;
    y[i] = (x[i] - mean) * invstd * g + bt;
  }
  if (save_mean) save_mean[k] = mean;
  if (save_invstd) save_invstd[k] = invstd;
}

// dx += gamma*invstd*(dy - mean_b(dy) - xhat*mean_b(dy*xhat)) (training) or gamma*invstd*dy (eval: constants);
// dgamma += sum_b dy*xhat ; dbeta += sum_b dy
__global__ void batchnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                     const float* __restrict__ save_mean, const float* __restrict__ save_invstd,
                                     const float* __restrict__ dy, int training, float* __restrict__ dx,
                                     float* __restrict__ dgamma, float* __restrict__ dbeta, int B, int d) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= d) return;
  const float mean = save_mean[k], invstd = save_invstd[k], g = gamma ? gamma[k] : 1.f;
  float s1 = 0.f, s2 = 0.f;
  for (int b = 0; b < B; ++b) {
    const size_t i = (size_t)b * d + k;
    const float gy = dy[i];
    s1 += gy;
    s2 = fmaf(gy, (x[i] - mean) * invstd, s2);
  }
  if (dx) {
    const float m1 = training ? s1 / (float)B : 0.f, m2 = training ? s2 / (float)B : 0.f;
    for (int b = 0; b < B; ++b) {
      const size_t i = (size_t)b * d + k;
      dx[i] += g * invstd * (dy[i] - m1 - (x[i] - mean) * invstd * m2);
    }
  }
  if (dgamma) dgamma[k] += s2;
  if (dbeta) dbeta[k] += s1;
}

static int launch_colsum(const float* x, float* out, int B, int N, int d, int accumulate, cudaStream_t stream) {
  dim3 grid((d + 127) / 128, B);
  colsum_kernel<<<grid, 256, 0, stream>>>(x, out, N, d, accumulate);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}
}  // namespace mac

// ================================================================================================ C ABI
extern "C" int mac_axpy(float* dst, const float* src, float alpha, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!dst || !src || n <= 0) return MAC_ERR_INVALID;
  axpy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dst, src, alpha, n);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_bcast_op_bwd(const float* x, const float* v, const float* out, const float* g, int mode, float mul_bias,
                                float* dx, float* dv, float* dbias_part, int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !v || !g || B <= 0 || N <= 0 || d <= 0 || mode < 0 || mode > 2 || (mode == 2 && !out)) return MAC_ERR_INVALID;
  bcast_op_bwd_kernel<<<dim3((d + 127) / 128, B), 256, 0, stream>>>(x, v, out, g, mode, mul_bias, dx, dv, dbias_part, N, d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" size_t mac_rowdot_bwd_workspace_bytes(long long R, int k_total) {
  return (size_t)((R + RD_ROWS - 1) / RD_ROWS) * (size_t)(k_total + 1) * sizeof(float) + 256;
}

extern "C" int mac_rowdot_bwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* w,
                              const float* g, float* const* dx_segs, const int* ld_dx, float* dw, float* db, void* workspace,
                              size_t workspace_bytes, long long R, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !ldx || nseg < 1 || nseg > 3 || !w || !g || !workspace || R <= 0) return MAC_ERR_INVALID;
  const float* x[3] = {nullptr, nullptr, nullptr};
  float* dx[3] = {nullptr, nullptr, nullptr};
  int k[3] = {0, 0, 0}, ld[3] = {0, 0, 0}, ldd[3] = {0, 0, 0};
  for (int i = 0; i < nseg; ++i) {
    x[i] = x_segs[i]; k[i] = k_segs[i]; ld[i] = ldx[i];
    if (!x[i] || k[i] <= 0) return MAC_ERR_INVALID;
    if (dx_segs && dx_segs[i]) { dx[i] = dx_segs[i]; ldd[i] = ld_dx ? ld_dx[i] : k[i]; }
  }
  const int Ktot = k[0] + k[1] + k[2];
  if (workspace_bytes < mac_rowdot_bwd_workspace_bytes(R, Ktot)) return MAC_ERR_WORKSPACE;
  float* part = reinterpret_cast<float*>(workspace);
  const int nblk = (int)((R + RD_ROWS - 1) / RD_ROWS);
  rowdot_bwd_kernel<<<dim3((Ktot + 1 + 127) / 128, nblk), 128, 0, stream>>>(x[0], x[1], x[2], k[0], k[1], k[2], ld[0], ld[1],
                                                                            ld[2], w, g, dx[0], dx[1], dx[2], ldd[0], ldd[1],
                                                                            ldd[2], part, R);
  MAC_LAUNCH_CHECK();
  rowdot_bwd_reduce_kernel<<<(Ktot + 1 + 127) / 128, 128, 0, stream>>>(part, nblk, Ktot, dw, db);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_batchnorm_fwd(const float* x, const float* gamma, const float* beta, float* moving_mean, float* moving_var,
                                 float decay, float eps, int training, float* y, float* save_mean, float* save_invstd, int B,
                                 int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !moving_mean || !moving_var || !y || B <= 0 || d <= 0 || !(eps > 0.f)) return MAC_ERR_INVALID;
  batchnorm_fwd_kernel<<<(d + 127) / 128, 128, 0, stream>>>(x, gamma, beta, moving_mean, moving_var, decay, eps, training, y,
                                                           save_mean, save_invstd, B, d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_batchnorm_bwd(const float* x, const float* gamma, const float* save_mean, const float* save_invstd,
                                 const float* dy, int training, float* dx, float* dgamma, float* dbeta, int B, int d,
                                 mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x || !save_mean || !save_invstd || !dy || B <= 0 || d <= 0) return MAC_ERR_INVALID;
  batchnorm_bwd_kernel<<<(d + 127) / 128, 128, 0, stream>>>(x, gamma, save_mean, save_invstd, dy, training, dx, dgamma, dbeta, B,
                                                           d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_activation_bwd(const float* y, const float* dy, int act, float* dx, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!y || !dy || !dx || n <= 0) return MAC_ERR_INVALID;
  act_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(y, dy, act, dx, n);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_colsum(const float* x, float* out, int B, int N, int d, int accumulate, mac_stream_t stream_) {
  if (!x || !out || B <= 0 || N <= 0 || d <= 0) return MAC_ERR_INVALID;
  return launch_colsum(x, out, B, N, d, accumulate, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int mac_gate_bwd(const float* g, const float* z, const float* mnew, const float* mprev, float* dmnew,
                            float* dmprev, float* dpre, long long n, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!g || !z || !mnew || !mprev || !dmnew || !dmprev || !dpre || n <= 0) return MAC_ERR_INVALID;
  gate_bwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(g, z, mnew, mprev, dmnew, dmprev, dpre, n);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// Backward of ops.linear on concatenated segments (ops.py:298-333):  y = concat(x_s) @ W + b
//   dx_s (+)= dy @ W[koff_s : koff_s+k_s, :]^T   (needs Wt = W^T [n_out, K], row-major)
//   dW  += concat(x_s)^T @ dy ;  db += colsum(dy)
extern "C" int mac_linear_bwd(const float* const* x_segs, const int* k_segs, const int* ldx, int nseg, const float* Wt,
                              const float* dy, int ldy, float* const* dx_segs, const int* ld_dx, const int* dx_accum,
                              float* dW, float* db, int M, int n_out, void* workspace, size_t workspace_bytes,
                              mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!x_segs || !k_segs || !dy || nseg < 1 || nseg > 4 || M <= 0 || n_out <= 0) return MAC_ERR_INVALID;
  char* ws = reinterpret_cast<char*>(workspace);
  const bool have_ws = ws != nullptr && workspace_bytes > BW_HEADER;
  unsigned int* counters = have_ws ? reinterpret_cast<unsigned int*>(ws) : nullptr;
  float* partial = have_ws ? reinterpret_cast<float*>(ws + BW_HEADER) : nullptr;
  const size_t pbytes = have_ws ? workspace_bytes - BW_HEADER : 0;
  int K = 0;
  for (int s = 0; s < nseg; ++s) K += k_segs[s];
  int koff = 0;
  for (int s = 0; s < nseg; ++s) {
    if (dx_segs && dx_segs[s]) {
      if (!Wt) return MAC_ERR_INVALID;
      SgemmParams p{};
      p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = dy; p.ak[0] = n_out; p.lda[0] = ldy;
      p.W = Wt + koff; p.ldw = K; p.M = M; p.N = k_segs[s]; p.K = n_out;
      p.epi = EPI_BIAS_ACT; p.act = MAC_ACT_NON; p.Y = dx_segs[s]; p.ldy = ld_dx[s]; p.accumulate = dx_accum ? dx_accum[s] : 0;
      int st = sgemm_launch(p, counters, partial, pbytes, stream);
      if (st != MAC_OK) return st;
    }
    if (dW) {
      SgemmParams p{};
      p.a_mode = A_TRANS; p.nseg = 1; p.a[0] = x_segs[s]; p.lda[0] = ldx[s];
      p.W = dy; p.ldw = ldy; p.M = k_segs[s]; p.N = n_out; p.K = M;
      p.epi = EPI_BIAS_ACT; p.act = MAC_ACT_NON; p.Y = dW + (size_t)koff * n_out; p.ldy = n_out; p.accumulate = 1;
      int st = sgemm_launch(p, counters, partial, pbytes, stream);
      if (st != MAC_OK) return st;
    }
    koff += k_segs[s];
  }
  if (db) {
    if (ldy != n_out) return MAC_ERR_UNSUPPORTED;
    int st = launch_colsum(dy, db, 1, M, n_out, 1, stream);
    if (st != MAC_OK) return st;
  }
  return MAC_OK;
}

extern "C" int mac_control_attend_bwd(const float* cc, long long cc_tstride, long long cc_bstride,
                                      const float* in_words, long long in_bstride, long long in_rstride,
                                      const float* out_words, long long out_bstride, long long out_rstride,
                                      const float* w_logit, const float* att, const float* g_out, long long g_tstride,
                                      long long g_bstride, float* d_in_words, float* d_out_words, float* dq,
                                      long long dq_tstride, long long dq_bstride, int dq_accumulate, float* dw_part,
                                      float* db_part, int nsteps, int B, int S, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!cc || !in_words || !out_words || !w_logit || !att || !g_out || !d_in_words || !d_out_words || !dq || !dw_part ||
      !db_part)
    return MAC_ERR_INVALID;
  if (nsteps <= 0 || B <= 0 || S <= 0 || d <= 0) return MAC_ERR_INVALID;
  const size_t smem = (size_t)3 * S * sizeof(float) + 16;
  control_attend_bwd_kernel<<<B, AB_THREADS, smem, stream>>>(cc, cc_tstride, cc_bstride, in_words, in_bstride, in_rstride,
                                                            out_words, out_bstride, out_rstride, w_logit, att, g_out,
                                                            g_tstride, g_bstride, d_in_words, d_out_words, dq, dq_tstride,
                                                            dq_bstride, dq_accumulate, dw_part, db_part, nsteps, B, S, d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

extern "C" int mac_kb_attend_bwd(const float* kb, const float* att, const float* dinfo, float* dka_scratch, float* dkl,
                                 float* dkb, float* dbr_part, int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!kb || !att || !dinfo || !dka_scratch || !dkl || B <= 0 || N <= 0 || d <= 0 || (d & 3)) return MAC_ERR_INVALID;
  kb_dot_kernel<<<dim3((N + 7) / 8, B), 256, 0, stream>>>(kb, dinfo, dka_scratch, N, d);
  MAC_LAUNCH_CHECK();
  kb_attend_bwd_kernel<<<dim3((N + 31) / 32, B), 256, 0, stream>>>(att, dka_scratch, dinfo, dkl, dkb, dbr_part, N, d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}


// ================================================================================================ read unit backward
// Backward of mac_read_fwd's training forms (mac_cell.py:209-277; see mac_read_bwd* in mac_b200.h) in three forms that run
// one seven-step schedule (read_bwd_run) and differ only in how they form its six [B*N, .] products:
//   RB_FP32  mac_read_bwd       on the FMA pipe (sgemm), data gradients from the transposed fp32 weights, with the fused
//                               prologues / epilogues of sgemm.cuh (P*y concat, KB dropout, * ELU'(H), dropout on dKB)
//   RB_TC    mac_read_bwd_tc    bf16 operands on wgmma tensor cores (fp32 accumulation)
//   RB_TC32  mac_read_bwd_tc32  split-bf16 operands on wgmma tensor cores (x = hi + lo, three of the four partial products)
// The tensor-core forms build their operands with the transposing pack of tc_gemm.cuh, which applies P*y and the forward's KB
// dropout mask on the way, and reach the tensor-core templates through the internal exports of units.cu below:
//   wgrad  dW[in, d] += X^T G  (K = B*N)   X^T and G^T packed into the workspace, one split-K launch; the pack of G also
//                                          leaves its row-major copy for the dgrad that follows
//   dgrad  dX[M, in] = G W^T               W fp32 in its own [in, d] layout, cast (tc) or split (tc32) on every call
// Every call is checked against everything its form reads and every limit of the kernels it launches (read_bwd_check), and
// only then run: a refusal never follows a launch or a write, and nothing behind the check checks anything.
extern "C" int mac_tc_wgrad_splitk_(const void* xT, const void* gT, float* dW, float* partial, int in_dim, int out_dim, int K,
                                    mac_stream_t stream_);
extern "C" size_t mac_tc_wgrad_partial_bytes_(int in_dim, int out_dim);
extern "C" int mac_pack_t_bf16_(int mode, const float* X, void* Xt, void* Xrm, int K, int N, const float* rowvec,
                                int rows_per_batch, uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                mac_stream_t stream_);
extern "C" int mac_pack_t_split_(int mode, const float* X, void* Xt, void* Xrm, int K, int N, int segs, const float* rowvec,
                                 int rows_per_batch, uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                 mac_stream_t stream_);
extern "C" int mac_tc3_wgrad_splitk_(const void* xT2, const void* gT3, float* dW, float* partial, int in_dim, int out_dim,
                                     int kp, mac_stream_t stream_);
extern "C" int mac_split3_rows_(const float* W, void* W3, int R, int C, mac_stream_t stream_);
extern "C" int mac_tc3_linear_(const void* a_split, const void* wt3, float* y, int M, int K, int n_out, mac_stream_t stream_);

namespace mac {
enum ReadBwdForm { RB_FP32, RB_TC, RB_TC32 };

// The workspace of every form, first the fp32 part (M = B*N; dka and dkl padded to a multiple of 4 floats):
//   [header 4 KB: split-K counters | bufA [M,d]: dI1, later dP | bufB [M,d]: dZ | bufC [M,2d]: dI0 | dka [M] | dkl [M] |
//    dy [B,d] | md [B,d]: dropout(memory_in) | dmd [B,d] | unused [B,d] and 4 KB | split-K partials of the fp32 form's
//    largest weight gradient, 32 x [2d, d]]
// (the unused slab and gap have always been part of mac_read_bwd_workspace_bytes, which must not change), then for the
// tensor-core forms, 1 KB aligned and each slab 1 KB aligned, with the contraction Mp = M (tc) or M rounded up to 64 (tc32):
//   g [M, 2d] bf16      G of the last wgrad, row-major: bf16(G) (tc) or [G_hi | G_lo] (tc32), the dgrad's A operand
//   xT [2d, Mp] bf16    the wgrad's activations transposed: X^T (tc) or [X_hi^T | X_lo^T] ([2d, 2Mp], tc32)
//   gT [d, Mp] bf16     G transposed: G^T (tc) or [G_hi^T | G_hi^T | G_lo^T] ([d, 3Mp], tc32)
//   w [2d, d] bf16      the dgrad's weight in its own layout: bf16(W) (tc) or [W_hi | W_hi | W_lo] per row ([2d, 3d], tc32)
//   tmp32 fp32          a dgrad's output before its element-wise pass: [M, 2d] (tc) or [M, d] (tc32)
//   dWtmp               split-K partials of the largest weight gradient
// ws may be NULL when only `bytes` is wanted.
struct ReadBwdWs {
  unsigned int* counters;
  float *bufA, *bufB, *bufC, *dka, *dkl, *dy, *md, *dmd, *partial;
  size_t partial_bytes;
  int Mp;
  __nv_bfloat16 *g, *xT, *gT, *w;
  float *tmp32, *dWtmp;
  size_t bytes;          // mac_read_bwd*_workspace_bytes
};
static ReadBwdWs read_bwd_layout(ReadBwdForm f, void* ws, int B, int N, int d) {
  const size_t M = (size_t)B * N, Md = M * d, Bd = (size_t)B * d, Mp4 = (M + 3) & ~(size_t)3;
  const uintptr_t base = reinterpret_cast<uintptr_t>(ws);
  auto fp = [&](size_t o) { return reinterpret_cast<float*>(base + o); };
  ReadBwdWs L{};
  L.counters = reinterpret_cast<unsigned int*>(base);
  L.bufA = fp(BW_HEADER);
  L.bufB = L.bufA + Md;
  L.bufC = L.bufB + Md;
  L.dka = L.bufC + 2 * Md;
  L.dkl = L.dka + Mp4;
  L.dy = L.dkl + Mp4;
  L.md = L.dy + Bd;
  L.dmd = L.md + Bd;
  L.partial = L.dmd + 2 * Bd + 1024;
  L.partial_bytes = (size_t)32 * 2 * d * d * 4;            // sgemm_launch cuts a product into at most 32 slices
  // (M + 4) * 8 bytes cover dka and dkl with their padding
  const size_t fp32 = BW_HEADER + 4 * Md * 4 + (M + 4) * 8 + 4 * Bd * 4 + 4096 + L.partial_bytes;
  const bool split = f == RB_TC32;
  L.Mp = split ? (int)((M + 63) & ~(size_t)63) : (int)M;
  L.bytes = fp32;
  if (f == RB_FP32) return L;
  const uintptr_t tc = (base + fp32 + 1023) & ~(uintptr_t)1023;
  size_t o = 0;
  auto take = [&](size_t bytes) { const size_t r = o; o += (bytes + 1023) & ~(size_t)1023; return tc + r; };
  L.g = reinterpret_cast<__nv_bfloat16*>(take(M * 2 * d * 2));
  L.xT = reinterpret_cast<__nv_bfloat16*>(take((size_t)2 * d * (split ? 2 : 1) * L.Mp * 2));
  L.gT = reinterpret_cast<__nv_bfloat16*>(take((size_t)d * (split ? 3 : 1) * L.Mp * 2));
  L.w = reinterpret_cast<__nv_bfloat16*>(take((size_t)2 * d * (split ? 3 : 1) * d * 2));
  L.tmp32 = reinterpret_cast<float*>(take(M * (split ? 1 : 2) * d * 4));
  L.dWtmp = reinterpret_cast<float*>(take(mac_tc_wgrad_partial_bytes_(2 * d, d)));
  L.bytes = fp32 + 1024 + o;
  return L;
}

// What one mac_read_bwd* call was given, with the layout, the dropout threshold and scale and the parts of `save` filled in
// by read_bwd_run.  Wx_t, Wm_t, Wm2_t: the fp32 form's dgrad weights (the tensor-core forms read w->Wx, w->Wm, w->Wm2).
struct ReadBwdCall {
  ReadBwdForm f;
  const float *kb, *memory_in, *control; const mac_read_weights* w;
  const float *Wx_t, *Wy_t, *Wm_t, *Wm2_t;
  const float *att, *save, *dinfo; float keep; uint64_t seed; int step;
  float *dkb, *dmem_in, *dcontrol, *dWx, *dbx_part, *dWy, *dby, *dWm, *dbm_part, *dWm2, *dbm2_part, *dwr_part, *dbr_part;
  void* ws; size_t ws_bytes; int B, N, d;
  cudaStream_t s;
  ReadBwdWs L; uint32_t thr; float scale;      // thr != 0 exactly when keep < 1
  const float *P, *H, *I1, *y;
};

// Everything a form can refuse, before any CUDA call.  Pointers:
//   required   kb, memory_in, control, w, w->wr, att, save, dinfo, dmem_in, dcontrol, Wy_t, dbx_part, dbm_part, dbm2_part,
//              dwr_part, workspace, the dgrad weights of dI1 and dZ (Wm2_t, Wm_t or w->Wm2, w->Wm), and with dkb that of
//              dP (Wx_t or w->Wx); dWx, dWm and dWm2 for the tensor-core forms
//   optional   dkb, dWy, dby, dbr_part; dWx, dWm, dWm2 for RB_FP32 (their products are skipped)
//   16-byte    kb, memory_in, control, w->wr, save, dinfo, dmem_in, Wy_t, workspace, the dgrad weights, and dkb, dWx, dWy,
//   aligned    dWm, dWm2 when given: the float4 / cp.async accesses of kb_dot, kb_attend_bwd, read_bwd_logits, read_bwd_p,
//              the sgemm and skinny products, elu_bwd_colsum, axpy_dropout, mac_cast_bf16, split3_rows and splitk_accum
// Shapes: B, N, d > 0 (INVALID); d % 128 == 0 for the tensor-core forms and (B*N) % 64 == 0 for RB_TC, whose weight
// gradients contract over B*N in 64-row k-blocks (UNSUPPORTED); d % 4 == 0 (INVALID).  keep_read in (0, 1] (INVALID).
// MAC_ERR_ARCH last.
static int read_bwd_check(const ReadBwdCall& c) {
  if (!c.kb || !c.memory_in || !c.control || !c.w || !c.w->wr || !c.att || !c.save || !c.dinfo || !c.dmem_in ||
      !c.dcontrol || !c.Wy_t || !c.dbx_part || !c.dbm_part || !c.dbm2_part || !c.dwr_part || !c.ws)
    return MAC_ERR_INVALID;
  const bool tc = c.f != RB_FP32;
  const float* Wx = c.dkb ? (tc ? c.w->Wx : c.Wx_t) : nullptr;
  const float *Wm = tc ? c.w->Wm : c.Wm_t, *Wm2 = tc ? c.w->Wm2 : c.Wm2_t;
  if (!Wm || !Wm2 || (c.dkb && !Wx) || (tc && (!c.dWx || !c.dWm || !c.dWm2))) return MAC_ERR_INVALID;
  if (c.B <= 0 || c.N <= 0 || c.d <= 0) return MAC_ERR_INVALID;
  if (tc && ((c.d % 128) || (c.f == RB_TC && (c.B * c.N) % 64))) return MAC_ERR_UNSUPPORTED;
  if ((c.d & 3) || !(c.keep > 0.f && c.keep <= 1.f)) return MAC_ERR_INVALID;
  const void* vec[] = {c.kb, c.memory_in, c.control, c.w->wr, c.save, c.dinfo, c.dmem_in, c.Wy_t, c.ws, Wx, Wm, Wm2,
                       c.dkb, c.dWx, c.dWy, c.dWm, c.dWm2};
  for (const void* p : vec)
    if (p && !mac_aligned16(p)) return MAC_ERR_ALIGN;
  if (c.ws_bytes < read_bwd_layout(c.f, nullptr, c.B, c.N, c.d).bytes) return MAC_ERR_WORKSPACE;
  return tc && !mac_b200_device_ok() ? MAC_ERR_ARCH : MAC_OK;
}

// ------------------------------------------------------------------------------------------------ the four form-specific steps
// The activation X of a weight gradient dW += X^T G: H, [P*y | P] (K = 2d) or dropout(KB) with the forward's mask
enum ReadBwdAct { RB_H, RB_PY_P, RB_KB };

// tensor-core forms: X [M, d] -> Xt (tc: bf16 X^T; tc32: `segs` split segments of Mp columns per row, see the layout) with
// x*y (mode 1) or the forward's KB dropout (mode 2) applied; Xrm (may be NULL) receives the row-major copy
static int rb_pack(const ReadBwdCall& c, int mode, const float* X, void* Xt, void* Xrm, int segs) {
  if (c.f == RB_TC)
    return mac_pack_t_bf16_(mode, X, Xt, Xrm, c.B * c.N, c.d, c.y, c.N, c.thr, c.scale, c.seed, MAC_SITE_READ_KB, c.step, c.s);
  return mac_pack_t_split_(mode, X, Xt, Xrm, c.B * c.N, c.d, segs, c.y, c.N, c.thr, c.scale, c.seed, MAC_SITE_READ_KB, c.step,
                           c.s);
}

// dW[in, d] += X^T G, skipped by RB_FP32 when dW is NULL
static int rb_wgrad(const ReadBwdCall& c, ReadBwdAct a, const float* G, float* dW) {
  const ReadBwdWs& L = c.L;
  const int M = c.B * c.N, d = c.d, in = a == RB_PY_P ? 2 * d : d;
  const float* X = a == RB_H ? c.H : a == RB_PY_P ? c.P : c.kb;
  const bool drop = a == RB_KB && c.thr;
  if (c.f == RB_FP32) {
    if (!dW) return MAC_OK;
    SgemmParams p{};
    p.a_mode = a == RB_PY_P ? A_TRANS_ROWSCALE_CONCAT : drop ? A_TRANS_DROPOUT : A_TRANS;
    p.nseg = 1; p.a[0] = X; p.lda[0] = d; p.rowvec = c.y; p.rows_per_batch = c.N;
    p.a_thresh = c.thr; p.a_scale = c.scale; p.seed = c.seed; p.a_site = MAC_SITE_READ_KB; p.step = c.step;
    p.W = G; p.ldw = d; p.M = in; p.N = d; p.K = M;
    p.epi = EPI_BIAS_ACT; p.Y = dW; p.ldy = d; p.accumulate = 1;
    return sgemm_launch(p, L.counters, L.partial, L.partial_bytes, c.s);
  }
  int st = rb_pack(c, a == RB_PY_P ? 1 : drop ? 2 : 0, X, L.xT, nullptr, 2);                   // rows 0..d-1: X or P*y
  if (st == MAC_OK && a == RB_PY_P)                                                            // rows d..2d-1: P
    st = rb_pack(c, 0, X, L.xT + (size_t)d * (c.f == RB_TC32 ? 2 : 1) * L.Mp, nullptr, 2);
  if (st == MAC_OK) st = rb_pack(c, 0, G, L.gT, L.g, 3);
  if (st != MAC_OK) return st;
  return c.f == RB_TC ? mac_tc_wgrad_splitk_(L.xT, L.gT, dW, L.dWtmp, in, d, M, c.s)
                      : mac_tc3_wgrad_splitk_(L.xT, L.gT, dW, L.dWtmp, in, d, L.Mp, c.s);
}

// out[M, in] = G W^T: RB_FP32 from G and the transposed weight Wt [d, in] with the sgemm epilogue `epi`; the tensor-core
// forms from the weight W [in, d] in its own layout and the copy of G the preceding rb_wgrad left in L.g, stored in fp32
static int rb_dgrad(const ReadBwdCall& c, const float* G, const float* Wt, const float* W, int in, int epi, float* out) {
  const int M = c.B * c.N, d = c.d;
  int st;
  switch (c.f) {
    case RB_FP32: {
      SgemmParams p{};
      p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = G; p.ak[0] = d; p.lda[0] = d;
      p.W = Wt; p.ldw = in; p.M = M; p.N = in; p.K = d;
      p.epi = epi; p.act = MAC_ACT_NON; p.Y = out; p.ldy = in;
      if (epi == EPI_MUL_ELUGRAD) { p.aux = c.H; p.ldaux = d; }
      p.e_thresh = c.thr; p.e_scale = c.scale; p.e_site = MAC_SITE_READ_KB; p.seed = c.seed; p.step = c.step;
      return sgemm_launch(p, nullptr, nullptr, 0, c.s, false);
    }
    case RB_TC:
      st = mac_cast_bf16(W, c.L.w, (long long)in * d, c.s);
      return st != MAC_OK ? st : mac_linear_tc_fwd(c.L.g, c.L.w, nullptr, MAC_ACT_NON, out, 0, M, d, in, c.s);
    default:
      st = mac_split3_rows_(W, c.L.w, in, d, c.s);
      return st != MAC_OK ? st : mac_tc3_linear_(c.L.g, c.L.w, out, M, d, in, c.s);
  }
}

// dZ = (dI1 @ Wm2^T) * ELU'(H) into bufB, dbm_part += its column sums
static int rb_dz(const ReadBwdCall& c) {
  const ReadBwdWs& L = c.L;
  if (c.f == RB_FP32) {
    const int st = rb_dgrad(c, L.bufA, c.Wm2_t, nullptr, c.d, EPI_MUL_ELUGRAD, L.bufB);
    return st != MAC_OK ? st : launch_colsum(L.bufB, c.dbm_part, c.B, c.N, c.d, 1, c.s);
  }
  const int st = rb_dgrad(c, nullptr, nullptr, c.w->Wm2, c.d, 0, L.tmp32);
  if (st != MAC_OK) return st;
  elu_bwd_colsum_kernel<<<dim3((c.d + 127) / 128, c.B), 256, 0, c.s>>>(c.H, L.tmp32, L.bufB, c.dbm_part, c.N, c.d);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// dKB += (dP @ Wx^T) * mask/keep
static int rb_dkb(const ReadBwdCall& c) {
  const ReadBwdWs& L = c.L;
  if (c.f == RB_FP32) return rb_dgrad(c, L.bufA, c.Wx_t, nullptr, c.d, EPI_ACCUM_DROPOUT, c.dkb);
  const int st = rb_dgrad(c, nullptr, nullptr, c.w->Wx, c.d, 0, L.tmp32);
  if (st != MAC_OK) return st;
  const long long n4 = (long long)c.B * c.N * c.d / 4;
  if (!c.thr) return mac_axpy(c.dkb, L.tmp32, 1.f, 4 * n4, c.s);
  axpy_dropout_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, c.s>>>(reinterpret_cast<float4*>(c.dkb),
                                                                     reinterpret_cast<const float4*>(L.tmp32), c.thr, c.scale,
                                                                     c.seed, MAC_SITE_READ_KB, c.step, n4);
  MAC_LAUNCH_CHECK();
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------ the schedule
static int read_bwd_run(ReadBwdCall c) {
  const int B = c.B, N = c.N, d = c.d;
  const size_t Md = (size_t)B * N * d;
  c.L = read_bwd_layout(c.f, c.ws, B, N, d);
  c.thr = c.keep < 1.f ? keep_threshold(c.keep) : 0u;
  c.scale = c.keep < 1.f ? 1.f / c.keep : 1.f;
  c.P = c.save; c.H = c.save + Md; c.I1 = c.save + 2 * Md; c.y = c.save + 3 * Md;     // `save` = [P | H | I1 | y]
  const ReadBwdWs& L = c.L;
  // (1) info = sum_n att*KB ; att = softmax(kl):  dkl, dKB += att (x) dinfo
  int st = mac_kb_attend_bwd(c.kb, c.att, c.dinfo, L.dka, L.dkl, c.dkb, c.dbr_part, B, N, d, c.s);
  if (st != MAC_OK) return st;
  // (2) logits epilogue backward -> dI1 (bufA), dcontrol, dwr, dbm2
  read_bwd_logits_kernel<<<dim3((d + 127) / 128, B), 256, 0, c.s>>>(c.I1, c.control, c.w->wr, L.dkl, c.thr, c.scale, c.seed,
                                                                    c.step, L.bufA, c.dcontrol, c.dwr_part, c.dbm2_part, N, d);
  MAC_LAUNCH_CHECK();
  // (3) I1 = H @ Wm2 + bm2:  dWm2 += H^T dI1 ;  dZ = (dI1 @ Wm2^T) * ELU'(H) ; dbm += colsum(dZ)
  st = rb_wgrad(c, RB_H, L.bufA, c.dWm2);
  if (st == MAC_OK) st = rb_dz(c);
  // (4) H = ELU([P*y, P] @ Wm + bm):  dWm += [P*y, P]^T dZ ;  dI0 = dZ @ Wm^T
  if (st == MAC_OK) st = rb_wgrad(c, RB_PY_P, L.bufB, c.dWm);
  if (st == MAC_OK) st = rb_dgrad(c, L.bufB, c.Wm_t, c.w->Wm, 2 * d, EPI_BIAS_ACT, L.bufC);
  if (st != MAC_OK) return st;
  // (5) I0 = [P*y, P]:  dP (bufA), dy, dbx
  read_bwd_p_kernel<<<dim3((d + 127) / 128, B), 256, 0, c.s>>>(L.bufC, c.P, c.y, L.bufA, L.dy, c.dbx_part, N, d);
  MAC_LAUNCH_CHECK();
  // (6) P = dropout(KB) @ Wx + bx:  dWx += Kd^T dP ;  dKB += (dP @ Wx^T) * mask/keep
  st = rb_wgrad(c, RB_KB, L.bufA, c.dWx);
  if (st == MAC_OK && c.dkb) st = rb_dkb(c);
  if (st != MAC_OK) return st;
  // (7) y = md @ Wy + by with md = dropout(memory_in):  dWy += md^T dy ; dby += colsum(dy) ; dmem_in = (dy @ Wy^T)*mask/keep
  // An M = B product in fp32 for every form.  mac_linear_bwd gets no workspace, so it runs without split-K: its partials
  // would start at bufA, and at small N (B*N*4 < splitk*d) they would overwrite its own inputs dy, md and dmd behind it.
  const bool drop = c.thr != 0;
  if (drop) {
    st = mac_dropout_fwd(c.memory_in, c.keep, c.seed, MAC_SITE_READ_MEM, c.step, L.md, (long long)B * d, c.s);
    if (st != MAC_OK) return st;
  }
  const float* xs[1] = {drop ? L.md : c.memory_in};
  const int ks[1] = {d}, acc0[1] = {0};
  float* dxs[1] = {drop ? L.dmd : c.dmem_in};
  st = mac_linear_bwd(xs, ks, ks, 1, c.Wy_t, L.dy, d, dxs, ks, acc0, c.dWy, c.dby, B, d, nullptr, 0, c.s);
  if (st != MAC_OK || !drop) return st;
  return mac_dropout_fwd(L.dmd, c.keep, c.seed, MAC_SITE_READ_MEM, c.step, c.dmem_in, (long long)B * d, c.s);
}

static int read_bwd(ReadBwdCall c) {
  const int st = read_bwd_check(c);
  return st != MAC_OK ? st : read_bwd_run(c);
}
}  // namespace mac

// ------------------------------------------------------------------------------------------------ entry points
extern "C" size_t mac_read_bwd_workspace_bytes(int B, int N, int d) { return read_bwd_layout(RB_FP32, nullptr, B, N, d).bytes; }
extern "C" size_t mac_read_bwd_tc_workspace_bytes(int B, int N, int d) { return read_bwd_layout(RB_TC, nullptr, B, N, d).bytes; }
extern "C" size_t mac_read_bwd_tc32_workspace_bytes(int B, int N, int d) {
  return read_bwd_layout(RB_TC32, nullptr, B, N, d).bytes;
}

extern "C" int mac_read_bwd(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                            const float* Wx_t, const float* Wy_t, const float* Wm_t, const float* Wm2_t,
                            const float* att, const float* save, const float* dinfo, float keep_read, uint64_t seed,
                            int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx, float* dbx_part,
                            float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2, float* dbm2_part,
                            float* dwr_part, float* dbr_part, void* workspace, size_t workspace_bytes, int B, int N,
                            int d, mac_stream_t stream_) {
  return read_bwd({RB_FP32, kb, memory_in, control, w, Wx_t, Wy_t, Wm_t, Wm2_t, att, save, dinfo, keep_read, seed, step, dkb,
                   dmem_in, dcontrol, dWx, dbx_part, dWy, dby, dWm, dbm_part, dWm2, dbm2_part, dwr_part, dbr_part, workspace,
                   workspace_bytes, B, N, d, reinterpret_cast<cudaStream_t>(stream_)});
}

extern "C" int mac_read_bwd_tc(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                               const float* Wy_t, const float* att, const float* save, const float* dinfo, float keep_read,
                               uint64_t seed, int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx,
                               float* dbx_part, float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2,
                               float* dbm2_part, float* dwr_part, float* dbr_part, void* workspace, size_t workspace_bytes,
                               int B, int N, int d, mac_stream_t stream_) {
  return read_bwd({RB_TC, kb, memory_in, control, w, nullptr, Wy_t, nullptr, nullptr, att, save, dinfo, keep_read, seed, step,
                   dkb, dmem_in, dcontrol, dWx, dbx_part, dWy, dby, dWm, dbm_part, dWm2, dbm2_part, dwr_part, dbr_part,
                   workspace, workspace_bytes, B, N, d, reinterpret_cast<cudaStream_t>(stream_)});
}

extern "C" int mac_read_bwd_tc32(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                                 const float* Wy_t, const float* att, const float* save, const float* dinfo, float keep_read,
                                 uint64_t seed, int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx,
                                 float* dbx_part, float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2,
                                 float* dbm2_part, float* dwr_part, float* dbr_part, void* workspace, size_t workspace_bytes,
                                 int B, int N, int d, mac_stream_t stream_) {
  return read_bwd({RB_TC32, kb, memory_in, control, w, nullptr, Wy_t, nullptr, nullptr, att, save, dinfo, keep_read, seed,
                   step, dkb, dmem_in, dcontrol, dWx, dbx_part, dWy, dby, dWm, dbm_part, dWm2, dbm2_part, dwr_part, dbr_part,
                   workspace, workspace_bytes, B, N, d, reinterpret_cast<cudaStream_t>(stream_)});
}
