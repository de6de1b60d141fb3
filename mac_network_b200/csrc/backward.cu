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

// dx = dy * act'(.) expressed through the saved OUTPUT y (tanh: 1-y^2; sigmoid: y(1-y); elu: y>0?1:y+1; relu: y>0)
__global__ void act_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, int act,
                               float* __restrict__ dx, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = y[i];
  float g = 1.f;
  if (act == MAC_ACT_TANH) g = 1.f - v * v;
  else if (act == MAC_ACT_SIGMOID) g = v * (1.f - v);
  else if (act == MAC_ACT_ELU) g = v > 0.f ? 1.f : v + 1.f;
  else if (act == MAC_ACT_RELU) g = v > 0.f ? 1.f : 0.f;
  dx[i] = dy[i] * g;
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

// Backward of mac_read_fwd (fp32 path).  `save` = [P | H | I1 | y] from the forward.  Gradients in:
//   dinfo [B,d].  Gradients out / accumulated:
//   dkb [B,N,d] += (may be NULL), dmem_in [B,d] = gradient w.r.t. memory_in (the tensor handed to mac_read_fwd),
//   dcontrol [B,d] +=, parameter gradients += (dWx..dWm2 full; bias / wr gradients as per-sample partials [B,d] that
//   the caller reduces over B once per backward pass; dbr_part [B]).
extern "C" size_t mac_read_bwd_workspace_bytes(int B, int N, int d) {
  const size_t Md = (size_t)B * N * d * 4;
  return BW_HEADER + 4 * Md /*dI1|dZ, dI0 (2x), dP*/ + ((size_t)B * N + 4) * 8 + (size_t)4 * B * d * 4 + 4096 +
         (size_t)32 * 2 * d * d * 4 /*split-K partials of the largest wgrad*/;
}

extern "C" int mac_read_bwd(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                            const float* Wx_t, const float* Wy_t, const float* Wm_t, const float* Wm2_t,
                            const float* att, const float* save, const float* dinfo, float keep_read, uint64_t seed,
                            int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx, float* dbx_part,
                            float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2, float* dbm2_part,
                            float* dwr_part, float* dbr_part, void* workspace, size_t workspace_bytes, int B, int N,
                            int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!kb || !memory_in || !control || !w || !att || !save || !dinfo || !dmem_in || !dcontrol || !workspace)
    return MAC_ERR_INVALID;
  if (workspace_bytes < mac_read_bwd_workspace_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const int M = B * N;
  const size_t Md = (size_t)M * d;
  char* ws = reinterpret_cast<char*>(workspace);
  unsigned int* counters = reinterpret_cast<unsigned int*>(ws);
  float* f = reinterpret_cast<float*>(ws + BW_HEADER);
  float* bufA = f;                 // dI1, then dZ (in place is not possible: separate GEMM output) -> dI1 here
  float* bufB = f + Md;            // dZ
  float* bufC = f + 2 * Md;        // dI0 [M, 2d]
  float* dka = f + 4 * Md;         // [B,N]
  const size_t BNp = ((size_t)B * N + 3) & ~(size_t)3;   // keep the [B,d] buffers behind it 16-byte aligned
  float* dkl = dka + BNp;
  float* dy = dkl + BNp;           // [B,d]
  float* md = dy + (size_t)B * d;  // [B,d] recomputed dropped memory
  float* dmd = md + (size_t)B * d; // [B,d]
  float* partial = dmd + (size_t)2 * B * d + 1024;
  const size_t pbytes = workspace_bytes - (reinterpret_cast<char*>(partial) - ws);
  const float* P = save;
  const float* H = save + Md;
  const float* I1 = save + 2 * Md;
  const float* y = save + 3 * Md;
  const bool drop = keep_read < 1.f;
  const uint32_t thr = drop ? keep_threshold(keep_read) : 0u;
  const float scale = drop ? 1.f / keep_read : 1.f;
  int st;
  // (1) info = sum_n att*KB ; att = softmax(kl):  dkl, dKB += att (x) dinfo
  st = mac_kb_attend_bwd(kb, att, dinfo, dka, dkl, dkb, dbr_part, B, N, d, stream_);
  if (st != MAC_OK) return st;
  // (2) logits epilogue backward -> dI1, dcontrol, dwr, dbm2
  read_bwd_logits_kernel<<<dim3((d + 127) / 128, B), 256, 0, stream>>>(I1, control, w->wr, dkl, thr, scale, seed, step,
                                                                      bufA, dcontrol, dwr_part, dbm2_part, N, d);
  MAC_LAUNCH_CHECK();
  // (3) I1 = H @ Wm2 + bm2:  dWm2 += H^T dI1 ;  dZ = (dI1 @ Wm2^T) * ELU'(Z)
  if (dWm2) {
    SgemmParams p{};
    p.a_mode = A_TRANS; p.nseg = 1; p.a[0] = H; p.lda[0] = d;
    p.W = bufA; p.ldw = d; p.M = d; p.N = d; p.K = M;
    p.epi = EPI_BIAS_ACT; p.Y = dWm2; p.ldy = d; p.accumulate = 1;
    st = sgemm_launch(p, counters, partial, pbytes, stream);
    if (st != MAC_OK) return st;
  }
  {
    SgemmParams p{};
    p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = bufA; p.ak[0] = d; p.lda[0] = d;
    p.W = Wm2_t; p.ldw = d; p.M = M; p.N = d; p.K = d;
    p.epi = EPI_MUL_ELUGRAD; p.aux = H; p.ldaux = d; p.Y = bufB; p.ldy = d;
    st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
    if (st != MAC_OK) return st;
  }
  st = launch_colsum(bufB, dbm_part, B, N, d, 1, stream);
  if (st != MAC_OK) return st;
  // (4) Z = [P*y, P] @ Wm + bm:  dWm += I0^T dZ ;  dI0 = dZ @ Wm^T
  if (dWm) {
    SgemmParams p{};
    p.a_mode = A_TRANS_ROWSCALE_CONCAT; p.nseg = 1; p.a[0] = P; p.lda[0] = d; p.rowvec = y; p.rows_per_batch = N;
    p.W = bufB; p.ldw = d; p.M = 2 * d; p.N = d; p.K = M;
    p.epi = EPI_BIAS_ACT; p.Y = dWm; p.ldy = d; p.accumulate = 1;
    st = sgemm_launch(p, counters, partial, pbytes, stream);
    if (st != MAC_OK) return st;
  }
  {
    SgemmParams p{};
    p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = bufB; p.ak[0] = d; p.lda[0] = d;
    p.W = Wm_t; p.ldw = 2 * d; p.M = M; p.N = 2 * d; p.K = d;
    p.epi = EPI_BIAS_ACT; p.act = MAC_ACT_NON; p.Y = bufC; p.ldy = 2 * d;
    st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
    if (st != MAC_OK) return st;
  }
  // (5) I0 = [P*y, P]:  dP, dy, dbx   (dP overwrites bufA)
  read_bwd_p_kernel<<<dim3((d + 127) / 128, B), 256, 0, stream>>>(bufC, P, y, bufA, dy, dbx_part, N, d);
  MAC_LAUNCH_CHECK();
  // (6) P = dropout(KB) @ Wx + bx:  dWx += Kd^T dP ;  dKB += (dP @ Wx^T) * mask/keep
  if (dWx) {
    SgemmParams p{};
    p.a_mode = drop ? A_TRANS_DROPOUT : A_TRANS; p.nseg = 1; p.a[0] = kb; p.lda[0] = d;
    p.a_thresh = thr; p.a_scale = scale; p.seed = seed; p.a_site = MAC_SITE_READ_KB; p.step = step;
    p.W = bufA; p.ldw = d; p.M = d; p.N = d; p.K = M;
    p.epi = EPI_BIAS_ACT; p.Y = dWx; p.ldy = d; p.accumulate = 1;
    st = sgemm_launch(p, counters, partial, pbytes, stream);
    if (st != MAC_OK) return st;
  }
  if (dkb) {
    SgemmParams p{};
    p.a_mode = A_SEGS; p.nseg = 1; p.a[0] = bufA; p.ak[0] = d; p.lda[0] = d;
    p.W = Wx_t; p.ldw = d; p.M = M; p.N = d; p.K = d;
    p.epi = EPI_ACCUM_DROPOUT; p.Y = dkb; p.ldy = d;
    p.e_thresh = thr; p.e_scale = scale; p.e_site = MAC_SITE_READ_KB; p.seed = seed; p.step = step;
    st = sgemm_launch(p, nullptr, nullptr, 0, stream, false);
    if (st != MAC_OK) return st;
  }
  // (7) y = md @ Wy + by with md = dropout(memory_in):  dWy += md^T dy ; dby += colsum(dy) ; dmem_in = (dy @ Wy^T)*mask/keep
  const float* mdp = memory_in;
  if (drop) {
    st = mac_dropout_fwd(memory_in, keep_read, seed, MAC_SITE_READ_MEM, step, md, (long long)B * d, stream_);
    if (st != MAC_OK) return st;
    mdp = md;
  }
  {
    const float* xs[1] = {mdp};
    const int ks[1] = {d};
    float* dxs[1] = {drop ? dmd : dmem_in};
    const int acc0[1] = {0};
    st = mac_linear_bwd(xs, ks, ks, 1, Wy_t, dy, d, dxs, ks, acc0, dWy, dby, B, d, ws, BW_HEADER + pbytes / 2, stream_);
    if (st != MAC_OK) return st;
    if (drop) {
      st = mac_dropout_fwd(dmd, keep_read, seed, MAC_SITE_READ_MEM, step, dmem_in, (long long)B * d, stream_);
      if (st != MAC_OK) return st;
    }
  }
  return MAC_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// Backward of the read unit with the six [B*N, .] x [., .] products on wgmma tensor cores (bf16 operands, fp32
// accumulation; everything element-wise stays fp32).  Same inputs, outputs and accumulation conventions as
// mac_read_bwd; the GEMMs go through the entry points the forward uses (mac_linear_tc_fwd), fed by the cast / transposing
// cast kernels (mac_cast_bf16, mac_pack_weight_bf16):
//   dgrad  dX[M, in]   = dY[M, out] @ W^T        x = bf16(dY) [M, out],  Wt operand = bf16(W) in its own [in, out] layout
//   wgrad  dW[in, out] = X^T[in, M] @ dY[M, out]  x = bf16(X)^T [in, M],  Wt operand = bf16(dY)^T [out, M]   (K = M = B*N)
// The prologue fusions of the fp32 kernels live in the transposing cast here (pack_t_bf16_kernel applies P*y / the KB dropout
// mask while it builds the bf16 operand, and writes the row-major bf16 copy of a gradient from the same read); * ELU'(H) with
// its column sums and the dropout mask on dKB are one fp32 pass each.  The arithmetic of every pass is the forward's, so the
// masks and saved tensors are shared.
// Requires d % 128 == 0 and (B*N) % 64 == 0 (the UMMA K block); otherwise MAC_ERR_UNSUPPORTED (use mac_read_bwd).
// ------------------------------------------------------------------------------------------------------------------
extern "C" int mac_tc_wgrad_splitk_(const void* xT, const void* gT, float* dW, float* partial, int in_dim, int out_dim, int K,
                                    mac_stream_t stream_);
extern "C" size_t mac_tc_wgrad_partial_bytes_(int in_dim, int out_dim);
extern "C" int mac_pack_t_bf16_(int mode, const float* X, void* Xt, void* Xrm, int K, int N, const float* rowvec,
                                int rows_per_batch, uint32_t thresh, float scale, uint64_t seed, int site, int step,
                                mac_stream_t stream_);
static size_t rbt_align(size_t x) { return (x + 1023) & ~(size_t)1023; }

extern "C" size_t mac_read_bwd_tc_workspace_bytes(int B, int N, int d) {
  const size_t M = (size_t)B * N;
  return mac_read_bwd_workspace_bytes(B, N, d) + 1024 + rbt_align(M * 2 * d * 2) /*g16*/ + rbt_align(2 * d * M * 2) /*xT16*/ +
         rbt_align(d * M * 2) /*gT16*/ + rbt_align((size_t)2 * d * d * 2) /*w16*/ + rbt_align(M * 2 * d * 4) /*tmp32*/ +
         rbt_align(mac_tc_wgrad_partial_bytes_(2 * d, d)) /*dWtmp: split-K partials of the largest weight gradient*/;
}

extern "C" int mac_read_bwd_tc(const float* kb, const float* memory_in, const float* control, const mac_read_weights* w,
                               const float* Wy_t, const float* att, const float* save, const float* dinfo, float keep_read,
                               uint64_t seed, int step, float* dkb, float* dmem_in, float* dcontrol, float* dWx,
                               float* dbx_part, float* dWy, float* dby, float* dWm, float* dbm_part, float* dWm2,
                               float* dbm2_part, float* dwr_part, float* dbr_part, void* workspace, size_t workspace_bytes,
                               int B, int N, int d, mac_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  if (!kb || !memory_in || !control || !w || !att || !save || !dinfo || !dmem_in || !dcontrol || !workspace || !dWx ||
      !dWm || !dWm2)
    return MAC_ERR_INVALID;
  const int M = B * N;
  if ((d % 128) || (M % 64)) return MAC_ERR_UNSUPPORTED;
  if (workspace_bytes < mac_read_bwd_tc_workspace_bytes(B, N, d)) return MAC_ERR_WORKSPACE;
  const size_t Md = (size_t)M * d;
  char* ws = reinterpret_cast<char*>(workspace);
  float* f = reinterpret_cast<float*>(ws + BW_HEADER);
  float* bufA = f;                 // dI1, later dP
  float* bufB = f + Md;            // dZ
  float* bufC = f + 2 * Md;        // dI0 [M, 2d]
  float* dka = f + 4 * Md;         // [B,N]
  const size_t BNp = ((size_t)B * N + 3) & ~(size_t)3;
  float* dkl = dka + BNp;
  float* dy = dkl + BNp;           // [B,d]
  float* md = dy + (size_t)B * d;  // [B,d]
  float* dmd = md + (size_t)B * d; // [B,d]
  // tensor-core operands behind the fp32 layout of mac_read_bwd
  char* x = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(ws + mac_read_bwd_workspace_bytes(B, N, d)) + 1023) &
                                    ~(uintptr_t)1023);
  void* g16 = x;   x += rbt_align((size_t)M * 2 * d * 2);        // bf16 [M, <=2d]   gradient as the A operand of a dgrad
  void* xT16 = x;  x += rbt_align((size_t)2 * d * M * 2);        // bf16 [<=2d, M]   activations, transposed
  void* gT16 = x;  x += rbt_align((size_t)d * M * 2);            // bf16 [d, M]      gradient, transposed
  void* w16 = x;   x += rbt_align((size_t)2 * d * d * 2);        // bf16 weight in its own [in, out] layout
  float* tmp32 = reinterpret_cast<float*>(x); x += rbt_align((size_t)M * 2 * d * 4);
  float* dWtmp = reinterpret_cast<float*>(x);
  const float* P = save;
  const float* H = save + Md;
  const float* I1 = save + 2 * Md;
  const float* y = save + 3 * Md;
  const bool drop = keep_read < 1.f;
  const uint32_t thr = drop ? keep_threshold(keep_read) : 0u;
  const float scale = drop ? 1.f / keep_read : 1.f;
  int st;
#define RBT(call)                 \
  do {                            \
    st = (call);                  \
    if (st != MAC_OK) return st;  \
  } while (0)
  // activations / gradients for the tensor-core operands: fp32 [M, d] -> bf16 transposed [d, M] (+ optionally the row-major
  // bf16 copy), with the forward's P*y scaling or KB dropout applied on the way (pack_t_bf16_kernel, csrc/tc_gemm.cuh)
  auto packT = [&](int mode, const float* X, void* Xt, void* Xrm, const float* rowvec) -> int {
    return mac_pack_t_bf16_(mode, X, Xt, Xrm, M, d, rowvec, N, thr, scale, seed, MAC_SITE_READ_KB, step, stream_);
  };
  // wgrad: dW[in, out] += X^T @ G with X^T already packed as xT [in, M]; leaves bf16(G) row-major in g16 for the dgrad below
  auto wgrad = [&](const void* xT, int in, const float* G, float* dW) -> int {
    int s = packT(0, G, gT16, g16, nullptr);                                                 // G [M, d] -> G^T [d, M], bf16(G)
    if (s != MAC_OK) return s;
    return mac_tc_wgrad_splitk_(xT, gT16, dW, dWtmp, in, d, M, stream_);                          // dW[in, d] += xT @ (G^T)^T, split-K
  };
  // dgrad: out[M, in] = G[M, d] @ W[in, d]^T   (W fp32 in its own [in, out = d] layout; G = the g16 of the preceding wgrad)
  auto dgrad = [&](const float* W, int in, float* out) -> int {
    int s = mac_cast_bf16(W, w16, (long long)in * d, stream_);
    if (s != MAC_OK) return s;
    return mac_linear_tc_fwd(g16, w16, nullptr, MAC_ACT_NON, out, 0, M, d, in, stream_);
  };
  // (1) info = sum_n att*KB ; att = softmax(kl):  dkl, dKB += att (x) dinfo
  RBT(mac_kb_attend_bwd(kb, att, dinfo, dka, dkl, dkb, dbr_part, B, N, d, stream_));
  // (2) logits epilogue backward -> dI1 (bufA), dcontrol, dwr, dbm2
  read_bwd_logits_kernel<<<dim3((d + 127) / 128, B), 256, 0, stream>>>(I1, control, w->wr, dkl, thr, scale, seed, step,
                                                                      bufA, dcontrol, dwr_part, dbm2_part, N, d);
  MAC_LAUNCH_CHECK();
  // (3) I1 = H @ Wm2 + bm2:  dWm2 += H^T dI1 ;  dZ = (dI1 @ Wm2^T) * ELU'(H) ; dbm += colsum(dZ)
  RBT(packT(0, H, xT16, nullptr, nullptr));
  RBT(wgrad(xT16, d, bufA, dWm2));
  RBT(dgrad(w->Wm2, d, tmp32));
  elu_bwd_colsum_kernel<<<dim3((d + 127) / 128, B), 256, 0, stream>>>(H, tmp32, bufB, dbm_part, N, d);
  MAC_LAUNCH_CHECK();
  // (4) Z = [P*y, P] @ Wm + bm:  dWm += [P*y, P]^T dZ ;  dI0 = dZ @ Wm^T
  RBT(packT(1, P, xT16, nullptr, y));                                                            // rows 0..d-1   of [2d, M]: (P*y)^T
  RBT(packT(0, P, reinterpret_cast<__nv_bfloat16*>(xT16) + (size_t)d * M, nullptr, nullptr));    // rows d..2d-1: P^T
  RBT(wgrad(xT16, 2 * d, bufB, dWm));
  RBT(dgrad(w->Wm, 2 * d, bufC));
  // (5) I0 = [P*y, P]:  dP (bufA), dy, dbx
  read_bwd_p_kernel<<<dim3((d + 127) / 128, B), 256, 0, stream>>>(bufC, P, y, bufA, dy, dbx_part, N, d);
  MAC_LAUNCH_CHECK();
  // (6) P = dropout(KB) @ Wx + bx:  dWx += Kd^T dP ;  dKB += (dP @ Wx^T) * mask/keep
  RBT(packT(drop ? 2 : 0, kb, xT16, nullptr, nullptr));                                          // dropout(KB)^T: the forward's mask
  RBT(wgrad(xT16, d, bufA, dWx));
  if (dkb) {
    RBT(dgrad(w->Wx, d, tmp32));
    if (drop) {
      axpy_dropout_kernel<<<(unsigned)((Md / 4 + 255) / 256), 256, 0, stream>>>(
          reinterpret_cast<float4*>(dkb), reinterpret_cast<const float4*>(tmp32), thr, scale, seed, MAC_SITE_READ_KB, step,
          (long long)(Md / 4));
      MAC_LAUNCH_CHECK();
    } else {
      RBT(mac_axpy(dkb, tmp32, 1.f, (long long)Md, stream_));
    }
  }
  // (7) y = md @ Wy + by with md = dropout(memory_in): an M = B product, fp32 (mac_linear_bwd)
  const float* mdp = memory_in;
  if (drop) {
    RBT(mac_dropout_fwd(memory_in, keep_read, seed, MAC_SITE_READ_MEM, step, md, (long long)B * d, stream_));
    mdp = md;
  }
  {
    const float* xs[1] = {mdp};
    const int ks[1] = {d};
    float* dxs[1] = {drop ? dmd : dmem_in};
    const int acc0[1] = {0};
    RBT(mac_linear_bwd(xs, ks, ks, 1, Wy_t, dy, d, dxs, ks, acc0, dWy, dby, B, d, nullptr, 0, stream_));
    if (drop) RBT(mac_dropout_fwd(dmd, keep_read, seed, MAC_SITE_READ_MEM, step, dmem_in, (long long)B * d, stream_));
  }
#undef RBT
  return MAC_OK;
}
