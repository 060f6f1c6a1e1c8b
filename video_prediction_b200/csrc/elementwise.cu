// HBM-bound kernels of the SAVP path (forward): instance norm, ConvLSTM gates, tile-concat, dense,
// CDNA kernel head / apply, mask softmax + compositing, small utilities.
// All tensors fp32 channels-last with an explicit channel stride so producers write straight into
// the concat buffers their consumers read (no tf.concat / tile_concat materialisation passes).
#include "common.h"
#include "ptx.cuh"

namespace vp {

__device__ __forceinline__ float act_fn(float v, int act, float alpha) {
  switch (act) {
    case VP_ACT_RELU: return fmaxf(v, 0.f);
    case VP_ACT_LRELU: return fmaxf(alpha * v, v);
    case VP_ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    case VP_ACT_TANH: return tanhf(v);
    default: return v;
  }
}
__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + __expf(-v)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// block-wide sum of kN values per thread; result broadcast to all threads. scratch: [kN][32] floats.
template <int kN>
__device__ __forceinline__ void block_sum(float* vals, float* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int i = 0; i < kN; ++i) vals[i] = warp_sum(vals[i]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < kN; ++i) scratch[i * 32 + warp] = vals[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kN; ++i) {
    float v = (lane < nw) ? scratch[i * 32 + lane] : 0.f;
    vals[i] = warp_sum(v);
  }
}

// ------------------------------------------------------------------------------------------------
// instance norm (+affine, +activation):  layers/normalization.py:34-196 (fused_batch_norm training
// mode on the [1,HW,1,N*C] view == per-(n,c) mean / biased variance), eps 1e-6.
// One CTA per (sample, group of 4 channels); three passes over a plane that lives in L2.
// ------------------------------------------------------------------------------------------------
// The (sample, 4-channel) plane is staged once in shared memory (16 B per position): one HBM/L2 read, one write.
__global__ void __launch_bounds__(512) inorm_act_kernel(const float* __restrict__ x, int xs, float* __restrict__ y,
                                                        int ys, int P, int C, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int act,
                                                        float alpha, float* __restrict__ stats, int staged) {
  extern __shared__ float4 splane[];
  __shared__ float scratch[4 * 32];
  const int n = blockIdx.y, c0 = blockIdx.x * 4;
  const float* xp = x + static_cast<long long>(n) * P * xs + c0;
  float* yp = y + static_cast<long long>(n) * P * ys + c0;
  float s[4] = {0.f, 0.f, 0.f, 0.f};
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float4 v = *reinterpret_cast<const float4*>(xp + static_cast<long long>(p) * xs);
    if (staged) splane[p] = v;
    s[0] += v.x; s[1] += v.y; s[2] += v.z; s[3] += v.w;
  }
  block_sum<4>(s, scratch);
  const float inv = 1.f / P;
  const float m[4] = {s[0] * inv, s[1] * inv, s[2] * inv, s[3] * inv};
  float q[4] = {0.f, 0.f, 0.f, 0.f};
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float4 v = staged ? splane[p] : *reinterpret_cast<const float4*>(xp + static_cast<long long>(p) * xs);
    q[0] += (v.x - m[0]) * (v.x - m[0]); q[1] += (v.y - m[1]) * (v.y - m[1]);
    q[2] += (v.z - m[2]) * (v.z - m[2]); q[3] += (v.w - m[3]) * (v.w - m[3]);
  }
  block_sum<4>(q, scratch);
  float r[4], g[4], b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    r[i] = rsqrtf(q[i] * inv + eps);
    g[i] = (gamma ? gamma[c0 + i] : 1.f) * r[i];
    b[i] = (beta ? beta[c0 + i] : 0.f) - m[i] * g[i];
  }
  if (stats && threadIdx.x < 4) {
    stats[(static_cast<long long>(n) * C + c0 + threadIdx.x) * 2 + 0] = m[threadIdx.x];
    stats[(static_cast<long long>(n) * C + c0 + threadIdx.x) * 2 + 1] = r[threadIdx.x];
  }
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float4 v = staged ? splane[p] : *reinterpret_cast<const float4*>(xp + static_cast<long long>(p) * xs);
    float4 o;
    o.x = act_fn(v.x * g[0] + b[0], act, alpha); o.y = act_fn(v.y * g[1] + b[1], act, alpha);
    o.z = act_fn(v.z * g[2] + b[2], act, alpha); o.w = act_fn(v.w * g[3] + b[3], act, alpha);
    *reinterpret_cast<float4*>(yp + static_cast<long long>(p) * ys) = o;
  }
}

// ------------------------------------------------------------------------------------------------
// ConvLSTM gates: rnn_ops.py:148-165.  pre = conv output [N,P,4F] (i,j,f,o).  One CTA per
// (sample, 4 state channels): the 16 gate planes + c are read once into shared memory, both
// instance norms (over the 4F concat and over new_c) complete on-chip.
//   i,j,f,o = IN(pre)*g1+b1 ; c' = c*sig(f+1) + sig(i)*tanh(j) ; cn = IN(c')*g2+b2 ; h = tanh(cn)*sig(o)
// ------------------------------------------------------------------------------------------------
constexpr int kGatesMaxP = 1024;
struct GateDst { float* ptr[3]; int stride[3]; int count; };

__global__ void __launch_bounds__(512) lstm_gates_fwd_kernel(const float* __restrict__ pre, int P, int F,
                                                             const float* __restrict__ c_prev,
                                                             const float* __restrict__ g1, const float* __restrict__ b1,
                                                             const float* __restrict__ g2, const float* __restrict__ b2,
                                                             float forget_bias, float eps, float* __restrict__ c_new,
                                                             GateDst hdst, float* __restrict__ stats1,
                                                             float* __restrict__ stats2) {
  extern __shared__ float sm[];            // [16][P] gates (float4-granular), then [4][P] c'
  __shared__ float scratch[16 * 32];
  float4* sg = reinterpret_cast<float4*>(sm);            // index [gate(4)][p] -> float4 of 4 channels
  float4* sc = sg + 4 * P;
  const int n = blockIdx.y, c0 = blockIdx.x * 4;
  const float* pp = pre + static_cast<long long>(n) * P * 4 * F;
  const float inv = 1.f / P;
  float s[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) s[i] = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 v = *reinterpret_cast<const float4*>(pp + static_cast<long long>(p) * 4 * F + g * F + c0);
      sg[g * P + p] = v;
      s[4 * g] += v.x; s[4 * g + 1] += v.y; s[4 * g + 2] += v.z; s[4 * g + 3] += v.w;
    }
  }
  block_sum<16>(s, scratch);
  float m[16], q[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) { m[i] = s[i] * inv; q[i] = 0.f; }
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 v = sg[g * P + p];
      q[4 * g] += (v.x - m[4 * g]) * (v.x - m[4 * g]);
      q[4 * g + 1] += (v.y - m[4 * g + 1]) * (v.y - m[4 * g + 1]);
      q[4 * g + 2] += (v.z - m[4 * g + 2]) * (v.z - m[4 * g + 2]);
      q[4 * g + 3] += (v.w - m[4 * g + 3]) * (v.w - m[4 * g + 3]);
    }
  }
  block_sum<16>(q, scratch);
  float ga[16], be[16];
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ch = g * F + c0 + k;
      const float r = rsqrtf(q[4 * g + k] * inv + eps);
      if (stats1 && threadIdx.x == 0) {
        stats1[(static_cast<long long>(n) * 4 * F + ch) * 2] = m[4 * g + k];
        stats1[(static_cast<long long>(n) * 4 * F + ch) * 2 + 1] = r;
      }
      ga[4 * g + k] = g1[ch] * r;
      be[4 * g + k] = b1[ch] - m[4 * g + k] * ga[4 * g + k];
    }
  // gates -> c' (pre-norm), kept in shared memory
  float cs[4] = {0.f, 0.f, 0.f, 0.f};
  const float* cp = c_prev + static_cast<long long>(n) * P * F + c0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float4 vi = sg[p], vj = sg[P + p], vf = sg[2 * P + p];
    const float4 c = *reinterpret_cast<const float4*>(cp + static_cast<long long>(p) * F);
    float4 o;
    o.x = c.x * sigmoidf_(vf.x * ga[8] + be[8] + forget_bias) + sigmoidf_(vi.x * ga[0] + be[0]) * tanhf(vj.x * ga[4] + be[4]);
    o.y = c.y * sigmoidf_(vf.y * ga[9] + be[9] + forget_bias) + sigmoidf_(vi.y * ga[1] + be[1]) * tanhf(vj.y * ga[5] + be[5]);
    o.z = c.z * sigmoidf_(vf.z * ga[10] + be[10] + forget_bias) + sigmoidf_(vi.z * ga[2] + be[2]) * tanhf(vj.z * ga[6] + be[6]);
    o.w = c.w * sigmoidf_(vf.w * ga[11] + be[11] + forget_bias) + sigmoidf_(vi.w * ga[3] + be[3]) * tanhf(vj.w * ga[7] + be[7]);
    sc[p] = o;
    cs[0] += o.x; cs[1] += o.y; cs[2] += o.z; cs[3] += o.w;
  }
  block_sum<4>(cs, scratch);
  float cm[4], cq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 4; ++k) cm[k] = cs[k] * inv;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float4 v = sc[p];
    cq[0] += (v.x - cm[0]) * (v.x - cm[0]); cq[1] += (v.y - cm[1]) * (v.y - cm[1]);
    cq[2] += (v.z - cm[2]) * (v.z - cm[2]); cq[3] += (v.w - cm[3]) * (v.w - cm[3]);
  }
  block_sum<4>(cq, scratch);
  float cg[4], cb[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float r = rsqrtf(cq[k] * inv + eps);
    if (stats2 && threadIdx.x == 0) {
      stats2[(static_cast<long long>(n) * F + c0 + k) * 2] = cm[k];
      stats2[(static_cast<long long>(n) * F + c0 + k) * 2 + 1] = r;
    }
    cg[k] = g2[c0 + k] * r;
    cb[k] = b2[c0 + k] - cm[k] * cg[k];
  }
  float* cn = c_new + static_cast<long long>(n) * P * F + c0;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float4 v = sc[p], vo = sg[3 * P + p];
    float4 c, h;
    c.x = v.x * cg[0] + cb[0]; c.y = v.y * cg[1] + cb[1]; c.z = v.z * cg[2] + cb[2]; c.w = v.w * cg[3] + cb[3];
    h.x = tanhf(c.x) * sigmoidf_(vo.x * ga[12] + be[12]); h.y = tanhf(c.y) * sigmoidf_(vo.y * ga[13] + be[13]);
    h.z = tanhf(c.z) * sigmoidf_(vo.z * ga[14] + be[14]); h.w = tanhf(c.w) * sigmoidf_(vo.w * ga[15] + be[15]);
    *reinterpret_cast<float4*>(cn + static_cast<long long>(p) * F) = c;
    for (int d = 0; d < hdst.count; ++d)
      *reinterpret_cast<float4*>(hdst.ptr[d] + (static_cast<long long>(n) * P + p) * hdst.stride[d] + c0) = h;
  }
}

// ------------------------------------------------------------------------------------------------
// small utilities
// ------------------------------------------------------------------------------------------------
// dst[n, p, c] = vec[n, c]  (ops.tile_concat, ops.py:968-1006: spatial broadcast of z / actions)
__global__ void broadcast_channels_kernel(const float* __restrict__ vec, int vs, float* __restrict__ dst, int ds,
                                          long long total, int P, int Cv) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % Cv);
  const long long np = idx / Cv;
  const long long n = np / P;
  dst[np * ds + c] = vec[n * vs + c];
}
// dst[.., c] = src[.., c] for c < C (channel-slice copy between channels-last buffers)
__global__ void copy_channels_kernel(const float* __restrict__ src, int ss, float* __restrict__ dst, int ds,
                                     long long total, int C) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % C);
  const long long np = idx / C;
  dst[np * ds + c] = src[np * ss + c];
}
// out[n] = sel[n] ? a[n] : b[n]   (tf.where(ground_truth[t], images, gen_image), savp_model.py:406)
__global__ void select_rows_kernel(const int32_t* __restrict__ sel, const float4* __restrict__ a,
                                   const float4* __restrict__ b, float4* __restrict__ out, long long per, long long total) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  out[idx] = sel[idx / per] ? a[idx] : b[idx];
}
// global average pool over P positions: [N,P,C] -> [N,C]  (networks.py:30-31)
__global__ void avgpool_kernel(const float* __restrict__ x, int xs, float* __restrict__ y, int P, int C) {
  const int n = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float* xp = x + static_cast<long long>(n) * P * xs + c;
  float s = 0.f;
  for (int p = 0; p < P; ++p) s += xp[static_cast<long long>(p) * xs];
  y[static_cast<long long>(n) * C + c] = s / P;
}

// ------------------------------------------------------------------------------------------------
// dense: y[b, j] (+)= sum_k x[b,k] W[k,j] (+ bias)   (ops.dense, ops.py:5-16).  Lanes run over j
// (coalesced rows of W), 4 batch rows share each W element, k is split over warps and CTAs.
// y must be zero-filled by the caller when gridDim.y > 1 (atomic accumulation).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dense_fwd_kernel(const float* __restrict__ x, int xs, const float* __restrict__ W,
                                                        const float* __restrict__ bias, const float* __restrict__ inv_scale,
                                                        float* __restrict__ y, int ys, int B, int K, int J, int kchunk) {
  const int b0 = blockIdx.x * 4;
  const int k_begin = blockIdx.y * kchunk, k_end = min(K, k_begin + kchunk);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __shared__ float red[8][4][32];
  const float sc = inv_scale ? 1.f / __ldg(inv_scale) : 1.f;
  for (int j0 = 0; j0 < J; j0 += 32) {
    const int j = j0 + lane;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (j < J) {
      for (int k = k_begin + warp; k < k_end; k += nw) {
        const float w = W[static_cast<long long>(k) * J + j];
#pragma unroll
        for (int r = 0; r < 4; ++r)
          if (b0 + r < B) acc[r] += x[static_cast<long long>(b0 + r) * xs + k] * w;
      }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) red[warp][r][lane] = acc[r];
    __syncthreads();
    if (warp < 4 && j < J && b0 + warp < B) {
      float t = 0.f;
      for (int w2 = 0; w2 < nw; ++w2) t += red[w2][warp][lane];
      t *= sc;
      if (bias && blockIdx.y == 0) t += bias[j];
      // with K split over blockIdx.y, y is a scratch buffer of dense [B][J] parts (ys = J), summed in block order by the host
      float* o = y + static_cast<long long>(blockIdx.y) * B * ys + static_cast<long long>(b0 + warp) * ys + j;
      *o = t;
    }
    __syncthreads();
  }
}


// Tiled forward for the wide CDNA-kernel dense layer (K = 8192 -> J = 100, B <= 64 rows): one CTA per 64 k, W tile and
// the transposed x slab staged in shared memory; every thread owns a 4 (rows) x 4 (outputs) register tile fed by two
// 16-byte shared loads per k; partial [B, J] products are reduced into the zero-filled y with atomics.
__global__ void __launch_bounds__(256) dense_fwd_tiled_kernel(const float* __restrict__ x, int xs, const float* __restrict__ W,
                                                              const float* __restrict__ bias, const float* __restrict__ inv_scale,
                                                              float* __restrict__ y, int ys, int B, int K, int J) {
  extern __shared__ __align__(16) float fsm[];
  const int BP = (B + 3) & ~3, JP = (J + 3) & ~3;
  float* Ws = fsm;              // [64][JP]
  float* xT = fsm + 64 * JP;    // [64][BP]  (k-major: a thread's four rows are one float4)
  const int k0 = blockIdx.x * 64;
  const int J4 = JP >> 2;
  if (J == JP && (reinterpret_cast<uintptr_t>(W) & 15) == 0) {
    for (int i = threadIdx.x; i < 64 * J4; i += blockDim.x) {
      const int kk = i / J4;
      reinterpret_cast<float4*>(Ws)[i] = (k0 + kk < K) ? reinterpret_cast<const float4*>(W + static_cast<long long>(k0) * J)[i]
                                                       : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else {
    for (int i = threadIdx.x; i < 64 * JP; i += blockDim.x) {
      const int kk = i / JP, j = i - kk * JP;
      Ws[i] = (j < J && k0 + kk < K) ? W[static_cast<long long>(k0 + kk) * J + j] : 0.f;
    }
  }
  for (int i = threadIdx.x; i < 64 * BP; i += blockDim.x) {
    const int b = i >> 6, kk = i & 63;
    xT[kk * BP + b] = (b < B && k0 + kk < K) ? x[static_cast<long long>(b) * xs + k0 + kk] : 0.f;
  }
  __syncthreads();
  const float sc = inv_scale ? 1.f / __ldg(inv_scale) : 1.f;
  const int BT = BP >> 2;
  for (int t = threadIdx.x; t < BT * J4; t += blockDim.x) {
    const int bt = t % BT, jt = t / BT;
    float acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
#pragma unroll 8
    for (int kk = 0; kk < 64; ++kk) {
      const float4 xv = *reinterpret_cast<const float4*>(xT + kk * BP + 4 * bt);
      const float4 wv = *reinterpret_cast<const float4*>(Ws + kk * JP + 4 * jt);
      const float xr[4] = {xv.x, xv.y, xv.z, xv.w}, wc[4] = {wv.x, wv.y, wv.z, wv.w};
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] += xr[r] * wc[c];
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int b = 4 * bt + r;
      if (b >= B) continue;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = 4 * jt + c;
        if (j >= J) continue;
        float v = acc[r][c] * sc;
        if (bias && blockIdx.x == 0) v += bias[j];
        y[(static_cast<long long>(blockIdx.x) * B + b) * ys + j] = v;      // this block's part of a K-split sum (dense rows)
      }
    }
  }
}

// dense LSTM cell on z (tf.nn.rnn_cell.LSTMCell, savp_model.py:354-362): gates [B,4U] (i,j,f,o)
__global__ void lstm_cell_fwd_kernel(const float* __restrict__ gates, const float* __restrict__ c_prev,
                                     float* __restrict__ c_new, float* __restrict__ h_new, int B, int U,
                                     float forget_bias) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * U) return;
  const int b = idx / U, u = idx % U;
  const float* g = gates + static_cast<long long>(b) * 4 * U;
  const float c = sigmoidf_(g[2 * U + u] + forget_bias) * c_prev[idx] + sigmoidf_(g[u]) * tanhf(g[U + u]);
  c_new[idx] = c;
  h_new[idx] = tanhf(c) * sigmoidf_(g[3 * U + u]);
}

// z = mu + sqrt(exp(clip(lss,-10,10))) * eps  (savp_model.py:49, 712); also writes the clipped lss
__global__ void sample_z_kernel(const float* __restrict__ mu, float* __restrict__ lss, const float* __restrict__ eps,
                                float* __restrict__ z, int total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const float l = fminf(fmaxf(lss[idx], -10.f), 10.f);
  lss[idx] = l;
  z[idx] = mu[idx] + sqrtf(expf(l)) * eps[idx];
}

// ------------------------------------------------------------------------------------------------
// CDNA (savp_model.py:546-559, 893-923) and compositing (savp_model.py:574-646)
// ------------------------------------------------------------------------------------------------
// raw [B, KK*NK] (dense output, index (i*kw+j)*NK + k) -> +identity, relu(.-1e-12)+1e-12, / sum over taps
__global__ void cdna_kernel_norm_kernel(const float* __restrict__ raw, float* __restrict__ out, int B, int KH, int KW,
                                        int NK) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * NK) return;
  const int b = idx / NK, k = idx % NK;
  const int KK = KH * KW;
  const float* r = raw + static_cast<long long>(b) * KK * NK + k;
  float* o = out + static_cast<long long>(b) * KK * NK + k;
  // identity_kernel (savp_model.py:968-980): odd sizes -> one-hot centre
  const int ci = KH / 2, cj = KW / 2;
  float s = 0.f;
  for (int t = 0; t < KK; ++t) {
    float idv = 0.f;
    const int i = t / KW, j = t % KW;
    const bool in_i = (KH % 2) ? (i == ci) : (i == ci - 1 || i == ci);
    const bool in_j = (KW % 2) ? (j == cj) : (j == cj - 1 || j == cj);
    if (in_i && in_j) idv = 1.f / (((KH % 2) ? 1 : 2) * ((KW % 2) ? 1 : 2));
    const float v = fmaxf(r[static_cast<long long>(t) * NK] + idv - 1e-12f, 0.f) + 1e-12f;
    o[static_cast<long long>(t) * NK] = v;
    s += v;
  }
  const float invs = 1.f / s;
  for (int t = 0; t < KK; ++t) o[static_cast<long long>(t) * NK] *= invs;
}

__device__ __forceinline__ int reflect_idx(int i, int n) {  // SYMMETRIC padding (edge pixel repeated)
  if (i < 0) i = -i - 1;
  if (i >= n) i = 2 * n - 1 - i;
  return i;
}
// image [N,H,W,4]; kern [N, KH*KW, NK]; writes NK transformed images + prev image + first image as
// float4 slots into the masks-conv concat buffer: layers[n,y,x, off + 4*l .. ] (l = 0..NK+1).
__global__ void __launch_bounds__(256) cdna_apply_kernel(const float4* __restrict__ image, const float4* __restrict__ first,
                                                         const float* __restrict__ kern, float* __restrict__ layers,
                                                         int ls, int N, int H, int W, int KH, int KW, int NK) {
  extern __shared__ float sk[];  // [KH*KW*NK]
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < KH * KW * NK; i += blockDim.x) sk[i] = kern[static_cast<long long>(n) * KH * KW * NK + i];
  __syncthreads();
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= H * W) return;
  const int y = p / W, x = p % W;
  const float4* img = image + static_cast<long long>(n) * H * W;
  float4 acc[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  const int ph = (KH - 1) / 2, pw = (KW - 1) / 2;  // SAME pad-before for stride 1
  for (int i = 0; i < KH; ++i) {
    const int yy = reflect_idx(y + i - ph, H);
    for (int j = 0; j < KW; ++j) {
      const int xx = reflect_idx(x + j - pw, W);
      const float4 v = img[yy * W + xx];
      const float* kk = sk + (i * KW + j) * NK;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < NK) {
          acc[k].x += v.x * kk[k]; acc[k].y += v.y * kk[k]; acc[k].z += v.z * kk[k]; acc[k].w += v.w * kk[k];
        }
      }
    }
  }
  float* lp = layers + (static_cast<long long>(n) * H * W + p) * ls;
  for (int k = 0; k < NK; ++k) *reinterpret_cast<float4*>(lp + 4 * k) = acc[k];
  *reinterpret_cast<float4*>(lp + 4 * NK) = img[p];
  *reinterpret_cast<float4*>(lp + 4 * NK + 4) = first[static_cast<long long>(n) * H * W + p];
}

// logits [N*P, lgs] (L valid) ; layers: L float4 slots at layers[np*ls + 4*l] ; masks out [N*P, 8];
// gen [N*P] float4 = sum_l softmax(logits)_l * layer_l
__global__ void composite_kernel(const float* __restrict__ logits, int lgs, const float* __restrict__ layers, int ls,
                                 float* __restrict__ masks, int ms, float4* __restrict__ gen, long long total, int L) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  float lg[8];
  float mx = -1e30f;
  for (int l = 0; l < L; ++l) { lg[l] = logits[idx * lgs + l]; mx = fmaxf(mx, lg[l]); }
  float s = 0.f;
  for (int l = 0; l < L; ++l) { lg[l] = __expf(lg[l] - mx); s += lg[l]; }
  const float invs = 1.f / s;
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int l = 0; l < L; ++l) {
    const float m = lg[l] * invs;
    if (masks) masks[idx * ms + l] = m;
    const float4 v = *reinterpret_cast<const float4*>(layers + idx * ls + 4 * l);
    o.x += m * v.x; o.y += m * v.y; o.z += m * v.z; o.w += m * v.w;
  }
  gen[idx] = o;
}

}  // namespace vp

using namespace vp;

extern "C" int vp_inorm_act(const float* x, int x_cstride, float* y, int y_cstride, int n, int positions, int c,
                            const float* gamma, const float* beta, float eps, int act, float alpha, float* stats,
                            vp_stream_t stream) {
  if (!x || !y) return set_error("vp_inorm_act: null pointer");
  if (c % 4 || x_cstride % 4 || y_cstride % 4) return set_error("vp_inorm_act: channels/strides must be multiples of 4");
  {
    const int rc = slab_inorm_act(x, x_cstride, y, y_cstride, n, positions, c, gamma, beta, eps, act, alpha, stats, stream);
    if (rc <= 0) return rc;
  }
  dim3 grid(c / 4, n);
  const int staged = positions <= 4096 ? 1 : 0;
  const size_t smem = staged ? static_cast<size_t>(positions) * 16 : 0;
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(inorm_act_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 4096 * 16);
    attr_set = true;
  }
  inorm_act_kernel<<<grid, positions >= 2048 ? 512 : 256, smem, as_stream(stream)>>>(x, x_cstride, y, y_cstride, positions, c, gamma, beta, eps, act,
                                                           alpha, stats, staged);
  return check_launch("inorm_act_kernel");
}

extern "C" int vp_lstm_gates_fwd(const float* pre, int n, int positions, int filters, const float* c_prev,
                                 const float* gamma1, const float* beta1, const float* gamma2, const float* beta2,
                                 float forget_bias, float eps, float* c_new, float* const* h_dst, const int* h_cstride,
                                 int num_h_dst, float* stats1, float* stats2, vp_stream_t stream) {
  if (!pre || !c_prev || !c_new || !h_dst) return set_error("vp_lstm_gates_fwd: null pointer");
  if (positions > kGatesMaxP) return set_error("vp_lstm_gates_fwd: plane of %d positions exceeds %d", positions, kGatesMaxP);
  if (filters % 4 || num_h_dst < 1 || num_h_dst > 3) return set_error("vp_lstm_gates_fwd: bad filters / destination count");
  {
    const int rc = slab_gates_fwd(pre, n, positions, filters, c_prev, gamma1, beta1, gamma2, beta2, forget_bias, eps, c_new, h_dst, h_cstride,
                                  num_h_dst, stats1, stats2, stream);
    if (rc <= 0) return rc;
  }
  GateDst d;
  d.count = num_h_dst;
  for (int i = 0; i < 3; ++i) { d.ptr[i] = i < num_h_dst ? h_dst[i] : nullptr; d.stride[i] = i < num_h_dst ? h_cstride[i] : 0; }
  const size_t smem = static_cast<size_t>(positions) * 20 * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    cudaFuncSetAttribute(lstm_gates_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGatesMaxP * 20 * 4);
    attr_set = true;
  }
  dim3 grid(filters / 4, n);
  lstm_gates_fwd_kernel<<<grid, positions >= 512 ? 512 : 256, smem, as_stream(stream)>>>(pre, positions, filters, c_prev, gamma1, beta1, gamma2, beta2,
                                                               forget_bias, eps, c_new, d, stats1, stats2);
  return check_launch("lstm_gates_fwd_kernel");
}

extern "C" int vp_broadcast_channels(const float* vec, int vec_stride, float* dst, int dst_cstride, int n, int positions,
                                     int c, vp_stream_t stream) {
  const long long total = static_cast<long long>(n) * positions * c;
  if (total == 0) return 0;
  broadcast_channels_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(vec, vec_stride, dst, dst_cstride, total,
                                                                                positions, c);
  return check_launch("broadcast_channels_kernel");
}

extern "C" int vp_copy_channels(const float* src, int src_cstride, float* dst, int dst_cstride, long long rows, int c,
                                vp_stream_t stream) {
  const long long total = rows * c;
  if (total == 0) return 0;
  copy_channels_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(src, src_cstride, dst, dst_cstride, total, c);
  return check_launch("copy_channels_kernel");
}

extern "C" int vp_select_rows(const int32_t* sel, const float* a, const float* b, float* out, int n, long long per_row,
                              vp_stream_t stream) {
  if (per_row % 4) return set_error("vp_select_rows: row length must be a multiple of 4");
  const long long total = static_cast<long long>(n) * per_row / 4;
  select_rows_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(sel, reinterpret_cast<const float4*>(a),
                                                                         reinterpret_cast<const float4*>(b),
                                                                         reinterpret_cast<float4*>(out), per_row / 4, total);
  return check_launch("select_rows_kernel");
}

extern "C" int vp_avgpool(const float* x, int x_cstride, float* y, int n, int positions, int c, vp_stream_t stream) {
  dim3 grid((c + 127) / 128, n);
  avgpool_kernel<<<grid, 128, 0, as_stream(stream)>>>(x, x_cstride, y, positions, c);
  return check_launch("avgpool_kernel");
}

extern "C" int vp_dense_fwd(const float* x, int x_stride, const float* w, const float* bias, const float* inv_scale,
                            float* y, int y_stride, int b, int k, int j, int k_splits, vp_stream_t stream) {
  if (!x || !w || !y) return set_error("vp_dense_fwd: null pointer");
  // wide layers called with k_splits > 1 (y zero-filled by the caller): tiled kernel
  const size_t tsm = (64 * static_cast<size_t>((j + 3) & ~3) + 64 * static_cast<size_t>((b + 3) & ~3)) * sizeof(float);
  if (k_splits > 1 && k >= 1024 && j <= 128 && tsm <= 48 * 1024) {
    // the K blocks write their parts into scratch rows, which are added to y in block order (run-to-run identical sums)
    const int parts = (k + 63) / 64;
    float* ws = nullptr;
    if (scratch_zeroed(&ws, static_cast<long long>(parts) * b * j, stream)) return -1;
    dense_fwd_tiled_kernel<<<parts, 256, tsm, as_stream(stream)>>>(x, x_stride, w, bias, inv_scale, ws, j, b, k, j);
    int rc = check_launch("dense_fwd_tiled_kernel");
    if (!rc) rc = reduce_parts_strided(ws, parts, b, j, y, y_stride, stream);
    scratch_free(ws, stream);
    return rc;
  }
  if (k_splits < 1) k_splits = 1;
  const int kchunk = (k + k_splits - 1) / k_splits;
  dim3 grid((b + 3) / 4, (k + kchunk - 1) / kchunk);
  if (grid.y == 1) {
    dense_fwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(x, x_stride, w, bias, inv_scale, y, y_stride, b, k, j, kchunk);
    return check_launch("dense_fwd_kernel");
  }
  float* ws = nullptr;
  if (scratch_zeroed(&ws, static_cast<long long>(grid.y) * b * j, stream)) return -1;
  dense_fwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(x, x_stride, w, bias, inv_scale, ws, j, b, k, j, kchunk);
  int rc = check_launch("dense_fwd_kernel");
  if (!rc) rc = reduce_parts_strided(ws, grid.y, b, j, y, y_stride, stream);
  scratch_free(ws, stream);
  return rc;
}

extern "C" int vp_lstm_cell_fwd(const float* gates, const float* c_prev, float* c_new, float* h_new, int b, int units,
                                float forget_bias, vp_stream_t stream) {
  lstm_cell_fwd_kernel<<<grid_for(static_cast<long long>(b) * units, 128), 128, 0, as_stream(stream)>>>(
      gates, c_prev, c_new, h_new, b, units, forget_bias);
  return check_launch("lstm_cell_fwd_kernel");
}

extern "C" int vp_sample_z(const float* mu, float* log_sigma_sq, const float* eps, float* z, int total,
                           vp_stream_t stream) {
  sample_z_kernel<<<grid_for(total, 128), 128, 0, as_stream(stream)>>>(mu, log_sigma_sq, eps, z, total);
  return check_launch("sample_z_kernel");
}

extern "C" int vp_cdna_kernel_norm(const float* raw, float* out, int b, int kh, int kw, int nk, vp_stream_t stream) {
  cdna_kernel_norm_kernel<<<grid_for(static_cast<long long>(b) * nk, 64), 64, 0, as_stream(stream)>>>(raw, out, b, kh, kw, nk);
  return check_launch("cdna_kernel_norm_kernel");
}

extern "C" int vp_cdna_apply(const float* image, const float* first_image, const float* kernels, float* layers,
                             int layers_cstride, int n, int h, int w, int kh, int kw, int nk, vp_stream_t stream) {
  if (nk > 4) return set_error("vp_cdna_apply: at most 4 transformations");
  if (layers_cstride % 4) return set_error("vp_cdna_apply: layers stride must be a multiple of 4");
  dim3 grid((h * w + 255) / 256, n);
  cdna_apply_kernel<<<grid, 256, kh * kw * nk * sizeof(float), as_stream(stream)>>>(
      reinterpret_cast<const float4*>(image), reinterpret_cast<const float4*>(first_image), kernels, layers, layers_cstride, n,
      h, w, kh, kw, nk);
  return check_launch("cdna_apply_kernel");
}

extern "C" int vp_composite(const float* logits, int logits_cstride, const float* layers, int layers_cstride, float* masks,
                            int masks_cstride, float* gen_image, long long positions, int num_layers, vp_stream_t stream) {
  if (num_layers > 8) return set_error("vp_composite: at most 8 layers");
  composite_kernel<<<grid_for(positions, 256), 256, 0, as_stream(stream)>>>(logits, logits_cstride, layers, layers_cstride, masks,
                                                                           masks_cstride, reinterpret_cast<float4*>(gen_image),
                                                                           positions, num_layers);
  return check_launch("composite_kernel");
}

// ------------------------------------------------------------------------------------------------
// flow_ops.image_warp (flow_ops.py:4-79): backward bilinear warp.  x = floor(flow_x), weights from the fractional
// part, the four neighbour indices are clipped to the image (tf.clip_by_value, :53-56), flow[...,0] = x, [...,1] = y.
// im / out: [N,H,W,cs] (C valid channels), flow: [N,H,W,2].  HBM-bound gather: one thread per (pixel, channel).
// ------------------------------------------------------------------------------------------------
namespace vp {
__global__ void image_warp_fwd_kernel(const float* __restrict__ im, int ims, const float* __restrict__ flow,
                                      float* __restrict__ out, int os, int N, int H, int W, int C) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(N) * H * W * C;
  if (idx >= total) return;
  const int c = static_cast<int>(idx % C);
  const long long p = idx / C;
  const int x = static_cast<int>(p % W), y = static_cast<int>((p / W) % H);
  const long long n = p / (static_cast<long long>(W) * H);
  const float fx = flow[p * 2], fy = flow[p * 2 + 1];
  const float flx = floorf(fx), fly = floorf(fy);
  const float xw = fx - flx, yw = fy - fly;
  const int x0 = min(max(x + static_cast<int>(flx), 0), W - 1), x1 = min(max(x + static_cast<int>(flx) + 1, 0), W - 1);
  const int y0 = min(max(y + static_cast<int>(fly), 0), H - 1), y1 = min(max(y + static_cast<int>(fly) + 1, 0), H - 1);
  const float* b = im + n * H * W * ims + c;
  const float Ia = b[(static_cast<long long>(y0) * W + x0) * ims], Ib = b[(static_cast<long long>(y1) * W + x0) * ims];
  const float Ic = b[(static_cast<long long>(y0) * W + x1) * ims], Id = b[(static_cast<long long>(y1) * W + x1) * ims];
  out[p * os + c] = (1.f - xw) * (1.f - yw) * Ia + (1.f - xw) * yw * Ib + xw * (1.f - yw) * Ic + xw * yw * Id;
}
// dim (+= atomics, zero-filled by the caller) and dflow (overwritten; floor has zero gradient, so only the weights carry it)
__global__ void image_warp_bwd_kernel(const float* __restrict__ im, int ims, const float* __restrict__ flow,
                                      const float* __restrict__ dout, int dos, float* __restrict__ dim, int dis,
                                      float* __restrict__ dflow, int N, int H, int W, int C) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(N) * H * W;
  if (p >= total) return;
  const int x = static_cast<int>(p % W), y = static_cast<int>((p / W) % H);
  const long long n = p / (static_cast<long long>(W) * H);
  const float fx = flow[p * 2], fy = flow[p * 2 + 1];
  const float flx = floorf(fx), fly = floorf(fy);
  const float xw = fx - flx, yw = fy - fly;
  const int x0 = min(max(x + static_cast<int>(flx), 0), W - 1), x1 = min(max(x + static_cast<int>(flx) + 1, 0), W - 1);
  const int y0 = min(max(y + static_cast<int>(fly), 0), H - 1), y1 = min(max(y + static_cast<int>(fly) + 1, 0), H - 1);
  const long long base = n * H * W;
  const long long ia = (base + static_cast<long long>(y0) * W + x0), ib = (base + static_cast<long long>(y1) * W + x0);
  const long long ic = (base + static_cast<long long>(y0) * W + x1), id = (base + static_cast<long long>(y1) * W + x1);
  float gx = 0.f, gy = 0.f;
  for (int c = 0; c < C; ++c) {
    const float d = dout[p * dos + c];
    const float Ia = im[ia * ims + c], Ib = im[ib * ims + c], Ic = im[ic * ims + c], Id = im[id * ims + c];
    gx += d * ((1.f - yw) * (Ic - Ia) + yw * (Id - Ib));
    gy += d * ((1.f - xw) * (Ib - Ia) + xw * (Id - Ic));
    if (dim) {
      atomicAdd(dim + ia * dis + c, d * (1.f - xw) * (1.f - yw));
      atomicAdd(dim + ib * dis + c, d * (1.f - xw) * yw);
      atomicAdd(dim + ic * dis + c, d * xw * (1.f - yw));
      atomicAdd(dim + id * dis + c, d * xw * yw);
    }
  }
  if (dflow) { dflow[p * 2] = gx; dflow[p * 2 + 1] = gy; }
}
}  // namespace vp

extern "C" int vp_image_warp_fwd(const float* im, int im_cstride, const float* flow, float* out, int out_cstride, int n, int h,
                                 int w, int c, vp_stream_t stream) {
  const long long total = static_cast<long long>(n) * h * w * c;
  vp::image_warp_fwd_kernel<<<vp::grid_for(total, 256), 256, 0, vp::as_stream(stream)>>>(im, im_cstride, flow, out, out_cstride, n, h, w, c);
  return vp::check_launch("image_warp_fwd_kernel");
}

extern "C" int vp_image_warp_bwd(const float* im, int im_cstride, const float* flow, const float* dout, int dout_cstride,
                                 float* dim, int dim_cstride, float* dflow, int n, int h, int w, int c, vp_stream_t stream) {
  const long long total = static_cast<long long>(n) * h * w;
  vp::image_warp_bwd_kernel<<<vp::grid_for(total, 256), 256, 0, vp::as_stream(stream)>>>(im, im_cstride, flow, dout, dout_cstride, dim,
                                                                                          dim_cstride, dflow, n, h, w, c);
  return vp::check_launch("image_warp_bwd_kernel");
}

// ------------------------------------------------------------------------------------------------
// transformation = 'flow' (savp_model.py:522-530, 577-578, 955-965): the transformed images are backward bilinear warps
// of the previous image by NK predicted flow fields.  `flows` is the 3x3 flows-conv output [N,H,W,2*NK] reshaped by the
// reference to [.., 2, NK]: channel k is the x-flow of transform k, channel NK + k its y-flow.  Writes the NK warped
// images + the previous image + the first image as consecutive float4 slots of the masks-conv concat buffer (same slot
// layout as cdna_apply_kernel).  flow_ops.image_warp semantics: floor, four neighbours clipped to the image.
// ------------------------------------------------------------------------------------------------
namespace vp {
__global__ void __launch_bounds__(256) flow_apply_kernel(const float4* __restrict__ image, const float4* __restrict__ first,
                                                         const float* __restrict__ flows, int fs, float* __restrict__ layers, int ls,
                                                         int N, int H, int W, int NK) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= static_cast<long long>(N) * H * W) return;
  const int x = static_cast<int>(p % W), y = static_cast<int>((p / W) % H);
  const long long base = p - (static_cast<long long>(y) * W + x);
  float* lp = layers + p * ls;
  for (int k = 0; k < NK; ++k) {
    const float fx = flows[p * fs + k], fy = flows[p * fs + NK + k];
    const float flx = floorf(fx), fly = floorf(fy);
    const float xw = fx - flx, yw = fy - fly;
    const int x0 = min(max(x + static_cast<int>(flx), 0), W - 1), x1 = min(max(x + static_cast<int>(flx) + 1, 0), W - 1);
    const int y0 = min(max(y + static_cast<int>(fly), 0), H - 1), y1 = min(max(y + static_cast<int>(fly) + 1, 0), H - 1);
    const float4 Ia = image[base + static_cast<long long>(y0) * W + x0], Ib = image[base + static_cast<long long>(y1) * W + x0];
    const float4 Ic = image[base + static_cast<long long>(y0) * W + x1], Id = image[base + static_cast<long long>(y1) * W + x1];
    const float wa = (1.f - xw) * (1.f - yw), wb = (1.f - xw) * yw, wc = xw * (1.f - yw), wd = xw * yw;
    *reinterpret_cast<float4*>(lp + 4 * k) = make_float4(wa * Ia.x + wb * Ib.x + wc * Ic.x + wd * Id.x, wa * Ia.y + wb * Ib.y + wc * Ic.y + wd * Id.y,
                                                          wa * Ia.z + wb * Ib.z + wc * Ic.z + wd * Id.z, wa * Ia.w + wb * Ib.w + wc * Ic.w + wd * Id.w);
  }
  *reinterpret_cast<float4*>(lp + 4 * NK) = image[p];
  *reinterpret_cast<float4*>(lp + 4 * NK + 4) = first[p];
}

// gradients of flow_apply: dT_k = dA[slot k] + dB[slot k] (through the masks conv and through the compositing);
// dimage += scatter of the bilinear weights (+ the previous-image slot NK); dflows (overwritten): only the fractional
// weights carry a gradient (floor has none, flow_ops.py:27-34).
__global__ void __launch_bounds__(256) flow_apply_bwd_kernel(const float4* __restrict__ image, const float* __restrict__ flows, int fs,
                                                             const float* __restrict__ dA, int das, const float* __restrict__ dB,
                                                             int dbs, float* __restrict__ dimage, float* __restrict__ dflows, int N,
                                                             int H, int W, int NK) {
  const long long p = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p >= static_cast<long long>(N) * H * W) return;
  const int x = static_cast<int>(p % W), y = static_cast<int>((p / W) % H);
  const long long base = p - (static_cast<long long>(y) * W + x);
  {
    const float4 a = *reinterpret_cast<const float4*>(dA + p * das + 4 * NK), b = *reinterpret_cast<const float4*>(dB + p * dbs + 4 * NK);
    atomicAdd(dimage + p * 4 + 0, a.x + b.x); atomicAdd(dimage + p * 4 + 1, a.y + b.y); atomicAdd(dimage + p * 4 + 2, a.z + b.z);
  }
  for (int k = 0; k < NK; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(dA + p * das + 4 * k), b = *reinterpret_cast<const float4*>(dB + p * dbs + 4 * k);
    const float d[3] = {a.x + b.x, a.y + b.y, a.z + b.z};
    const float fx = flows[p * fs + k], fy = flows[p * fs + NK + k];
    const float flx = floorf(fx), fly = floorf(fy);
    const float xw = fx - flx, yw = fy - fly;
    const int x0 = min(max(x + static_cast<int>(flx), 0), W - 1), x1 = min(max(x + static_cast<int>(flx) + 1, 0), W - 1);
    const int y0 = min(max(y + static_cast<int>(fly), 0), H - 1), y1 = min(max(y + static_cast<int>(fly) + 1, 0), H - 1);
    const long long ia = base + static_cast<long long>(y0) * W + x0, ib = base + static_cast<long long>(y1) * W + x0;
    const long long ic = base + static_cast<long long>(y0) * W + x1, id = base + static_cast<long long>(y1) * W + x1;
    const float4 A = image[ia], B = image[ib], Cc = image[ic], D = image[id];
    const float va[3] = {A.x, A.y, A.z}, vb[3] = {B.x, B.y, B.z}, vc[3] = {Cc.x, Cc.y, Cc.z}, vd[3] = {D.x, D.y, D.z};
    float gx = 0.f, gy = 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      gx += d[c] * ((1.f - yw) * (vc[c] - va[c]) + yw * (vd[c] - vb[c]));
      gy += d[c] * ((1.f - xw) * (vb[c] - va[c]) + xw * (vd[c] - vc[c]));
      atomicAdd(dimage + ia * 4 + c, d[c] * (1.f - xw) * (1.f - yw));
      atomicAdd(dimage + ib * 4 + c, d[c] * (1.f - xw) * yw);
      atomicAdd(dimage + ic * 4 + c, d[c] * xw * (1.f - yw));
      atomicAdd(dimage + id * 4 + c, d[c] * xw * yw);
    }
    dflows[p * fs + k] = gx;
    dflows[p * fs + NK + k] = gy;
  }
}
}  // namespace vp

extern "C" int vp_flow_apply(const float* image, const float* first_image, const float* flows, int flows_cstride, float* layers,
                             int layers_cstride, int n, int h, int w, int nk, vp_stream_t stream) {
  if (nk < 1 || nk > 6 || flows_cstride < 2 * nk) return vp::set_error("vp_flow_apply: bad nk / flows_cstride");
  const long long total = static_cast<long long>(n) * h * w;
  vp::flow_apply_kernel<<<vp::grid_for(total, 256), 256, 0, vp::as_stream(stream)>>>(
      reinterpret_cast<const float4*>(image), reinterpret_cast<const float4*>(first_image), flows, flows_cstride, layers, layers_cstride,
      n, h, w, nk);
  return vp::check_launch("flow_apply_kernel");
}

extern "C" int vp_flow_apply_bwd(const float* image, const float* flows, int flows_cstride, const float* d_a, int d_a_cstride,
                                 const float* d_b, int d_b_cstride, float* dimage, float* dflows, int n, int h, int w, int nk,
                                 vp_stream_t stream) {
  if (nk < 1 || nk > 6 || flows_cstride < 2 * nk) return vp::set_error("vp_flow_apply_bwd: bad nk / flows_cstride");
  const long long total = static_cast<long long>(n) * h * w;
  vp::flow_apply_bwd_kernel<<<vp::grid_for(total, 256), 256, 0, vp::as_stream(stream)>>>(
      reinterpret_cast<const float4*>(image), flows, flows_cstride, d_a, d_a_cstride, d_b, d_b_cstride, dimage, dflows, n, h, w, nk);
  return vp::check_launch("flow_apply_bwd_kernel");
}
