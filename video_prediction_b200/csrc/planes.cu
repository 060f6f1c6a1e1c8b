// Plane kernels of the SAVP path in the SLAB mapping: instance norm (+activation) and the ConvLSTM gate math
// (rnn_ops.py:148-165, layers/normalization.py:146-170), forward and backward.
//
// The first versions (elementwise.cu / backward.cu) give one CTA a (sample, 4 channels) plane: every thread reads 16 bytes
// at a stride of the full channel count, i.e. a warp instruction touches 32 different 128-byte lines.  ncu showed them
// L1TEX-bound at 15 - 24 % of the HBM roofline with only 8 x N CTAs for the 32-channel layers.  Here
//   * a CTA owns (sample, 32-channel slab, slice of the plane's positions); thread = (position, quad of 4 channels), so 8
//     neighbouring lanes read one contiguous 128-byte line: fully coalesced, 4x fewer L1TEX wavefronts;
//   * the slices of one (sample, slab) form a thread-block CLUSTER (up to 8 CTAs): the per-channel statistics of instance
//     norm are reduced across the cluster through distributed shared memory, so a 32x32 or 64x64 plane is spread over 4 - 8
//     SMs instead of one;
//   * mean and variance come from ONE pass (sums of (x - k) and (x - k)^2 with k = the value at position 0 of the sample,
//     which keeps the subtraction well conditioned), and the forward kernels keep their operands in registers between the
//     passes instead of re-reading them.
// Shapes outside the fast path (channels not a multiple of 32, non-power-of-two planes) fall back to the first versions.
#include <cooperative_groups.h>

#include <cstdlib>
#include <map>
#include <mutex>
#include <tuple>

#include "common.h"
#include "ptx.cuh"

namespace cg = cooperative_groups;

namespace vp {

__device__ __forceinline__ float p_sigm(float v) { return 1.f / (1.f + __expf(-v)); }
__device__ __forceinline__ float p_act(float v, int act, float alpha) {
  switch (act) {
    case VP_ACT_RELU: return fmaxf(v, 0.f);
    case VP_ACT_LRELU: return fmaxf(alpha * v, v);
    case VP_ACT_SIGMOID: return p_sigm(v);
    case VP_ACT_TANH: return tanhf(v);
    default: return v;
  }
}
__device__ __forceinline__ float p_act_grad(float yp, int act, float alpha) {
  switch (act) {
    case VP_ACT_RELU: return yp > 0.f ? 1.f : 0.f;
    case VP_ACT_LRELU: return yp > 0.f ? 1.f : alpha;
    default: return 1.f;
  }
}

constexpr int kSlabMaxWarps = 16;

// Sum of NV per-thread values over every thread of the CLUSTER that has the same quad q = threadIdx.x & 7; the totals come
// back in v.  s_warp: [kSlabMaxWarps * 8 * NV] scratch, s_part: this CTA's partials [8 * NV] (read by the other CTAs of the
// cluster through DSMEM; callers alternate between two buffers so that one cluster barrier per reduction suffices), s_tot: [8 * NV].
template <int NV>
__device__ __forceinline__ void slab_reduce(float (&v)[NV], float* s_warp, float* s_part, float* s_tot, int cs) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5, q = threadIdx.x & 7;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    v[i] += __shfl_xor_sync(0xffffffffu, v[i], 8);
    v[i] += __shfl_xor_sync(0xffffffffu, v[i], 16);
  }
  if (lane < 8) {
#pragma unroll
    for (int i = 0; i < NV; ++i) s_warp[(warp * 8 + q) * NV + i] = v[i];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 8 * NV; t += blockDim.x) {
    float acc = 0.f;
    for (int w = 0; w < nw; ++w) acc += s_warp[w * 8 * NV + t];
    s_part[t] = acc;
  }
  if (cs > 1) {
    cg::cluster_group cluster = cg::this_cluster();
    cluster.sync();
    for (int t = threadIdx.x; t < 8 * NV; t += blockDim.x) {
      float acc = 0.f;
      for (int r = 0; r < cs; ++r) acc += *cluster.map_shared_rank(s_part + t, r);
      s_tot[t] = acc;
    }
  } else {
    __syncthreads();
    for (int t = threadIdx.x; t < 8 * NV; t += blockDim.x) s_tot[t] = s_part[t];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = s_tot[q * NV + i];
}

struct SlabSrcs {
  const float* ptr[4];
  int stride[4];
  int count;
};
struct SlabDsts {
  float* ptr[3];
  int stride[3];
  int count;
};

// ------------------------------------------------------------------------------------------------ instance norm forward
// grid (cluster rank = position slice, slab, sample); block = 8 * lanes; every thread owns ITERS positions x 4 channels.
template <int ITERS>
__global__ void __launch_bounds__(512) slab_inorm_act_kernel(const float* __restrict__ x, int xs, float* __restrict__ y, int ys, int P, int C,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                             int act, float alpha, float* __restrict__ stats, int cs) {
  __shared__ float s_warp[kSlabMaxWarps * 8 * 8], s_part[8 * 8], s_tot[8 * 8];
  const int q = threadIdx.x & 7, pl = threadIdx.x >> 3, lanes = blockDim.x >> 3;
  const int n = blockIdx.z, c0 = blockIdx.y * 32 + q * 4;
  const int p0 = blockIdx.x * lanes * ITERS;
  const float* xp = x + static_cast<long long>(n) * P * xs + c0;
  const float4 k4 = *reinterpret_cast<const float4*>(xp);          // shift: the sample's value at position 0
  float4 v[ITERS];
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    v[it] = *reinterpret_cast<const float4*>(xp + static_cast<long long>(p0 + pl + it * lanes) * xs);
    const float d0 = v[it].x - k4.x, d1 = v[it].y - k4.y, d2 = v[it].z - k4.z, d3 = v[it].w - k4.w;
    s[0] += d0; s[1] += d1; s[2] += d2; s[3] += d3;
    s[4] += d0 * d0; s[5] += d1 * d1; s[6] += d2 * d2; s[7] += d3 * d3;
  }
  slab_reduce<8>(s, s_warp, s_part, s_tot, cs);
  const float inv = 1.f / P;
  const float kk[4] = {k4.x, k4.y, k4.z, k4.w};
  float g[4], b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float md = s[i] * inv;                                   // mean - k
    const float var = fmaxf(s[4 + i] * inv - md * md, 0.f);
    const float m = kk[i] + md, r = rsqrtf(var + eps);
    g[i] = (gamma ? gamma[c0 + i] : 1.f) * r;
    b[i] = (beta ? beta[c0 + i] : 0.f) - m * g[i];
    if (stats && blockIdx.x == 0 && pl == 0) {
      stats[(static_cast<long long>(n) * C + c0 + i) * 2 + 0] = m;
      stats[(static_cast<long long>(n) * C + c0 + i) * 2 + 1] = r;
    }
  }
  float* yp = y + static_cast<long long>(n) * P * ys + c0;
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    float4 o;
    o.x = p_act(v[it].x * g[0] + b[0], act, alpha); o.y = p_act(v[it].y * g[1] + b[1], act, alpha);
    o.z = p_act(v[it].z * g[2] + b[2], act, alpha); o.w = p_act(v[it].w * g[3] + b[3], act, alpha);
    *reinterpret_cast<float4*>(yp + static_cast<long long>(p0 + pl + it * lanes) * ys) = o;
  }
  if (cs > 1) cg::this_cluster().sync();      // keep this CTA's shared memory alive until every peer has read its partials
}

// ------------------------------------------------------------------------------------------------ instance norm backward
// dx = r*g*(dyp - mean(dyp) - xh*mean(dyp*xh)),  dyp = dy*act'(g*xh+b); dgamma += sum dyp*xh, dbeta += sum dyp
template <int ITERS>
__global__ void __launch_bounds__(512) slab_inorm_act_bwd_kernel(const float* __restrict__ x, int xs, SlabSrcs srcs, float* __restrict__ dx,
                                                                 int dxs, int P, int C, const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, const float* __restrict__ stats, int act,
                                                                 float alpha, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                 int cs) {
  __shared__ float s_warp[kSlabMaxWarps * 8 * 8], s_part[8 * 8], s_tot[8 * 8];
  const int q = threadIdx.x & 7, pl = threadIdx.x >> 3, lanes = blockDim.x >> 3;
  const int n = blockIdx.z, c0 = blockIdx.y * 32 + q * 4;
  const int p0 = blockIdx.x * lanes * ITERS;
  const float* xp = x + static_cast<long long>(n) * P * xs + c0;
  float m[4], r[4], g[4], b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = stats[(static_cast<long long>(n) * C + c0 + i) * 2];
    r[i] = stats[(static_cast<long long>(n) * C + c0 + i) * 2 + 1];
    g[i] = gamma[c0 + i];
    b[i] = beta[c0 + i];
  }
  float xh[ITERS][4], dyp[ITERS][4];
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    const long long p = p0 + pl + it * lanes;
    const float4 xv = *reinterpret_cast<const float4*>(xp + p * xs);
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sI = 0; sI < srcs.count; ++sI) {
      const float4 t = *reinterpret_cast<const float4*>(srcs.ptr[sI] + (static_cast<long long>(n) * P + p) * srcs.stride[sI] + c0);
      d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
    }
    const float xv4[4] = {xv.x, xv.y, xv.z, xv.w}, dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      xh[it][i] = (xv4[i] - m[i]) * r[i];
      dyp[it][i] = dv[i] * p_act_grad(g[i] * xh[it][i] + b[i], act, alpha);
      s[i] += dyp[it][i];
      s[4 + i] += dyp[it][i] * xh[it][i];
    }
  }
  slab_reduce<8>(s, s_warp, s_part, s_tot, cs);
  if (blockIdx.x == 0 && pl == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      dbeta[static_cast<long long>(n) * C + c0 + i] = s[i];
      dgamma[static_cast<long long>(n) * C + c0 + i] = s[4 + i];
    }
  }
  const float inv = 1.f / P;
  float* dp = dx + static_cast<long long>(n) * P * dxs + c0;
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    float o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = r[i] * g[i] * (dyp[it][i] - s[i] * inv - xh[it][i] * s[4 + i] * inv);
    *reinterpret_cast<float4*>(dp + static_cast<long long>(p0 + pl + it * lanes) * dxs) = make_float4(o[0], o[1], o[2], o[3]);
  }
  if (cs > 1) cg::this_cluster().sync();
}

// The same for CTAs that walk more positions than fit in registers (64x64 planes in clusters of 4 = 1024 positions per CTA, so
// that all 128 CTAs of a 32-sample launch are resident at once): two passes over x and dy, the second one served by the L2.
__global__ void __launch_bounds__(512) slab_inorm_act_bwd_loop_kernel(const float* __restrict__ x, int xs, SlabSrcs srcs, float* __restrict__ dx,
                                                                      int dxs, int P, int C, const float* __restrict__ gamma,
                                                                      const float* __restrict__ beta, const float* __restrict__ stats, int act,
                                                                      float alpha, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                                      int cs, int ppc) {
  __shared__ float s_warp[kSlabMaxWarps * 8 * 8], s_part[8 * 8], s_tot[8 * 8];
  const int q = threadIdx.x & 7, pl = threadIdx.x >> 3, lanes = blockDim.x >> 3;
  const int n = blockIdx.z, c0 = blockIdx.y * 32 + q * 4;
  const int p0 = blockIdx.x * ppc;
  const float* xp = x + static_cast<long long>(n) * P * xs + c0;
  float m[4], r[4], g[4], b[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m[i] = stats[(static_cast<long long>(n) * C + c0 + i) * 2];
    r[i] = stats[(static_cast<long long>(n) * C + c0 + i) * 2 + 1];
    g[i] = gamma[c0 + i];
    b[i] = beta[c0 + i];
  }
  auto load = [&](long long p, float* xh, float* dyp) {
    const float4 xv = *reinterpret_cast<const float4*>(xp + p * xs);
    float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int sI = 0; sI < srcs.count; ++sI) {
      const float4 t = *reinterpret_cast<const float4*>(srcs.ptr[sI] + (static_cast<long long>(n) * P + p) * srcs.stride[sI] + c0);
      d.x += t.x; d.y += t.y; d.z += t.z; d.w += t.w;
    }
    const float xv4[4] = {xv.x, xv.y, xv.z, xv.w}, dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      xh[i] = (xv4[i] - m[i]) * r[i];
      dyp[i] = dv[i] * p_act_grad(g[i] * xh[i] + b[i], act, alpha);
    }
  };
  float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
  for (int l = pl; l < ppc; l += lanes) {
    float xh[4], dyp[4];
    load(p0 + l, xh, dyp);
#pragma unroll
    for (int i = 0; i < 4; ++i) { s[i] += dyp[i]; s[4 + i] += dyp[i] * xh[i]; }
  }
  slab_reduce<8>(s, s_warp, s_part, s_tot, cs);
  if (blockIdx.x == 0 && pl == 0) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      dbeta[static_cast<long long>(n) * C + c0 + i] = s[i];
      dgamma[static_cast<long long>(n) * C + c0 + i] = s[4 + i];
    }
  }
  const float inv = 1.f / P;
  float* dp = dx + static_cast<long long>(n) * P * dxs + c0;
#pragma unroll 4
  for (int l = pl; l < ppc; l += lanes) {
    float xh[4], dyp[4], o[4];
    load(p0 + l, xh, dyp);
#pragma unroll
    for (int i = 0; i < 4; ++i) o[i] = r[i] * g[i] * (dyp[i] - s[i] * inv - xh[i] * s[4 + i] * inv);
    *reinterpret_cast<float4*>(dp + static_cast<long long>(p0 + l) * dxs) = make_float4(o[0], o[1], o[2], o[3]);
  }
  if (cs > 1) cg::this_cluster().sync();
}

// ------------------------------------------------------------------------------------------------ ConvLSTM gates forward
// pre [N,P,4F] (i,j,f,o); i,j,f,o = IN(pre)*g1+b1 ; c' = c*sig(f+fb) + sig(i)*tanh(j) ; cn = IN(c')*g2+b2 ; h = tanh(cn)*sig(o)
template <int ITERS, int THREADS = 256>
__global__ void __launch_bounds__(THREADS) slab_gates_fwd_kernel(const float* __restrict__ pre, int P, int F, const float* __restrict__ c_prev,
                                                             const float* __restrict__ g1, const float* __restrict__ b1,
                                                             const float* __restrict__ g2, const float* __restrict__ b2, float forget_bias,
                                                             float eps, float* __restrict__ c_new, SlabDsts hdst, float* __restrict__ stats1,
                                                             float* __restrict__ stats2, int cs) {
  __shared__ float s_warp[kSlabMaxWarps * 8 * 32], s_partA[8 * 32], s_partB[8 * 8], s_tot[8 * 32];
  const int q = threadIdx.x & 7, pl = threadIdx.x >> 3, lanes = blockDim.x >> 3;
  const int n = blockIdx.z, c0 = blockIdx.y * 32 + q * 4;
  const int p0 = blockIdx.x * lanes * ITERS;
  const float* pp = pre + static_cast<long long>(n) * P * 4 * F + c0;
  const float* cp = c_prev + static_cast<long long>(n) * P * F + c0;
  float kg[16];                                                    // shifts: the gates at position 0 of the sample
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const float4 t = *reinterpret_cast<const float4*>(pp + g * F);
    kg[4 * g] = t.x; kg[4 * g + 1] = t.y; kg[4 * g + 2] = t.z; kg[4 * g + 3] = t.w;
  }
  float v[ITERS][16];
  float s[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) s[i] = 0.f;
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    const long long p = p0 + pl + it * lanes;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 t = *reinterpret_cast<const float4*>(pp + p * 4 * F + g * F);
      v[it][4 * g] = t.x; v[it][4 * g + 1] = t.y; v[it][4 * g + 2] = t.z; v[it][4 * g + 3] = t.w;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float d = v[it][i] - kg[i];
      s[i] += d;
      s[16 + i] += d * d;
    }
  }
  slab_reduce<32>(s, s_warp, s_partA, s_tot, cs);
  const float inv = 1.f / P;
  float ga[16], be[16];
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int i = 4 * g + k, ch = g * F + c0 + k;
      const float md = s[i] * inv;
      const float var = fmaxf(s[16 + i] * inv - md * md, 0.f);
      const float m = kg[i] + md, r = rsqrtf(var + eps);
      if (stats1 && blockIdx.x == 0 && pl == 0) {
        stats1[(static_cast<long long>(n) * 4 * F + ch) * 2] = m;
        stats1[(static_cast<long long>(n) * 4 * F + ch) * 2 + 1] = r;
      }
      ga[i] = g1[ch] * r;
      be[i] = b1[ch] - m * ga[i];
    }
  // c' of position 0 of the sample = the shift of the state norm (recomputed by every thread for its 4 channels)
  float kc[4];
  {
    const float4 c4 = *reinterpret_cast<const float4*>(cp);
    const float cv[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
      kc[k] = cv[k] * p_sigm(kg[8 + k] * ga[8 + k] + be[8 + k] + forget_bias) +
              p_sigm(kg[k] * ga[k] + be[k]) * tanhf(kg[4 + k] * ga[4 + k] + be[4 + k]);
  }
  float cpre[ITERS][4], so[ITERS][4];
  float t2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    const long long p = p0 + pl + it * lanes;
    const float4 c4 = *reinterpret_cast<const float4*>(cp + p * F);
    const float cv[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float gi = v[it][k] * ga[k] + be[k], gj = v[it][4 + k] * ga[4 + k] + be[4 + k];
      const float gf = v[it][8 + k] * ga[8 + k] + be[8 + k], go = v[it][12 + k] * ga[12 + k] + be[12 + k];
      cpre[it][k] = cv[k] * p_sigm(gf + forget_bias) + p_sigm(gi) * tanhf(gj);
      so[it][k] = p_sigm(go);
      const float d = cpre[it][k] - kc[k];
      t2[k] += d;
      t2[4 + k] += d * d;
    }
  }
  slab_reduce<8>(t2, s_warp, s_partB, s_tot, cs);
  float cg2[4], cb2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float md = t2[k] * inv;
    const float var = fmaxf(t2[4 + k] * inv - md * md, 0.f);
    const float m = kc[k] + md, r = rsqrtf(var + eps);
    if (stats2 && blockIdx.x == 0 && pl == 0) {
      stats2[(static_cast<long long>(n) * F + c0 + k) * 2] = m;
      stats2[(static_cast<long long>(n) * F + c0 + k) * 2 + 1] = r;
    }
    cg2[k] = g2[c0 + k] * r;
    cb2[k] = b2[c0 + k] - m * cg2[k];
  }
  float* cn = c_new + static_cast<long long>(n) * P * F + c0;
#pragma unroll
  for (int it = 0; it < ITERS; ++it) {
    const long long p = p0 + pl + it * lanes;
    float c[4], h[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      c[k] = cpre[it][k] * cg2[k] + cb2[k];
      h[k] = tanhf(c[k]) * so[it][k];
    }
    *reinterpret_cast<float4*>(cn + p * F) = make_float4(c[0], c[1], c[2], c[3]);
    for (int d = 0; d < hdst.count; ++d)
      *reinterpret_cast<float4*>(hdst.ptr[d] + (static_cast<long long>(n) * P + p) * hdst.stride[d] + c0) = make_float4(h[0], h[1], h[2], h[3]);
  }
  if (cs > 1) cg::this_cluster().sync();
}

// ------------------------------------------------------------------------------------------------ ConvLSTM gates backward
// Shared-memory staged like the first version (see lstm_gates_bwd_kernel), slab-mapped: index = local position * 8 + quad.
__global__ void __launch_bounds__(512) slab_gates_bwd_kernel(
    const float* __restrict__ pre, int P, int F, const float* __restrict__ c_prev, const float* __restrict__ g1, const float* __restrict__ b1,
    const float* __restrict__ g2, const float* __restrict__ b2, const float* __restrict__ stats1, const float* __restrict__ stats2,
    float forget_bias, SlabSrcs dh_srcs, const float* __restrict__ dc_next, float* __restrict__ dpre, float* __restrict__ dc_prev,
    float* __restrict__ dg1, float* __restrict__ db1, float* __restrict__ dg2, float* __restrict__ db2, int cs, int ppc) {
  extern __shared__ float4 sm4[];   // ([4][ppc*8] staged pre-activations if ppc <= 128,) [4][ppc*8] gate gradients, [ppc*8] dcn, [ppc*8] chat
  __shared__ float s_warp[kSlabMaxWarps * 8 * 32], s_partA[8 * 8], s_partB[8 * 32], s_tot[8 * 32];
  const int items = ppc * 8;
  const bool stage_pre = ppc <= 128;   // larger CTAs re-read the pre-activations from global memory (L2) in passes B and C
  float4* spre = sm4;
  float4* sdg = stage_pre ? spre + 4 * items : sm4;
  float4* sdc = sdg + 4 * items;
  float4* sch = sdc + items;
  const int q = threadIdx.x & 7, pl = threadIdx.x >> 3, lanes = blockDim.x >> 3;
  const int n = blockIdx.z, c0 = blockIdx.y * 32 + q * 4;
  const int p0 = blockIdx.x * ppc;
  const float inv = 1.f / P;
  float ga[16], be[16], m1[16], r1[16];
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int ch = g * F + c0 + k;
      m1[4 * g + k] = stats1[(static_cast<long long>(n) * 4 * F + ch) * 2];
      r1[4 * g + k] = stats1[(static_cast<long long>(n) * 4 * F + ch) * 2 + 1];
      ga[4 * g + k] = g1[ch];
      be[4 * g + k] = b1[ch];
    }
  float m2[4], r2[4], cg2[4], cb2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    m2[k] = stats2[(static_cast<long long>(n) * F + c0 + k) * 2];
    r2[k] = stats2[(static_cast<long long>(n) * F + c0 + k) * 2 + 1];
    cg2[k] = g2[c0 + k];
    cb2[k] = b2[c0 + k];
  }
  const float* pp = pre + static_cast<long long>(n) * P * 4 * F + c0;
  const float* cp = c_prev + static_cast<long long>(n) * P * F + c0;
  auto gate = [&](const float4 v, int g, float* out) {
    out[0] = (v.x - m1[4 * g]) * r1[4 * g] * ga[4 * g] + be[4 * g];
    out[1] = (v.y - m1[4 * g + 1]) * r1[4 * g + 1] * ga[4 * g + 1] + be[4 * g + 1];
    out[2] = (v.z - m1[4 * g + 2]) * r1[4 * g + 2] * ga[4 * g + 2] + be[4 * g + 2];
    out[3] = (v.w - m1[4 * g + 3]) * r1[4 * g + 3] * ga[4 * g + 3] + be[4 * g + 3];
  };
  // ---- pass A: dcn, chat, dgo; sums for the state norm
  float sA[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int l = pl; l < ppc; l += lanes) {
    const long long p = p0 + l;
    const int si = l * 8 + q;
    float4 pv[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      pv[g] = *reinterpret_cast<const float4*>(pp + p * 4 * F + g * F);
      if (stage_pre) spre[g * items + si] = pv[g];
    }
    float gi[4], gj[4], gf[4], go[4];
    gate(pv[0], 0, gi); gate(pv[1], 1, gj); gate(pv[2], 2, gf); gate(pv[3], 3, go);
    const float4 c4 = *reinterpret_cast<const float4*>(cp + p * F);
    const float cpv[4] = {c4.x, c4.y, c4.z, c4.w};
    float dh[4] = {0.f, 0.f, 0.f, 0.f};
    for (int s = 0; s < dh_srcs.count; ++s) {
      const float4 t = *reinterpret_cast<const float4*>(dh_srcs.ptr[s] + (static_cast<long long>(n) * P + p) * dh_srcs.stride[s] + c0);
      dh[0] += t.x; dh[1] += t.y; dh[2] += t.z; dh[3] += t.w;
    }
    float4 dcn4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (dc_next) dcn4 = *reinterpret_cast<const float4*>(dc_next + (static_cast<long long>(n) * P + p) * F + c0);
    const float dcx[4] = {dcn4.x, dcn4.y, dcn4.z, dcn4.w};
    float dcn[4], chat[4], dgo[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float cpre = cpv[k] * p_sigm(gf[k] + forget_bias) + p_sigm(gi[k]) * tanhf(gj[k]);
      chat[k] = (cpre - m2[k]) * r2[k];
      const float cn = chat[k] * cg2[k] + cb2[k];
      const float th = tanhf(cn), so = p_sigm(go[k]);
      dgo[k] = dh[k] * th * so * (1.f - so);
      dcn[k] = dh[k] * so * (1.f - th * th) + dcx[k];
      sA[k] += dcn[k];
      sA[4 + k] += dcn[k] * chat[k];
    }
    sdc[si] = make_float4(dcn[0], dcn[1], dcn[2], dcn[3]);
    sch[si] = make_float4(chat[0], chat[1], chat[2], chat[3]);
    sdg[3 * items + si] = make_float4(dgo[0], dgo[1], dgo[2], dgo[3]);
  }
  slab_reduce<8>(sA, s_warp, s_partA, s_tot, cs);
  if (blockIdx.x == 0 && pl == 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      db2[static_cast<long long>(n) * F + c0 + k] = sA[k];
      dg2[static_cast<long long>(n) * F + c0 + k] = sA[4 + k];
    }
  }
  // ---- pass B: dc' -> gate gradients (w.r.t. the normalised + affine gates); sums for the gate norm
  float sB[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) sB[i] = 0.f;
  float* dcp = dc_prev + static_cast<long long>(n) * P * F + c0;
  for (int l = pl; l < ppc; l += lanes) {
    const long long p = p0 + l;
    const int si = l * 8 + q;
    float4 pv0, pv1, pv2, pv3;
    if (stage_pre) {
      pv0 = spre[si]; pv1 = spre[items + si]; pv2 = spre[2 * items + si]; pv3 = spre[3 * items + si];
    } else {
      const float* g = pp + p * 4 * F;
      pv0 = *reinterpret_cast<const float4*>(g); pv1 = *reinterpret_cast<const float4*>(g + F);
      pv2 = *reinterpret_cast<const float4*>(g + 2 * F); pv3 = *reinterpret_cast<const float4*>(g + 3 * F);
    }
    float gi[4], gj[4], gf[4];
    gate(pv0, 0, gi); gate(pv1, 1, gj); gate(pv2, 2, gf);
    const float4 c4 = *reinterpret_cast<const float4*>(cp + p * F);
    const float cpv[4] = {c4.x, c4.y, c4.z, c4.w};
    const float4 dcn4 = sdc[si], ch4 = sch[si], dgo4 = sdg[3 * items + si];
    const float dcn[4] = {dcn4.x, dcn4.y, dcn4.z, dcn4.w}, chat[4] = {ch4.x, ch4.y, ch4.z, ch4.w};
    const float dgo[4] = {dgo4.x, dgo4.y, dgo4.z, dgo4.w};
    float di[4], dj[4], df[4], dcpv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float dcpre = r2[k] * cg2[k] * (dcn[k] - sA[k] * inv - chat[k] * sA[4 + k] * inv);
      const float si_ = p_sigm(gi[k]), tj = tanhf(gj[k]), sf = p_sigm(gf[k] + forget_bias);
      di[k] = dcpre * tj * si_ * (1.f - si_);
      dj[k] = dcpre * si_ * (1.f - tj * tj);
      df[k] = dcpre * cpv[k] * sf * (1.f - sf);
      dcpv[k] = dcpre * sf;
    }
    *reinterpret_cast<float4*>(dcp + p * F) = make_float4(dcpv[0], dcpv[1], dcpv[2], dcpv[3]);
    sdg[si] = make_float4(di[0], di[1], di[2], di[3]);
    sdg[items + si] = make_float4(dj[0], dj[1], dj[2], dj[3]);
    sdg[2 * items + si] = make_float4(df[0], df[1], df[2], df[3]);
    const float* dall[4] = {di, dj, df, dgo};
    const float4 pvs[4] = {pv0, pv1, pv2, pv3};
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float xv[4] = {pvs[g].x, pvs[g].y, pvs[g].z, pvs[g].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xh = (xv[k] - m1[4 * g + k]) * r1[4 * g + k];
        sB[4 * g + k] += dall[g][k];
        sB[16 + 4 * g + k] += dall[g][k] * xh;
      }
    }
  }
  slab_reduce<32>(sB, s_warp, s_partB, s_tot, cs);
  if (blockIdx.x == 0 && pl == 0) {
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        db1[static_cast<long long>(n) * 4 * F + g * F + c0 + k] = sB[4 * g + k];
        dg1[static_cast<long long>(n) * 4 * F + g * F + c0 + k] = sB[16 + 4 * g + k];
      }
  }
  // ---- pass C: gate-norm backward -> dpre
  float* dpp = dpre + static_cast<long long>(n) * P * 4 * F + c0;
  for (int l = pl; l < ppc; l += lanes) {
    const long long p = p0 + l;
    const int si = l * 8 + q;
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      const float4 v = stage_pre ? spre[g * items + si] : *reinterpret_cast<const float4*>(pp + p * 4 * F + g * F);
      const float4 d4 = sdg[g * items + si];
      const float xv[4] = {v.x, v.y, v.z, v.w}, dv[4] = {d4.x, d4.y, d4.z, d4.w};
      float o[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float xh = (xv[k] - m1[4 * g + k]) * r1[4 * g + k];
        o[k] = r1[4 * g + k] * ga[4 * g + k] * (dv[k] - sB[4 * g + k] * inv - xh * sB[16 + 4 * g + k] * inv);
      }
      *reinterpret_cast<float4*>(dpp + p * 4 * F + g * F) = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
  if (cs > 1) cg::this_cluster().sync();
}

// ------------------------------------------------------------------------------------------------ host side
static bool slab_enabled() {
  const char* e = getenv("VP_SLAB");
  return !(e && atoi(e) == 0);
}
static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

// Decomposition of a plane of P positions for `units` = slabs * samples independent (sample, slab) units:
// cluster size cs (1..8), positions per CTA ppc = P / cs, and for the register-resident kernels lanes * iters = ppc.
//
// The candidates are ranked by how many ROUNDS of resident clusters the launch needs: these kernels hold one CTA per SM
// (registers or 160-200 KB of staging), and a cluster of 8 is placed inside a GPC, so fewer CTAs than SMs are co-resident
// in clusters of 8; launching more clusters than fit runs extra rounds of a latency-bound kernel.  cudaOccupancyMaxActiveClusters
// gives the resident cluster count of each candidate; cost = rounds * (1 + ppc / ppc_ref): a round is a fixed latency chain
// (loads, two cluster-wide reductions, stores) plus a part that grows with the positions a CTA walks.
struct SlabPlan { int cs, ppc, lanes, iters; };

static int max_active_clusters(const void* kernel, int cs, int threads, size_t smem) {
  static std::map<std::tuple<const void*, int, int, size_t>, int> cache;
  static std::mutex cache_mutex;                       // ctypes releases the GIL: the C ABI may be entered from several host threads
  std::lock_guard<std::mutex> lock(cache_mutex);
  const auto key = std::make_tuple(kernel, cs, threads, smem);
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(cs * 64);
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess || n < 1) {
    cudaGetLastError();
    n = std::max(1, device_sms() / cs);
  }
  cache[key] = n;
  return n;
}

// `describe(ppc, lanes, iters, &kernel, &threads, &smem)` returns false when the kernel family has no variant for that shape.
template <typename Describe>
static bool plan_slab(int P, long long units, int max_lanes, double ppc_ref, Describe describe, SlabPlan* best) {
  if (!is_pow2(P) || P < 8) return false;
  double best_cost = 1e30;
  for (int cs = 1; cs <= 8; cs *= 2) {
    if (P % cs) continue;
    const int ppc = P / cs;
    const int lanes = ppc < max_lanes ? ppc : max_lanes;
    if (lanes < 4) continue;                                                       // block of at least 32 threads
    const int iters = ppc / lanes;
    const void* kernel = nullptr;
    int threads = 0;
    size_t smem = 0;
    if (!describe(ppc, lanes, iters, &kernel, &threads, &smem)) continue;
    const long long resident = max_active_clusters(kernel, cs, threads, smem);
    const long long rounds = (units + resident - 1) / resident;
    const double cost = static_cast<double>(rounds) * (1.0 + ppc / ppc_ref);
    if (cost < best_cost - 1e-9) { best_cost = cost; best->cs = cs; best->ppc = ppc; best->lanes = lanes; best->iters = iters; }
  }
  return best_cost < 1e29;
}

template <typename... Args>
static int launch_cluster(void (*kernel)(Args...), dim3 grid, int threads, size_t smem, int cs, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cs;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (cudaLaunchKernelEx(&cfg, kernel, args...) != cudaSuccess)
    return set_error("cluster launch failed: %s", cudaGetErrorString(cudaGetLastError()));
  count_launch(1);
  return 0;
}

int slab_inorm_act(const float* x, int xs, float* y, int ys, int n, int P, int C, const float* gamma, const float* beta, float eps, int act,
                   float alpha, float* stats, vp_stream_t stream) {
  if (!slab_enabled() || C % 32 || (xs & 3) || (ys & 3)) return 1;
  typedef void (*K)(const float*, int, float*, int, int, int, const float*, const float*, float, int, float, float*, int);
  auto pick = [](int iters) -> K {
    switch (iters) {
      case 1: return slab_inorm_act_kernel<1>;
      case 2: return slab_inorm_act_kernel<2>;
      case 4: return slab_inorm_act_kernel<4>;
      case 8: return slab_inorm_act_kernel<8>;
      case 16: return slab_inorm_act_kernel<16>;
      default: return nullptr;
    }
  };
  SlabPlan pl;
  if (!plan_slab(P, static_cast<long long>(C / 32) * n, 64, 2048.0,
                 [&](int, int lanes, int iters, const void** kern, int* threads, size_t* smem) {
                   K kk = pick(iters);
                   *kern = reinterpret_cast<const void*>(kk); *threads = lanes * 8; *smem = 0;
                   return kk != nullptr;
                 }, &pl)) return 1;
  dim3 grid(pl.cs, C / 32, n);
  K k = pick(pl.iters);
  return launch_cluster(k, grid, pl.lanes * 8, 0, pl.cs, as_stream(stream), x, xs, y, ys, P, C, gamma, beta, eps, act, alpha, stats, pl.cs);
}

int slab_inorm_act_bwd(const float* x, int xs, const float* const* dy, const int* dy_cs, int num_dy, float* dx, int dxs, int n, int P, int C,
                       const float* gamma, const float* beta, const float* stats, int act, float alpha, float* dgamma, float* dbeta,
                       vp_stream_t stream) {
  if (!slab_enabled() || C % 32 || (xs & 3) || (dxs & 3)) return 1;
  typedef void (*K)(const float*, int, SlabSrcs, float*, int, int, int, const float*, const float*, const float*, int, float, float*, float*, int);
  auto pick = [](int iters) -> K {
    switch (iters) {
      case 1: return slab_inorm_act_bwd_kernel<1>;
      case 2: return slab_inorm_act_bwd_kernel<2>;
      case 4: return slab_inorm_act_bwd_kernel<4>;
      case 8: return slab_inorm_act_bwd_kernel<8>;
      default: return nullptr;
    }
  };
  // dx may alias one of the gradient sources only in the register-resident kernels (everything is read before anything is written)
  bool aliased = false;
  for (int i = 0; i < num_dy; ++i) aliased = aliased || dy[i] == dx;
  SlabPlan pl;
  if (!plan_slab(P, static_cast<long long>(C / 32) * n, 64, 1024.0,
                 [&](int ppc, int lanes, int iters, const void** kern, int* threads, size_t* smem) {
                   K kk = pick(iters);
                   *threads = lanes * 8; *smem = 0;
                   if (kk) { *kern = reinterpret_cast<const void*>(kk); return true; }
                   *kern = reinterpret_cast<const void*>(slab_inorm_act_bwd_loop_kernel);
                   return !aliased && ppc <= 2048;
                 }, &pl)) return 1;
  SlabSrcs s;
  s.count = num_dy;
  for (int i = 0; i < 4; ++i) { s.ptr[i] = i < num_dy ? dy[i] : nullptr; s.stride[i] = i < num_dy ? dy_cs[i] : 0; }
  dim3 grid(pl.cs, C / 32, n);
  K k = pick(pl.iters);
  // per-sample partials of dgamma / dbeta (rows of the scratch buffer), added to the outputs in sample order
  float* ws = nullptr;
  if (scratch_alloc(&ws, 2LL * n * C, stream)) return -1;
  float *wg = ws, *wb = ws + static_cast<long long>(n) * C;
  int rc;
  if (!k)
    rc = launch_cluster(slab_inorm_act_bwd_loop_kernel, grid, pl.lanes * 8, 0, pl.cs, as_stream(stream), x, xs, s, dx, dxs, P, C, gamma, beta,
                        stats, act, alpha, wg, wb, pl.cs, pl.ppc);
  else
    rc = launch_cluster(k, grid, pl.lanes * 8, 0, pl.cs, as_stream(stream), x, xs, s, dx, dxs, P, C, gamma, beta, stats, act, alpha, wg, wb,
                        pl.cs);
  if (rc == 0) rc = reduce_parts(wg, n, C, dgamma, stream);
  if (rc == 0) rc = reduce_parts(wb, n, C, dbeta, stream);
  scratch_free(ws, stream);
  return rc;
}

int slab_gates_fwd(const float* pre, int n, int P, int F, const float* c_prev, const float* g1, const float* b1, const float* g2,
                   const float* b2, float forget_bias, float eps, float* c_new, float* const* h_dst, const int* h_cs, int num_h, float* stats1,
                   float* stats2, vp_stream_t stream) {
  if (!slab_enabled() || F % 32) return 1;
  for (int i = 0; i < num_h; ++i) if (h_cs[i] & 3) return 1;
  typedef void (*K)(const float*, int, int, const float*, const float*, const float*, const float*, const float*, float, float, float*, SlabDsts,
                    float*, float*, int);
  auto pick = [](int iters) -> K {                                                   // 256 threads x <= 4 positions: operands stay in registers
    switch (iters) {
      case 1: return slab_gates_fwd_kernel<1>;
      case 2: return slab_gates_fwd_kernel<2>;
      case 4: return slab_gates_fwd_kernel<4>;
      case 8: return slab_gates_fwd_kernel<4, 512>;                                  // lanes = 64: 512 threads x 4 positions
      default: return nullptr;
    }
  };
  SlabPlan pl;
  if (!plan_slab(P, static_cast<long long>(F / 32) * n, 32, 256.0,
                 [&](int, int lanes, int iters, const void** kern, int* threads, size_t* smem) {
                   K kk = pick(iters);
                   *kern = reinterpret_cast<const void*>(kk); *threads = iters == 8 ? 512 : lanes * 8; *smem = 0;
                   return kk != nullptr;
                 }, &pl)) return 1;
  SlabDsts d;
  d.count = num_h;
  for (int i = 0; i < 3; ++i) { d.ptr[i] = i < num_h ? h_dst[i] : nullptr; d.stride[i] = i < num_h ? h_cs[i] : 0; }
  dim3 grid(pl.cs, F / 32, n);
  K k = pick(pl.iters);
  return launch_cluster(k, grid, pl.iters == 8 ? 512 : pl.lanes * 8, 0, pl.cs, as_stream(stream), pre, P, F, c_prev, g1, b1, g2, b2, forget_bias, eps, c_new, d,
                        stats1, stats2, pl.cs);
}

int slab_gates_bwd(const float* pre, int n, int P, int F, const float* c_prev, const float* g1, const float* b1, const float* g2,
                   const float* b2, const float* stats1, const float* stats2, float forget_bias, const float* const* dh, const int* dh_cs,
                   int num_dh, const float* dc_next, float* dpre, float* dc_prev, float* dg1, float* db1, float* dg2, float* db2,
                   vp_stream_t stream) {
  if (!slab_enabled() || F % 32) return 1;
  for (int i = 0; i < num_dh; ++i) if (dh_cs[i] & 3) return 1;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(slab_gates_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 256 * 8 * 6 * 16) != cudaSuccess)
      return set_error("cudaFuncSetAttribute(slab_gates_bwd_kernel) failed");
    attr_set = true;
  }
  // ppc <= 128: pre-activations staged too (10 float4 per position and quad = 160 KB); ppc = 256: they are re-read from
  // global memory (L2) in the second and third pass and only the six derived float4 are staged (192 KB)
  auto staging = [](int ppc) { return static_cast<size_t>(ppc) * 8 * (ppc <= 128 ? 10 : 6) * sizeof(float4); };
  SlabPlan pl;
  if (!plan_slab(P, static_cast<long long>(F / 32) * n, 64, 256.0,
                 [&](int ppc, int lanes, int, const void** kern, int* threads, size_t* smem) {
                   *kern = reinterpret_cast<const void*>(slab_gates_bwd_kernel); *threads = lanes * 8; *smem = staging(ppc);
                   return ppc <= 256;
                 }, &pl)) return 1;
  SlabSrcs s;
  s.count = num_dh;
  for (int i = 0; i < 4; ++i) { s.ptr[i] = i < num_dh ? dh[i] : nullptr; s.stride[i] = i < num_dh ? dh_cs[i] : 0; }
  dim3 grid(pl.cs, F / 32, n);
  // per-sample partials of the four norm-parameter gradients, added to the outputs in sample order
  float* ws = nullptr;
  if (scratch_alloc(&ws, 10LL * n * F, stream)) return -1;
  const long long nf = static_cast<long long>(n) * F;
  float *w_dg1 = ws, *w_db1 = ws + 4 * nf, *w_dg2 = ws + 8 * nf, *w_db2 = ws + 9 * nf;
  int rc = launch_cluster(slab_gates_bwd_kernel, grid, pl.lanes * 8, staging(pl.ppc), pl.cs, as_stream(stream), pre, P, F, c_prev, g1, b1, g2, b2,
                          stats1, stats2, forget_bias, s, dc_next, dpre, dc_prev, w_dg1, w_db1, w_dg2, w_db2, pl.cs, pl.ppc);
  if (rc == 0) rc = reduce_parts(w_dg1, n, 4LL * F, dg1, stream);
  if (rc == 0) rc = reduce_parts(w_db1, n, 4LL * F, db1, stream);
  if (rc == 0) rc = reduce_parts(w_dg2, n, F, dg2, stream);
  if (rc == 0) rc = reduce_parts(w_db2, n, F, db2, stream);
  scratch_free(ws, stream);
  return rc;
}

}  // namespace vp
