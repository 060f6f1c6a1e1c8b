// Weight packing for the tensor-core engine and its adjoint.
//
// The trainable kernels stay in the reference's layouts (HWIO / DHWIO, ops.py:513, 768; rnn_ops.py:118).
// Once per optimizer step they are turned into "effective tap matrices" Keff[tap][ci][co]:
//   PLAIN      Keff = w
//   POOLED     conv_pool2d (ops.py:838-842): the 2x2 average pool is applied to the kernel
//   UPSAMPLED  upsample_conv2d (ops.py:698-704): bilinear 4x4 (x) kernel, FULL correlation
// and stored K-major, zero padded and rounded to TF32 (round-to-nearest), in the layout the wgmma
// descriptors read:  FWD  [tap][co -> n_pad][ci -> kc*32],  DGRAD [tap][ci -> n_pad][co -> kc*32].
// A channel map lets the engine's internal (16-byte aligned, padded) concat layouts differ from the
// reference's channel order.
#include <algorithm>
#include <cstdint>

#include "common.h"
#include "ptx.cuh"

namespace vp {

__device__ __forceinline__ float bil4(int i) {  // [.25,.75,.75,.25], zero outside
  return (i == 0 || i == 3) ? 0.25f : ((i == 1 || i == 2) ? 0.75f : 0.f);
}

// effective tap value for reference channel ci, output co
__device__ __forceinline__ float keff(const float* __restrict__ w, int kind, int kd, int kh, int kw, int ci_ref,
                                      int co_n, int tap, int ci, int co) {
  if (kind == VP_WKIND_PLAIN) {
    return w[(static_cast<long long>(tap) * ci_ref + ci) * co_n + co];
  } else if (kind == VP_WKIND_POOLED) {
    const int P = kw + 1;
    const int p = tap / P, q = tap % P;
    float s = 0.f;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int i = p - a, j = q - b;
        if (i >= 0 && i < kh && j >= 0 && j < kw) s += w[((static_cast<long long>(i) * kw + j) * ci_ref + ci) * co_n + co];
      }
    return 0.25f * s;
  } else {
    const int P = kw + 3;
    const int p = tap / P, q = tap % P;
    float s = 0.f;
    for (int i = 0; i < kh; ++i)
      for (int j = 0; j < kw; ++j) {
        const float bw = bil4(p + i - (kh - 1)) * bil4(q + j - (kw - 1));
        if (bw != 0.f) s += bw * w[((static_cast<long long>(i) * kw + j) * ci_ref + ci) * co_n + co];
      }
    return s;
  }
}

__device__ __forceinline__ void pack_element(const float* __restrict__ w, int kd, int kh, int kw, int ci_ref, int co_n, int kind, int layout,
                                             const int32_t* __restrict__ cmap, int ci_int, const float* __restrict__ inv_scale,
                                             float* __restrict__ wp, int n_pad, int kpad, long long idx) {
  const int k = static_cast<int>(idx % kpad);
  const int n = static_cast<int>((idx / kpad) % n_pad);
  const int tap = static_cast<int>(idx / (static_cast<long long>(kpad) * n_pad));
  const int co = (layout & 3) == VP_WLAYOUT_FWD ? n : k;
  const int ci = (layout & 3) == VP_WLAYOUT_FWD ? k : n;
  float v = 0.f;
  if (co < co_n && ci < ci_int) {
    const int cr = cmap ? cmap[ci] : ci;
    if (cr >= 0) {
      v = keff(w, kind, kd, kh, kw, ci_ref, co_n, tap, cr, co);
      if (inv_scale) v = v / __ldg(inv_scale);
    }
  }
  // VP_WLAYOUT_RESIDUAL: the part of the weight the TF32 rounding dropped (the "lo" term of the fp32-exact 3xTF32 mode)
  wp[idx] = (layout & VP_WLAYOUT_RESIDUAL) ? round_tf32(v - round_tf32(v)) : round_tf32(v);
}

__global__ void pack_weights_kernel(const float* __restrict__ w, int kd, int kh, int kw, int ci_ref, int co_n,
                                    int kind, int layout, const int32_t* __restrict__ cmap, int ci_int,
                                    const float* __restrict__ inv_scale, float* __restrict__ wp, int taps, int n_pad,
                                    int kpad) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(taps) * n_pad * kpad;
  if (idx >= total) return;
  pack_element(w, kd, kh, kw, ci_ref, co_n, kind, layout, cmap, ci_int, inv_scale, wp, n_pad, kpad, idx);
}

// All weight tensors of an optimizer in ONE launch (the generator repacks ~60 small tensors after every Adam step: 60
// launches of a few microseconds each): a device table of jobs, each owning the blocks [block_begin, next block_begin).
__global__ void pack_weights_batch_kernel(const vp_pack_job* __restrict__ jobs, int njobs) {
  __shared__ vp_pack_job j;                                      // one table lookup per block, not per thread
  const int b = static_cast<int>(blockIdx.x);
  if (threadIdx.x == 0) {
    int lo = 0, hi = njobs - 1;
    while (lo < hi) {                                            // last job with block_begin <= b
      const int mid = (lo + hi + 1) >> 1;
      if (jobs[mid].block_begin <= b) lo = mid; else hi = mid - 1;
    }
    j = jobs[lo];
  }
  __syncthreads();
  const long long idx = static_cast<long long>(b - j.block_begin) * blockDim.x + threadIdx.x;
  const int kpad = j.kc * 32;
  const int taps = j.kind == VP_WKIND_POOLED ? (j.kh + 1) * (j.kw + 1) : (j.kind == VP_WKIND_UPSAMPLED ? (j.kh + 3) * (j.kw + 3) : j.kd * j.kh * j.kw);
  if (idx >= static_cast<long long>(taps) * j.n_pad * kpad) return;
  pack_element(j.w, j.kd, j.kh, j.kw, j.ci_ref, j.co, j.kind, j.layout, j.cmap, j.ci_int, j.inv_scale, j.wpacked, j.n_pad, kpad, idx);
}

// lo = x - tf32_truncate(x): what the tensor core does not see of an fp32 activation (it reads the top 19 bits)
__global__ void tf32_residual_kernel(const float4* __restrict__ x, float4* __restrict__ lo, long long n4) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = x[i];
    float4 r;
    r.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
    r.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
    r.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
    r.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
    lo[i] = r;
  }
}

// dw[i][j][cmap[ci]][co] += sum_taps dKeff/dw * dwp[tap][co][ci]   (dwp in FWD layout)
__global__ void unpack_wgrad_kernel(const float* __restrict__ dwp, int kd, int kh, int kw, int ci_ref, int co_n,
                                    int kind, const int32_t* __restrict__ cmap, int ci_int, float* __restrict__ dw,
                                    int n_pad, int kpad) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int rtaps = kd * kh * kw;
  const long long total = static_cast<long long>(rtaps) * ci_int * co_n;
  if (idx >= total) return;
  const int co = static_cast<int>(idx % co_n);
  const int ci = static_cast<int>((idx / co_n) % ci_int);
  const int rt = static_cast<int>(idx / (static_cast<long long>(co_n) * ci_int));
  const int cr = cmap ? cmap[ci] : ci;
  if (cr < 0) return;
  auto at = [&](int tap) { return dwp[(static_cast<long long>(tap) * n_pad + co) * kpad + ci]; };
  float g = 0.f;
  if (kind == VP_WKIND_PLAIN) {
    g = at(rt);
  } else if (kind == VP_WKIND_POOLED) {
    const int i = rt / kw, j = rt % kw, P = kw + 1;
    g = 0.25f * (at(i * P + j) + at(i * P + j + 1) + at((i + 1) * P + j) + at((i + 1) * P + j + 1));
  } else {
    const int i = rt / kw, j = rt % kw, P = kw + 3;
    for (int p = 0; p < kh + 3; ++p)
      for (int q = 0; q < kw + 3; ++q) {
        const float bw = bil4(p + i - (kh - 1)) * bil4(q + j - (kw - 1));
        if (bw != 0.f) g += bw * at(p * P + q);
      }
  }
  dw[(static_cast<long long>(rt) * ci_ref + cr) * co_n + co] += g;
}

}  // namespace vp

using namespace vp;

static int eff_taps(int kd, int kh, int kw, int kind) {
  if (kind == VP_WKIND_POOLED) return (kh + 1) * (kw + 1);
  if (kind == VP_WKIND_UPSAMPLED) return (kh + 3) * (kw + 3);
  return kd * kh * kw;
}

extern "C" int vp_pack_weights(const float* w, int kd, int kh, int kw, int ci_ref, int co, int kind, int layout,
                               const int32_t* cmap, int ci_int, const float* inv_scale, float* wpacked, int n_pad,
                               int kc, vp_stream_t stream) {
  if (!w || !wpacked) return set_error("vp_pack_weights: null pointer");
  if (kind != VP_WKIND_PLAIN && kd != 1) return set_error("vp_pack_weights: pooled/upsampled kernels are 2-D");
  const int taps = eff_taps(kd, kh, kw, kind);
  const int kpad = kc * 32;
  const int rows = (layout & 3) == VP_WLAYOUT_FWD ? co : ci_int, cols = (layout & 3) == VP_WLAYOUT_FWD ? ci_int : co;
  if (rows > n_pad || cols > kpad) return set_error("vp_pack_weights: n_pad/kc too small (%d>%d or %d>%d)", rows, n_pad, cols, kpad);
  const long long total = static_cast<long long>(taps) * n_pad * kpad;
  pack_weights_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(w, kd, kh, kw, ci_ref, co, kind, layout, cmap,
                                                                         ci_int, inv_scale, wpacked, taps, n_pad, kpad);
  return check_launch("pack_weights_kernel");
}

extern "C" int vp_pack_weights_batch(const vp_pack_job* jobs_device, int njobs, int total_blocks, vp_stream_t stream) {
  if (!jobs_device || njobs < 1 || total_blocks < 1) return set_error("vp_pack_weights_batch: empty job table");
  pack_weights_batch_kernel<<<total_blocks, 256, 0, as_stream(stream)>>>(jobs_device, njobs);
  return check_launch("pack_weights_batch_kernel");
}

extern "C" int vp_unpack_wgrad(const float* dwpacked, int kd, int kh, int kw, int ci_ref, int co, int kind,
                               const int32_t* cmap, int ci_int, float* dw, int n_pad, int kc, vp_stream_t stream) {
  if (!dwpacked || !dw) return set_error("vp_unpack_wgrad: null pointer");
  const long long total = static_cast<long long>(kd) * kh * kw * ci_int * co;
  unpack_wgrad_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(dwpacked, kd, kh, kw, ci_ref, co, kind, cmap,
                                                                         ci_int, dw, n_pad, kc * 32);
  return check_launch("unpack_wgrad_kernel");
}

extern "C" int vp_tf32_residual(const float* x, float* lo, long long n, vp_stream_t stream) {
  if (!x || !lo || (n & 3) || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(lo) & 15))
    return set_error("vp_tf32_residual: pointers must be 16B aligned and n a multiple of 4");
  const long long n4 = n / 4;
  const int blocks = static_cast<int>(std::min<long long>(8LL * device_sms(), (n4 + 255) / 256));
  tf32_residual_kernel<<<std::max(blocks, 1), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(x),
                                                                          reinterpret_cast<float4*>(lo), n4);
  return check_launch("tf32_residual_kernel");
}
