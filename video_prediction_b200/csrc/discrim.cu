// Discriminator-side helpers: spectral normalisation (ops.py:1020-1049, one power iteration,
// differentiable through the iteration) and per-sample clip gather/scatter (savp_model.py:97-102).
#include <algorithm>

#include "common.h"
#include "ptx.cuh"

namespace vp {

__device__ __forceinline__ float wsum2(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ float block_reduce(float v, float* scratch) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = wsum2(v);
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  float t = (lane < nw) ? scratch[lane] : 0.f;
  return wsum2(t);
}

// out[r] = sum_c W[r][c] * vec[c]     (one warp per row)
__global__ void __launch_bounds__(256) sn_rowdot_kernel(const float* __restrict__ W, const float* __restrict__ vec,
                                                        float* __restrict__ out, int R, int C) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (r >= R) return;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += W[static_cast<long long>(r) * C + c] * vec[c];
  s = wsum2(s);
  if (lane == 0) out[r] = s;
}
// part[blockIdx.y][c] = sum_{r in the block's rows} vec[r] * W[r][c]   (rows split over blockIdx.y; summed in block order)
__global__ void __launch_bounds__(256) sn_coldot_kernel(const float* __restrict__ W, const float* __restrict__ vec,
                                                        float* __restrict__ out, int R, int C, int rows_per_block) {
  const int c = blockIdx.x * 32 + (threadIdx.x & 31), sub = threadIdx.x >> 5;
  const int r0 = blockIdx.y * rows_per_block, r1 = min(R, r0 + rows_per_block);
  float s = 0.f;
  if (c < C)
    for (int r = r0 + sub; r < r1; r += 8) s += vec[r] * W[static_cast<long long>(r) * C + c];
  __shared__ float red[8][32];
  red[sub][threadIdx.x & 31] = s;
  __syncthreads();
  if (sub == 0 && c < C) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i][threadIdx.x & 31];
    out[static_cast<long long>(blockIdx.y) * C + c] = t;
  }
}
// v = t/(|t|+eps) in place; scal[0] = |t|
__global__ void __launch_bounds__(1024) sn_normalize_kernel(float* __restrict__ t, int n, float* __restrict__ scal, int slot) {
  __shared__ float scratch[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += t[i] * t[i];
  const float nrm = sqrtf(block_reduce(s, scratch));
  if (threadIdx.x == 0) scal[slot] = nrm;
  const float inv = 1.f / (nrm + 1e-12f);
  for (int i = threadIdx.x; i < n; i += blockDim.x) t[i] *= inv;
}
// s -> u' = s/(|s|+eps); sigma = s.u' ; scal[1] = |s|, scal[2] = sigma
__global__ void __launch_bounds__(1024) sn_finish_kernel(const float* __restrict__ s, float* __restrict__ u_new, int n,
                                                         float* __restrict__ scal) {
  __shared__ float scratch[32];
  float q = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) q += s[i] * s[i];
  q = block_reduce(q, scratch);
  const float nrm = sqrtf(q);
  const float inv = 1.f / (nrm + 1e-12f);
  for (int i = threadIdx.x; i < n; i += blockDim.x) u_new[i] = s[i] * inv;
  if (threadIdx.x == 0) { scal[1] = nrm; scal[2] = q * inv; }
}
// part[blockIdx.x] = this block's share of <G, W>
__global__ void __launch_bounds__(256) sn_dot_kernel(const float* __restrict__ G, const float* __restrict__ W, long long n,
                                                     float* __restrict__ scal) {
  __shared__ float scratch[32];
  float s = 0.f;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    s += G[i] * W[i];
  s = block_reduce(s, scratch);
  if (threadIdx.x == 0) scal[blockIdx.x] = s;
}
// gs[c] = a * s_hat[c] * gsigma, gsigma = -<G,W>/sigma^2, a = (|s|^2+2 eps |s|)/(|s|+eps)^2, s_hat = s/|s|
__global__ void sn_bwd_gs_kernel(const float* __restrict__ s, float* __restrict__ gs, int n, const float* __restrict__ scal) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float ns = scal[1], sigma = scal[2], dot = scal[3];
  const float gsig = -dot / (sigma * sigma);
  const float a = (ns * ns + 2e-12f * ns) / ((ns + 1e-12f) * (ns + 1e-12f));
  gs[i] = ns > 0.f ? a * (s[i] / ns) * gsig : 0.f;
}
// gt = gv/(n+eps) - t*(t.gv)/(n*(n+eps)^2), t = v*(n+eps);  in place on gv
__global__ void __launch_bounds__(1024) sn_bwd_gt_kernel(const float* __restrict__ v, float* __restrict__ gv, int n,
                                                         const float* __restrict__ scal) {
  __shared__ float scratch[32];
  const float nt = scal[0];
  float d = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) d += v[i] * gv[i];
  d = block_reduce(d, scratch);   // v.gv
  const float ne = nt + 1e-12f;
  // t.gv = ne * (v.gv);  t_i*(t.gv)/(n*ne^2) = v_i*ne*ne*(v.gv)/(n*ne^2) = v_i*(v.gv)/n
  const float coef = nt > 0.f ? d / nt : 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) gv[i] = gv[i] / ne - v[i] * coef;
}
// dW[r][c] += G[r][c]/sigma + v[r]*gs[c] + gt[r]*u[c]
__global__ void sn_bwd_final_kernel(const float* __restrict__ G, const float* __restrict__ v, const float* __restrict__ gs,
                                    const float* __restrict__ gt, const float* __restrict__ u, float* __restrict__ dW,
                                    long long n, int C, const float* __restrict__ scal) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = static_cast<int>(i % C);
  const long long r = i / C;
  dW[i] += G[i] / scal[2] + v[r] * gs[c] + gt[r] * u[c];
}

// clip[b][j][p] = video[t_start[b] + j][b][p]  (float4 pixels; video time-major [T][NBv][P], sample offset b_off)
__global__ void gather_clip_kernel(const float4* __restrict__ video, const int32_t* __restrict__ t_start,
                                   float4* __restrict__ clip, int Bc, int clip_len, long long P, int NBv, int b_off) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(Bc) * clip_len * P;
  if (idx >= total) return;
  const long long p = idx % P;
  const int j = static_cast<int>((idx / P) % clip_len);
  const int b = static_cast<int>(idx / (P * clip_len));
  clip[idx] = video[(static_cast<long long>(t_start[b] + j) * NBv + b_off + b) * P + p];
}
__global__ void scatter_clip_kernel(const float4* __restrict__ dclip, const int32_t* __restrict__ t_start,
                                    float4* __restrict__ dvideo, int Bc, int clip_len, long long P, int NBv, int b_off) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(Bc) * clip_len * P;
  if (idx >= total) return;
  const long long p = idx % P;
  const int j = static_cast<int>((idx / P) % clip_len);
  const int b = static_cast<int>(idx / (P * clip_len));
  float4* o = dvideo + (static_cast<long long>(t_start[b] + j) * NBv + b_off + b) * P + p;
  const float4 d = dclip[idx];
  // towers of different kinds (image / video) on the same unroll run as parallel graph branches and add into the same rows
  red_add_v4(reinterpret_cast<float*>(o), d.x, d.y, d.z, d.w);
}

}  // namespace vp

using namespace vp;

extern "C" int vp_spectral_norm_fwd(const float* w, const float* u, int rows, int cols, float* v, float* s, float* u_new,
                                    float* scal, vp_stream_t stream) {
  cudaStream_t st = as_stream(stream);
  sn_rowdot_kernel<<<(rows + 7) / 8, 256, 0, st>>>(w, u, v, rows, cols);            // t = W u
  sn_normalize_kernel<<<1, 1024, 0, st>>>(v, rows, scal, 0);                          // v = l2n(t)
  cudaMemsetAsync(s, 0, sizeof(float) * cols, st);
  const int rpb = 512;
  dim3 grid((cols + 31) / 32, (rows + rpb - 1) / rpb);
  {
    float* ws = nullptr;
    if (scratch_alloc(&ws, static_cast<long long>(grid.y) * cols, stream)) return -1;
    sn_coldot_kernel<<<grid, 256, 0, st>>>(w, v, ws, rows, cols, rpb);                  // s = v W, block partials
    const int rc = reduce_parts(ws, grid.y, cols, s, stream);
    scratch_free(ws, stream);
    if (rc) return rc;
  }
  sn_finish_kernel<<<1, 1024, 0, st>>>(s, u_new, cols, scal);                         // u' = l2n(s), sigma
  count_launch(3);
  return check_launch("spectral_norm_fwd");
}

extern "C" int vp_spectral_norm_bwd(const float* w, const float* u, const float* g_wbar, int rows, int cols, const float* v,
                                    const float* s, float* scal, float* gs, float* gt, float* dw, vp_stream_t stream) {
  cudaStream_t st = as_stream(stream);
  const long long n = static_cast<long long>(rows) * cols;
  cudaMemsetAsync(scal + 3, 0, sizeof(float), st);
  {
    const int blocks = static_cast<int>(std::min<long long>(592, (n + 255) / 256));
    float* ws = nullptr;
    if (scratch_alloc(&ws, blocks, stream)) return -1;
    sn_dot_kernel<<<blocks, 256, 0, st>>>(g_wbar, w, n, ws);
    const int rc = reduce_parts(ws, blocks, 1, scal + 3, stream);
    scratch_free(ws, stream);
    if (rc) return rc;
  }
  sn_bwd_gs_kernel<<<(cols + 127) / 128, 128, 0, st>>>(s, gs, cols, scal);
  sn_rowdot_kernel<<<(rows + 7) / 8, 256, 0, st>>>(w, gs, gt, rows, cols);            // gv = W gs
  sn_bwd_gt_kernel<<<1, 1024, 0, st>>>(v, gt, rows, scal);
  sn_bwd_final_kernel<<<grid_for(n, 256), 256, 0, st>>>(g_wbar, v, gs, gt, u, dw, n, cols, scal);
  count_launch(4);
  return check_launch("spectral_norm_bwd");
}

extern "C" int vp_gather_clip(const float* video, const int32_t* t_start, float* clip, int clips, int clip_len,
                              long long pixels, int video_batch, int batch_offset, vp_stream_t stream) {
  const long long total = static_cast<long long>(clips) * clip_len * pixels;
  gather_clip_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(video), t_start,
                                                                         reinterpret_cast<float4*>(clip), clips, clip_len, pixels,
                                                                         video_batch, batch_offset);
  return check_launch("gather_clip_kernel");
}

extern "C" int vp_scatter_clip(const float* dclip, const int32_t* t_start, float* dvideo, int clips, int clip_len,
                               long long pixels, int video_batch, int batch_offset, vp_stream_t stream) {
  const long long total = static_cast<long long>(clips) * clip_len * pixels;
  scatter_clip_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(reinterpret_cast<const float4*>(dclip), t_start,
                                                                          reinterpret_cast<float4*>(dvideo), clips, clip_len, pixels,
                                                                          video_batch, batch_offset);
  return check_launch("scatter_clip_kernel");
}

// ------------------------------------------------------------------------------------------------
// Weight gradient of the first discriminator layer (networks.py:83-84: conv3d 3x3x3, stride 1, zero pad 1, C_in = colour
// channels <= 3, C_out = ndf = 32) on the CUDA cores, in exact fp32: the fp32-exact mode's kernel, and the fallback for
// widths the tensor-core kernel (d0_layer.cu) does not tile.  lane = output channel; a warp walks a chunk of voxels keeping
// the 27*C_in partial sums in registers.
// ------------------------------------------------------------------------------------------------
namespace vp {

// gw[(t*CI + ci)*32 + co] += sum_v x[v + tap_t][ci] * dy[v][co]
// blockIdx.y selects the temporal tap dz (9 of the 27 taps -> 27 accumulators per lane, high occupancy); lane = output
// channel; a warp walks one contiguous chunk of voxels (9 broadcast neighbour loads + 1 dy load + 27 FMAs per voxel).
__global__ void __launch_bounds__(256, 3) conv3d_c4_wgrad_kernel(const float4* __restrict__ x, const float* __restrict__ dy,
                                                                 float* __restrict__ gw, int N, int D, int H, int W, int CI,
                                                                 int chunk) {
  const int lane = threadIdx.x & 31;
  const int dz = static_cast<int>(blockIdx.y) - 1;
  const long long warp_id = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  const long long total = static_cast<long long>(N) * D * H * W;
  const long long v0 = min(total, warp_id * chunk), v1 = min(total, v0 + chunk);      // (empty ranges still take part in the block reduction)
  float acc[27];
#pragma unroll
  for (int i = 0; i < 27; ++i) acc[i] = 0.f;
  int xw = static_cast<int>(v0 % W);
  int yh = static_cast<int>((v0 / W) % H);
  int zd = static_cast<int>((v0 / (static_cast<long long>(W) * H)) % D);
  const long long zoff = static_cast<long long>(dz) * H * W;
  for (long long v = v0; v < v1; ++v) {
    const float d = __ldg(dy + v * 32 + lane);
    const bool zin = static_cast<unsigned>(zd + dz) < static_cast<unsigned>(D);
    float4 nb[9];
#pragma unroll
    for (int dyy = -1; dyy <= 1; ++dyy) {
      const bool yin = zin && static_cast<unsigned>(yh + dyy) < static_cast<unsigned>(H);
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const bool in = yin && static_cast<unsigned>(xw + dx) < static_cast<unsigned>(W);
        nb[(dyy + 1) * 3 + dx + 1] = in ? __ldg(x + v + zoff + dyy * W + dx) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      acc[t * 3 + 0] += nb[t].x * d;
      acc[t * 3 + 1] += nb[t].y * d;
      acc[t * 3 + 2] += nb[t].z * d;
    }
    if (++xw == W) { xw = 0; if (++yh == H) { yh = 0; if (++zd == D) zd = 0; } }
  }
  // the 8 warps of the block are summed in shared memory first: 81 x 32 output addresses receive one atomic per BLOCK instead
  // of one per warp (the first version issued 80 M same-address atomics per launch, half of its run time)
  __shared__ float red[8][27][32];
  const int warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < 27; ++i) red[warp][i][lane] = acc[i];
  __syncthreads();
  for (int i = threadIdx.x; i < 27 * 32; i += blockDim.x) {
    const int t3 = i >> 5, co = i & 31;
    float sum = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) sum += red[w][t3][co];
    const int t = t3 / 3, ci = t3 % 3;
    if (ci < CI) atomicAdd(gw + (((dz + 1) * 9 + t) * CI + ci) * 32 + co, sum);
  }
}

}  // namespace vp

extern "C" int vp_conv3d_c4_wgrad(const float* x, const float* dy, float* gw, int n, int d, int h, int wd, int ci,
                                  vp_stream_t stream) {
  if (ci < 1 || ci > 3) return set_error("vp_conv3d_c4_wgrad: 1..3 input channels");
  const long long total = static_cast<long long>(n) * d * h * wd;
  // ~3 resident blocks per SM per temporal tap: each warp walks one contiguous chunk of voxels
  const long long target_warps = 24LL * device_sms();
  const int chunk = static_cast<int>(std::max<long long>(64, (total + target_warps - 1) / target_warps));
  const long long warps = (total + chunk - 1) / chunk;
  dim3 grid(static_cast<unsigned>((warps + 7) / 8), 3);
  conv3d_c4_wgrad_kernel<<<grid, 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(x), dy, gw, n, d, h, wd, ci, chunk);
  return check_launch("conv3d_c4_wgrad_kernel");
}
