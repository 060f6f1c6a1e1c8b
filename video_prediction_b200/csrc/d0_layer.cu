// Weight gradient of the FIRST video-discriminator layer (conv3d 3x3x3, stride 1, zero pad 1, <= 4 input channels
// stored as float4 voxels, 32 output channels; networks.py:83-84) on the tensor cores.
//
//   gw[tap][ci][co] += sum_v x[v + tap][ci] * dy[v][co]            GEMM-K = voxels, M = (dx, ci), N = co
//
// With 4 input channels the generic wgrad engine wastes 7/8 of every 32-channel operand box, and the CUDA-core kernel
// (conv3d_c4_wgrad_kernel, discrim.cu) is latency bound.  Here a line segment of 64 voxels is one pipeline stage: TMA
// brings the 64 x 32 dy tile and the nine halo rows (dz, dy) of x, each 80 float4 voxels from x0 - 8 (borders are zero
// fill = the convolution's padding).  For halo row r the three taps dx and the four channels are the 12 (of 16) M rows of
// one m16n8k8 MMA whose A element (m = 4 dx + ci, k = v) is x_row[v + dx + 7][ci]: the overlapping voxels of the row are the
// operand without any im2col.  Nine MMA warps (one per halo row) issue 4 x 8 MMAs per stage and keep their 16 x 32
// accumulators in registers over the CTA's whole voxel range; each CTA stores its sum into its own scratch row, and the rows
// are added to gw in CTA order (reduce_parts).
#include <algorithm>
#include <cstdint>
#include <cstdlib>

#include "common.h"
#include "ptx.cuh"
#include "tensormap.h"

namespace vp {

constexpr int kD0Pix = 64;                                   // voxels (GEMM-K) per stage
constexpr int kD0RowOct = 10;                                // halo row box: voxels x0 - 8 .. x0 + 71
constexpr int kD0RowBytes = kD0RowOct * 128;
constexpr int kD0DyBytes = kD0Pix * 128;
constexpr int kD0StageBytes = 20 * 1024;                     // dy tile (8 KB) + 9 rows (11520 B)
constexpr int kD0Stages = 8;
constexpr int kD0Threads = 320;                              // warp 0: TMA; warps 1..9: one halo row each

struct D0WgradArgs {
  CUtensorMap xmap, dymap;
  float* gw;                                                 // [gridDim.x][27 * CI * 32] per-CTA partial sums
  int tiles_w, H, D, N, CI;
  int total;                                                 // line segments = N * D * H * tiles_w
};

__global__ void __launch_bounds__(kD0Threads, 1) d0_wgrad_kernel(const __grid_constant__ D0WgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[kD0Stages], empty_bar[kD0Stages];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int it0 = static_cast<int>(static_cast<long long>(a.total) * blockIdx.x / gridDim.x);
  const int it1 = static_cast<int>(static_cast<long long>(a.total) * (blockIdx.x + 1) / gridDim.x);
  if (it1 <= it0) return;

  if (threadIdx.x == 0) {
    for (int i = 0; i < kD0Stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 9); }
    fence_barrier_init();
  }
  __syncthreads();
  const uint32_t smem0 = smem_u32(smem);

  if (warp == 0) {
    // lanes 0..8: the nine halo rows, lane 9: the dy tile
    int mt = it0;
    int tw = mt % a.tiles_w; mt /= a.tiles_w;
    int line = mt;                                             // (n * D + z) * H + y
    int y = mt % a.H; mt /= a.H;
    int z = mt % a.D;
    int n = mt / a.D;
    const int rz = lane / 3 - 1, ry = lane % 3 - 1;
    uint32_t stage = 0, ph = 0;
#pragma unroll 1
    for (int it = it0; it < it1; ++it) {
      mbar_wait(&empty_bar[stage], ph ^ 1);
      const uint32_t dst = smem0 + stage * kD0StageBytes;
      const uint32_t fb = smem_u32(&full_bar[stage]);
      if (lane == 0) mbar_expect_tx(&full_bar[stage], 9 * kD0RowBytes + kD0DyBytes);
      __syncwarp();
      if (lane < 9) {
        tma_load_5d_addr(dst + kD0DyBytes + lane * kD0RowBytes, &a.xmap, fb, 0, tw * (kD0Pix / 8) - 1, y + ry, z + rz, n);
      } else if (lane == 9) {
        tma_load_2d_addr(dst, &a.dymap, fb, 0, line * (a.tiles_w * kD0Pix) + tw * kD0Pix);
      }
      if (++tw == a.tiles_w) {
        tw = 0; ++line;
        if (++y == a.H) { y = 0; if (++z == a.D) { z = 0; ++n; } }
      }
      if (++stage == kD0Stages) { stage = 0; ph ^= 1; }
    }
    return;
  }

  const int r = warp - 1;                                      // halo row (dz, dy) = (r / 3, r % 3)
  const int g = lane >> 2, t = lane & 3;
  const int dx0 = g >> 2, ci = g & 3;                          // M row g = (dx0, ci); M row g + 8 = (dx0 + 2, ci)
  float acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  uint32_t stage = 0, ph = 0;
#pragma unroll 1
  for (int it = it0; it < it1; ++it) {
    mbar_wait(&full_bar[stage], ph);
    const uint32_t dyb = smem0 + stage * kD0StageBytes;
    const uint32_t xr = dyb + kD0DyBytes + r * kD0RowBytes + static_cast<uint32_t>((dx0 + 7) * 4 + ci) * 4u;
#pragma unroll
    for (int k0 = 0; k0 < kD0Pix; k0 += 8) {
      uint32_t af[4];
      af[0] = lds_u32(xr + (k0 + t) * 16);
      af[1] = lds_u32(xr + (k0 + t + 2) * 16);
      af[2] = lds_u32(xr + (k0 + t + 4) * 16);
      af[3] = lds_u32(xr + (k0 + t + 6) * 16);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint32_t bf[2];
        bf[0] = lds_u32(dyb + (k0 + t) * 128 + (8 * j + g) * 4);
        bf[1] = lds_u32(dyb + (k0 + t + 4) * 128 + (8 * j + g) * 4);
        mma_tf32_16x8x8(acc[j], af, bf);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == kD0Stages) { stage = 0; ph ^= 1; }
  }
  if (ci >= a.CI) return;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int dx = dx0 + 2 * h;
    if (dx > 2) continue;
    float* o = a.gw + static_cast<long long>(blockIdx.x) * 27 * a.CI * 32 + (static_cast<long long>(r * 3 + dx) * a.CI + ci) * 32 + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j) *reinterpret_cast<float2*>(o + 8 * j) = make_float2(acc[j][2 * h], acc[j][2 * h + 1]);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// FORWARD of the same layer: out[v][co] = lrelu(bias[co] + sum_{dz,dy,dx,ci} x[v + (dz,dy,dx)][ci] * w[dz][dy][dx][ci][co] / sigma).
//
// GEMM M = voxels, N = 32, K = (tap, ci).  The un-swizzled K-major wgmma layout has core matrices of 8 rows x 16 bytes
// stored as 128 contiguous bytes, i.e. eight consecutive float4 voxels are eight A rows whose first four K elements are the
// voxel's channels; the next four K elements sit LBO bytes further, and LBO = 16 makes them the NEXT voxel (tap dx + 1):
// the overlapping rows x[v-1 .. v+2] are the K = 16 operand of one kernel row (the dx = +2 column meets zero weights) without
// any im2col.  To give 128 consecutive A rows a uniform 16-byte pitch the halo tile is kept FLAT: TMA writes (L + 2) lines
// of (W + 2) voxels back to back, a 128-row M tile is 128 consecutive flat positions (about two lines) and the two halo
// positions per line produce outputs that are not stored (3 %).  The generic engine needed 27 taps x 32 padded channels
// (8x the MMAs); this kernel issues 18 MMAs (K = 8) per 64 voxels and warpgroup.
// Work item = (sample, frame, block of L lines): three TMA boxes (the planes z-1, z, z+1), double buffered; weights / sigma,
// TF32-rounded, are laid out once per CTA as the B operand.  Warpgroup 0 loads, warpgroups 1 and 2 each own one 64-row half
// of every 128-row tile and apply bias + leaky relu from their accumulator registers.
constexpr int kF0Threads = 384;

struct D0FwdArgs {
  CUtensorMap xmap;
  const float* w;            // [3][3][3][CI][32]
  const float* inv_scale;    // sigma (device scalar) or null
  const float* bias;         // [32] or null
  float* out;                // [N][D][H][W][32]
  float alpha;
  int N, D, H, W, CI, L;     // L lines per work item
  int pitch, plane_bytes, plane_stride, stage_bytes, tiles, items, hblocks;   // plane_stride: plane_bytes rounded to the 128 B TMA alignment
};

__global__ void __launch_bounds__(kF0Threads, 1) d0_fwd_kernel(const __grid_constant__ D0FwdArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[2], empty_bar[2];
  const int wg = threadIdx.x >> 7;
  const int lane = threadIdx.x & 31;
  constexpr int kWBytes = 18 * 1024;                                  // B operand: [row 9][k-step 2][32 n x 8 k = 1 KB]
  if (static_cast<int>(blockIdx.x) >= a.items) return;

  // B operand, K-major un-swizzled core matrices: element (n, kk) of block (r, s) at (n / 8) * 256 + (kk / 4) * 128 + (n % 8) * 16 + (kk % 4) * 4
  {
    const float sigma = a.inv_scale ? __ldg(a.inv_scale) : 1.f;
    float* wb = reinterpret_cast<float*>(smem);
    for (int i = threadIdx.x; i < 18 * 256; i += blockDim.x) {
      const int blk = i >> 8, e = i & 255;
      const int n = e >> 3, kk = e & 7;
      const int r = blk >> 1, dx = 2 * (blk & 1) + (kk >> 2), ci = kk & 3;
      float v = 0.f;
      if (dx < 3 && ci < a.CI) v = round_tf32(__ldg(a.w + ((r * 3 + dx) * a.CI + ci) * 32 + n) / sigma);
      wb[blk * 256 + (n >> 3) * 64 + (kk >> 2) * 32 + (n & 7) * 4 + (kk & 3)] = v;
    }
    // The zero-weight K column (dx = +2) of the LAST voxel of a plane reads one voxel past what TMA writes (alignment gap, the
    // next stage before its first load, or the tail): 0 x garbage must not be 0 x NaN, so the tile area starts out as zeros.
    float4* tiles = reinterpret_cast<float4*>(smem + kWBytes);
    const int n16 = (2 * a.stage_bytes + (128 + 2 * a.pitch + 8) * 16) / 16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) tiles[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    fence_proxy_async();
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();
  const uint32_t smem0 = smem_u32(smem);
  const uint32_t stage0 = smem0 + kWBytes;

  if (wg == 0) {
    if (threadIdx.x < 32) {
      uint32_t stage = 0, ph = 0;
#pragma unroll 1
      for (int item = blockIdx.x; item < a.items; item += gridDim.x) {
        int t = item;
        const int hb = t % a.hblocks; t /= a.hblocks;
        const int z = t % a.D;
        const int n = t / a.D;
        mbar_wait(&empty_bar[stage], ph ^ 1);
        if (lane == 0) mbar_expect_tx(&full_bar[stage], 3u * static_cast<uint32_t>(a.plane_bytes));
        __syncwarp();
        if (lane < 3)
          tma_load_5d_addr(stage0 + stage * a.stage_bytes + lane * a.plane_stride, &a.xmap, smem_u32(&full_bar[stage]), 0, -1, hb * a.L - 1,
                           z + lane - 1, n);
        if (++stage == 2) { stage = 0; ph ^= 1; }
      }
    }
    return;
  }

  const int h = wg - 1, wq = (threadIdx.x >> 5) & 3;
  const uint64_t a_base = make_wgmma_desc(stage0 + h * 64 * 16, 16, 128, kWgmmaInterleave);   // LBO 16 B: K elements 4..7 = the next voxel; SBO: 8 voxels
  const uint64_t b_base = make_wgmma_desc(smem0, 128, 256, kWgmmaInterleave);
  float bv[8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int co = 8 * i + 2 * (lane & 3);
    bv[2 * i] = a.bias ? __ldg(a.bias + co) : 0.f;
    bv[2 * i + 1] = a.bias ? __ldg(a.bias + co + 1) : 0.f;
  }
  uint32_t stage = 0, ph = 0;
  float acc[16];
#pragma unroll 1
  for (int item = blockIdx.x; item < a.items; item += gridDim.x) {
    int t = item;
    const int hb = t % a.hblocks; t /= a.hblocks;
    const int z = t % a.D;
    const int n = t / a.D;
    float* obase = a.out + ((static_cast<long long>(n) * a.D + z) * a.H + static_cast<long long>(hb) * a.L) * a.W * 32;
    mbar_wait(&full_bar[stage], ph);
    const uint32_t sadv = stage * (static_cast<uint32_t>(a.stage_bytes) >> 4);
#pragma unroll 1
    for (int tile = 0; tile < a.tiles; ++tile) {
      // A row m of this tile = flat position p0 + m; tap (dz, dy, dx) reads flat voxel p + (dy + 1) * pitch + dx + 1 of plane dz + 1
      const uint32_t p0 = sadv + static_cast<uint32_t>(tile) * 128u;          // in 16-byte units = voxels
      wgmma_fence();
#pragma unroll
      for (int r = 0; r < 9; ++r) {
        const uint32_t row_off = static_cast<uint32_t>(r / 3) * (static_cast<uint32_t>(a.plane_stride) >> 4) +
                                 static_cast<uint32_t>(r % 3) * static_cast<uint32_t>(a.pitch);
#pragma unroll
        for (int s = 0; s < 2; ++s)
          Wgmma<32>::mma(acc, a_base + p0 + row_off + 2 * s, b_base + (r * 2 + s) * (1024 >> 4), (r | s) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int p = tile * 128 + 64 * h + 16 * wq + (lane >> 2) + 8 * rr;
        const int line = p / a.pitch, i = p - line * a.pitch;
        if (line < a.L && i < a.W) {
          float* o = obase + (static_cast<long long>(line) * a.W + i) * 32 + 2 * (lane & 3);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const float u0 = acc[4 * q + 2 * rr] + bv[2 * q], u1 = acc[4 * q + 2 * rr + 1] + bv[2 * q + 1];
            *reinterpret_cast<float2*>(o + 8 * q) = make_float2(fmaxf(u0, a.alpha * u0), fmaxf(u1, a.alpha * u1));
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == 2) { stage = 0; ph ^= 1; }
  }
}

static int encode_map(CUtensorMap* m, const float* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides, const cuuint32_t* box,
                      CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_NONE) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point not found");
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank, const_cast<float*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled(first discriminator layer) failed with %d", static_cast<int>(r));
  return 0;
}

}  // namespace vp

using namespace vp;

extern "C" int vp_conv3d_c4_wgrad_tc(const float* x, const float* dy, float* gw, int n, int d, int h, int wd, int ci, vp_stream_t stream) {
  if (!x || !dy || !gw) return set_error("vp_conv3d_c4_wgrad_tc: null pointer");
  if (ci < 1 || ci > 4) return set_error("vp_conv3d_c4_wgrad_tc: ci must be 1..4");
  if (wd % kD0Pix) return set_error("vp_conv3d_c4_wgrad_tc: width %d is not a multiple of %d (use vp_conv3d_c4_wgrad)", wd, kD0Pix);
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(gw)) & 15)
    return set_error("vp_conv3d_c4_wgrad_tc: pointers must be 16-byte aligned");
  const long long total = static_cast<long long>(n) * d * h * (wd / kD0Pix);
  if (total <= 0 || total > 0x7fffffffLL) return set_error("vp_conv3d_c4_wgrad_tc: bad dims");
  D0WgradArgs A;
  {
    // x: (octet of float4 voxels, w / 8, h, d, n), halo row boxes of 10 octets; dy: (channel, voxel of all lines), 64-voxel boxes
    const cuuint64_t W = wd, H = h, Dd = d;
    cuuint64_t xd[5] = {32, W / 8, H, Dd, static_cast<cuuint64_t>(n)};
    cuuint64_t xs[4] = {128, 16 * W, 16 * W * H, 16 * W * H * Dd};
    cuuint32_t xb[5] = {32, kD0RowOct, 1, 1, 1};
    if (encode_map(&A.xmap, x, 5, xd, xs, xb)) return -1;
    cuuint64_t yd[2] = {32, static_cast<cuuint64_t>(n) * Dd * H * W};
    cuuint64_t ys[1] = {128};
    cuuint32_t yb[2] = {32, kD0Pix};
    if (encode_map(&A.dymap, dy, 2, yd, ys, yb)) return -1;
  }
  A.tiles_w = wd / kD0Pix; A.H = h; A.D = d; A.N = n; A.CI = ci;
  A.total = static_cast<int>(total);
  const size_t smem = static_cast<size_t>(kD0Stages) * kD0StageBytes + 1024;
  static bool configured = false;
  if (!configured) {
    if (cudaFuncSetAttribute(d0_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) != cudaSuccess)
      return set_error("cudaFuncSetAttribute(d0_wgrad_kernel) failed: %s", cudaGetErrorString(cudaGetLastError()));
    configured = true;
  }
  const int sms = device_sms();
  const int grid = static_cast<int>(std::min<long long>(sms, total));
  const long long part = 27LL * ci * 32;
  float* ws = nullptr;
  if (scratch_zeroed(&ws, grid * part, stream)) return -1;     // a CTA with no line segment leaves its row zero
  A.gw = ws;
  d0_wgrad_kernel<<<grid, kD0Threads, smem, as_stream(stream)>>>(A);
  int rc = check_launch("d0_wgrad_kernel");
  if (!rc) rc = reduce_parts(ws, grid, part, gw, stream);
  scratch_free(ws, stream);
  return rc;
}

extern "C" int vp_conv3d_c4_fwd_tc(const float* x, const float* w, const float* inv_scale, const float* bias, float* out, int n, int d, int h,
                                   int wd, int ci, float lrelu_alpha, vp_stream_t stream) {
  if (!x || !w || !out) return set_error("vp_conv3d_c4_fwd_tc: null pointer");
  if (ci < 1 || ci > 4) return set_error("vp_conv3d_c4_fwd_tc: ci must be 1..4");
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15) return set_error("vp_conv3d_c4_fwd_tc: pointers must be 16-byte aligned");
  if (lrelu_alpha < 0.f || lrelu_alpha > 1.f) return set_error("vp_conv3d_c4_fwd_tc: leaky-relu slope must be in [0, 1]");
  D0FwdArgs A;
  A.pitch = wd + 2;
  // lines per work item: three planes of (L + 2) x (W + 2) voxels, two stages, 18 KB of weights
  int L = 0;
  for (int cand : {16, 8, 4}) {
    if (h % cand == 0 && 3LL * (cand + 2) * A.pitch * 16 <= 90 * 1024) { L = cand; break; }
  }
  if (!L || A.pitch > 256) return set_error("vp_conv3d_c4_fwd_tc: %d x %d frames do not tile (use vp_conv3d_c4_fwd)", h, wd);
  A.L = L;
  A.plane_bytes = (L + 2) * A.pitch * 16;
  A.plane_stride = (A.plane_bytes + 127) / 128 * 128;
  A.stage_bytes = (3 * A.plane_stride + 1023) / 1024 * 1024;
  A.tiles = (L * A.pitch + 127) / 128;
  A.hblocks = h / L;
  const long long items = static_cast<long long>(n) * d * A.hblocks;
  if (items <= 0 || items > 0x7fffffffLL) return set_error("vp_conv3d_c4_fwd_tc: bad dims");
  A.items = static_cast<int>(items);
  A.N = n; A.D = d; A.H = h; A.W = wd; A.CI = ci;
  A.w = w; A.inv_scale = inv_scale; A.bias = bias; A.out = out; A.alpha = lrelu_alpha;
  {
    const cuuint64_t W = wd, H = h, Dd = d;
    cuuint64_t xd[5] = {4, W, H, Dd, static_cast<cuuint64_t>(n)};
    cuuint64_t xs[4] = {16, 16 * W, 16 * W * H, 16 * W * H * Dd};
    cuuint32_t xb[5] = {4, static_cast<cuuint32_t>(A.pitch), static_cast<cuuint32_t>(L + 2), 1, 1};
    if (encode_map(&A.xmap, x, 5, xd, xs, xb, CU_TENSOR_MAP_SWIZZLE_NONE)) return -1;
  }
  // tail: the last M tile's junk rows read up to 128 + 2 * pitch + 4 voxels past the third plane
  const size_t smem = 18 * 1024 + 2 * static_cast<size_t>(A.stage_bytes) + (128 + 2 * A.pitch + 8) * 16 + 1024;
  if (smem + 20 * 1024 > 227 * 1024) return set_error("vp_conv3d_c4_fwd_tc: tile does not fit in shared memory");
  static size_t configured = 0;
  if (smem > configured) {
    if (cudaFuncSetAttribute(d0_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)) != cudaSuccess)
      return set_error("cudaFuncSetAttribute(d0_fwd_kernel) failed: %s", cudaGetErrorString(cudaGetLastError()));
    configured = smem;
  }
  const int sms = device_sms();
  const int grid = static_cast<int>(std::min<long long>(sms, items));
  d0_fwd_kernel<<<grid, kF0Threads, smem, as_stream(stream)>>>(A);
  return check_launch("d0_fwd_kernel");
}
