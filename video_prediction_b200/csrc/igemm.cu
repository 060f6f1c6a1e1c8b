// Tensor-core implicit-GEMM convolution engine for H100 (sm_90a).
//
//   D[pixels, Cout] = sum_taps  A_tap[pixels, Cin] * W_tap[Cin, Cout]          (fwd / dgrad)
//   dW_tap[Cout, Cin] = sum_pixels dY[pixels, Cout]^T * X_tap[pixels, Cin]     (wgrad)
//
// Operands are fp32 in HBM/shared memory and are consumed as TF32 by the tensor cores with fp32 accumulation in
// registers.  Activation tiles are fetched with 5-D TMA boxes straight from the NDHWC tensor: a box of bw x bh x bd x bn
// output positions is one 128-row (64-row for wgrad) operand tile whose rows are 32 channels = 128 bytes, written by TMA
// with the 128-byte swizzle.  A filter tap is a coordinate shift of the box; TMA zero-fills out-of-bounds rows/channels,
// which *is* the convolution's zero padding.  Strided convolutions read one of s_d*s_h*s_w "parity" sub-lattices of the
// input (one tensor map each); transposed convolutions (upsample_conv2d forward, dgrad of strided convs) are split into
// output phases.
//
// Forward / dgrad: both operands are K-major (channels contiguous), which is what wgmma needs for TF32: warpgroup 0 is
// the TMA producer, warpgroups 1 and 2 each issue wgmma.m64nBNk8 on one 64-row half of the 128-pixel tile and run the
// epilogue (bias / activation / fused activation gradient) from their accumulator registers.
// Weight gradient: GEMM-K is the pixel dimension, so both shared-memory tiles are MN-major, which wgmma does not accept
// for TF32; eight warps read their fragments from the swizzled TMA tiles and issue mma.sync.m16n8k8 instead.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>

#include "common.h"
#include "ptx.cuh"
#include "tensormap.h"

namespace vp {

constexpr int kMaxTaps = 128;
constexpr int kMaxMaps = 8;
constexpr int kMaxStagesFwd = 8;
constexpr int kWgPix = 64;  // pixels (GEMM-K) per wgrad pipeline stage

struct Tap {
  int8_t map, cd, ch, cw;
  int32_t wslot;
};

struct alignas(64) IgemmArgs {
  CUtensorMap amap[kMaxMaps];  // shifted operand, one map per stride parity
  CUtensorMap bmap;            // fwd: packed weights (2-D);  wgrad: the un-shifted operand (5-D)
  int32_t tiles_w, tiles_h, tiles_d, tiles_n;
  int32_t bw, bh, bd, bn;
  int32_t kc, n_pad, bn_tile;
  int32_t num_phases, splits;
  int32_t phase_begin[9];
  int8_t phase_ooff[8][4];
  int32_t os_d, os_h, os_w;
  float* out;
  long long so_n, so_d, so_h, so_w;
  int32_t out_n, out_d, out_h, out_w, out_c;
  const float* bias;
  int32_t act;
  float alpha;
  int32_t accumulate;
  const float* aux_y;    // optional: activation OUTPUT with the layout of `out`; result is multiplied by act'(aux_y)
  const float* aux_add;  // optional addend (same layout), added before the multiplication
  int32_t aux_act;
  // wgrad only
  int32_t rows_from_shifted, m_tiles, n_tiles, kpad;
  int32_t num_taps, rows_valid, stages;
  int32_t k_tail;        // MMAs (K = 8 channels each) that hold real channels in the LAST k-chunk of a tap (1..4)
  Tap taps[kMaxTaps];
};

__device__ __forceinline__ float apply_act(float v, int act, float alpha) {
  switch (act) {
    case VP_ACT_RELU: return fmaxf(v, 0.f);
    case VP_ACT_LRELU: return fmaxf(alpha * v, v);
    case VP_ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    case VP_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

// Epilogue of one accumulator element: output element `ooff + col` of a valid row.
__device__ __forceinline__ void fwd_store(const IgemmArgs& a, long long ooff, int col, float v, bool add_bias) {
  if (col >= a.out_c) return;
  float* o = a.out + ooff + col;
  if (a.accumulate == 2) v += *o;      // last pass of a multi-pass accumulation: the partial sum is added BEFORE bias / activation
  if (add_bias) v += __ldg(a.bias + col);
  if (a.splits > 1) { atomicAdd(o, v); return; }
  v = apply_act(v, a.act, a.alpha);
  if (a.aux_y != nullptr) {            // fused backward of the previous layer's activation: (v + add) * act'(y)
    const float yv = __ldg(a.aux_y + ooff + col);
    if (a.aux_add != nullptr) v += __ldg(a.aux_add + ooff + col);
    if (a.aux_act == VP_ACT_LRELU) v = yv > 0.f ? v : a.alpha * v;
    else if (a.aux_act == VP_ACT_RELU) v = yv > 0.f ? v : 0.f;
    else if (a.aux_act == VP_ACT_SIGMOID) v *= yv * (1.f - yv);
    else if (a.aux_act == VP_ACT_TANH) v *= (1.f - yv * yv);
  }
  *o = a.accumulate == 1 ? *o + v : v;
}

// ------------------------------------------------------------------------------------------------
// forward / dgrad kernel.  A CTA owns one (BN-column tile, phase, k-split) and walks the 128-pixel tiles
// m = blockIdx.x, blockIdx.x + gridDim.x, ... (persistent): the TMA ring keeps streaming across tiles, so the loads of
// tile i+1 overlap the epilogue of tile i.  A ring stage is one 32-channel k-chunk: a 16 KB activation tile (128 rows)
// and a BN x 128 B weight tile, both 128B-swizzled.
// ------------------------------------------------------------------------------------------------
constexpr int kFwdThreads = 384;
template <int BN>
__global__ void __launch_bounds__(kFwdThreads, 1) igemm_fwd_kernel(const __grid_constant__ IgemmArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[kMaxStagesFwd], empty_bar[kMaxStagesFwd];

  const int wg = threadIdx.x >> 7;
  constexpr uint32_t kABytes = 16384u, kStageBytes = kABytes + BN * 128u;
  const int num_mtiles = a.tiles_w * a.tiles_h * a.tiles_d * a.tiles_n;
  const int n0 = blockIdx.y * BN;
  const int phase = blockIdx.z / a.splits, split = blockIdx.z % a.splits;
  const int tb = a.phase_begin[phase], te = a.phase_begin[phase + 1];
  const int total = (te - tb) * a.kc;
  const int it0 = static_cast<int>(static_cast<long long>(total) * split / a.splits);
  const int it1 = static_cast<int>(static_cast<long long>(total) * (split + 1) / a.splits);
  if (it1 <= it0) return;

  if (threadIdx.x == 0) {
    // full: one arrive (expect_tx) by the producer; empty: one arrive per consumer warp
    for (int i = 0; i < a.stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  const uint32_t smem0 = smem_u32(smem);
  const uint32_t full0 = smem_u32(&full_bar[0]), empty0 = smem_u32(&empty_bar[0]);
  const uint32_t ring_end = static_cast<uint32_t>(a.stages) * 8u;
  if (wg == 0) {
    if (threadIdx.x == 0) {
      // one 5-D activation box and one 2-D weight box per k-chunk; the tap is a coordinate shift, padding is the OOB zero fill
      uint32_t s_off = 0, b_off = 0, ph = 0;
      const int tap0 = it0 / a.kc, c00 = (it0 - tap0 * a.kc) * 32, c0_end = a.kc * 32;
#pragma unroll 1
      for (int mtile = blockIdx.x; mtile < num_mtiles; mtile += gridDim.x) {
        int mt = mtile;
        const int tw = mt % a.tiles_w; mt /= a.tiles_w;
        const int th = mt % a.tiles_h; mt /= a.tiles_h;
        const int td = mt % a.tiles_d;
        const int tn = mt / a.tiles_d;
        const int x0 = tw * a.bw, y0 = th * a.bh, d0 = td * a.bd, s0 = tn * a.bn;
        int tap = tb + tap0, c0 = c00;
#pragma unroll 1
        for (int it = it0; it < it1; ++it) {
          const Tap tp = a.taps[tap];
          mbar_wait_addr(empty0 + b_off, ph ^ 1);
          const uint32_t fb = full0 + b_off;
          mbar_expect_tx_addr(fb, kStageBytes);
          tma_load_5d_addr(smem0 + s_off, &a.amap[tp.map], fb, c0, x0 + tp.cw, y0 + tp.ch, d0 + tp.cd, s0);
          tma_load_2d_addr(smem0 + s_off + kABytes, &a.bmap, fb, c0, tp.wslot * a.n_pad + n0);
          c0 += 32;
          if (c0 == c0_end) { c0 = 0; ++tap; }
          s_off += kStageBytes; b_off += 8;
          if (b_off == ring_end) { s_off = 0; b_off = 0; ph ^= 1; }
        }
      }
    }
    return;
  }

  // ---- consumers: warpgroup h = wg - 1 owns rows 64 h .. 64 h + 63 of the tile
  const int h = wg - 1;
  const int wq = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const uint64_t ad_base = make_wgmma_desc(smem0 + h * 8192u, 16, 1024, kWgmmaSwizzle128B);
  const uint64_t bd_base = make_wgmma_desc(smem0 + kABytes, 16, 1024, kWgmmaSwizzle128B);
  constexpr uint32_t kStageAdv = kStageBytes >> 4;
  const int kq_last = a.kc - 1;
  const bool add_bias = (a.bias != nullptr) && (split == 0);
  // the two rows of this thread inside the tile, as box coordinates
  int lw[2], lh[2], ld[2], ln[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    int row = 64 * h + 16 * wq + (lane >> 2) + 8 * r;
    lw[r] = row % a.bw; row /= a.bw;
    lh[r] = row % a.bh; row /= a.bh;
    ld[r] = row % a.bd;
    ln[r] = row / a.bd;
  }
  uint32_t b_off = 0, ph = 0, adv = 0;
  float acc[BN / 2];
#pragma unroll 1
  for (int mtile = blockIdx.x; mtile < num_mtiles; mtile += gridDim.x) {
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int kq = it0 % a.kc;
#pragma unroll 1
    for (int it = it0; it < it1; ++it) {
      mbar_wait_addr(full0 + b_off, ph);
      // the last k-chunk of a tap may hold fewer than 32 real channels (e.g. 72 = 32 + 32 + 8): the zero-filled K = 8
      // slices are not multiplied at all
      const int nk = kq == kq_last ? a.k_tail : 4;
      const uint64_t ad = ad_base + adv, bd = bd_base + adv;
      wgmma_fence();
      Wgmma<BN>::mma(acc, ad, bd, 1u);
      if (nk > 1) Wgmma<BN>::mma(acc, ad + 2, bd + 2, 1u);
      if (nk > 2) Wgmma<BN>::mma(acc, ad + 4, bd + 4, 1u);
      if (nk > 3) Wgmma<BN>::mma(acc, ad + 6, bd + 6, 1u);
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive_addr(empty0 + b_off);
      kq = kq == kq_last ? 0 : kq + 1;
      adv += kStageAdv; b_off += 8;
      if (b_off == ring_end) { b_off = 0; ph ^= 1; adv = 0; }
    }
    int mt = mtile;
    const int tw = mt % a.tiles_w; mt /= a.tiles_w;
    const int th = mt % a.tiles_h; mt /= a.tiles_h;
    const int td = mt % a.tiles_d;
    const int tn = mt / a.tiles_d;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int ow = (tw * a.bw + lw[r]) * a.os_w + a.phase_ooff[phase][2];
      const int oh = (th * a.bh + lh[r]) * a.os_h + a.phase_ooff[phase][1];
      const int od = (td * a.bd + ld[r]) * a.os_d + a.phase_ooff[phase][0];
      const int on = tn * a.bn + ln[r];
      if (ow < a.out_w && oh < a.out_h && od < a.out_d && on < a.out_n) {
        const long long ooff = on * a.so_n + od * a.so_d + oh * a.so_h + ow * a.so_w;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int col = n0 + 8 * i + 2 * (lane & 3);
          fwd_store(a, ooff, col, acc[4 * i + 2 * r], add_bias);
          fwd_store(a, ooff, col + 1, acc[4 * i + 2 * r + 1], add_bias);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// wgrad kernel: one CTA = (128 dy-channels x up-to-128 x-channels) x ONE filter tap x a range of 64-pixel boxes.
// Per box, warp 0 loads the dy and x tiles (<= 4 + 4 boxes of 64 pixels x 32 channels, 128B-swizzled); the shifted
// operand (x for a conv, dy for a transposed conv) is read at the tap's coordinate shift.  Warps 1..8 own 16 dy channels
// each and accumulate their 16 x (32 nb) slice of dW over the CTA's whole pixel range in registers.  Every dW element has
// one owner per pixel-range split, which adds its sum without atomics: into dW itself when there is one split, otherwise
// into the split's own zero-filled scratch plane (so_n floats apart), which reduce_parts then adds to dW in split order.
// ------------------------------------------------------------------------------------------------
constexpr int kWgMaxStages = 4;
constexpr int kWgThreads = 288;
__global__ void __launch_bounds__(kWgThreads, 1) igemm_wgrad_kernel(const __grid_constant__ IgemmArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[kWgMaxStages], empty_bar[kWgMaxStages];
  constexpr uint32_t kSub = kWgPix * 128;  // bytes of one 64-pixel x 32-channel box

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mtile = blockIdx.x % a.m_tiles, ntile = blockIdx.x / a.m_tiles;
  const int m0 = mtile * 128;                                   // dy channel (row) origin
  const int c0 = ntile * 128;                                   // x channel (col) origin
  const int nb = min(4, a.kc - ntile * 4);                      // 32-channel boxes of x in this tile
  const int na = min(4, (a.rows_valid - m0 + 31) / 32);         // 32-channel boxes of dy that hold real channels
  const Tap tp = a.taps[blockIdx.y];
  const uint32_t stage_bytes = static_cast<uint32_t>(na + nb) * kSub;
  const int total = a.tiles_w * a.tiles_h * a.tiles_d * a.tiles_n;
  const int it0 = static_cast<int>(static_cast<long long>(total) * blockIdx.z / a.splits);
  const int it1 = static_cast<int>(static_cast<long long>(total) * (blockIdx.z + 1) / a.splits);
  if (it1 <= it0 || na <= 0) return;

  if (threadIdx.x == 0) {
    for (int i = 0; i < a.stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  const uint32_t full0 = smem_u32(&full_bar[0]), empty0 = smem_u32(&empty_bar[0]);
  const uint32_t ring_end = static_cast<uint32_t>(a.stages) * 8u;
  const uint32_t smem0 = smem_u32(smem);
  if (warp == 0) {
    if (lane == 0) {
      // dy boxes first, then the x boxes; the plain operand (bmap) is un-shifted, the other one is read at the tap's shift
      const bool dy_shifted = a.rows_from_shifted != 0;
      const CUtensorMap* map = &a.amap[tp.map];
      int mt = it0;
      int tw = mt % a.tiles_w; mt /= a.tiles_w;
      int th = mt % a.tiles_h; mt /= a.tiles_h;
      int td = mt % a.tiles_d;
      int tn = mt / a.tiles_d;
      uint32_t s_off = 0, b_off = 0, ph = 0;
#pragma unroll 1
      for (int it = it0; it < it1; ++it) {
        const int x0 = tw * a.bw, y0 = th * a.bh, d0 = td * a.bd, s0 = tn * a.bn;
        mbar_wait_addr(empty0 + b_off, ph ^ 1);
        const uint32_t fb = full0 + b_off;
        uint32_t dst = smem0 + s_off;
        mbar_expect_tx_addr(fb, stage_bytes);
        for (int i = 0; i < na; ++i, dst += kSub) {
          if (dy_shifted) tma_load_5d_addr(dst, map, fb, m0 + 32 * i, x0 + tp.cw, y0 + tp.ch, d0 + tp.cd, s0);
          else tma_load_5d_addr(dst, &a.bmap, fb, m0 + 32 * i, x0, y0, d0, s0);
        }
        for (int i = 0; i < nb; ++i, dst += kSub) {
          if (dy_shifted) tma_load_5d_addr(dst, &a.bmap, fb, c0 + 32 * i, x0, y0, d0, s0);
          else tma_load_5d_addr(dst, map, fb, c0 + 32 * i, x0 + tp.cw, y0 + tp.ch, d0 + tp.cd, s0);
        }
        if (++tw == a.tiles_w) { tw = 0; if (++th == a.tiles_h) { th = 0; if (++td == a.tiles_d) { td = 0; ++tn; } } }
        s_off += stage_bytes; b_off += 8;
        if (b_off == ring_end) { s_off = 0; b_off = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ---- MMA warps: warp w (1..8) owns dy channels m0 + 16 (w - 1) .. + 15, all 32 nb x channels
  const int cw = warp - 1;
  const int g = lane >> 2, t = lane & 3;
  const bool active = 16 * cw < 32 * na;
  const uint32_t a_box = static_cast<uint32_t>(cw >> 1) * kSub;
  const int a_c = (cw & 1) * 16 + g;
  const int nfr = 4 * nb;
  float acc[16][4];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
  uint32_t s_off = 0, b_off = 0, ph = 0;
#pragma unroll 1
  for (int it = it0; it < it1; ++it) {
    mbar_wait_addr(full0 + b_off, ph);
    if (active) {
      const uint32_t abase = smem0 + s_off + a_box;
      const uint32_t xbase = smem0 + s_off + static_cast<uint32_t>(na) * kSub;
#pragma unroll 2
      for (int k0 = 0; k0 < kWgPix; k0 += 8) {
        uint32_t af[4];
        af[0] = lds_u32(abase + sw128_offset(k0 + t, a_c));
        af[1] = lds_u32(abase + sw128_offset(k0 + t, a_c + 8));
        af[2] = lds_u32(abase + sw128_offset(k0 + t + 4, a_c));
        af[3] = lds_u32(abase + sw128_offset(k0 + t + 4, a_c + 8));
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          if (j < nfr) {
            const uint32_t xb = xbase + static_cast<uint32_t>(j >> 2) * kSub;
            const int c = (j & 3) * 8 + g;
            uint32_t bf[2];
            bf[0] = lds_u32(xb + sw128_offset(k0 + t, c));
            bf[1] = lds_u32(xb + sw128_offset(k0 + t + 4, c));
            mma_tf32_16x8x8(acc[j], af, bf);
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive_addr(empty0 + b_off);
    s_off += stage_bytes; b_off += 8;
    if (b_off == ring_end) { s_off = 0; b_off = 0; ph ^= 1; }
  }
  if (!active) return;
  const int row_end = min(a.n_pad, a.rows_valid);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = m0 + 16 * cw + g + 8 * r;
    if (row >= row_end) continue;
    float* orow = a.out + blockIdx.z * a.so_n + (static_cast<long long>(tp.wslot) * a.n_pad + row) * a.kpad + c0 + 2 * t;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      if (j < nfr) {
        float2* o = reinterpret_cast<float2*>(orow + 8 * j);
        const float2 e = *o;
        *o = make_float2(e.x + acc[j][2 * r], e.y + acc[j][2 * r + 1]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int floor_pow2(int v) { int p = 1; while (p * 2 <= v) p *= 2; return p; }
static int ceil_div(int a, int b) { return (a + b - 1) / b; }
static int pos_mod(int a, int b) { int r = a % b; return r < 0 ? r + b : r; }
static int floor_div(int a, int b) { return (a - pos_mod(a, b)) / b; }

// 5-D map over the (sd,sh,sw)-strided sub-lattice with parity (qd,qh,qw) of an NDHWC view.
static int make_act_map(CUtensorMap* m, const vp_tensor* t, int qd, int qh, int qw, int sd, int sh, int sw,
                        const int box[4] /*w,h,d,n*/) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return set_error("cuTensorMapEncodeTiled entry point not found");
  const long long cs = t->cstride;
  float* base = t->ptr + ((static_cast<long long>(qd) * t->h + qh) * t->w + qw) * cs;
  cuuint64_t dims[5] = {static_cast<cuuint64_t>(t->c), static_cast<cuuint64_t>(std::max(1, ceil_div(t->w - qw, sw))),
                        static_cast<cuuint64_t>(std::max(1, ceil_div(t->h - qh, sh))),
                        static_cast<cuuint64_t>(std::max(1, ceil_div(t->d - qd, sd))), static_cast<cuuint64_t>(t->n)};
  cuuint64_t strides[4] = {static_cast<cuuint64_t>(cs * sw * 4), static_cast<cuuint64_t>(cs * t->w * sh * 4),
                           static_cast<cuuint64_t>(cs * t->w * t->h * sd * 4),
                           static_cast<cuuint64_t>(cs * t->w * t->h * t->d * 4)};
  cuuint32_t boxd[5] = {32, static_cast<cuuint32_t>(box[0]), static_cast<cuuint32_t>(box[1]),
                        static_cast<cuuint32_t>(box[2]), static_cast<cuuint32_t>(box[3])};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, base, dims, strides, boxd, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled(activation) failed with %d", static_cast<int>(r));
  return 0;
}

static int check_tensor(const vp_tensor* t, const char* what) {
  if (!t || !t->ptr) return set_error("%s: null tensor", what);
  if ((reinterpret_cast<uintptr_t>(t->ptr) & 15) || (t->cstride & 3))
    return set_error("%s: pointer must be 16B aligned and cstride a multiple of 4", what);
  if (t->n < 1 || t->d < 1 || t->h < 1 || t->w < 1 || t->c < 1 || t->c > t->cstride)
    return set_error("%s: bad dims", what);
  return 0;
}

// Fills taps / phases / output strides of the geometry; `lat` (w,h,d,n) is divided by the stride for transposed convs.
static int build_taps(IgemmArgs& A, const vp_conv_geom* g, int lat[4]) {
  int ntaps = 0;
  const int K = g->kd * g->kh * g->kw;
  if (K > kMaxTaps) return set_error("too many filter taps (%d)", K);
  if (!g->transposed) {
    if (g->sd * g->sh * g->sw > kMaxMaps) return set_error("stride product too large");
    A.num_phases = 1;
    A.phase_begin[0] = 0;
    A.os_d = A.os_h = A.os_w = 1;
    std::memset(A.phase_ooff, 0, sizeof(A.phase_ooff));
    for (int rd = 0; rd < g->kd; ++rd)
      for (int rh = 0; rh < g->kh; ++rh)
        for (int rw = 0; rw < g->kw; ++rw) {
          Tap& t = A.taps[ntaps++];
          const int qd = pos_mod(rd - g->pd, g->sd), qh = pos_mod(rh - g->ph, g->sh), qw = pos_mod(rw - g->pw, g->sw);
          t.map = static_cast<int8_t>((qd * g->sh + qh) * g->sw + qw);
          t.cd = static_cast<int8_t>(floor_div(rd - g->pd, g->sd));
          t.ch = static_cast<int8_t>(floor_div(rh - g->ph, g->sh));
          t.cw = static_cast<int8_t>(floor_div(rw - g->pw, g->sw));
          t.wslot = (rd * g->kh + rh) * g->kw + rw;
        }
    A.phase_begin[1] = ntaps;
  } else {
    const int P = g->sd * g->sh * g->sw;
    if (P > 8) return set_error("stride product too large");
    A.num_phases = P;
    A.os_d = g->sd; A.os_h = g->sh; A.os_w = g->sw;
    int p = 0;
    for (int fd = 0; fd < g->sd; ++fd)
      for (int fh = 0; fh < g->sh; ++fh)
        for (int fw = 0; fw < g->sw; ++fw, ++p) {
          A.phase_begin[p] = ntaps;
          A.phase_ooff[p][0] = static_cast<int8_t>(fd);
          A.phase_ooff[p][1] = static_cast<int8_t>(fh);
          A.phase_ooff[p][2] = static_cast<int8_t>(fw);
          A.phase_ooff[p][3] = 0;
          const int r0d = pos_mod(fd + g->pd, g->sd), r0h = pos_mod(fh + g->ph, g->sh), r0w = pos_mod(fw + g->pw, g->sw);
          for (int rd = r0d; rd < g->kd; rd += g->sd)
            for (int rh = r0h; rh < g->kh; rh += g->sh)
              for (int rw = r0w; rw < g->kw; rw += g->sw) {
                if (ntaps >= kMaxTaps) return set_error("too many taps");
                Tap& t = A.taps[ntaps++];
                t.map = 0;
                t.cd = static_cast<int8_t>((fd + g->pd - rd) / g->sd);   // exact: (f+p-r) is a multiple of s
                t.ch = static_cast<int8_t>((fh + g->ph - rh) / g->sh);
                t.cw = static_cast<int8_t>((fw + g->pw - rw) / g->sw);
                t.wslot = (rd * g->kh + rh) * g->kw + rw;
              }
        }
    A.phase_begin[P] = ntaps;
    lat[0] = ceil_div(lat[0], g->sw); lat[1] = ceil_div(lat[1], g->sh); lat[2] = ceil_div(lat[2], g->sd);
  }
  return 0;
}

// Fills taps / phases / maps for the tap-shifted tensor `sh_t`; the iteration lattice has dims `lat`.
static int build_geometry(IgemmArgs& A, const vp_conv_geom* g, const vp_tensor* sh_t, int rows_per_tile,
                          const int lat_in[4] /*w,h,d,n*/) {
  int lat[4] = {lat_in[0], lat_in[1], lat_in[2], lat_in[3]};
  if (build_taps(A, g, lat)) return -1;
  // box shape: product == rows_per_tile, powers of two, w fastest
  int rem = rows_per_tile;
  A.bw = std::min(floor_pow2(lat[0]), rem); rem /= A.bw;
  A.bh = std::min(floor_pow2(lat[1]), rem); rem /= A.bh;
  A.bd = std::min(floor_pow2(lat[2]), rem); rem /= A.bd;
  A.bn = rem;
  A.tiles_w = ceil_div(lat[0], A.bw); A.tiles_h = ceil_div(lat[1], A.bh);
  A.tiles_d = ceil_div(lat[2], A.bd); A.tiles_n = ceil_div(lat[3], A.bn);
  const int box[4] = {A.bw, A.bh, A.bd, A.bn};
  if (!g->transposed) {
    for (int qd = 0; qd < g->sd; ++qd)
      for (int qh = 0; qh < g->sh; ++qh)
        for (int qw = 0; qw < g->sw; ++qw) {
          int rc = make_act_map(&A.amap[(qd * g->sh + qh) * g->sw + qw], sh_t, qd, qh, qw, g->sd, g->sh, g->sw, box);
          if (rc) return rc;
        }
  } else {
    int rc = make_act_map(&A.amap[0], sh_t, 0, 0, 0, 1, 1, 1, box);
    if (rc) return rc;
  }
  return 0;
}


}  // namespace vp

using namespace vp;

static int conv_igemm_impl(const vp_tensor* in, const vp_conv_geom* g, const float* wpacked, int n_pad, int kc,
                           const vp_tensor* out, const float* bias, int act, float alpha, int split_k, int accumulate,
                           const float* aux_y, const float* aux_add, int aux_act, vp_stream_t stream) {
  if (check_tensor(in, "vp_conv_igemm(in)") || check_tensor(out, "vp_conv_igemm(out)")) return -1;
  if (!g || !wpacked) return set_error("vp_conv_igemm: null argument");
  if (n_pad % 16 || n_pad < 16) return set_error("vp_conv_igemm: n_pad must be a positive multiple of 16");
  if (kc < 1 || kc * 32 < in->c) return set_error("vp_conv_igemm: kc*32 must cover in->c");
  if (out->c > n_pad) return set_error("vp_conv_igemm: out->c exceeds n_pad");
  if (in->n != out->n) return set_error("vp_conv_igemm: batch mismatch");
  if (split_k > 1 && act != VP_ACT_NONE) return set_error("vp_conv_igemm: split_k needs act NONE");
  if (aux_y && split_k > 1) return set_error("vp_conv_igemm: the fused activation gradient needs split_k <= 1");
  static thread_local IgemmArgs A;  // large POD; per-thread host-side scratch (ctypes releases the GIL during calls)
  std::memset(&A, 0, sizeof(A));
  const int lat[4] = {out->w, out->h, out->d, out->n};
  if (build_geometry(A, g, in, 128, lat)) return -1;
  A.kc = kc; A.n_pad = n_pad;
  A.k_tail = std::min(4, std::max(1, ceil_div(in->c - (kc - 1) * 32, 8)));
  // N tiling: the wgmma N of the tile (32, 64 or 128) whose tiles cover n_pad with the fewest padded columns (ties: the
  // wider tile, which reads the activations fewer times).  A last tile that reaches past n_pad multiplies rows of the next
  // tap's weights (or TMA zero fill) into columns that are never stored.
  {
    int best = 1 << 30;
    for (int bn : {128, 64, 32}) {
      const int cols = ceil_div(n_pad, bn) * bn;
      if (cols < best) { best = cols; A.bn_tile = bn; }
    }
  }
  const int n_tiles = ceil_div(n_pad, A.bn_tile);
  int min_iters = 1 << 30;
  for (int p = 0; p < A.num_phases; ++p) min_iters = std::min(min_iters, (A.phase_begin[p + 1] - A.phase_begin[p]) * kc);
  if (min_iters < 1) return set_error("vp_conv_igemm: a phase has no taps");
  const int sms = device_sms();
  // split_k == 0 (automatic) runs unsplit: split partial sums are added with atomics, whose order (and so the fp32 result)
  // would change from run to run
  if (split_k <= 0) split_k = 1;
  A.splits = std::max(1, std::min(split_k, min_iters));
  A.aux_y = aux_y; A.aux_add = aux_add; A.aux_act = aux_act;
  A.out = out->ptr;
  A.so_w = out->cstride; A.so_h = A.so_w * out->w; A.so_d = A.so_h * out->h; A.so_n = A.so_d * out->d;
  A.out_n = out->n; A.out_d = out->d; A.out_h = out->h; A.out_w = out->w; A.out_c = out->c;
  A.bias = bias; A.act = act; A.alpha = alpha; A.accumulate = accumulate;
  if (accumulate == 1 && act != VP_ACT_NONE) return set_error("vp_conv_igemm: accumulate = 1 needs act NONE");
  // weights: 2-D [slots*n_pad rows][kc*32]
  {
    EncodeTiledFn enc = get_encode();
    if (!enc) return set_error("cuTensorMapEncodeTiled entry point not found");
    const int slots = g->kd * g->kh * g->kw;
    // logical width = the real channel count: the zero padding of the last k-chunk is OOB-filled, not fetched
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(std::min(kc * 32, (in->c + 3) / 4 * 4)), static_cast<cuuint64_t>(slots) * n_pad};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(kc) * 128};
    cuuint32_t box[2] = {32, static_cast<cuuint32_t>(A.bn_tile)};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&A.bmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(wpacked), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error("cuTensorMapEncodeTiled(weights) failed with %d", static_cast<int>(r));
  }
  // ring depth: as many one-chunk stages as fit next to the static shared memory
  const size_t stage_bytes = 16384 + static_cast<size_t>(A.bn_tile) * 128;
  const size_t smem_max = 227 * 1024 - 2048;
  A.stages = static_cast<int>(std::min<size_t>(kMaxStagesFwd, (smem_max - 1024) / stage_bytes));
  const size_t smem = static_cast<size_t>(A.stages) * stage_bytes + 1024;
  typedef void (*FwdKernel)(const IgemmArgs);
  static const FwdKernel kernels[3] = {igemm_fwd_kernel<32>, igemm_fwd_kernel<64>, igemm_fwd_kernel<128>};
  static bool attr_set = false;
  if (!attr_set) {
    for (FwdKernel k : kernels)
      if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)) != cudaSuccess)
        return set_error("cudaFuncSetAttribute(igemm_fwd_kernel) failed: %s", cudaGetErrorString(cudaGetLastError()));
    attr_set = true;
  }
  const FwdKernel kernel = kernels[A.bn_tile == 32 ? 0 : A.bn_tile == 64 ? 1 : 2];
  // persistent over the pixel tiles: one CTA per SM in total; each CTA strides through the M tiles
  const int m_tiles = A.tiles_w * A.tiles_h * A.tiles_d * A.tiles_n;
  const int other = n_tiles * A.num_phases * A.splits;
  const int gx = std::min(m_tiles, std::max(1, sms / other));
  dim3 grid(gx, n_tiles, A.num_phases * A.splits);
  kernel<<<grid, kFwdThreads, smem, static_cast<cudaStream_t>(stream)>>>(A);
  return check_launch("igemm_fwd_kernel");
}

extern "C" int vp_conv_igemm(const vp_tensor* in, const vp_conv_geom* g, const float* wpacked, int n_pad, int kc,
                             const vp_tensor* out, const float* bias, int act, float alpha, int split_k,
                             int accumulate, vp_stream_t stream) {
  return conv_igemm_impl(in, g, wpacked, n_pad, kc, out, bias, act, alpha, split_k, accumulate, nullptr, nullptr, 0, stream);
}

extern "C" int vp_conv_igemm_actgrad(const vp_tensor* in, const vp_conv_geom* g, const float* wpacked, int n_pad, int kc,
                                     const vp_tensor* out, const float* act_output, const float* addend, int act,
                                     float alpha, int accumulate, vp_stream_t stream) {
  if (!act_output) return set_error("vp_conv_igemm_actgrad: act_output is required");
  if (out->c != out->cstride) return set_error("vp_conv_igemm_actgrad: dense output required");
  if (accumulate != 0 && accumulate != 2) return set_error("vp_conv_igemm_actgrad: accumulate must be 0 or 2");
  return conv_igemm_impl(in, g, wpacked, n_pad, kc, out, nullptr, VP_ACT_NONE, alpha, 1, accumulate, act_output, addend, act, stream);
}

extern "C" int vp_conv_wgrad(const vp_tensor* x, const vp_tensor* dy, const vp_conv_geom* g, float* dwpacked,
                             int n_pad, int kc, int split_k, vp_stream_t stream) {
  if (check_tensor(x, "vp_conv_wgrad(x)") || check_tensor(dy, "vp_conv_wgrad(dy)")) return -1;
  if (!g || !dwpacked) return set_error("vp_conv_wgrad: null argument");
  if (n_pad % 16 || dy->c > n_pad || kc * 32 < x->c) return set_error("vp_conv_wgrad: bad n_pad / kc");
  static thread_local IgemmArgs A;
  std::memset(&A, 0, sizeof(A));
  // conv:  dW[r] += sum_o dy[o]^T x[s*o+r-p]   (x shifted, lattice = dy)
  // tconv: dW[r] += sum_o dy[s*o+r-p]^T x[o]   (dy shifted, lattice = x); as a gather this is a
  //        plain (non-transposed) strided access pattern, so build the geometry with transposed=0.
  vp_conv_geom gg = *g;
  gg.transposed = 0;
  const vp_tensor* shifted = g->transposed ? dy : x;
  const vp_tensor* plain = g->transposed ? x : dy;
  const int lat[4] = {plain->w, plain->h, plain->d, plain->n};
  if (build_geometry(A, &gg, shifted, kWgPix, lat)) return -1;
  const int box[4] = {A.bw, A.bh, A.bd, A.bn};
  if (make_act_map(&A.bmap, plain, 0, 0, 0, 1, 1, 1, box)) return -1;
  A.rows_from_shifted = g->transposed ? 1 : 0;
  A.kc = kc; A.n_pad = n_pad; A.kpad = kc * 32;
  A.rows_valid = dy->c;
  A.m_tiles = ceil_div(std::min(n_pad, ceil_div(dy->c, 32) * 32), 128);
  A.n_tiles = ceil_div(kc, 4);
  A.num_taps = A.phase_begin[1];
  const int na_max = std::min(4, ceil_div(dy->c, 32)), nb_max = std::min(4, kc);
  const size_t stage_bytes = static_cast<size_t>(na_max + nb_max) * kWgPix * 128;
  const size_t smem_max = 227 * 1024 - 2048;
  A.stages = static_cast<int>(std::min<size_t>(kWgMaxStages, (smem_max - 1024) / stage_bytes));
  const int total = A.tiles_w * A.tiles_h * A.tiles_d * A.tiles_n;
  const int ctas = A.m_tiles * A.n_tiles * A.num_taps;
  if (split_k <= 0) split_k = std::max(1, (2 * device_sms()) / ctas);  // auto: at most two full waves (never a third partial wave)
  A.splits = std::max(1, std::min(split_k, std::max(1, total / 4)));
  const long long plane = static_cast<long long>(A.num_taps) * n_pad * A.kpad;
  float* ws = nullptr;
  if (A.splits > 1 && scratch_zeroed(&ws, A.splits * plane, stream)) return -1;
  A.out = A.splits > 1 ? ws : dwpacked;
  A.so_n = plane;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(igemm_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)) != cudaSuccess)
      return set_error("cudaFuncSetAttribute(igemm_wgrad_kernel) failed: %s", cudaGetErrorString(cudaGetLastError()));
    attr_set = true;
  }
  const size_t smem = static_cast<size_t>(A.stages) * stage_bytes + 1024;
  dim3 grid(A.m_tiles * A.n_tiles, A.num_taps, A.splits);
  igemm_wgrad_kernel<<<grid, kWgThreads, smem, static_cast<cudaStream_t>(stream)>>>(A);
  int rc = check_launch("igemm_wgrad_kernel");
  if (ws) {
    if (!rc) rc = reduce_parts(ws, A.splits, plane, dwpacked, stream);
    scratch_free(ws, stream);
  }
  return rc;
}
