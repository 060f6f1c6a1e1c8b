// Tensor-core implicit-GEMM convolution engine for H100 (sm_90a).
//
//   D[pixels, Cout] = sum_taps  A_tap[pixels, Cin] * W_tap[Cin, Cout]          (fwd / dgrad)
//   dW_tap[Cout, Cin] = sum_pixels dY[pixels, Cout]^T * X_tap[pixels, Cin]     (wgrad)
//
// Operands are fp32 in HBM/shared memory and are consumed as TF32 by the tensor cores with fp32 accumulation in
// registers.  Activation tiles are fetched with 5-D TMA boxes straight from the NDHWC tensor: a box of bw x bh x bd x bn
// positions is one 128-row (64-row for the wgrad's dy) operand tile whose rows are 32 channels = 128 bytes, written by TMA
// with the 128-byte swizzle.  A filter tap is a coordinate shift of the box; TMA zero-fills out-of-bounds rows/channels,
// which *is* the convolution's zero padding.  Strided convolutions read one of s_d*s_h*s_w "parity" sub-lattices of the
// input (one tensor map each); transposed convolutions (upsample_conv2d forward, dgrad of strided convs) are split into
// output phases.
//
// Forward / dgrad: both operands are K-major (channels contiguous), which is what wgmma needs for TF32: warpgroup 0 is
// the TMA producer, warpgroups 1 and 2 each issue wgmma.m64nBNk8 on one 64-row half of the 128-pixel tile and run the
// epilogue (bias / activation / fused activation gradient) from their accumulator registers.
// Weight gradient: GEMM-K is the pixel dimension, so both NDHWC operands are MN-major, which wgmma does not accept from
// shared memory for TF32.  A pre-pass copies the un-shifted operand channel-major in tile order (the K-major B operand);
// the tap-shifted one stays channel-minor and reaches wgmma through registers (the register-A form), with the filter taps
// folded into GEMM-M.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <vector>

#include "act.cuh"
#include "common.h"
#include "ptx.cuh"
#include "tensormap.h"

namespace vp {

constexpr int kMaxTaps = 128;
constexpr int kMaxMaps = 8;
constexpr int kMaxStagesFwd = 8;

struct Tap {
  int8_t map, cd, ch, cw;
  int32_t wslot;
};

struct alignas(64) IgemmArgs {
  CUtensorMap amap[kMaxMaps];  // shifted operand, one map per stride parity
  CUtensorMap bmap;            // packed weights (2-D)
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
  int32_t stages;
  int32_t k_tail;        // MMAs (K = 8 channels each) that hold real channels in the LAST k-chunk of a tap (1..4)
  // ConvLSTM epilogue (vp_conv_lstm_fwd): `out` is the natural-order gate pre-activation z [pixels][4F]; GEMM column
  // 128 t + 32 g + c of the GATES pack is gate g of cell channel 32 t + c
  int32_t lstm_f, num_h;
  float forget_bias;
  const float* c_prev;
  float* c_new;
  float* h_dst[3];
  int32_t h_cs[3];
  Tap taps[kMaxTaps];
};

// Epilogue of one accumulator element: output element `ooff + col` of a valid row.
template <bool kElu>
__device__ __forceinline__ void fwd_store(const IgemmArgs& a, long long ooff, int col, float v, bool add_bias) {
  if (col >= a.out_c) return;
  float* o = a.out + ooff + col;
  if (a.accumulate == 2) v += *o;      // last pass of a multi-pass accumulation: the partial sum is added BEFORE bias / activation
  if (add_bias) v += __ldg(a.bias + col);
  if (a.splits > 1) { atomicAdd(o, v); return; }
  v = act_fwd<kElu>(v, a.act, a.alpha);
  if (a.aux_y != nullptr) {            // fused backward of the previous layer's activation: (v + add) * act'(y)
    const float yv = __ldg(a.aux_y + ooff + col);
    if (a.aux_add != nullptr) v += __ldg(a.aux_add + ooff + col);
    v = act_grad_mul<kElu>(v, yv, a.aux_act, a.alpha);
  }
  *o = a.accumulate == 1 ? *o + v : v;
}

__device__ __forceinline__ float sigm_fast(float v) { return 1.f / (1.f + __expf(-v)); }
__device__ __forceinline__ float2 ld2(const float* p) { return *reinterpret_cast<const float2*>(p); }
__device__ __forceinline__ void st2(float* p, float x, float y) { *reinterpret_cast<float2*>(p) = make_float2(x, y); }

// ConvLSTM epilogue of one pixel row (rnn_ops.py:137-171 without normalizer_fn).  With the GATES pack and BN = 128 the
// thread's accumulators acc[4 (4 g + k) + 2 r + e] are gate g of cell channel 32 blockIdx.y + 8 k + 2 (lane % 4) + e, so
// the whole cell runs from registers:  z = conv + bias (natural order [i|j|f|o], kept for the backward),
// c' = c sigmoid(f + forget_bias) + sigmoid(i) tanh(j),  h = tanh(c') sigmoid(o).
// accumulate = 1 is a partial pass of the fp32-exact mode (z += conv, nothing else); accumulate = 2 adds z first.
__device__ __forceinline__ void lstm_store(const IgemmArgs& a, long long pix, const float* acc, int r, int lane) {
  const int F = a.lstm_f;
  float* z = a.out + pix * 4 * F;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int ch = 32 * blockIdx.y + 8 * k + 2 * (lane & 3);
    float zx[4], zy[4];
#pragma unroll
    for (int g = 0; g < 4; ++g) { zx[g] = acc[4 * (4 * g + k) + 2 * r]; zy[g] = acc[4 * (4 * g + k) + 2 * r + 1]; }
    if (a.accumulate == 1) {
#pragma unroll
      for (int g = 0; g < 4; ++g) { const float2 o = ld2(z + g * F + ch); st2(z + g * F + ch, o.x + zx[g], o.y + zy[g]); }
      continue;
    }
#pragma unroll
    for (int g = 0; g < 4; ++g) {
      if (a.accumulate == 2) { const float2 o = ld2(z + g * F + ch); zx[g] += o.x; zy[g] += o.y; }
      const float2 b = __ldg(reinterpret_cast<const float2*>(a.bias + g * F + ch));
      zx[g] += b.x; zy[g] += b.y;
      st2(z + g * F + ch, zx[g], zy[g]);
    }
    const float2 cp = ld2(a.c_prev + pix * F + ch);
    const float cx = cp.x * sigm_fast(zx[2] + a.forget_bias) + sigm_fast(zx[0]) * tanhf(zx[1]);
    const float cy = cp.y * sigm_fast(zy[2] + a.forget_bias) + sigm_fast(zy[0]) * tanhf(zy[1]);
    st2(a.c_new + pix * F + ch, cx, cy);
    const float hx = tanhf(cx) * sigm_fast(zx[3]), hy = tanhf(cy) * sigm_fast(zy[3]);
    for (int d = 0; d < a.num_h; ++d) st2(a.h_dst[d] + pix * a.h_cs[d] + ch, hx, hy);
  }
}

// ------------------------------------------------------------------------------------------------
// forward / dgrad kernel.  A CTA owns one (BN-column tile, phase, k-split) and walks the 128-pixel tiles
// m = blockIdx.x, blockIdx.x + gridDim.x, ... (persistent): the TMA ring keeps streaming across tiles, so the loads of
// tile i+1 overlap the epilogue of tile i.  A ring stage is one 32-channel k-chunk: a 16 KB activation tile (128 rows)
// and a BN x 128 B weight tile, both 128B-swizzled.  One wgmma group per consumer stays in flight: a stage is released
// once the group that read it has completed, while the next chunk's MMAs are already queued.
// ------------------------------------------------------------------------------------------------
constexpr int kFwdThreads = 384;
template <int BN, bool kLstm, bool kElu = false>
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
    uint32_t held = 0;     // empty barrier of the stage read by the wgmma group still in flight
#pragma unroll 1
    for (int it = it0; it < it1; ++it) {
      mbar_wait_addr(full0 + b_off, ph);
      // the last k-chunk of a tap may hold fewer than 32 real channels (e.g. 72 = 32 + 32 + 8): the zero-filled K = 8
      // slices are not multiplied at all.  kq is the same in every thread, but only a vote makes that visible to ptxas:
      // a wgmma behind a branch it cannot prove warp-uniform is serialised (a wait after every MMA, ptxas advisory C7520)
      const int nk = __all_sync(0xffffffffu, kq == kq_last) ? a.k_tail : 4;
      const uint64_t ad = ad_base + adv, bd = bd_base + adv;
      wgmma_fence();
      Wgmma<BN>::mma(acc, ad, bd, 1u);
      if (nk > 1) Wgmma<BN>::mma(acc, ad + 2, bd + 2, 1u);
      if (nk > 2) Wgmma<BN>::mma(acc, ad + 4, bd + 4, 1u);
      if (nk > 3) Wgmma<BN>::mma(acc, ad + 6, bd + 6, 1u);
      wgmma_commit();
      // one group stays in flight: the previous chunk's group has completed, so its stage goes back to the producer
      wgmma_wait<1>();
      if (it > it0) {
        __syncwarp();
        if (lane == 0) mbar_arrive_addr(empty0 + held);
      }
      held = b_off;
      kq = kq == kq_last ? 0 : kq + 1;
      adv += kStageAdv; b_off += 8;
      if (b_off == ring_end) { b_off = 0; ph ^= 1; adv = 0; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive_addr(empty0 + held);
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
        if constexpr (kLstm) {
          lstm_store(a, ((static_cast<long long>(on) * a.out_d + od) * a.out_h + oh) * a.out_w + ow, acc, r, lane);
          continue;
        }
        const long long ooff = on * a.so_n + od * a.so_d + oh * a.so_h + ow * a.so_w;
#pragma unroll
        for (int i = 0; i < BN / 8; ++i) {
          const int col = n0 + 8 * i + 2 * (lane & 3);
          fwd_store<kElu>(a, ooff, col, acc[4 * i + 2 * r], add_bias);
          fwd_store<kElu>(a, ooff, col + 1, acc[4 * i + 2 * r + 1], add_bias);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Weight gradient.  Of the two operands one is read at a per-tap shift ("shifted": x of a conv, which reads x at
// s*o + r - p; dy of a transposed conv, which writes dy there) and the other without one ("plain": dy of a conv, x of a
// transposed conv); the sum runs over the plain operand's pixels o, and tap r reads the shifted operand at position o + c_r
// of its stride-parity lattice q_r (q_r = (r - p) mod s, c_r = floor((r - p) / s)).
// wgrad_xt_kernel copies the plain operand once per call into scratch as T[c][pixel], channel-major, pixels in the main
// kernel's 64-pixel tile order and zero outside the lattice: a K-major wgmma B operand (N = plain channels, K = pixels),
// fetched with 32-pixel x BN-channel TMA boxes (channels past the view are TMA zero fill).  The filter taps are folded into
// GEMM-M: a CTA owns four 32-row blocks, each a (tap, 32-channel chunk of the shifted operand) pair whose rows are a 5-D
// TMA box of the tap's parity lattice at the tap's shift (channel-minor, 128B swizzle, zero fill = the padding), so one B
// tile per 64 pixels serves all of a CTA's taps.  Each thread loads its A fragments from the box with lds and issues
// wgmma.m64nBNk8 in the register-A form.  The products of a dW element are summed in pixel order, 8 pixels per MMA, over
// the tiles of its pixel-range split.
// ------------------------------------------------------------------------------------------------
constexpr int kWgTile = 64;        // pixels (GEMM-K) per pipeline stage
constexpr int kWgBlocks = 4;       // 32-row (tap, channel chunk) blocks per CTA: two per consumer warpgroup
constexpr int kWgMaxStages = 6;
constexpr int kWgThreads = 384;

struct alignas(64) WgradArgs {
  CUtensorMap amap[kMaxMaps];      // shifted operand, one map per stride parity; box: 32 channels x the pixel box
  CUtensorMap tmap;                // plain operand transposed, 2-D [channel][pixel]
  int32_t bw, bh, bd, bn;          // pixel box, w fastest, bw * bh * bd * bn = kWgTile
  int32_t tiles_w, tiles_h, tiles_d, tiles_n;
  int32_t num_taps, chunks, n_tiles, splits, stages;
  int32_t rows_valid, cols_valid;  // channels of the shifted (GEMM-M) and plain (GEMM-N) operands
  int32_t rows_are_ci;             // 1: GEMM-M is x's channels (conv), 0: dy's channels (transposed conv)
  int32_t n_pad, kpad;
  float* out;
  long long so_n;
  Tap taps[kMaxTaps];
};

// Row rho (0..31) of a row block holds channel 4 (rho / 8) + (rho % 4) + 16 ((rho % 8) / 4): lanes g = 0..7 of one
// fragment load then read channels {x..x+3, x+16..x+19}, whose 16-byte chunks under the 128B swizzle fall on 32 different
// banks for the four pixel rows t = 0..3 (a contiguous 8 channels would be a 2-way conflict).
__device__ __forceinline__ int wg_row_channel(int rho) { return 4 * (rho >> 3) + (rho & 3) + 16 * ((rho >> 2) & 1); }

template <int BN>
__global__ void __launch_bounds__(kWgThreads, 1) igemm_wgrad_kernel(const __grid_constant__ WgradArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full_bar[kWgMaxStages], empty_bar[kWgMaxStages];
  constexpr uint32_t kBox = kWgTile * 128;                  // one row block: 64 pixels x 32 channels
  constexpr uint32_t kTHalf = BN * 128;                     // 32 pixels of the B tile: BN channel rows of 128 B
  constexpr uint32_t kStage = kWgBlocks * kBox + 2 * kTHalf;

  const int wg = threadIdx.x >> 7;
  const int ntile = blockIdx.x % a.n_tiles;
  const int blk0 = (blockIdx.x / a.n_tiles) * kWgBlocks;
  const int nblk = min(kWgBlocks, a.num_taps * a.chunks - blk0);
  const int c0 = ntile * BN;
  const int total = a.tiles_w * a.tiles_h * a.tiles_d * a.tiles_n;
  const int it0 = static_cast<int>(static_cast<long long>(total) * blockIdx.y / a.splits);
  const int it1 = static_cast<int>(static_cast<long long>(total) * (blockIdx.y + 1) / a.splits);
  if (it1 <= it0) return;

  if (threadIdx.x == 0) {
    for (int i = 0; i < a.stages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    fence_barrier_init();
  }
  __syncthreads();

  const uint32_t smem0 = smem_u32(smem);
  const uint32_t full0 = smem_u32(&full_bar[0]), empty0 = smem_u32(&empty_bar[0]);
  const uint32_t ring_end = static_cast<uint32_t>(a.stages) * 8u;
  if (wg == 0) {
    if (threadIdx.x == 0) {
      int rem = it0;
      int tw = rem % a.tiles_w; rem /= a.tiles_w;
      int th = rem % a.tiles_h; rem /= a.tiles_h;
      int td = rem % a.tiles_d;
      int tn = rem / a.tiles_d;
      const uint32_t stage_tx = static_cast<uint32_t>(nblk) * kBox + 2 * kTHalf;
      uint32_t s_off = 0, b_off = 0, ph = 0;
#pragma unroll 1
      for (int it = it0; it < it1; ++it) {
        const int x0 = tw * a.bw, y0 = th * a.bh, d0 = td * a.bd, s0 = tn * a.bn;
        mbar_wait_addr(empty0 + b_off, ph ^ 1);
        const uint32_t fb = full0 + b_off, dst = smem0 + s_off;
        mbar_expect_tx_addr(fb, stage_tx);
        for (int j = 0; j < nblk; ++j) {
          const int b = blk0 + j;
          const Tap tp = a.taps[b / a.chunks];
          tma_load_5d_addr(dst + j * kBox, &a.amap[tp.map], fb, 32 * (b % a.chunks), x0 + tp.cw, y0 + tp.ch, d0 + tp.cd, s0);
        }
        tma_load_2d_addr(dst + kWgBlocks * kBox, &a.tmap, fb, it * kWgTile, c0);
        tma_load_2d_addr(dst + kWgBlocks * kBox + kTHalf, &a.tmap, fb, it * kWgTile + 32, c0);
        if (++tw == a.tiles_w) { tw = 0; if (++th == a.tiles_h) { th = 0; if (++td == a.tiles_d) { td = 0; ++tn; } } }
        s_off += kStage; b_off += 8;
        if (b_off == ring_end) { s_off = 0; b_off = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ---- consumers: warpgroup h owns row blocks 2h, 2h + 1; warp w of it rows 16 (w % 2) .. + 15 of block 2h + w / 2
  const int h = wg - 1, w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int j = 2 * h + (w >> 1);
  const bool live = j < nblk;
  const int c_lo = wg_row_channel(16 * (w & 1) + g), c_hi = wg_row_channel(16 * (w & 1) + 8 + g);
  const uint64_t bd_base = make_wgmma_desc(smem0 + kWgBlocks * kBox, 16, 1024, kWgmmaSwizzle128B);
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  uint32_t s_off = 0, b_off = 0, ph = 0;
#pragma unroll 1
  for (int it = it0; it < it1; ++it) {
    mbar_wait_addr(full0 + b_off, ph);
    uint32_t af[8][4];
    const uint32_t ab = smem0 + s_off + static_cast<uint32_t>(j) * kBox;
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int k = 8 * ks + t;
      af[ks][0] = live ? lds_u32(ab + sw128_offset(k, c_lo)) : 0u;
      af[ks][1] = live ? lds_u32(ab + sw128_offset(k, c_hi)) : 0u;
      af[ks][2] = live ? lds_u32(ab + sw128_offset(k + 4, c_lo)) : 0u;
      af[ks][3] = live ? lds_u32(ab + sw128_offset(k + 4, c_hi)) : 0u;
    }
    const uint64_t bd = bd_base + (s_off >> 4);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks)
      WgmmaRS<BN>::mma(acc, af[ks], bd + (ks < 4 ? 2 * ks : kTHalf / 16 + 2 * (ks - 4)));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive_addr(empty0 + b_off);
    s_off += kStage; b_off += 8;
    if (b_off == ring_end) { s_off = 0; b_off = 0; ph ^= 1; }
  }
  if (!live) return;
  // every dW element has one owner per pixel-range split, which adds its sum without atomics: into dW itself when there is
  // one split, otherwise into the split's own zero-filled scratch plane, which reduce_parts adds to dW in split order
  const int b = blk0 + j;
  const Tap tp = a.taps[b / a.chunks];
  float* plane = a.out + blockIdx.y * a.so_n + static_cast<long long>(tp.wslot) * a.n_pad * a.kpad;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int row = 32 * (b % a.chunks) + (r ? c_hi : c_lo);
    if (row >= a.rows_valid) continue;
#pragma unroll
    for (int i = 0; i < BN / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = c0 + 8 * i + 2 * t + e;
        if (col >= a.cols_valid) continue;
        // dW is [co][ci]: GEMM rows are x channels (ci) for a conv and dy channels (co) for a transposed conv
        float* o = a.rows_are_ci ? plane + static_cast<long long>(col) * a.kpad + row : plane + static_cast<long long>(row) * a.kpad + col;
        *o += acc[4 * i + 2 * r + e];
      }
    }
  }
}

// T[c][tile * 64 + k] = the plain operand at pixel k of tile `tile` (0 outside the tensor).  One block transposes one tile
// x 32 channels through shared memory: reads run along channels, writes along pixels.
struct TransposeArgs {
  const float* src;
  long long cstride;
  int32_t n, d, h, w, c;
  int32_t bw, bh, bd, bn;
  int32_t tiles_w, tiles_h, tiles_d;
  float* dst;
  long long p_pad;                 // pixels per channel row of T
};

__global__ void __launch_bounds__(256) wgrad_transpose_kernel(const __grid_constant__ TransposeArgs a) {
  __shared__ float tile_s[32][kWgTile + 1];
  const int tile = blockIdx.x;
  const int tw = tile % a.tiles_w, th = (tile / a.tiles_w) % a.tiles_h, td = (tile / (a.tiles_w * a.tiles_h)) % a.tiles_d;
  const int tn = tile / (a.tiles_w * a.tiles_h * a.tiles_d);
  const int c0 = blockIdx.y * 32;
  for (int e = threadIdx.x; e < kWgTile * 32; e += blockDim.x) {
    const int k = e >> 5, c = e & 31;
    const int pw = tw * a.bw + k % a.bw, ph = th * a.bh + (k / a.bw) % a.bh;
    const int pd = td * a.bd + (k / (a.bw * a.bh)) % a.bd, pn = tn * a.bn + k / (a.bw * a.bh * a.bd);
    float v = 0.f;
    if (pw < a.w && ph < a.h && pd < a.d && pn < a.n && c0 + c < a.c) {
      const long long pix = ((static_cast<long long>(pn) * a.d + pd) * a.h + ph) * a.w + pw;
      v = __ldg(a.src + pix * a.cstride + c0 + c);
    }
    tile_s[c][k] = v;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < kWgTile * 32; e += blockDim.x) {
    const int c = e / kWgTile, k = e % kWgTile;
    if (c0 + c < a.c) a.dst[static_cast<long long>(c0 + c) * a.p_pad + static_cast<long long>(tile) * kWgTile + k] = tile_s[c][k];
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

// Taps of a (non-transposed) convolution in weight-slot order: tap r reads the input at s * o + r - p, i.e. at lattice
// position o + c_r of the stride-parity sub-lattice q_r (map = q_r, (cd, ch, cw) = c_r).  Returns the count, -1 on error.
static int conv_taps(const vp_conv_geom* g, Tap* taps) {
  const int K = g->kd * g->kh * g->kw;
  if (K > kMaxTaps) return set_error("too many filter taps (%d)", K);
  if (g->sd * g->sh * g->sw > kMaxMaps) return set_error("stride product too large");
  int n = 0;
  for (int rd = 0; rd < g->kd; ++rd)
    for (int rh = 0; rh < g->kh; ++rh)
      for (int rw = 0; rw < g->kw; ++rw) {
        Tap& t = taps[n++];
        const int qd = pos_mod(rd - g->pd, g->sd), qh = pos_mod(rh - g->ph, g->sh), qw = pos_mod(rw - g->pw, g->sw);
        t.map = static_cast<int8_t>((qd * g->sh + qh) * g->sw + qw);
        t.cd = static_cast<int8_t>(floor_div(rd - g->pd, g->sd));
        t.ch = static_cast<int8_t>(floor_div(rh - g->ph, g->sh));
        t.cw = static_cast<int8_t>(floor_div(rw - g->pw, g->sw));
        t.wslot = (rd * g->kh + rh) * g->kw + rw;
      }
  return n;
}

// Fills taps / phases / output strides of the geometry; `lat` (w,h,d,n) is divided by the stride for transposed convs.
static int build_taps(IgemmArgs& A, const vp_conv_geom* g, int lat[4]) {
  int ntaps = 0;
  if (!g->transposed) {
    ntaps = conv_taps(g, A.taps);
    if (ntaps < 0) return -1;
    A.num_phases = 1;
    A.phase_begin[0] = 0;
    A.os_d = A.os_h = A.os_w = 1;
    std::memset(A.phase_ooff, 0, sizeof(A.phase_ooff));
    A.phase_begin[1] = ntaps;
  } else {
    if (g->kd * g->kh * g->kw > kMaxTaps) return set_error("too many filter taps (%d)", g->kd * g->kh * g->kw);
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

// The cell of vp_conv_lstm_fwd, for conv_igemm_impl (nullptr: a plain convolution).
struct LstmCell {
  const float* c_prev;
  float* c_new;
  float* const* h_dst;
  const int* h_cs;
  int num_h;
  float forget_bias;
};

static int conv_igemm_impl(const vp_tensor* in, const vp_conv_geom* g, const float* wpacked, int n_pad, int kc,
                           const vp_tensor* out, const float* bias, int act, float alpha, int split_k, int accumulate,
                           const float* aux_y, const float* aux_add, int aux_act, vp_stream_t stream,
                           const LstmCell* cell = nullptr) {
  if (check_tensor(in, "vp_conv_igemm(in)") || check_tensor(out, "vp_conv_igemm(out)")) return -1;
  if (!g || !wpacked) return set_error("vp_conv_igemm: null argument");
  if (n_pad % 16 || n_pad < 16) return set_error("vp_conv_igemm: n_pad must be a positive multiple of 16");
  if (kc < 1 || kc * 32 < in->c) return set_error("vp_conv_igemm: kc*32 must cover in->c");
  if (out->c > n_pad) return set_error("vp_conv_igemm: out->c exceeds n_pad");
  if (in->n != out->n) return set_error("vp_conv_igemm: batch mismatch");
  if (check_act(act, "vp_conv_igemm") || check_act(aux_act, "vp_conv_igemm_actgrad")) return -1;
  if (split_k > 1 && act != VP_ACT_NONE) return set_error("vp_conv_igemm: split_k needs act NONE");
  if (aux_y && split_k > 1) return set_error("vp_conv_igemm: the fused activation gradient needs split_k <= 1");
  if (accumulate < 0 || accumulate > 2) return set_error("vp_conv_igemm: accumulate must be 0, 1 or 2 (got %d)", accumulate);
  // every split would read the existing partial sum and add it again, as many times as there are splits
  if (accumulate == 2 && split_k > 1)
    return set_error("vp_conv_igemm: accumulate = 2 needs split_k <= 1 (got split_k = %d)", split_k);
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
  if (cell) {     // a 128-column tile holds all four gates of 32 cell channels
    A.bn_tile = 128;
    A.lstm_f = out->c / 4;
    A.c_prev = cell->c_prev; A.c_new = cell->c_new; A.num_h = cell->num_h; A.forget_bias = cell->forget_bias;
    for (int i = 0; i < cell->num_h; ++i) { A.h_dst[i] = cell->h_dst[i]; A.h_cs[i] = cell->h_cs[i]; }
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
  static const FwdKernel kernels[7] = {igemm_fwd_kernel<32, false>, igemm_fwd_kernel<64, false>, igemm_fwd_kernel<128, false>,
                                       igemm_fwd_kernel<128, true>, igemm_fwd_kernel<32, false, true>,
                                       igemm_fwd_kernel<64, false, true>, igemm_fwd_kernel<128, false, true>};
  static bool attr_set = false;
  if (!attr_set) {
    for (FwdKernel k : kernels)
      if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)) != cudaSuccess)
        return set_error("cudaFuncSetAttribute(igemm_fwd_kernel) failed: %s", cudaGetErrorString(cudaGetLastError()));
    attr_set = true;
  }
  const bool elu = act == VP_ACT_ELU || (aux_y && aux_act == VP_ACT_ELU);
  const FwdKernel kernel = kernels[cell ? 3 : (A.bn_tile == 32 ? 0 : A.bn_tile == 64 ? 1 : 2) + (elu ? 4 : 0)];
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

extern "C" int vp_conv_lstm_fwd(const vp_tensor* in, const vp_conv_geom* g, const float* wpacked, int n_pad, int kc,
                                const vp_tensor* z, const float* bias, const float* c_prev, float* c_new, float* const* h_dst,
                                const int* h_cstride, int num_h_dst, float forget_bias, int accumulate, vp_stream_t stream) {
  if (check_tensor(z, "vp_conv_lstm_fwd(z)")) return -1;
  if (z->c % 128) return set_error("vp_conv_lstm_fwd: the cell needs filters %% 32 == 0 (got %d)", z->c / 4);
  if (z->c != z->cstride || n_pad != z->c) return set_error("vp_conv_lstm_fwd: z must be dense [pixels][4F] and n_pad == 4F");
  if (!bias || !c_prev || !c_new || !h_dst || !h_cstride) return set_error("vp_conv_lstm_fwd: null argument");
  if (num_h_dst < 1 || num_h_dst > 3) return set_error("vp_conv_lstm_fwd: 1 to 3 h destinations (got %d)", num_h_dst);
  if ((reinterpret_cast<uintptr_t>(bias) | reinterpret_cast<uintptr_t>(c_prev) | reinterpret_cast<uintptr_t>(c_new)) & 15)
    return set_error("vp_conv_lstm_fwd: bias / c pointers must be 16B aligned");
  for (int i = 0; i < num_h_dst; ++i)
    if (!h_dst[i] || (reinterpret_cast<uintptr_t>(h_dst[i]) & 15) || h_cstride[i] < z->c / 4 || (h_cstride[i] & 3))
      return set_error("vp_conv_lstm_fwd: h destination %d: null, unaligned, or channel stride below F / not a multiple of 4", i);
  if (accumulate < 0 || accumulate > 2) return set_error("vp_conv_lstm_fwd: accumulate must be 0, 1 or 2 (got %d)", accumulate);
  const LstmCell cell{c_prev, c_new, h_dst, h_cstride, num_h_dst, forget_bias};
  return conv_igemm_impl(in, g, wpacked, n_pad, kc, z, bias, VP_ACT_NONE, 0.f, 1, accumulate, nullptr, nullptr, 0, stream, &cell);
}

extern "C" int vp_conv_wgrad(const vp_tensor* x, const vp_tensor* dy, const vp_conv_geom* g, float* dwpacked,
                             int n_pad, int kc, int split_k, vp_stream_t stream) {
  if (check_tensor(x, "vp_conv_wgrad(x)") || check_tensor(dy, "vp_conv_wgrad(dy)")) return -1;
  if (!g || !dwpacked) return set_error("vp_conv_wgrad: null argument");
  if (n_pad % 16 || dy->c > n_pad || kc * 32 < x->c) return set_error("vp_conv_wgrad: bad n_pad / kc");
  static thread_local WgradArgs A;
  std::memset(&A, 0, sizeof(A));
  // conv:  dW[r] += sum_o x[s*o+r-p]^T dy[o]   (x shifted, lattice = dy)
  // tconv: dW[r] += sum_o dy[s*o+r-p]^T x[o]   (dy shifted, lattice = x); as a gather this is a plain (non-transposed)
  //        strided access pattern, so the taps are those of the geometry with transposed = 0.
  vp_conv_geom gg = *g;
  gg.transposed = 0;
  const vp_tensor* shifted = g->transposed ? dy : x;
  const vp_tensor* plain = g->transposed ? x : dy;
  const int ntaps = conv_taps(&gg, A.taps);
  if (ntaps < 0) return -1;
  A.num_taps = ntaps;
  int rem = kWgTile;
  A.bw = std::min(floor_pow2(plain->w), rem); rem /= A.bw;
  A.bh = std::min(floor_pow2(plain->h), rem); rem /= A.bh;
  A.bd = std::min(floor_pow2(plain->d), rem); rem /= A.bd;
  A.bn = rem;
  A.tiles_w = ceil_div(plain->w, A.bw); A.tiles_h = ceil_div(plain->h, A.bh);
  A.tiles_d = ceil_div(plain->d, A.bd); A.tiles_n = ceil_div(plain->n, A.bn);
  const long long total = static_cast<long long>(A.tiles_w) * A.tiles_h * A.tiles_d * A.tiles_n;
  if (total * kWgTile > (1LL << 31) - 1) return set_error("vp_conv_wgrad: too many pixels");
  const int box[4] = {A.bw, A.bh, A.bd, A.bn};
  for (int qd = 0; qd < g->sd; ++qd)
    for (int qh = 0; qh < g->sh; ++qh)
      for (int qw = 0; qw < g->sw; ++qw)
        if (make_act_map(&A.amap[(qd * g->sh + qh) * g->sw + qw], shifted, qd, qh, qw, g->sd, g->sh, g->sw, box)) return -1;
  A.chunks = ceil_div(shifted->c, 32);
  A.rows_valid = shifted->c; A.cols_valid = plain->c;
  A.rows_are_ci = g->transposed ? 0 : 1;
  A.n_pad = n_pad; A.kpad = kc * 32;
  const int m_tiles = ceil_div(ntaps * A.chunks, kWgBlocks);
  // N tile (GEMM-N = plain channels): the wgmma N whose tiles cover them with the fewest padded columns (ties: the wider)
  int bn_tile = 32;
  {
    int best = 1 << 30;
    for (int bn : {136, 128, 72, 64, 32}) {
      const int cols = ceil_div(plain->c, bn) * bn;
      if (cols < best) { best = cols; bn_tile = bn; }
    }
  }
  A.n_tiles = ceil_div(plain->c, bn_tile);
  const size_t stage_bytes = static_cast<size_t>(kWgBlocks) * kWgTile * 128 + 2 * static_cast<size_t>(bn_tile) * 128;
  const size_t smem_max = 227 * 1024 - 2048;
  A.stages = static_cast<int>(std::min<size_t>(kWgMaxStages, (smem_max - 1024) / stage_bytes));
  // The pixel range is split by a rule of the layer's shape alone -- two waves of (taps x 128-row dy tiles x 128-column x
  // tiles) CTAs, at least four tiles per split -- not of the kernel's tiling, so the grouping of every dW sum (and with
  // it the fp32 result) depends only on the layer.
  if (split_k <= 0) {
    const int ctas = ntaps * ceil_div(std::min(n_pad, ceil_div(dy->c, 32) * 32), 128) * ceil_div(kc, 4);
    split_k = std::max(1, (2 * device_sms()) / ctas);
  }
  A.splits = static_cast<int>(std::max<long long>(1, std::min<long long>(split_k, std::max<long long>(1, total / 4))));

  TransposeArgs T;
  std::memset(&T, 0, sizeof(T));
  T.src = plain->ptr; T.cstride = plain->cstride;
  T.n = plain->n; T.d = plain->d; T.h = plain->h; T.w = plain->w; T.c = plain->c;
  T.bw = A.bw; T.bh = A.bh; T.bd = A.bd; T.bn = A.bn;
  T.tiles_w = A.tiles_w; T.tiles_h = A.tiles_h; T.tiles_d = A.tiles_d;
  T.p_pad = total * kWgTile;
  float* tbuf = nullptr;
  if (scratch_alloc(&tbuf, static_cast<long long>(plain->c) * T.p_pad, stream)) return -1;
  T.dst = tbuf;
  {
    EncodeTiledFn enc = get_encode();
    if (!enc) { scratch_free(tbuf, stream); return set_error("cuTensorMapEncodeTiled entry point not found"); }
    cuuint64_t dims[2] = {static_cast<cuuint64_t>(T.p_pad), static_cast<cuuint64_t>(plain->c)};
    cuuint64_t strides[1] = {static_cast<cuuint64_t>(T.p_pad) * 4};
    cuuint32_t boxd[2] = {32, static_cast<cuuint32_t>(bn_tile)};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(&A.tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, tbuf, dims, strides, boxd, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { scratch_free(tbuf, stream); return set_error("cuTensorMapEncodeTiled(transposed operand) failed with %d", static_cast<int>(r)); }
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  wgrad_transpose_kernel<<<dim3(static_cast<unsigned>(total), ceil_div(plain->c, 32)), 256, 0, st>>>(T);
  int rc = check_launch("wgrad_transpose_kernel");
  const long long plane = static_cast<long long>(ntaps) * n_pad * A.kpad;
  float* ws = nullptr;
  if (!rc && A.splits > 1) rc = scratch_zeroed(&ws, A.splits * plane, stream);
  if (!rc) {
    A.out = A.splits > 1 ? ws : dwpacked;
    A.so_n = plane;
    typedef void (*WgKernel)(const WgradArgs);
    static const WgKernel kernels[5] = {igemm_wgrad_kernel<32>, igemm_wgrad_kernel<64>, igemm_wgrad_kernel<72>,
                                        igemm_wgrad_kernel<128>, igemm_wgrad_kernel<136>};
    static bool attr_set = false;
    if (!attr_set) {
      for (WgKernel k : kernels)
        if (cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem_max)) != cudaSuccess)
          rc = set_error("cudaFuncSetAttribute(igemm_wgrad_kernel) failed: %s", cudaGetErrorString(cudaGetLastError()));
      attr_set = rc == 0;
    }
    if (!rc) {
      const WgKernel kernel = kernels[bn_tile == 32 ? 0 : bn_tile == 64 ? 1 : bn_tile == 72 ? 2 : bn_tile == 128 ? 3 : 4];
      const size_t smem = static_cast<size_t>(A.stages) * stage_bytes + 1024;
      kernel<<<dim3(m_tiles * A.n_tiles, A.splits), kWgThreads, smem, st>>>(A);
      rc = check_launch("igemm_wgrad_kernel");
    }
  }
  if (ws) {
    if (!rc) rc = reduce_parts(ws, A.splits, plane, dwpacked, stream);
    scratch_free(ws, stream);
  }
  scratch_free(tbuf, stream);
  return rc;
}
