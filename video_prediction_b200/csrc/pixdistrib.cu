// Pixel distributions (savp_model.py:408-410, 598-621, 648-653): the probability maps of designated pixels are moved with
// the transformation and the masks the image path computed for the same time step, then renormalised per plane.
//
// One thread-block cluster of kPixClusterCtas CTAs owns one (row n, channel d) plane.  Each CTA composites a contiguous slice of
// the plane's positions, writes the unnormalised values and sums them in a fixed order (thread, warp tree, warps in order);
// the CTAs then read the cluster's partials through distributed shared memory in rank order, so every CTA holds the same
// plane sum and two runs are bit-identical.  Each thread finally divides the values it wrote itself.
#include <cooperative_groups.h>

#include "common.h"

namespace cg = cooperative_groups;

namespace vp {

constexpr int kPixClusterCtas = 8;
constexpr int kPixThreads = 256;

__device__ __forceinline__ int pd_reflect(int i, int n) {  // SYMMETRIC padding (edge pixel repeated), as cdna_apply_kernel
  if (i < 0) i = -i - 1;
  if (i >= n) i = 2 * n - 1 - i;
  return i;
}

// The slots of one step: transform k < NK of history map k / (NK / NF) (map NF - 1 = this step's selected map p, maps
// f < NF - 1 = tab.ptr[f], earlier steps' selected maps), then background b < NBG = tab.ptr[VP_SLOT_MAX_FRAMES + b] or, when
// that pointer is NULL, p itself, then p again in the scratch slot when SCRATCH.  kMaxSlots bounds NK + NBG + SCRATCH; the
// 8-slot instantiation is the default model's.
template <int kMaxSlots>
__global__ void __cluster_dims__(kPixClusterCtas, 1, 1) __launch_bounds__(kPixThreads)
pix_distrib_fwd_kernel(const __grid_constant__ VpSlotTable tab, const int32_t* __restrict__ sel, const float* __restrict__ gt, int gts,
                       const float* __restrict__ prev, const float* __restrict__ kern, const float* __restrict__ flows, int fs,
                       const float* __restrict__ masks, int ms, float* __restrict__ gen, int gs, float* __restrict__ tr, int trs,
                       int tr_slot, float* __restrict__ cur_out, int H, int W, int KH, int KW, int NK, int NF, int NBG, int SCRATCH) {
  extern __shared__ float sk[];  // [KH*KW*NK] CDNA kernels of this row
  __shared__ float s_warp[kPixThreads / 32];
  __shared__ float s_part;
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = static_cast<int>(cluster.block_rank());
  const int n = blockIdx.y, d = blockIdx.z;
  const int P = H * W;
  const long long row = static_cast<long long>(n) * P;
  if (kern) {
    for (int i = threadIdx.x; i < KH * KW * NK; i += blockDim.x) sk[i] = kern[static_cast<long long>(n) * KH * KW * NK + i];
    __syncthreads();
  }
  // select (savp_model.py:409): ground truth where sel[n], else the previous generated map; no previous map at t = 0
  const bool use_gt = prev == nullptr || sel[n] != 0;
  const float* src = use_gt ? gt + row * gts + d : prev + row * gs + d;
  const int ss = use_gt ? gts : gs;
  const int G = NK ? NK / NF : 1;
  const int nslots = NK + NBG + SCRATCH;
  const int ppc = (P + kPixClusterCtas - 1) / kPixClusterCtas;
  const int p_end = min(P, (rank + 1) * ppc);
  float acc = 0.f;
  for (int p = rank * ppc + threadIdx.x; p < p_end; p += blockDim.x) {
    const int y = p / W, x = p % W;
    float slot[kMaxSlots];
    if (kern) {  // apply_cdna_kernels (savp_model.py:893-923), group f on history map f (apply_kernels, :939-943)
      for (int k = 0; k < NK; ++k) slot[k] = 0.f;
      const int ph = (KH - 1) / 2, pw = (KW - 1) / 2;
      for (int i = 0; i < KH; ++i) {
        const int yy = pd_reflect(y + i - ph, H);
        for (int j = 0; j < KW; ++j) {
          const long long q = yy * W + pd_reflect(x + j - pw, W);
          const float* kk = sk + (i * KW + j) * NK;
          for (int f = 0; f < NF; ++f) {
            const float v = f == NF - 1 ? src[q * ss] : tab.ptr[f][(row + q) * gts + d];
            for (int k = f * G; k < (f + 1) * G; ++k) slot[k] += v * kk[k];
          }
        }
      }
    } else {  // apply_flows (savp_model.py:955-965), flow_ops.image_warp
      const float* fp = flows + (row + p) * fs;
      for (int k = 0; k < NK; ++k) {
        const int f = k / G;
        const float* m = f == NF - 1 ? src : tab.ptr[f] + row * gts + d;
        const int mst = f == NF - 1 ? ss : gts;
        const float fx = fp[k], fy = fp[NK + k];
        const float flx = floorf(fx), fly = floorf(fy);
        const float xw = fx - flx, yw = fy - fly;
        const int x0 = min(max(x + static_cast<int>(flx), 0), W - 1), x1 = min(max(x + static_cast<int>(flx) + 1, 0), W - 1);
        const int y0 = min(max(y + static_cast<int>(fly), 0), H - 1), y1 = min(max(y + static_cast<int>(fly) + 1, 0), H - 1);
        const float Ia = m[static_cast<long long>(y0 * W + x0) * mst], Ib = m[static_cast<long long>(y1 * W + x0) * mst];
        const float Ic = m[static_cast<long long>(y0 * W + x1) * mst], Id = m[static_cast<long long>(y1 * W + x1) * mst];
        slot[k] = (1.f - xw) * (1.f - yw) * Ia + (1.f - xw) * yw * Ib + xw * (1.f - yw) * Ic + xw * yw * Id;
      }
    }
    // background slots (:606-621): ground-truth maps, or the selected map itself; the scratch slot takes the map too
    const float pv = src[static_cast<long long>(p) * ss];
    if (cur_out) cur_out[(row + p) * gts + d] = pv;
    for (int b = 0; b < NBG; ++b) {
      const float* bp = tab.ptr[VP_SLOT_MAX_FRAMES + b];
      slot[NK + b] = bp ? bp[(row + p) * gts + d] : pv;
    }
    if (SCRATCH) slot[NK + NBG] = pv;
    // composite (:648-652) with the image path's softmax masks
    const float* mp = masks + (row + p) * ms;
    float* tp = tr + (row + p) * trs + d;
    float g = 0.f;
    for (int l = 0; l < nslots; ++l) {
      tp[static_cast<long long>(l) * tr_slot] = slot[l];
      g += slot[l] * mp[l];
    }
    gen[(row + p) * gs + d] = g;
    acc += g;
  }
  // plane sum in a fixed order: warp tree, warps in order, cluster ranks in order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < kPixThreads / 32; ++i) s += s_warp[i];
    s_part = s;
  }
  cluster.sync();
  float total = 0.f;
  for (int r = 0; r < kPixClusterCtas; ++r) total += *cluster.map_shared_rank(&s_part, r);
  // normalise (:653): the same division as the reference, no epsilon; each thread rescales the values it wrote
  for (int p = rank * ppc + threadIdx.x; p < p_end; p += blockDim.x) {
    float* gp = gen + (row + p) * gs + d;
    *gp = *gp / total;
  }
  cluster.sync();  // keep s_part alive until every CTA of the cluster has read it
}

}  // namespace vp

extern "C" int vp_pix_slots_fwd(const int32_t* sel, const float* pix_gt, int pix_cstride, const float* gen_prev,
                                const float* const* frames, int nframes, const float* kernels, const float* flows, int flows_cstride,
                                int nk, const float* const* backgrounds, int nbg, int scratch, const float* masks, int masks_cstride,
                                float* gen, int gen_cstride, float* transformed, int transformed_cstride, int slot_stride,
                                float* cur_out, int n, int h, int w, int d, int kh, int kw, vp_stream_t stream) {
  using namespace vp;
  const int nslots = nk + nbg + (scratch ? 1 : 0);
  if (nk < 0 || nk > VP_SLOT_MAX_TRANSFORMS || nbg < 0 || nslots < 1 || nslots > VP_SLOT_MAX_LAYERS)
    return set_error("vp_pix_slots_fwd: bad nk / backgrounds (nk <= %d, 1 <= slots <= %d)", VP_SLOT_MAX_TRANSFORMS, VP_SLOT_MAX_LAYERS);
  if (nk && (nframes < 1 || nframes > VP_SLOT_MAX_FRAMES || nk % nframes))
    return set_error("vp_pix_slots_fwd: the %d transforms must split evenly over 1..%d maps, got %d", nk, VP_SLOT_MAX_FRAMES, nframes);
  if (!pix_gt || !masks || !gen || !transformed) return set_error("vp_pix_slots_fwd: null pointer");
  if (nk && (kernels == nullptr) == (flows == nullptr)) return set_error("vp_pix_slots_fwd: pass exactly one of kernels and flows");
  if (!nk && (kernels || flows)) return set_error("vp_pix_slots_fwd: kernels / flows without transforms");
  if (gen_prev && !sel) return set_error("vp_pix_slots_fwd: gen_prev needs sel");
  if (masks_cstride < nslots) return set_error("vp_pix_slots_fwd: masks_cstride < %d slots", nslots);
  if (flows && flows_cstride < 2 * nk) return set_error("vp_pix_slots_fwd: flows_cstride < 2 * nk");
  if (kernels && (kh < 1 || kw < 1 || kh / 2 > h || kw / 2 > w)) return set_error("vp_pix_slots_fwd: kernel larger than the image");
  if (n < 1 || h < 1 || w < 1 || d < 1 || n > 65535 || d > 65535) return set_error("vp_pix_slots_fwd: bad n / h / w / d");
  if (pix_cstride % 4 || gen_cstride % 4 || transformed_cstride % 4 || slot_stride % 4)
    return set_error("vp_pix_slots_fwd: channel strides must be multiples of 4");
  if (pix_cstride < d || gen_cstride < d || slot_stride < d || static_cast<long long>(nslots - 1) * slot_stride + d > transformed_cstride)
    return set_error("vp_pix_slots_fwd: channel strides too small for d");
  if ((nk && nframes > 1 && !frames) || (nbg && !backgrounds)) return set_error("vp_pix_slots_fwd: null pointer");
  VpSlotTable tab{};
  for (int f = 0; nk && f < nframes - 1; ++f) {
    if (!frames[f]) return set_error("vp_pix_slots_fwd: null map %d", f);
    tab.ptr[f] = frames[f];
  }
  for (int b = 0; b < nbg; ++b) tab.ptr[VP_SLOT_MAX_FRAMES + b] = backgrounds[b];   // NULL: the step's selected map
  const int nf = nk ? nframes : 1;
  const dim3 grid(kPixClusterCtas, n, d);
  const size_t smem = kernels ? static_cast<size_t>(kh) * kw * nk * sizeof(float) : 0;
  if (nslots <= 8)
    pix_distrib_fwd_kernel<8><<<grid, kPixThreads, smem, as_stream(stream)>>>(tab, sel, pix_gt, pix_cstride, gen_prev, kernels, flows,
                                                                             flows_cstride, masks, masks_cstride, gen, gen_cstride,
                                                                             transformed, transformed_cstride, slot_stride, cur_out, h, w,
                                                                             kh, kw, nk, nf, nbg, scratch ? 1 : 0);
  else
    pix_distrib_fwd_kernel<VP_SLOT_MAX_LAYERS><<<grid, kPixThreads, smem, as_stream(stream)>>>(
        tab, sel, pix_gt, pix_cstride, gen_prev, kernels, flows, flows_cstride, masks, masks_cstride, gen, gen_cstride, transformed,
        transformed_cstride, slot_stride, cur_out, h, w, kh, kw, nk, nf, nbg, scratch ? 1 : 0);
  return check_launch("pix_distrib_fwd_kernel");
}

extern "C" int vp_pix_distrib_fwd(const int32_t* sel, const float* pix_gt, const float* pix_first, int pix_cstride,
                                  const float* gen_prev, const float* kernels, const float* flows, int flows_cstride,
                                  const float* masks, int masks_cstride, float* gen, int gen_cstride, float* transformed,
                                  int transformed_cstride, int slot_stride, int n, int h, int w, int d, int kh, int kw, int nk,
                                  vp_stream_t stream) {
  using namespace vp;
  if (!pix_gt || !pix_first || !masks || !gen || !transformed) return set_error("vp_pix_distrib_fwd: null pointer");
  if ((kernels == nullptr) == (flows == nullptr)) return set_error("vp_pix_distrib_fwd: pass exactly one of kernels and flows");
  if (nk < 1 || nk + 3 > 8 || masks_cstride < nk + 3) return set_error("vp_pix_distrib_fwd: bad nk / masks_cstride");
  const float* bg[2] = {nullptr, pix_first};     // the selected map, the first ground-truth map; then the scratch slot
  return vp_pix_slots_fwd(sel, pix_gt, pix_cstride, gen_prev, nullptr, 1, kernels, flows, flows_cstride, nk, bg, 2, 1, masks,
                          masks_cstride, gen, gen_cstride, transformed, transformed_cstride, slot_stride, nullptr, n, h, w, d, kh, kw,
                          stream);
}
