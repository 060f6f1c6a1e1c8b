// Robot-state recurrence of the action-conditioned SAVP cell (savp_model.py:411-412, 655-658): for every unroll row the state
// the cell is conditioned on is the ground truth or the cell's own previous prediction, and the next state is a dense layer
// of [actions | state].  The recurrence reads no image, so the whole unroll runs as one launch before the convolutions.
//
// One thread owns one row for all steps.  Each output is bias + sum_i x_i * K[i][j], added in increasing i, so two runs
// give identical bits.
#include "common.h"

namespace vp {

constexpr int kStateThreads = 128;
constexpr int kStateMaxWeights = 12 * 1024;  // (a + sd) * sd + sd floats staged in shared memory (48 KB)

__global__ void __launch_bounds__(kStateThreads)
state_pred_fwd_kernel(const int32_t* __restrict__ sel, const float* __restrict__ states, int states_stride,
                      const float* __restrict__ kernel, const float* __restrict__ bias, float* __restrict__ zvec, int zs,
                      float* __restrict__ gen, int S, int N, int A, int SD) {
  extern __shared__ float sw[];  // [(A + SD) * SD] kernel, then [SD] bias
  const int nw = (A + SD) * SD;
  for (int i = threadIdx.x; i < nw + SD; i += blockDim.x) sw[i] = i < nw ? kernel[i] : bias[i - nw];
  __syncthreads();
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  for (int t = 0; t < S; ++t) {
    const long long r = static_cast<long long>(t) * N + n;
    float* z = zvec + r * zs;
    // state_t = sel ? ground truth : previous prediction (:411-412); before the first step the prediction is the zero state
    const bool use_gt = sel[r] != 0;
    for (int j = 0; j < SD; ++j)
      z[A + j] = use_gt ? states[r * states_stride + j] : (t ? gen[(r - N) * SD + j] : 0.f);
    // gen_state_t = [actions_t | state_t] @ K + b (:655-658); the actions are already in z[0, A)
    for (int j = 0; j < SD; ++j) {
      float acc = 0.f;
      for (int i = 0; i < A + SD; ++i) acc = fmaf(z[i], sw[i * SD + j], acc);
      gen[r * SD + j] = acc + sw[nw + j];
    }
  }
}

}  // namespace vp

extern "C" int vp_state_pred_fwd(const int32_t* sel, const float* states, int states_stride, const float* kernel,
                                 const float* bias, float* zvec, int zvec_stride, float* gen_states, int s, int n, int a,
                                 int sd, vp_stream_t stream) {
  using namespace vp;
  if (!sel || !states || !kernel || !bias || !zvec || !gen_states) return set_error("vp_state_pred_fwd: null pointer");
  if (s < 1 || n < 1 || a < 0 || sd < 1) return set_error("vp_state_pred_fwd: bad s / n / a / sd");
  if (states_stride < sd) return set_error("vp_state_pred_fwd: states_stride < sd");
  if (zvec_stride < a + sd) return set_error("vp_state_pred_fwd: zvec_stride < a + sd");
  if (static_cast<long long>(a + sd + 1) * sd > kStateMaxWeights) return set_error("vp_state_pred_fwd: dense layer too large");
  const size_t smem = static_cast<size_t>(a + sd + 1) * sd * sizeof(float);
  state_pred_fwd_kernel<<<grid_for(n, kStateThreads), kStateThreads, smem, as_stream(stream)>>>(
      sel, states, states_stride, kernel, bias, zvec, zvec_stride, gen_states, s, n, a, sd);
  return check_launch("state_pred_fwd_kernel");
}
