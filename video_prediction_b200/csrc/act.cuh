// The fused activations (VP_ACT_*) of the engine epilogue, the norm kernels and vp_act_bwd, and their derivatives.
//
// Every kernel that applies one is instantiated twice, on kElu: launch sites pick the kElu = true instantiation only
// when an activation of the call is VP_ACT_ELU.  With kElu = false the ELU case is not compiled at all, so the relu /
// lrelu / sigmoid / tanh kernels keep exactly the code they have without it; an ELU case in their unrolled per-element
// code grows it by up to 2x.
#pragma once
#include "vp_b200.h"

namespace vp {

template <bool kElu>
__device__ __forceinline__ float act_fwd(float v, int act, float alpha) {
  if (kElu && act == VP_ACT_ELU) return v > 0.f ? v : expm1f(v);       // tf.nn.elu
  switch (act) {
    case VP_ACT_RELU: return fmaxf(v, 0.f);
    case VP_ACT_LRELU: return fmaxf(alpha * v, v);
    case VP_ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
    case VP_ACT_TANH: return tanhf(v);
    default: return v;
  }
}

// d * act'(x), taken from the activation's OUTPUT y = act(x).  relu / lrelu / elu: y > 0 exactly where x > 0 (alpha >= 0);
// elu below 0: exp(x) = y + 1.
template <bool kElu>
__device__ __forceinline__ float act_grad_mul(float d, float y, int act, float alpha) {
  if (kElu && act == VP_ACT_ELU) return y > 0.f ? d : d * (y + 1.f);
  if (act == VP_ACT_LRELU) d = y > 0.f ? d : alpha * d;
  else if (act == VP_ACT_RELU) d = y > 0.f ? d : 0.f;
  else if (act == VP_ACT_SIGMOID) d *= y * (1.f - y);
  else if (act == VP_ACT_TANH) d *= (1.f - y * y);
  return d;
}

// act'(x) from the pre-activation x, for the norm backward kernels, which keep x: their activations are none, relu, lrelu
// and elu.  ELU goes through its output, as act_grad_mul takes it.
template <bool kElu>
__device__ __forceinline__ float act_grad_pre(float x, int act, float alpha) {
  if (kElu && act == VP_ACT_ELU) return act_grad_mul<true>(1.f, act_fwd<true>(x, act, alpha), act, alpha);
  switch (act) {
    case VP_ACT_RELU: return x > 0.f ? 1.f : 0.f;
    case VP_ACT_LRELU: return x > 0.f ? 1.f : alpha;
    default: return 1.f;
  }
}

}  // namespace vp
