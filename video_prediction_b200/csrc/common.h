// Shared host-side helpers for libvp_b200 (error reporting, launch checks).
#pragma once
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cuda_runtime.h>

#include "vp_b200.h"

namespace vp {
int set_error(const char* fmt, ...);
void count_launch(int n);
inline int check_launch(const char* what) {
  count_launch(1);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error("%s launch failed: %s", what, cudaGetErrorString(e));
  return 0;
}
inline cudaStream_t as_stream(vp_stream_t s) { return static_cast<cudaStream_t>(s); }
// Sums that many blocks contribute to are made independent of block scheduling: every block writes its partial into its own
// row of a stream-ordered scratch buffer (cudaMallocAsync, also valid inside a CUDA-graph capture) and reduce_parts adds
// the rows in a fixed order: out[i] += sum_{q < parts} ws[q * n + i].  Float atomics would make two identical runs differ.
int scratch_alloc(float** p, long long count, vp_stream_t stream);
int scratch_zeroed(float** p, long long count, vp_stream_t stream);
void scratch_free(float* p, vp_stream_t stream);
int reduce_parts(const float* ws, int parts, long long n, float* out, vp_stream_t stream);
// The same for a [rows][cols] result stored with a row stride: out[r * out_stride + c] += sum_q ws[(q * rows + r) * cols + c].
int reduce_parts_strided(const float* ws, int parts, long long rows, long long cols, float* out, long long out_stride, vp_stream_t stream);
// slab-mapped plane kernels (planes.cu): return 0 = launched, 1 = shape outside the fast path (caller falls back), -1 = error
int slab_inorm_act(const float* x, int xs, float* y, int ys, int n, int P, int C, const float* gamma, const float* beta, float eps, int act,
                   float alpha, float* stats, vp_stream_t stream);
int slab_inorm_act_bwd(const float* x, int xs, const float* const* dy, const int* dy_cs, int num_dy, float* dx, int dxs, int n, int P, int C,
                       const float* gamma, const float* beta, const float* stats, int act, float alpha, float* dgamma, float* dbeta,
                       vp_stream_t stream);
int slab_gates_fwd(const float* pre, int n, int P, int F, const float* c_prev, const float* g1, const float* b1, const float* g2,
                   const float* b2, float forget_bias, float eps, float* c_new, float* const* h_dst, const int* h_cs, int num_h, float* stats1,
                   float* stats2, vp_stream_t stream);
int slab_gates_bwd(const float* pre, int n, int P, int F, const float* c_prev, const float* g1, const float* b1, const float* g2,
                   const float* b2, const float* stats1, const float* stats2, float forget_bias, const float* const* dh, const int* dh_cs,
                   int num_dh, const float* dc_next, float* dpre, float* dc_prev, float* dg1, float* db1, float* dg2, float* db2,
                   vp_stream_t stream);
inline int grid_for(long long n, int block) { return static_cast<int>((n + block - 1) / block); }
// Streaming multiprocessors of the current device (sizes persistent and split grids).
inline int device_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) {
    cudaGetLastError();
    n = 1;
  }
  return n;
}
}  // namespace vp
