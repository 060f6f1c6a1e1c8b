// Error reporting + version for the C ABI; scratch memory and the order-fixed reduction of per-block partial sums.
#include "common.h"

namespace vp {
static thread_local char g_err[512] = "";
int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return -1;
}
static long long g_launches = 0;
void count_launch(int n) { g_launches += n; }

int scratch_alloc(float** p, long long count, vp_stream_t stream) {
  *p = nullptr;
  if (cudaMallocAsync(reinterpret_cast<void**>(p), static_cast<size_t>(count) * sizeof(float), as_stream(stream)) != cudaSuccess)
    return set_error("cudaMallocAsync of %lld floats failed: %s", count, cudaGetErrorString(cudaGetLastError()));
  return 0;
}
int scratch_zeroed(float** p, long long count, vp_stream_t stream) {
  if (scratch_alloc(p, count, stream)) return -1;
  if (cudaMemsetAsync(*p, 0, static_cast<size_t>(count) * sizeof(float), as_stream(stream)) != cudaSuccess)
    return set_error("cudaMemsetAsync of scratch failed: %s", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
void scratch_free(float* p, vp_stream_t stream) {
  if (p) cudaFreeAsync(p, as_stream(stream));
}

__global__ void reduce_parts_kernel(const float* __restrict__ ws, int parts, long long rows, long long cols, float* __restrict__ out,
                                    long long out_stride) {
  const long long n = rows * cols;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float s = 0.f;
    for (int q = 0; q < parts; ++q) s += ws[q * n + i];
    const long long r = i / cols;
    out[r * out_stride + (i - r * cols)] += s;
  }
}
int reduce_parts_strided(const float* ws, int parts, long long rows, long long cols, float* out, long long out_stride, vp_stream_t stream) {
  if (rows * cols <= 0) return 0;
  const int grid = static_cast<int>(std::min<long long>((rows * cols + 255) / 256, 8LL * device_sms()));
  reduce_parts_kernel<<<grid, 256, 0, as_stream(stream)>>>(ws, parts, rows, cols, out, out_stride);
  return check_launch("reduce_parts_kernel");
}
int reduce_parts(const float* ws, int parts, long long n, float* out, vp_stream_t stream) {
  return reduce_parts_strided(ws, parts, 1, n, out, n, stream);
}
}  // namespace vp

extern "C" long long vp_launch_count(void) { return vp::g_launches; }
extern "C" const char* vp_last_error(void) { return vp::g_err; }
extern "C" int vp_version(void) { return 100; }
