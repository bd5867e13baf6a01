// Library-level state: error string, launch counter, small utility kernels.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace sb {
static thread_local char g_err[512] = "";
long long g_launch_count = 0;
bool pdl_enabled() {
  static int v = -1;
  // on unless SB_PDL=0 (read once per process)
  if (v < 0) { const char* e = getenv("SB_PDL"); v = (e == nullptr || atoi(e) != 0) ? 1 : 0; }
  return v != 0;
}
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

__global__ void cast_f32_f16_kernel(const float* __restrict__ s, elem_t* __restrict__ d, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) d[i] = __float2half_rn(s[i]);
}
}  // namespace sb

extern "C" const char* sb_last_error(void) { return sb::g_err; }
extern "C" int sb_version(void) { return 1; }
extern "C" int64_t sb_launch_count(void) { return sb::g_launch_count; }
extern "C" int sb_pdl_enabled(void) { return sb::pdl_enabled() ? 1 : 0; }

extern "C" int sb_cast_f32_to_f16(const float* src, void* dst, int64_t n, sb_stream_t stream) {
  SB_REQUIRE(src && dst && n >= 0, SB_EINVAL, "sb_cast_f32_to_f16: bad args");
  if (n == 0) return SB_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > (long long)sb::sm_count() * 16) blocks = (long long)sb::sm_count() * 16;  // grid-stride loop
  sb::cast_f32_f16_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(src, (sb::elem_t*)dst, n);
  SB_LAUNCH_OK();
  return SB_OK;
}

extern "C" int sb_fill_zero(void* dst, int64_t bytes, sb_stream_t stream) {
  SB_REQUIRE(dst && bytes >= 0, SB_EINVAL, "sb_fill_zero: bad args");
  SB_CUDA_OK(cudaMemsetAsync(dst, 0, (size_t)bytes, (cudaStream_t)stream));
  return SB_OK;
}
