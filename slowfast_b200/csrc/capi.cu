// Small C-ABI entry points that do not belong to a kernel file.
#include "../../include/slowfast_b200.h"
#include "runtime.h"

#ifndef SFB_BUILD_ARCH
#define SFB_BUILD_ARCH "unknown"
#endif

extern "C" const char* sfb_last_error(void) { return sfb::last_error(); }
extern "C" int sfb_abi_version(void) { return 1; }
extern "C" const char* sfb_build_arch(void) { return SFB_BUILD_ARCH; }

// Zero a [rows, c] fp32 view with row pitch `pitch` (elements) on the caller's stream.
extern "C" int sfb_zero_f32_2d(float* ptr, int64_t rows, int64_t c, int64_t pitch, void* stream) {
  if (rows <= 0 || c <= 0) return 0;
  cudaError_t e = (pitch == c)
                      ? cudaMemsetAsync(ptr, 0, size_t(rows) * size_t(c) * 4, (cudaStream_t)stream)
                      : cudaMemset2DAsync(ptr, size_t(pitch) * 4, 0, size_t(c) * 4, size_t(rows), (cudaStream_t)stream);
  if (e != cudaSuccess) {
    sfb::set_error("sfb_zero_f32_2d failed: %s", cudaGetErrorString(e));
    return -20;
  }
  return 0;
}
