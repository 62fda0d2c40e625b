// Host-side runtime shared by every kernel file: error reporting, device limits, launch checks, grid clamps and the
// construction of TMA tensor maps (tiled and im2col) through driver entry points resolved at run time, so the library
// links without libcuda.
#pragma once
#include <cstdint>
#include <cuda.h>

namespace sfb {

// Error plumbing shared by the C-ABI: every entry point returns 0 on success or a negative code and leaves a
// message retrievable with sfb_last_error().
void set_error(const char* fmt, ...);
const char* last_error();

// The SM count the fixed launch geometry was tuned and validated with: 148, a B200's count, kept from the port.  It
// caps the grids of the grid-strided kernels, sets the X3D channelwise tile heuristics and fixes the deterministic slab
// counts (sfb_flat_sumsq_blocks, sfb_rowslab_blocks, sfb_dwpool_wgrad_blocks, dw2_block_split), so it also fixes the
// summation order of those reductions.  It is not the device's SM count (132 on an H100): changing it is a performance
// change that needs measuring on the GPU.
constexpr int kGridSms = 148;

// Multiprocessor count and opt-in shared memory per block of the current device, queried once per process.  Either
// output may be null.  Returns 0, or -1 with the error set and the outputs untouched when there is no device.
int device_limits(int* sms, int* smem_optin);

// Status of the launch just issued on this thread: 0, or -20 with the error "<what> launch failed: <cuda error>",
// followed by " (<context>)" when ctx_fmt is given (a printf format of the launch's geometry).
int launch_status(const char* what, const char* ctx_fmt = nullptr, ...) __attribute__((format(printf, 2, 3)));

// ceil(items / block) blocks, clamped to [1, cap].
inline int capped_grid(int64_t items, int block, int64_t cap) {
  const int64_t want = (items + block - 1) / block;
  return int(want < 1 ? 1 : (want > cap ? cap : want));
}

enum SwizzleBytes { SWZ_NONE = 0, SWZ_32 = 32, SWZ_64 = 64, SWZ_128 = 128 };

// Tiled bf16 map of `rank` dimensions (innermost first) with byte strides of the outer rank - 1 dimensions; element
// strides 1, no interleave, 128-byte L2 promotion, no NaN fill.  `what` names the map in the error message.
int encode_tiled_bf16(CUtensorMap* out, uint32_t rank, const void* base, const cuuint64_t* dims,
                      const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle, const char* what);

// 2-D row-major bf16 matrix [rows, cols] with row pitch `pitch_elems`; box = [box_rows, box_cols].
int make_tmap_2d_bf16(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols, uint64_t pitch_elems,
                      uint32_t box_rows, uint32_t box_cols, SwizzleBytes swz);

// 3-D map over bf16 [batch][rows][cols] (cols contiguous, row pitch ld, batch stride bs), box = [1][box_rows][64],
// 128-byte swizzle.
int make_tmap_3d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t batch, uint64_t ld,
                 uint64_t bs, uint32_t box_rows);

// W-shift folded stem input X'[n, t, h, w', 8] bf16, box = [1,1,1,pix,8], no swizzle.
int make_tmap_fold(CUtensorMap* out, const void* base, int n, int t, int h, int w2, uint32_t pix);

// Stem output gradient dY [rows, OW, cout] bf16 (cout contiguous), box = [1][64 ow][64 co], 128-byte swizzle.
int make_tmap_dy3(CUtensorMap* out, const void* base, int64_t rows, int ow, int cout);

// 5-D im2col map over a channels-last bf16 activation [N, D, H, W, C] (C contiguous, channel pitch
// `c_pitch` >= C elements).  lower/upper corners and traversal strides are given in (W, H, D) order, exactly as
// the driver consumes them.
int make_tmap_im2col_bf16(CUtensorMap* out, const void* base, int n, int d, int h, int w, int c, int64_t c_pitch,
                          const int lower_whd[3], const int upper_whd[3], const int stride_whd[3],
                          uint32_t channels_per_pixel, uint32_t pixels_per_column, SwizzleBytes swz);

}  // namespace sfb
