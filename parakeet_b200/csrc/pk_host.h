// Host-side helpers shared by the C-ABI translation units: error reporting, TMA descriptor encoding.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/parakeet_b200.h"

namespace pk {

// thread-local last-error string (pk_last_error)
void set_error(const char* fmt, ...);
int fail(int code, const char* fmt, ...);

#define PK_CHECK_ARG(cond, ...)                                   \
  do {                                                            \
    if (!(cond)) return ::pk::fail(PK_ERR_INVALID_ARG, __VA_ARGS__); \
  } while (0)

#define PK_CHECK_CUDA(expr)                                                                          \
  do {                                                                                               \
    cudaError_t _e = (expr);                                                                         \
    if (_e != cudaSuccess) return ::pk::fail(PK_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(_e)); \
  } while (0)

// Encode a 3-D bf16 tiled tensor map (innermost dim = channels) with 128B swizzle and zero OOB fill.
//   dims   = {cols, rows, batches}; strides in ELEMENTS for rows / batches; box = {64, box_rows, 1}.
int encode_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t batches,
                        uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows);

// Both planes of a split-bf16 tensor as ONE 4-D map: dims {cols, rows, batches, 2}, box {box_cols, box_rows, 1, 2} - one TMA
// load then delivers [hi tile | lo tile] back to back.  Requires lo = hi + a positive 16-byte multiple (one allocation).
// box_cols 64 / 16 selects a 128 / 32-byte swizzle (the box row is exactly one swizzle atom wide).
int encode_tmap_bf16_planes(CUtensorMap* out, const void* hi, const void* lo, uint64_t cols, uint64_t rows, uint64_t batches,
                            uint64_t row_stride_elems, uint64_t batch_stride_elems, uint32_t box_rows, uint32_t box_cols = 64);

// A 3-D fp32 tiled tensor map of 128-byte lines (32 floats, one 128B-swizzle atom) with zero OOB fill:
//   dims = {32, rows, batches}; batch stride in ELEMENTS (0: 32 * rows); box = {32, box_rows, 1}.  A tensor whose rows are
//   wider than 32 floats is described with rows = its rows x (row width / 32).
int encode_tmap_f32_3d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t batches, uint64_t batch_stride_elems,
                       uint32_t box_rows);

int sm_count();
void count_launch(int n = 1);

}  // namespace pk
