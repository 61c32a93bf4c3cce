// Host-side helpers shared by the C-ABI translation units: error reporting, TMA descriptor encoding, launch setup.
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

// Grid size for n items, one thread per item: ceil(n / threads) blocks.
inline int nblk(long long n, int threads) { return static_cast<int>((n + threads - 1) / threads); }
// The same capped at 2^20 blocks.  Only for grid-stride kernels (PK_GRID_STRIDE), which cover any n with a capped grid.
inline int grid_stride_blocks(long long n, int threads) {
  const long long b = (n + threads - 1) / threads;
  return static_cast<int>(b < (1 << 20) ? b : (1 << 20));
}

// The stream argument of a C entry point, and its tail after the last of `n` launches.
#define PK_STREAM static_cast<cudaStream_t>(stream)
#define PK_LAUNCH_DONE(n)            \
  PK_CHECK_CUDA(cudaGetLastError()); \
  ::pk::count_launch(n);             \
  return PK_OK

// Readies a kernel for a launch with `threads` threads and `smem` bytes of dynamic shared memory on the current device: raises
// its dynamic shared-memory limit to cover smem (a CUDA call only the first time the kernel needs more on that device).  With
// resident_ctas, also returns how many such CTAs the device holds at once (occupancy x SMs, queried once per kernel, device and
// smem).  Thread-safe; a failed call is not remembered, so the next one tries again.
int prepare_kernel(const void* kernel, int threads, size_t smem, int* resident_ctas = nullptr);
template <class... Args>
int prepare_kernel(void (*kernel)(Args...), int threads, size_t smem, int* resident_ctas = nullptr) {
  return prepare_kernel(reinterpret_cast<const void*>(kernel), threads, smem, resident_ctas);
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// The PWG / WaveFlow gated activation tanh(a + b_a) * sigmoid(g + b_g) runs on ex2: tanh from exp2(kGateKa * a + gate_c[i]),
// sigmoid from exp2(kGateKg * g + gate_c[64 + i]).  fold_gate_bias fills gate_c from the gate biases bias1 (per 64-channel
// block: 64 a biases, then 64 g biases) for `channels` residual channels.
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kGateKa = -2.f * kLog2e, kGateKg = -kLog2e;
inline void fold_gate_bias(float* gate_c, const float* bias1, int channels) {
  for (int blk = 0; blk < channels / 64; ++blk) {
    for (int i = 0; i < 64; ++i) {
      gate_c[128 * blk + i] = -2.f * kLog2e * bias1[128 * blk + i];
      gate_c[128 * blk + 64 + i] = -kLog2e * bias1[128 * blk + 64 + i];
    }
  }
}

}  // namespace pk
