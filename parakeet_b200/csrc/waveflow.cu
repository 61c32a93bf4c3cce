// WaveFlow inference helpers (reference parakeet/models/waveflow.py): transposed-conv upsampler, and the small
// row-wise kernels around the per-row residual net whose GEMMs run through pk_conv_gemm:
//   input_proj (1 -> C), gated activation, residual / skip update, output_proj (C -> 2) + affine inverse of the row.
#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {

// Conv2DTranspose(1, 1, (3, 2f), stride (1, f), padding (1, f/2)) + trim of the last `trim` columns + leaky_relu(slope)
// x (B, C, Tin) -> y (B, C, Tout), Tout = Tin * f - trim.   weight [3][2f] (paddle [in=1, out=1, 3, 2f]).
__global__ void wf_upsample_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                                   int c, int t_in, int f, int t_out, float slope, long long n, float* __restrict__ y) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int t = i % t_out;
  const int m = (i / t_out) % c;
  const long long b = i / (static_cast<long long>(t_out) * c);
  const int kw_total = 2 * f, pad = f / 2;
  float acc = __ldg(bias);
  // out[m, t] = sum_{kh, j} in[m + 1 - kh, j] * w[kh][t + pad - j * f]
  const int j_hi = (t + pad) / f;
  for (int j = j_hi; j >= 0 && (t + pad - j * f) < kw_total; --j) {
    if (j >= t_in) continue;
    const int kw = t + pad - j * f;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int mi = m + 1 - kh;
      if (mi >= 0 && mi < c) acc = fmaf(__ldg(x + (b * c + mi) * t_in + j), __ldg(w + kh * kw_total + kw), acc);
    }
  }
  y[i] = acc > 0.f ? acc : acc * slope;
}

// state[b,w,c] = wi[c] * x_row[b,w] + bi[c]; also written as split planes into a (B, W, ld) buffer at column col0
__global__ void wf_input_proj_kernel(const float* __restrict__ x_row, long long x_batch_stride, const float* __restrict__ wi,
                                     const float* __restrict__ bi, int w_len, int c, long long n, float* __restrict__ state,
                                     __nv_bfloat16* __restrict__ buf_hi, __nv_bfloat16* __restrict__ buf_lo, int ld, int col0) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int ch = i % c;
  const long long row = i / c;
  const long long b = row / w_len;
  const int w = row % w_len;
  const float v = fmaf(__ldg(wi + ch), __ldg(x_row + b * x_batch_stride + w), __ldg(bi + ch));
  state[i] = v;
  __nv_bfloat16 h, l;
  split_bf16(v, h, l);
  buf_hi[row * ld + col0 + ch] = h;
  buf_lo[row * ld + col0 + ch] = l;
}

// z = tanh(h[:, :c]) * sigmoid(h[:, c:])  (rows, 2c) fp32 -> split planes (rows, c)
__global__ void gate_kernel(const float* __restrict__ h, int c, long long n, __nv_bfloat16* __restrict__ z_hi,
                            __nv_bfloat16* __restrict__ z_lo) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int ch = i % c;
  const long long row = i / c;
  const float a = h[row * 2 * c + ch], g = h[row * 2 * c + c + ch];
  const float v = tanhf(a) * (1.f / (1.f + expf(-g)));
  __nv_bfloat16 hh, ll;
  split_bf16(v, hh, ll);
  z_hi[i] = hh;
  z_lo[i] = ll;
}

// o (rows, 2c): state += o[:, :c]; skip (+)= o[:, c:]; optional split copy of the new state into the next layer's buffer
__global__ void wf_layer_update_kernel(const float* __restrict__ o, int c, long long n, float* __restrict__ state,
                                       float* __restrict__ skip, int skip_init, __nv_bfloat16* __restrict__ buf_hi,
                                       __nv_bfloat16* __restrict__ buf_lo, int ld, int col0) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int ch = i % c;
  const long long row = i / c;
  const float v = state[i] + o[row * 2 * c + ch];
  state[i] = v;
  const float s = o[row * 2 * c + c + ch];
  skip[i] = skip_init ? s : skip[i] + s;
  if (buf_hi) {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    buf_hi[row * ld + col0 + ch] = h;
    buf_lo[row * ld + col0 + ch] = l;
  }
}

// (logs, b) = output_proj(skip) (C -> 2); x_next = (z_row - b) * exp(-logs); one warp per (b, w)
__global__ void __launch_bounds__(256)
wf_row_out_kernel(const float* __restrict__ skip, const float* __restrict__ wo /*[2][c]*/, const float* __restrict__ bo /*[2]*/,
                  const float* __restrict__ z_row, long long z_batch_stride, int w_len, int c, long long rows,
                  float* __restrict__ x_next, long long x_batch_stride) {
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  float s0 = 0.f, s1 = 0.f;
  for (int k = lane; k < c; k += 32) {
    const float v = skip[row * c + k];
    s0 = fmaf(__ldg(wo + k), v, s0);
    s1 = fmaf(__ldg(wo + c + k), v, s1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
  }
  if (lane == 0) {
    const long long b = row / w_len;
    const int w = row % w_len;
    const float logs = s0 + __ldg(bo), bb = s1 + __ldg(bo + 1);
    x_next[b * x_batch_stride + w] = (z_row[b * z_batch_stride + w] - bb) * expf(-logs);
  }
}

static inline int nblocks(long long n, int threads) { return static_cast<int>((n + threads - 1) / threads); }

}  // namespace pk

using namespace pk;

extern "C" int pk_waveflow_upsample(const float* x, const float* w, const float* bias, int32_t batch, int32_t c, int32_t t_in,
                                    int32_t factor, int32_t trim, float slope, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(x && w && bias && y && batch > 0 && c > 0 && t_in > 0 && factor >= 2 && (factor % 2) == 0, "bad arguments");
  const int t_out = t_in * factor - (trim ? factor : 0);
  PK_CHECK_ARG(t_out > 0, "empty output");
  const long long n = static_cast<long long>(batch) * c * t_out;
  wf_upsample_kernel<<<nblocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, w, bias, c, t_in, factor, t_out, slope, n, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_input_proj(const float* x_row, int64_t x_batch_stride, const float* w, const float* bias, int32_t batch,
                                      int32_t width, int32_t c, float* state, void* buf_hi, void* buf_lo, int32_t ld, int32_t col0,
                                      pk_stream_t stream) {
  PK_CHECK_ARG(x_row && w && bias && state && buf_hi && buf_lo && batch > 0 && width > 0 && c > 0 && ld >= col0 + c, "bad arguments");
  const long long n = static_cast<long long>(batch) * width * c;
  wf_input_proj_kernel<<<nblocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x_row, x_batch_stride, w, bias, width, c, n, state, static_cast<__nv_bfloat16*>(buf_hi), static_cast<__nv_bfloat16*>(buf_lo), ld, col0);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_gated_activation(const float* h, int64_t rows, int32_t c, void* z_hi, void* z_lo, pk_stream_t stream) {
  PK_CHECK_ARG(h && z_hi && z_lo && rows > 0 && c > 0, "bad arguments");
  const long long n = rows * c;
  gate_kernel<<<nblocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(h, c, n, static_cast<__nv_bfloat16*>(z_hi),
                                                                              static_cast<__nv_bfloat16*>(z_lo));
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_layer_update(const float* o, int64_t rows, int32_t c, float* state, float* skip, int32_t skip_init,
                                        void* buf_hi, void* buf_lo, int32_t ld, int32_t col0, pk_stream_t stream) {
  PK_CHECK_ARG(o && state && skip && rows > 0 && c > 0, "bad arguments");
  PK_CHECK_ARG((buf_hi == nullptr) == (buf_lo == nullptr), "buf_hi and buf_lo must both be set or both NULL");
  const long long n = rows * c;
  wf_layer_update_kernel<<<nblocks(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      o, c, n, state, skip, skip_init, static_cast<__nv_bfloat16*>(buf_hi), static_cast<__nv_bfloat16*>(buf_lo), ld, col0);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_row_out(const float* skip, const float* w, const float* bias, const float* z_row, int64_t z_batch_stride,
                                   int32_t batch, int32_t width, int32_t c, float* x_next, int64_t x_batch_stride, pk_stream_t stream) {
  PK_CHECK_ARG(skip && w && bias && z_row && x_next && batch > 0 && width > 0 && c > 0, "bad arguments");
  const long long rows = static_cast<long long>(batch) * width;
  wf_row_out_kernel<<<nblocks(rows * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(skip, w, bias, z_row, z_batch_stride, width,
                                                                                           c, rows, x_next, x_batch_stride);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
