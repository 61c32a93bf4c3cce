// WaveFlow inference helpers (reference parakeet/models/waveflow.py): transposed-conv upsampler, and the small
// row-wise kernels around the per-row residual net whose GEMMs run through pk_conv_gemm:
//   input_proj (1 -> C), output_proj (C -> 2) + affine inverse of the row;
// and of the density direction: the tail of Flow.forward (output_proj, transform, log-det, permutation, next input_proj)
// and WaveFlowLoss.
#include <algorithm>
#include <mutex>

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

// ---------------------------------------------------------------- density direction (Flow.forward tail, WaveFlowLoss)
constexpr int kFwdMaxGroup = 16;
constexpr int kFwdTailThreads = 256;
constexpr int kFwdTailMaxBlocks = 1024;          // = the partials scratch of pk_waveflow_forward_tail_args

template <int C>
struct FwdTailArgs {
  int w, n_group;
  long long positions;                           // batch * n_group * w: one warp each
  int inv[kFwdMaxGroup];                         // x_next height of z height j (the inverse permutation)
  float po_w[2 * C], po_b[2];                    // output_proj (C -> logs, b)
  float in_w[C], in_b[C];                        // next flow's input_proj (1 -> C)
  const float* skip;
  const float* x;
  float* x_next;
  __nv_bfloat16* next_hi;
  __nv_bfloat16* next_lo;
  float* log_det;
  float* partials;
  unsigned* counter;
};

// One warp per (utterance, height j, column): output_proj over the C skip channels (lane owns channels 2 lane + 64 k + {0, 1}),
// the affine transform, the permuted store and the next input_proj.  Every block reduces the logs of its warps in a fixed
// order into partials[block]; the last block to finish sums the partials in a fixed order (the grid depends on the shape
// only) and adds the total to *log_det.
template <int C>
__global__ void __launch_bounds__(kFwdTailThreads)
wf_forward_tail_kernel(const __grid_constant__ FwdTailArgs<C> p) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int kWarps = kFwdTailThreads / 32;
  float lsum = 0.f;
  for (long long q = static_cast<long long>(blockIdx.x) * kWarps + warp; q < p.positions; q += static_cast<long long>(gridDim.x) * kWarps) {
    const int col = static_cast<int>(q % p.w);
    const long long bj = q / p.w;
    const int j = static_cast<int>(bj % p.n_group);
    const long long b = bj / p.n_group;
    const float xv = p.x[q];
    float zv = xv;
    if (p.skip != nullptr && j > 0) {
      const float* s = p.skip + ((b * (p.n_group - 1) + j - 1) * p.w + col) * C;
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int c = 2 * lane; c < C; c += 64) {
        const float2 v = *reinterpret_cast<const float2*>(s + c);
        s0 = fmaf(p.po_w[c], v.x, fmaf(p.po_w[c + 1], v.y, s0));
        s1 = fmaf(p.po_w[C + c], v.x, fmaf(p.po_w[C + c + 1], v.y, s1));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s0 += __shfl_xor_sync(0xffffffffu, s0, o);
        s1 += __shfl_xor_sync(0xffffffffu, s1, o);
      }
      const float logs = s0 + p.po_b[0], bb = s1 + p.po_b[1];
      zv = xv * expf(logs) + bb;
      lsum += logs;
    }
    const int h = p.inv[j];
    if (p.x_next != nullptr && lane == 0) p.x_next[(b * p.n_group + h) * p.w + col] = zv;
    if (p.next_hi != nullptr && h < p.n_group - 1) {
      const long long off = ((b * (p.n_group + 1) + 2 + h) * p.w + col) * C;
#pragma unroll
      for (int c = 2 * lane; c < C; c += 64) {
        __nv_bfloat16 h0, l0, h1, l1;
        split_bf16(fmaf(p.in_w[c], zv, p.in_b[c]), h0, l0);
        split_bf16(fmaf(p.in_w[c + 1], zv, p.in_b[c + 1]), h1, l1);
        *reinterpret_cast<uint32_t*>(p.next_hi + off + c) = pack_bf16x2(h0, h1);
        *reinterpret_cast<uint32_t*>(p.next_lo + off + c) = pack_bf16x2(l0, l1);
      }
    }
  }
  if (p.skip == nullptr) return;                                // no transform: nothing to add to log_det (uniform branch)
  __shared__ float wsum[kWarps];
  __shared__ double red[kFwdTailThreads];
  __shared__ bool is_last;
  if (lane == 0) wsum[warp] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < kWarps; ++i) s += wsum[i];
    p.partials[blockIdx.x] = s;
    __threadfence();
    is_last = atomicAdd(p.counter, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double acc = 0.0;
  for (int i = threadIdx.x; i < static_cast<int>(gridDim.x); i += kFwdTailThreads) acc += __ldcg(p.partials + i);
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kFwdTailThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    *p.log_det += static_cast<float>(red[0]);
    *p.counter = 0u;                                            // ready for the next call
  }
}

template <int C>
static int forward_tail_launch(const pk_waveflow_forward_tail_args* a, pk_stream_t stream) {
  static FwdTailArgs<C> p;                                      // filled under the caller's lock, copied by the launch
  p.w = a->width; p.n_group = a->n_group;
  p.positions = static_cast<long long>(a->batch) * a->n_group * a->width;
  bool seen[kFwdMaxGroup] = {};
  for (int i = 0; i < a->n_group; ++i) {
    PK_CHECK_ARG(a->perm[i] >= 0 && a->perm[i] < a->n_group && !seen[a->perm[i]], "perm is not a permutation of 0..n_group-1");
    seen[a->perm[i]] = true;
    p.inv[a->perm[i]] = i;
  }
  for (int i = 0; i < 2 * C; ++i) p.po_w[i] = a->skip ? a->out_w[i] : 0.f;
  p.po_b[0] = a->skip ? a->out_b[0] : 0.f;
  p.po_b[1] = a->skip ? a->out_b[1] : 0.f;
  for (int i = 0; i < C; ++i) {
    p.in_w[i] = a->next_hi ? a->in_w[i] : 0.f;
    p.in_b[i] = a->next_hi ? a->in_b[i] : 0.f;
  }
  p.skip = a->skip; p.x = a->x; p.x_next = a->x_next;
  p.next_hi = static_cast<__nv_bfloat16*>(a->next_hi); p.next_lo = static_cast<__nv_bfloat16*>(a->next_lo);
  p.log_det = a->log_det; p.partials = a->partials; p.counter = a->counter;
  constexpr int kWarps = kFwdTailThreads / 32;
  const int grid = static_cast<int>(std::min<long long>((p.positions + kWarps - 1) / kWarps, kFwdTailMaxBlocks));
  wf_forward_tail_kernel<C><<<grid, kFwdTailThreads, 0, static_cast<cudaStream_t>(stream)>>>(p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

__global__ void wf_nll_kernel(const double* __restrict__ sq_sum, const float* __restrict__ log_det, double n, double sigma,
                              float* __restrict__ loss) {
  const double kHalfLog2Pi = 0.91893853320467274178;
  loss[0] = static_cast<float>((sq_sum[0] / (2.0 * sigma * sigma) - static_cast<double>(log_det[0])) / n + kHalfLog2Pi + log(sigma));
}

}  // namespace pk

using namespace pk;

extern "C" int pk_waveflow_upsample(const float* x, const float* w, const float* bias, int32_t batch, int32_t c, int32_t t_in,
                                    int32_t factor, int32_t trim, float slope, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(x && w && bias && y && batch > 0 && c > 0 && t_in > 0 && factor >= 2 && (factor % 2) == 0, "bad arguments");
  const int t_out = t_in * factor - (trim ? factor : 0);
  PK_CHECK_ARG(t_out > 0, "empty output");
  const long long n = static_cast<long long>(batch) * c * t_out;
  wf_upsample_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, w, bias, c, t_in, factor, t_out, slope, n, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_input_proj(const float* x_row, int64_t x_batch_stride, const float* w, const float* bias, int32_t batch,
                                      int32_t width, int32_t c, float* state, void* buf_hi, void* buf_lo, int32_t ld, int32_t col0,
                                      pk_stream_t stream) {
  PK_CHECK_ARG(x_row && w && bias && state && buf_hi && buf_lo && batch > 0 && width > 0 && c > 0 && ld >= col0 + c, "bad arguments");
  const long long n = static_cast<long long>(batch) * width * c;
  wf_input_proj_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x_row, x_batch_stride, w, bias, width, c, n, state, static_cast<__nv_bfloat16*>(buf_hi), static_cast<__nv_bfloat16*>(buf_lo), ld, col0);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_row_out(const float* skip, const float* w, const float* bias, const float* z_row, int64_t z_batch_stride,
                                   int32_t batch, int32_t width, int32_t c, float* x_next, int64_t x_batch_stride, pk_stream_t stream) {
  PK_CHECK_ARG(skip && w && bias && z_row && x_next && batch > 0 && width > 0 && c > 0, "bad arguments");
  const long long rows = static_cast<long long>(batch) * width;
  wf_row_out_kernel<<<nblk(rows * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(skip, w, bias, z_row, z_batch_stride, width,
                                                                                           c, rows, x_next, x_batch_stride);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_forward_tail(const pk_waveflow_forward_tail_args* a, pk_stream_t stream) {
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  PK_CHECK_ARG(a->batch > 0 && a->width > 0 && a->n_group >= 2 && a->n_group <= kFwdMaxGroup, "bad batch/width/n_group");
  PK_CHECK_ARG(a->channels == 64 || a->channels == 128, "the WaveFlow forward tail is built for 64 or 128 channels (got %d)", a->channels);
  PK_CHECK_ARG(a->x && a->perm, "NULL x / perm");
  PK_CHECK_ARG(a->x_next != a->x, "x_next must not alias x");
  PK_CHECK_ARG(a->skip == nullptr || (a->out_w && a->out_b && a->log_det && a->partials && a->counter),
               "output_proj weights, log_det, partials and counter are needed with skip");
  PK_CHECK_ARG((a->next_hi == nullptr) == (a->next_lo == nullptr), "next_hi / next_lo: both or neither");
  PK_CHECK_ARG(a->next_hi == nullptr || (a->in_w && a->in_b), "input_proj weights are needed with next_hi");
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  return a->channels == 128 ? forward_tail_launch<128>(a, stream) : forward_tail_launch<64>(a, stream);
}

extern "C" int pk_waveflow_nll(const double* sq_sum, const float* log_det, int64_t n, float sigma, float* loss, pk_stream_t stream) {
  PK_CHECK_ARG(sq_sum && log_det && loss && n > 0 && sigma > 0.f, "bad arguments");
  wf_nll_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(sq_sum, log_det, static_cast<double>(n), static_cast<double>(sigma), loss);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
