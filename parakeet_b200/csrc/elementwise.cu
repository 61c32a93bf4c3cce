// HBM-bound helper kernels: fp32 -> split-bf16, length regulator (integer prefix-sum + row gather).
#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {

__global__ void split_f32_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                                 long long n) {
  const long long n8 = n >> 3;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(hi) & 15) == 0) &&
                       ((reinterpret_cast<uintptr_t>(lo) & 15) == 0);
  long long start8 = 0;
  if (aligned) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8; i += stride) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(x) + 2 * i);
      const float4 b = __ldg(reinterpret_cast<const float4*>(x) + 2 * i + 1);
      const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      uint4 h, l;
      split8(v, h, l);
      reinterpret_cast<uint4*>(hi)[i] = h;
      reinterpret_cast<uint4*>(lo)[i] = l;
    }
    start8 = n8 << 3;
  }
  for (long long i = start8 + blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += stride) {
    __nv_bfloat16 h, l;
    split_bf16(x[i], h, l);
    hi[i] = h;
    lo[i] = l;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Length regulator
// ---------------------------------------------------------------------------------------------------------------
constexpr int kLrThreads = 256;
constexpr int kLrMaxTokens = 8192;

// inclusive prefix sum of max(d,0) for one utterance into smem `cum` (int32), returns total. All threads call.
__device__ int lr_block_scan(const int64_t* __restrict__ dur, int t_in, int* cum, int* warp_sums) {
  const int tid = threadIdx.x;
  const int per = (t_in + kLrThreads - 1) / kLrThreads;
  const int beg = min(tid * per, t_in), end = min(beg + per, t_in);
  int local = 0;
  for (int j = beg; j < end; ++j) {
    const long long d = dur[j];
    local += d > 0 ? static_cast<int>(d) : 0;
    cum[j] = local;
  }
  // exclusive scan of `local` across threads
  int incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if ((tid & 31) >= o) incl += y;
  }
  if ((tid & 31) == 31) warp_sums[tid >> 5] = incl;
  __syncthreads();
  if (tid < 32) {
    int w = tid < kLrThreads / 32 ? warp_sums[tid] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (tid >= o) w += y;
    }
    if (tid < kLrThreads / 32) warp_sums[tid] = w;  // inclusive over warps
  }
  __syncthreads();
  const int warp_off = (tid >> 5) > 0 ? warp_sums[(tid >> 5) - 1] : 0;
  const int off = warp_off + incl - local;
  for (int j = beg; j < end; ++j) cum[j] += off;
  __syncthreads();
  return warp_sums[kLrThreads / 32 - 1];
}

__global__ void __launch_bounds__(kLrThreads) lr_lens_kernel(const int64_t* __restrict__ dur, int t_in, int32_t* __restrict__ out_lens) {
  __shared__ int warp_sums[kLrThreads / 32];
  const int64_t* d = dur + static_cast<long long>(blockIdx.x) * t_in;
  int local = 0;
  for (int j = threadIdx.x; j < t_in; j += kLrThreads) {
    const long long v = d[j];
    local += v > 0 ? static_cast<int>(v) : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    int s = 0;
    for (int w = 0; w < kLrThreads / 32; ++w) s += warp_sums[w];
    out_lens[blockIdx.x] = s;
  }
}

// grid = (row_blocks, batch); each CTA expands `rows_per_cta` consecutive output frames of one utterance.
__global__ void __launch_bounds__(kLrThreads)
lr_expand_kernel(const float* __restrict__ x, const int64_t* __restrict__ dur, int t_in, int c, int t_out, int rows_per_cta,
                 float* __restrict__ y, __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
  extern __shared__ int lr_smem[];
  int* cum = lr_smem;                 // [t_in] inclusive prefix sums
  __shared__ int warp_sums[kLrThreads / 32];
  const int b = blockIdx.y;
  const int total = lr_block_scan(dur + static_cast<long long>(b) * t_in, t_in, cum, warp_sums);
  const int row0 = blockIdx.x * rows_per_cta;
  const int row1 = min(row0 + rows_per_cta, t_out);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool vec = (c & 3) == 0;
  for (int r = row0 + warp; r < row1; r += kLrThreads / 32) {
    // source token: smallest j with cum[j] > r  (frames of token j are [cum[j-1], cum[j]))
    int j = -1;
    if (r < total) {
      int lo = 0, hi = t_in - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cum[mid] > r) hi = mid; else lo = mid + 1;
      }
      j = lo;
    }
    const long long yo = (static_cast<long long>(b) * t_out + r) * c;
    const float* src = j >= 0 ? x + (static_cast<long long>(b) * t_in + j) * c : nullptr;
    if (vec) {
      for (int q = lane; q < (c >> 2); q += 32) {
        const float4 v = src ? __ldg(reinterpret_cast<const float4*>(src) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (y) reinterpret_cast<float4*>(y + yo)[q] = v;
        if (y_hi) {
          __nv_bfloat16 h[4], l[4];
          split_bf16(v.x, h[0], l[0]); split_bf16(v.y, h[1], l[1]); split_bf16(v.z, h[2], l[2]); split_bf16(v.w, h[3], l[3]);
          reinterpret_cast<uint2*>(y_hi + yo)[q] = make_uint2(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]));
          reinterpret_cast<uint2*>(y_lo + yo)[q] = make_uint2(pack_bf16x2(l[0], l[1]), pack_bf16x2(l[2], l[3]));
        }
      }
    } else {
      for (int q = lane; q < c; q += 32) {
        const float v = src ? __ldg(src + q) : 0.f;
        if (y) y[yo + q] = v;
        if (y_hi) {
          __nv_bfloat16 h, l;
          split_bf16(v, h, l);
          y_hi[yo + q] = h;
          y_lo[yo + q] = l;
        }
      }
    }
  }
}

}  // namespace pk

extern "C" int pk_split_f32(const float* x, void* hi, void* lo, int64_t n, pk_stream_t stream) {
  PK_CHECK_ARG(x && hi && lo, "NULL pointer");
  PK_CHECK_ARG(n >= 0, "negative size");
  if (n == 0) return PK_OK;
  const int threads = 256;
  const long long want = (n / 8 + threads - 1) / threads + 1;
  const int blocks = static_cast<int>(want < pk::sm_count() * 8LL ? want : pk::sm_count() * 8LL);
  pk::split_f32_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(
      x, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), n);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}

extern "C" int pk_length_regulator_lens(const int64_t* dur, int32_t batch, int32_t t_in, int32_t* out_lens, pk_stream_t stream) {
  PK_CHECK_ARG(dur && out_lens, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && t_in > 0, "batch and t_in must be > 0");
  pk::lr_lens_kernel<<<batch, pk::kLrThreads, 0, static_cast<cudaStream_t>(stream)>>>(dur, t_in, out_lens);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}

extern "C" int pk_length_regulate(const float* x, const int64_t* dur, int32_t batch, int32_t t_in, int32_t c, int32_t t_out,
                                  float* y, void* y_hi, void* y_lo, pk_stream_t stream) {
  PK_CHECK_ARG(x && dur, "NULL pointer");
  PK_CHECK_ARG(y || y_hi, "no output requested");
  PK_CHECK_ARG((y_hi == nullptr) == (y_lo == nullptr), "y_hi and y_lo must both be set or both NULL");
  PK_CHECK_ARG(batch > 0 && t_in > 0 && c > 0 && t_out >= 0, "bad sizes");
  PK_CHECK_ARG(t_in <= pk::kLrMaxTokens, "t_in %d exceeds the supported maximum %d", t_in, pk::kLrMaxTokens);
  if (t_out == 0) return PK_OK;  // every duration is zero: empty output (reference: t_dec = 0)
  const int rows_per_cta = 32;
  dim3 grid((t_out + rows_per_cta - 1) / rows_per_cta, batch);
  pk::lr_expand_kernel<<<grid, pk::kLrThreads, t_in * sizeof(int), static_cast<cudaStream_t>(stream)>>>(
      x, dur, t_in, c, t_out, rows_per_cta, y, static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo));
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}
