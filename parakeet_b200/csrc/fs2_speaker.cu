// Speaker conditioning of the FastSpeech2 training step (reference: FastSpeech2._forward, parakeet/models/fastspeech2/
// fastspeech2.py:395-401 and _integrate_with_spk_embed :560-590; spk_embedding_table = nn.Embedding(num_speakers, D,
// padding_idx=0), F.normalize(p=2, axis=1, epsilon=1e-12)).
//
//   e[b] = table[id_b] / max(||table[id_b]||, eps)          (zeros where id_b == padding_idx)
//   concat: hs' = Linear(A + D -> A)([hs | e broadcast over time])       add: hs' = hs + Linear(D -> A)(e) broadcast over time
//
// The projection's GEMMs (forward, data gradient, weight gradient) run through pk_conv_gemm; these are the row-wise pieces
// around them.  Speaker ids are read on the device only, so a captured CUDA graph replays correctly for any ids of the same
// batch size.  No reduction uses atomics: every sum has a fixed order, and the step stays bit-for-bit reproducible.
// Ids outside [0, num_speakers) are treated like padding_idx (zero embedding, no gradient): the device cannot raise.
#include "pk_host.h"

namespace pk {
namespace {

constexpr int kRowThreads = 128;

// fixed-order sum over a block of kRowThreads threads (warp butterflies, then the 4 warp totals in order)
__device__ __forceinline__ float block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();                                   // red may still be read by the previous call
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  return (red[0] + red[1]) + (red[2] + red[3]);
}

__device__ __forceinline__ bool live_id(long long id, int num, int padding_idx) { return id >= 0 && id < num && id != padding_idx; }

// one block per utterance: lookup, L2 norm, e = x / max(norm, eps); norms[b] = ||x|| (0 for padding ids)
__global__ void __launch_bounds__(kRowThreads)
spk_embed_fwd_kernel(const float* __restrict__ table, int num, int d, const int64_t* __restrict__ ids, int padding_idx, float eps,
                     float* __restrict__ e, float* __restrict__ norms) {
  __shared__ float red[kRowThreads / 32];
  const int b = blockIdx.x;
  const long long id = ids[b];
  const bool live = live_id(id, num, padding_idx);
  const float* x = table + (live ? id : 0) * static_cast<long long>(d);
  float ss = 0.f;
  for (int c = threadIdx.x; c < d; c += kRowThreads) {
    const float v = live ? x[c] : 0.f;
    ss = fmaf(v, v, ss);
  }
  const float nrm = sqrtf(block_sum(ss, red));
  const float den = fmaxf(nrm, eps);
  for (int c = threadIdx.x; c < d; c += kRowThreads) e[static_cast<long long>(b) * d + c] = live ? x[c] / den : 0.f;
  if (threadIdx.x == 0) norms[b] = nrm;
}

// Per-utterance sum over ALL t rows of columns [col0, col0 + ncols) of dx (batch, t, c); columns [0, dhs_cols) are copied to
// the contiguous dhs (batch, t, dhs_cols) in the same pass, so a 640-wide concat gradient is read once.
// block = 32 columns x 8 row phases; grid = (ceil(cols_used / 32), batch)
__global__ void __launch_bounds__(256)
spk_time_sum_kernel(const float* __restrict__ dx, int t, int c, int col0, int ncols, float* __restrict__ dhs, int dhs_cols,
                    float* __restrict__ out) {
  __shared__ float part[8][33];
  const int b = blockIdx.y;
  const int lane = threadIdx.x & 31, ph = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + lane;
  const bool copy = dhs != nullptr && col < dhs_cols;
  const bool sum = col >= col0 && col < col0 + ncols;
  float s = 0.f;
  if (col < c && (copy || sum)) {
    for (int r = ph; r < t; r += 8) {
      const long long row = static_cast<long long>(b) * t + r;
      const float v = dx[row * c + col];
      if (copy) dhs[row * dhs_cols + col] = v;
      s += v;
    }
  }
  part[ph][lane] = s;
  __syncthreads();
  if (ph == 0 && sum && col < c) {
    float a = part[0][lane];
#pragma unroll
    for (int k = 1; k < 8; ++k) a += part[k][lane];
    out[static_cast<long long>(b) * ncols + (col - col0)] = a;
  }
}

// backward of e = x / max(||x||, eps): dx = (g - e (e.g)) / ||x|| where ||x|| > eps, g / eps otherwise; exact zeros for
// padding ids (their embedding is a constant zero).  One block per utterance.
__global__ void __launch_bounds__(kRowThreads)
spk_normalize_bwd_kernel(const float* __restrict__ e, const float* __restrict__ norms, const float* __restrict__ g,
                         const int64_t* __restrict__ ids, int num, int padding_idx, int d, float eps, float* __restrict__ dx) {
  __shared__ float red[kRowThreads / 32];
  const int b = blockIdx.x;
  const bool live = live_id(ids[b], num, padding_idx);
  const long long o = static_cast<long long>(b) * d;
  const float nrm = norms[b];
  float dot = 0.f;
  if (live && nrm > eps)
    for (int c = threadIdx.x; c < d; c += kRowThreads) dot = fmaf(e[o + c], g[o + c], dot);
  dot = block_sum(dot, red);              // every thread takes part (uniform control flow)
  for (int c = threadIdx.x; c < d; c += kRowThreads) {
    float v = 0.f;
    if (live) v = nrm > eps ? (g[o + c] - e[o + c] * dot) / nrm : g[o + c] / eps;
    dx[o + c] = v;
  }
}

// dense gradient of the table: dtable[r, c] = sum over b ascending with ids[b] == r of de[b, c]; every row is written (rows of
// absent speakers and padding_idx as zeros).  One thread per element.
__global__ void __launch_bounds__(256)
spk_table_grad_kernel(const float* __restrict__ de, const int64_t* __restrict__ ids, int batch, int num, int d, int padding_idx,
                      float* __restrict__ dtable) {
  const long long i = blockIdx.x * 256LL + threadIdx.x;
  if (i >= static_cast<long long>(num) * d) return;
  const int r = static_cast<int>(i / d), c = static_cast<int>(i % d);
  float s = 0.f;
  if (r != padding_idx)
    for (int b = 0; b < batch; ++b)
      if (ids[b] == r) s += de[static_cast<long long>(b) * d + c];
  dtable[i] = s;
}

}  // namespace
}  // namespace pk

using namespace pk;

extern "C" int pk_spk_embed_fwd(const float* table, int32_t num_speakers, int32_t d, const int64_t* ids, int32_t batch,
                                int32_t padding_idx, float eps, float* e, float* norms, pk_stream_t stream) {
  PK_CHECK_ARG(table && ids && e && norms, "NULL pointer");
  PK_CHECK_ARG(num_speakers > 0 && d > 0 && batch > 0 && eps > 0.f, "bad sizes");
  spk_embed_fwd_kernel<<<batch, kRowThreads, 0, PK_STREAM>>>(table, num_speakers, d, ids, padding_idx, eps, e, norms);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_spk_time_sum(const float* dx, int32_t batch, int32_t t, int32_t c, int32_t col0, int32_t ncols, float* dhs,
                               int32_t dhs_cols, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(dx && out, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && t > 0 && c > 0 && ncols > 0 && col0 >= 0 && col0 + ncols <= c, "bad column range");
  PK_CHECK_ARG(dhs == nullptr || (dhs_cols > 0 && dhs_cols <= c), "bad dhs width");
  const int used = dhs && dhs_cols > col0 + ncols ? dhs_cols : col0 + ncols;
  dim3 grid((used + 31) / 32, batch);
  spk_time_sum_kernel<<<grid, 256, 0, PK_STREAM>>>(dx, t, c, col0, ncols, dhs, dhs ? dhs_cols : 0, out);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_spk_normalize_bwd(const float* e, const float* norms, const float* g, const int64_t* ids, int32_t batch,
                                    int32_t num_speakers, int32_t padding_idx, int32_t d, float eps, float* dx, pk_stream_t stream) {
  PK_CHECK_ARG(e && norms && g && ids && dx, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && num_speakers > 0 && d > 0 && eps > 0.f, "bad sizes");
  spk_normalize_bwd_kernel<<<batch, kRowThreads, 0, PK_STREAM>>>(e, norms, g, ids, num_speakers, padding_idx, d, eps, dx);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_spk_table_grad(const float* de, const int64_t* ids, int32_t batch, int32_t num_speakers, int32_t d,
                                 int32_t padding_idx, float* dtable, pk_stream_t stream) {
  PK_CHECK_ARG(de && ids && dtable, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && num_speakers > 0 && d > 0, "bad sizes");
  const long long n = static_cast<long long>(num_speakers) * d;
  spk_table_grad_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, PK_STREAM>>>(de, ids, batch, num_speakers, d, padding_idx,
                                                                                      dtable);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
