// FastSpeech2 row-wise / element-wise kernels (HBM-bound): embedding + scaled positional encoding, LayerNorm,
// masked softmax, head transpose, duration post-op, variance embeddings, z-score.  The GEMM-shaped work of the model
// goes through pk_conv_gemm (conv_gemm.cu).
#include <math_constants.h>

#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {

// ---------------------------------------------------------------------------------------------------------------
// x[b,t,:] = (ids ? W[ids[b,t]] (zeros for id == padding_idx) : x_in[b,t,:]) + alpha * PE[t,:]
// PE[t, 2i] = sin(t * exp(2i * -ln(1e4)/d)), PE[t, 2i+1] = cos(...)   (embedding.py:46-62, fp32 arithmetic)
// one warp per row
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
embed_pe_kernel(const int64_t* __restrict__ ids, const float* __restrict__ table, int vocab, int padding_idx,
                const float* __restrict__ x_in, const float* __restrict__ alpha_p, const int32_t* __restrict__ lens, int rows_per_b,
                long long rows, int d, float* __restrict__ y) {
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int b = row / rows_per_b, t = row % rows_per_b;
  const float alpha = __ldg(alpha_p);
  const bool live = lens == nullptr || t < __ldg(lens + b);
  const float* src = nullptr;
  if (ids != nullptr) {
    const long long id = ids[row];
    if (id != padding_idx && id >= 0 && id < vocab) src = table + id * d;
  } else {
    src = x_in + row * d;
  }
  const float neg = -(logf(10000.0f) / static_cast<float>(d));
  for (int c = lane; c < d; c += 32) {
    const float div = expf(static_cast<float>(c & ~1) * neg);
    const float ang = static_cast<float>(t) * div;
    const float pe = (c & 1) ? cosf(ang) : sinf(ang);
    const float v = (src ? __ldg(src + c) : 0.f) + alpha * pe;
    y[row * d + c] = live ? v : 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (eps inside sqrt), one warp per row; outputs fp32 and/or split planes;
// rows t >= lens[b] are written as zero.
// ---------------------------------------------------------------------------------------------------------------
template <int MAX_PER_LANE>
__global__ void __launch_bounds__(256)
layer_norm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                  const int32_t* __restrict__ lens, int rows_per_b, long long rows, int d, float* __restrict__ y,
                  __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int b = row / rows_per_b, t = row % rows_per_b;
  const bool live = lens == nullptr || t < __ldg(lens + b);
  const float* xr = x + row * d;
  float v[MAX_PER_LANE];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAX_PER_LANE; ++i) {
    const int c = lane + 32 * i;
    v[i] = c < d ? xr[c] : 0.f;
    s += v[i];
  }
  const float mean = warp_sum(s) / static_cast<float>(d);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAX_PER_LANE; ++i) {
    const int c = lane + 32 * i;
    const float dv = c < d ? v[i] - mean : 0.f;
    q += dv * dv;
  }
  const float rstd = rsqrtf(warp_sum(q) / static_cast<float>(d) + eps);
#pragma unroll
  for (int i = 0; i < MAX_PER_LANE; ++i) {
    const int c = lane + 32 * i;
    if (c < d) {
      const float o = live ? (v[i] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c) : 0.f;
      if (y) y[row * d + c] = o;
      if (y_hi) {
        __nv_bfloat16 h, l;
        split_bf16(o, h, l);
        y_hi[row * d + c] = h;
        y_lo[row * d + c] = l;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Masked softmax over keys, optionally causal: s (batch * heads, rows, ld) fp32 -> p split planes of the same shape.  Query row
// i of utterance b attends keys j < key_lens[b] (all `keys` when key_lens is NULL) and, when causal, j <= i: attention.py:107-119
// and the TransformerTTS decoder's non_pad(olens) & tril mask (transformer_tts.py:692 _target_mask).  Masked and padding
// columns get 0; a row with no key left is all zeros (masked_fill(min) -> softmax -> masked_fill(0)).  One warp per row.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
masked_softmax_kernel(const float* __restrict__ s, const int32_t* __restrict__ klens, int heads, int rows_per_z, int keys, int ld,
                      int causal, long long rows, __nv_bfloat16* __restrict__ p_hi, __nv_bfloat16* __restrict__ p_lo) {
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int z = static_cast<int>(row / rows_per_z), i = static_cast<int>(row % rows_per_z);
  int klen = klens ? min(__ldg(klens + z / heads), keys) : keys;
  if (causal) klen = min(klen, i + 1);
  const float* sr = s + row * ld;
  float m = -CUDART_INF_F;
  for (int c = lane; c < klen; c += 32) m = fmaxf(m, sr[c]);
  m = warp_max(m);
  float sum = 0.f;
  for (int c = lane; c < klen; c += 32) sum += expf(sr[c] - m);
  sum = warp_sum(sum);
  const float inv = klen > 0 ? 1.f / sum : 0.f;
  for (int c = lane; c < ld; c += 32) {
    const float pv = c < klen ? expf(sr[c] - m) * inv : 0.f;
    __nv_bfloat16 h, l;
    split_bf16(pv, h, l);
    p_hi[row * ld + c] = h;
    p_lo[row * ld + c] = l;
  }
}

// V^T for the P.V matmul: src planes (B, T, ld_src) at column offset col0 + h*dk  ->  dst planes (B*H, dk, ld_dst)
// (keys contiguous; columns t >= T are zero-filled up to ld_dst).  32x32 tile transpose through shared memory.
__global__ void __launch_bounds__(256)
transpose_heads_kernel(const __nv_bfloat16* __restrict__ src_hi, const __nv_bfloat16* __restrict__ src_lo, int t_len, int ld_src,
                       int col0, int dk, int heads, int ld_dst, __nv_bfloat16* __restrict__ dst_hi,
                       __nv_bfloat16* __restrict__ dst_lo) {
  __shared__ __nv_bfloat16 th[32][34], tl[32][34];
  const int z = blockIdx.z, b = z / heads, h = z % heads;
  const int t0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int t = t0 + i, dcol = d0 + tx;
    __nv_bfloat16 vh = __float2bfloat16(0.f), vl = vh;
    if (t < t_len && dcol < dk) {
      const long long o = (static_cast<long long>(b) * t_len + t) * ld_src + col0 + h * dk + dcol;
      vh = src_hi[o];
      vl = src_lo[o];
    }
    th[i][tx] = vh;
    tl[i][tx] = vl;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int dcol = d0 + i, t = t0 + tx;
    if (dcol < dk && t < ld_dst) {
      const long long o = (static_cast<long long>(z) * dk + dcol) * ld_dst + t;
      dst_hi[o] = th[tx][i];
      dst_lo[o] = tl[tx][i];
    }
  }
}

// durations = clip(round_half_away(exp(x) - offset), 0), padded tokens -> 0 (duration_predictor.py:94-101)
__global__ void duration_post_kernel(const float* __restrict__ x, const int32_t* __restrict__ lens, int t_len, long long n,
                                     float offset, float* __restrict__ d_f32, int64_t* __restrict__ d_i64) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int b = i / t_len, t = i % t_len;
  float v = roundf(expf(x[i]) - offset);  // roundf: half away from zero == paddle.round
  v = fmaxf(v, 0.f);
  if (lens != nullptr && t >= __ldg(lens + b)) v = 0.f;
  if (d_f32) d_f32[i] = v;
  if (d_i64) d_i64[i] = static_cast<int64_t>(v);
}

// ds = round_half_away(ds * alpha) as int64 (length_regulator.py:85-88)
__global__ void duration_scale_kernel(const int64_t* __restrict__ d, float alpha, long long n, int64_t* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) out[i] = static_cast<int64_t>(roundf(static_cast<float>(d[i]) * alpha));
}

// masked fill of a (B, T) or (B, T, 1) tensor: x[b,t] = 0 for t >= lens[b]
__global__ void mask_rows_kernel(float* __restrict__ x, const int32_t* __restrict__ lens, int t_len, int inner, long long n) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const long long row = i / inner;
  const int b = row / t_len, t = row % t_len;
  if (t >= __ldg(lens + b)) x[i] = 0.f;
}

// hs[b,t,c] += conv1d(p)[b,t,c] + conv1d(e)[b,t,c], Conv1D(1 -> C, k, pad (k-1)/2) on scalar tracks p, e (B, T)
// (fastspeech2.py:426-430 / :436-440); zero padding at the ends of the (padded) batch rows, like the reference.
__global__ void __launch_bounds__(256)
variance_embed_add_kernel(const float* __restrict__ hs, const float* __restrict__ p, const float* __restrict__ e,
                          const float* __restrict__ wp, const float* __restrict__ bp, int kp, const float* __restrict__ we,
                          const float* __restrict__ be, int ke, const int32_t* __restrict__ lens, int t_len, int c, long long n,
                          float* __restrict__ y) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int ch = i % c;
  const long long row = i / c;
  const int b = row / t_len, t = row % t_len;
  const int tmax = lens ? __ldg(lens + b) : t_len;   // independent-utterance mode: the track ends at lens[b]
  float acc = hs[i] + __ldg(bp + ch) + __ldg(be + ch);
  for (int q = 0; q < kp; ++q) {
    const int tt = t + q - (kp - 1) / 2;
    if (tt >= 0 && tt < tmax) acc = fmaf(__ldg(wp + ch * kp + q), __ldg(p + static_cast<long long>(b) * t_len + tt), acc);
  }
  for (int q = 0; q < ke; ++q) {
    const int tt = t + q - (ke - 1) / 2;
    if (tt >= 0 && tt < tmax) acc = fmaf(__ldg(we + ch * ke + q), __ldg(e + static_cast<long long>(b) * t_len + tt), acc);
  }
  y[i] = (lens == nullptr || t < tmax) ? acc : 0.f;
}

// y = x * scale[c] + shift[c] over the last dim (ZScore.forward with scale = 1/sigma, shift = -mu/sigma is NOT used:
// to keep the reference's rounding the two forms are separate)   mode 0: (x - mu) / sigma ; mode 1: x * sigma + mu
__global__ void zscore_kernel(const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ sigma, int c,
                              long long n, int mode, float* __restrict__ y) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int ch = i % c;
  y[i] = mode == 0 ? (x[i] - __ldg(mu + ch)) / __ldg(sigma + ch) : fmaf(x[i], __ldg(sigma + ch), __ldg(mu + ch));
}

}  // namespace pk

using namespace pk;

extern "C" int pk_embed_pe(const int64_t* ids, const float* table, int32_t vocab, int32_t padding_idx, const float* x_in,
                           const float* alpha, const int32_t* lens, int32_t batch, int32_t t, int32_t d, float* y,
                           pk_stream_t stream) {
  PK_CHECK_ARG((ids != nullptr) != (x_in != nullptr), "exactly one of ids / x_in must be given");
  PK_CHECK_ARG(ids == nullptr || table != nullptr, "table is NULL");
  PK_CHECK_ARG(alpha && y && batch > 0 && t > 0 && d > 0, "bad arguments");
  const long long rows = static_cast<long long>(batch) * t;
  embed_pe_kernel<<<nblk(rows * 32, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ids, table, vocab, padding_idx, x_in,
                                                                                       alpha, lens, t, rows, d, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_layer_norm(const float* x, const float* gamma, const float* beta, float eps, const int32_t* lens, int32_t batch,
                             int32_t t, int32_t d, float* y, void* y_hi, void* y_lo, pk_stream_t stream) {
  PK_CHECK_ARG(x && gamma && beta && batch > 0 && t > 0 && d > 0, "bad arguments");
  PK_CHECK_ARG(y || y_hi, "no output requested");
  PK_CHECK_ARG((y_hi == nullptr) == (y_lo == nullptr), "y_hi and y_lo must both be set or both NULL");
  PK_CHECK_ARG(d <= 2048, "layer_norm supports d <= 2048 (got %d)", d);
  const long long rows = static_cast<long long>(batch) * t;
  const int blocks = nblk(rows * 32, 256);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  auto* hi = static_cast<__nv_bfloat16*>(y_hi);
  auto* lo = static_cast<__nv_bfloat16*>(y_lo);
  if (d <= 256) layer_norm_kernel<8><<<blocks, 256, 0, s>>>(x, gamma, beta, eps, lens, t, rows, d, y, hi, lo);
  else if (d <= 512) layer_norm_kernel<16><<<blocks, 256, 0, s>>>(x, gamma, beta, eps, lens, t, rows, d, y, hi, lo);
  else layer_norm_kernel<64><<<blocks, 256, 0, s>>>(x, gamma, beta, eps, lens, t, rows, d, y, hi, lo);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_masked_softmax(const float* s, const int32_t* key_lens, int32_t batch, int32_t heads, int32_t rows, int32_t keys,
                                 int32_t ld, int32_t causal, void* p_hi, void* p_lo, pk_stream_t stream) {
  PK_CHECK_ARG(s && p_hi && p_lo && batch > 0 && heads > 0 && rows > 0 && keys > 0 && ld >= keys, "bad arguments to pk_masked_softmax");
  const long long total = static_cast<long long>(batch) * heads * rows;
  masked_softmax_kernel<<<nblk(total * 32, 256), 256, 0, PK_STREAM>>>(s, key_lens, heads, rows, keys, ld, causal ? 1 : 0, total,
                                                                       static_cast<__nv_bfloat16*>(p_hi), static_cast<__nv_bfloat16*>(p_lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_transpose_heads(const void* src_hi, const void* src_lo, int32_t batch, int32_t t, int32_t ld_src, int32_t col0,
                                  int32_t dk, int32_t heads, int32_t ld_dst, void* dst_hi, void* dst_lo, pk_stream_t stream) {
  PK_CHECK_ARG(src_hi && src_lo && dst_hi && dst_lo && batch > 0 && t > 0 && dk > 0 && heads > 0 && ld_dst >= t, "bad arguments");
  dim3 grid((ld_dst + 31) / 32, (dk + 31) / 32, batch * heads);
  transpose_heads_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(src_hi), static_cast<const __nv_bfloat16*>(src_lo), t, ld_src, col0, dk, heads, ld_dst,
      static_cast<__nv_bfloat16*>(dst_hi), static_cast<__nv_bfloat16*>(dst_lo));
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_duration_post(const float* x, const int32_t* lens, int32_t batch, int32_t t, float offset, float* d_f32,
                                int64_t* d_i64, pk_stream_t stream) {
  PK_CHECK_ARG(x && (d_f32 || d_i64) && batch > 0 && t > 0, "bad arguments");
  const long long n = static_cast<long long>(batch) * t;
  duration_post_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, lens, t, n, offset, d_f32, d_i64);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_duration_scale(const int64_t* d, float alpha, int64_t n, int64_t* out, pk_stream_t stream) {
  PK_CHECK_ARG(d && out && n > 0 && alpha > 0.f, "bad arguments");
  duration_scale_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(d, alpha, n, out);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_mask_rows(float* x, const int32_t* lens, int32_t batch, int32_t t, int32_t inner, pk_stream_t stream) {
  PK_CHECK_ARG(x && lens && batch > 0 && t > 0 && inner > 0, "bad arguments");
  const long long n = static_cast<long long>(batch) * t * inner;
  mask_rows_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, lens, t, inner, n);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_variance_embed_add(const float* hs, const float* pitch, const float* energy, const float* wp, const float* bp,
                                     int32_t kp, const float* we, const float* be, int32_t ke, const int32_t* lens, int32_t batch,
                                     int32_t t, int32_t c, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(hs && pitch && energy && wp && bp && we && be && y, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && t > 0 && c > 0 && kp >= 1 && ke >= 1 && (kp & 1) && (ke & 1), "bad sizes (odd kernel sizes only)");
  const long long n = static_cast<long long>(batch) * t * c;
  variance_embed_add_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(hs, pitch, energy, wp, bp, kp, we, be,
                                                                                         ke, lens, t, c, n, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_zscore(const float* x, const float* mu, const float* sigma, int32_t c, int64_t n, int32_t inverse, float* y,
                         pk_stream_t stream) {
  PK_CHECK_ARG(x && mu && sigma && y && c > 0 && n > 0, "bad arguments");
  zscore_kernel<<<nblk(n, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(x, mu, sigma, c, n, inverse ? 1 : 0, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// FastSpeech2Loss.forward (fastspeech2.py:701-812) with use_masking=True: masked means in one pass.
//   out[0] = mean_{valid frames x odim} |before - ys| + mean |after - ys|     (L1Loss on masked_select'ed tensors)
//   out[1] = mean_{valid tokens} (d_outs - log(ds + 1))^2                       (DurationPredictorLoss, offset 1)
//   out[2] = mean_{valid tokens} (p_outs - ps)^2 ;  out[3] = mean (e_outs - es)^2
// sums are accumulated in fp32 per block and combined with atomics into 6 accumulators, finalised by the last block.
// ---------------------------------------------------------------------------------------------------------------
namespace pk {
__global__ void __launch_bounds__(256)
fs2_loss_kernel(const float* __restrict__ before, const float* __restrict__ after, const float* __restrict__ ys,
                const int32_t* __restrict__ olens, int l_max, int odim, const float* __restrict__ d_outs,
                const int64_t* __restrict__ ds, const float* __restrict__ p_outs, const float* __restrict__ ps,
                const float* __restrict__ e_outs, const float* __restrict__ es, const int32_t* __restrict__ ilens, int t_max,
                int batch, float* __restrict__ acc /*[8]*/, unsigned int* __restrict__ counter, float* __restrict__ out /*[4]*/) {
  float s[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
  const long long n_mel = static_cast<long long>(batch) * l_max * odim;
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_mel; i += stride) {
    const long long row = i / odim;
    const int b = row / l_max, t = row % l_max;
    if (t < __ldg(olens + b)) {
      const float y = ys[i];
      s[0] += fabsf(before[i] - y);
      s[1] += fabsf(after[i] - y);
    }
  }
  const long long n_tok = static_cast<long long>(batch) * t_max;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_tok; i += stride) {
    const int b = i / t_max, t = i % t_max;
    if (t < __ldg(ilens + b)) {
      const float dd = d_outs[i] - logf(static_cast<float>(ds[i]) + 1.0f);
      const float dp = p_outs[i] - ps[i];
      const float de = e_outs[i] - es[i];
      s[2] += dd * dd; s[3] += dp * dp; s[4] += de * de;
    }
  }
  __shared__ float red[5][8];
#pragma unroll
  for (int k = 0; k < 5; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = s[k];
  }
  __syncthreads();
  if (threadIdx.x < 5) {
    float v = 0.f;
    for (int w = 0; w < 8; ++w) v += red[threadIdx.x][w];
    atomicAdd(acc + threadIdx.x, v);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int done = atomicAdd(counter, 1u);
    if (done == gridDim.x - 1) {   // last block: finalise
      long long frames = 0, toks = 0;
      for (int b = 0; b < batch; ++b) { frames += min(olens[b], l_max); toks += min(ilens[b], t_max); }
      const float nm = static_cast<float>(frames) * odim, nt = static_cast<float>(toks);
      volatile float* a = acc;
      out[0] = a[0] / nm + a[1] / nm;
      out[1] = a[2] / nt;
      out[2] = a[3] / nt;
      out[3] = a[4] / nt;
    }
  }
}
}  // namespace pk

extern "C" int pk_fs2_loss(const float* before, const float* after, const float* ys, const int32_t* olens, int32_t l_max,
                           int32_t odim, const float* d_outs, const int64_t* ds, const float* p_outs, const float* ps,
                           const float* e_outs, const float* es, const int32_t* ilens, int32_t t_max, int32_t batch,
                           float* workspace12, float* out4, pk_stream_t stream) {
  PK_CHECK_ARG(before && after && ys && olens && d_outs && ds && p_outs && ps && e_outs && es && ilens && workspace12 && out4,
               "NULL pointer");
  PK_CHECK_ARG(l_max > 0 && odim > 0 && t_max > 0 && batch > 0, "bad sizes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PK_CHECK_CUDA(cudaMemsetAsync(workspace12, 0, 12 * sizeof(float), s));
  const long long n = static_cast<long long>(batch) * l_max * odim;
  const int blocks = static_cast<int>(std::min<long long>((n + 255) / 256, sm_count() * 4LL));
  fs2_loss_kernel<<<blocks, 256, 0, s>>>(before, after, ys, olens, l_max, odim, d_outs, ds, p_outs, ps, e_outs, es, ilens, t_max,
                                         batch, workspace12, reinterpret_cast<unsigned int*>(workspace12 + 8), out4);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

// ----------------------------------------------------------------------------------------------------------------
// paddle.nn.functional.normalize(x, p=2, axis=1, epsilon=1e-12) on a tensor viewed as (outer, n, inner): y = x / max(||x||_2, eps)
// with the norm taken over the middle axis.  FastSpeech2 applies it to speaker embeddings (B, D): outer = B, n = D, inner = 1 -
// and, in the batched forward, to tone embeddings (B, T, D) where axis 1 is TIME (fastspeech2.py:577,581,606,611): outer = B,
// n = T, inner = D.  One block per (outer, 32-wide slice of inner); tiny tensors, latency bound.
// ----------------------------------------------------------------------------------------------------------------
namespace pk {
__global__ void l2_normalize_kernel(const float* __restrict__ x, int n, int inner, float eps, float* __restrict__ y) {
  const int o = blockIdx.x, i = blockIdx.y * 32 + (threadIdx.x & 31), part = threadIdx.x >> 5, parts = blockDim.x >> 5;
  __shared__ float red[8][33];
  const float* xo = x + static_cast<long long>(o) * n * inner;
  float acc = 0.f;
  if (i < inner)
    for (int k = part; k < n; k += parts) {
      const float v = xo[static_cast<long long>(k) * inner + i];
      acc = fmaf(v, v, acc);
    }
  red[part][threadIdx.x & 31] = acc;
  __syncthreads();
  float tot = 0.f;
  for (int q = 0; q < parts; ++q) tot += red[q][threadIdx.x & 31];
  const float inv = 1.f / fmaxf(sqrtf(tot), eps);
  float* yo = y + static_cast<long long>(o) * n * inner;
  if (i < inner)
    for (int k = part; k < n; k += parts) yo[static_cast<long long>(k) * inner + i] = xo[static_cast<long long>(k) * inner + i] * inv;
}
}  // namespace pk

extern "C" int pk_l2_normalize(const float* x, int32_t outer, int32_t n, int32_t inner, float eps, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(x && y && outer > 0 && n > 0 && inner > 0, "bad arguments");
  dim3 grid(outer, (inner + 31) / 32);
  pk::l2_normalize_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(x, n, inner, eps, y);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}
