// SpeedySpeech training step (reference: SpeedySpeechUpdater.update_core, parakeet/models/speedyspeech/speedyspeech_updater.py:48-85):
// the train-mode BatchNorm1D of every Conv1D -> ReLU -> BatchNorm1D unit (speedyspeech.py:21-39) forward and backward, and the
// three losses (masked L1 modules/losses.py:60-100, Huber on log durations, SSIM modules/ssim.py:21-80) with their gradients.
// The convolutions themselves, their data and weight gradients run through pk_conv_gemm.
// No reduction uses atomics: every sum is a per-block partial written to a scratch array and added up in a fixed order, so two
// steps from the same state give identical bits.
#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace {

constexpr int kC = 128;          // channels of every SpeedySpeech hidden layer
constexpr int kRows = 128;       // rows per block of the column kernels
constexpr int kThreads = 256;    // thread = (column, row parity)
constexpr int kFinalThreads = 1024;

__device__ __forceinline__ void put_split(__nv_bfloat16* hi, __nv_bfloat16* lo, long long i, float v) {
  __nv_bfloat16 h, l;
  split_bf16(v, h, l);
  hi[i] = h;
  lo[i] = l;
}

// part[b * nv + v], b < nblk, summed over b in double: blockDim / nv contiguous segments of b, then the segments in order.
// Returns the total in the threads of segment 0 (threadIdx.x < nv); every thread of the block must call it.
__device__ double reduce_partials(const float* __restrict__ part, int nblk, int nv, double* sh) {
  const int v = threadIdx.x % nv, seg = threadIdx.x / nv, segs = blockDim.x / nv;
  const int b0 = static_cast<int>(static_cast<long long>(nblk) * seg / segs);
  const int b1 = static_cast<int>(static_cast<long long>(nblk) * (seg + 1) / segs);
  double s = 0.0;
  for (int b = b0; b < b1; ++b) s += part[static_cast<long long>(b) * nv + v];
  sh[threadIdx.x] = s;
  __syncthreads();
  double t = 0.0;
  if (seg == 0)
    for (int k = 0; k < segs; ++k) t += sh[k * nv + v];
  return t;
}

// ---------------------------------------------------------------------------------------------------------------
// BatchNorm1D, training mode, on r (rows, 128)
// ---------------------------------------------------------------------------------------------------------------
// part[blk][0][c] = sum r, part[blk][1][c] = sum r^2 over the block's rows
__global__ void __launch_bounds__(kThreads) ss_bn_stats_kernel(const float* __restrict__ r, long long rows, float* __restrict__ part) {
  __shared__ float sh[2][kC];
  const int col = threadIdx.x & (kC - 1), half = threadIdx.x >> 7;
  const long long r0 = blockIdx.x * static_cast<long long>(kRows), r1 = min(rows, r0 + kRows);
  float s = 0.f, q = 0.f;
  for (long long i = r0 + half; i < r1; i += 2) {
    const float v = r[i * kC + col];
    s += v;
    q = fmaf(v, v, q);
  }
  if (half) { sh[0][col] = s; sh[1][col] = q; }
  __syncthreads();
  if (!half) {
    part[blockIdx.x * 2LL * kC + col] = s + sh[0][col];
    part[blockIdx.x * 2LL * kC + kC + col] = q + sh[1][col];
  }
}

// mean, rstd (biased variance) and Paddle's running update: running = momentum * running + (1 - momentum) * batch
__global__ void __launch_bounds__(kFinalThreads)
ss_bn_finalize_kernel(const float* __restrict__ part, int nblk, long long rows, float eps, float momentum, float* __restrict__ run_mean,
                      float* __restrict__ run_var, float* __restrict__ mean, float* __restrict__ rstd) {
  __shared__ double sh[kFinalThreads];
  __shared__ double tot[2 * kC];
  const double t = reduce_partials(part, nblk, 2 * kC, sh);
  if (threadIdx.x < 2 * kC) tot[threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.x < kC) {
    const int c = threadIdx.x;
    const double m = tot[c] / rows;
    const double var = fmax(tot[kC + c] / rows - m * m, 0.0);
    mean[c] = static_cast<float>(m);
    rstd[c] = static_cast<float>(1.0 / sqrt(var + eps));
    if (run_mean) {
      run_mean[c] = momentum * run_mean[c] + (1.f - momentum) * static_cast<float>(m);
      run_var[c] = momentum * run_var[c] + (1.f - momentum) * static_cast<float>(var);
    }
  }
}

// y = gamma * (r - mean) * rstd + beta (+ residual), fp32 and / or split planes
__global__ void __launch_bounds__(kThreads)
ss_bn_apply_kernel(const float* __restrict__ r, long long rows, const float* __restrict__ mean, const float* __restrict__ rstd,
                   const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ residual,
                   float* __restrict__ y, __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
  const int col = threadIdx.x & (kC - 1), half = threadIdx.x >> 7;
  const long long r0 = blockIdx.x * static_cast<long long>(kRows), r1 = min(rows, r0 + kRows);
  const float m = mean[col], k = gamma[col] * rstd[col], b = beta[col];
  for (long long i = r0 + half; i < r1; i += 2) {
    const long long o = i * kC + col;
    float v = fmaf(r[o] - m, k, b);
    if (residual) v += residual[o];
    if (y) y[o] = v;
    if (y_hi) put_split(y_hi, y_lo, o, v);
  }
}

// backward, pass 1: part[blk][0][c] = sum dy, part[blk][1][c] = sum dy * xhat
__global__ void __launch_bounds__(kThreads)
ss_bn_bwd_stats_kernel(const float* __restrict__ dy, const float* __restrict__ r, const float* __restrict__ mean,
                       const float* __restrict__ rstd, long long rows, float* __restrict__ part) {
  __shared__ float sh[2][kC];
  const int col = threadIdx.x & (kC - 1), half = threadIdx.x >> 7;
  const long long r0 = blockIdx.x * static_cast<long long>(kRows), r1 = min(rows, r0 + kRows);
  const float m = mean[col], rs = rstd[col];
  float s = 0.f, q = 0.f;
  for (long long i = r0 + half; i < r1; i += 2) {
    const float g = dy[i * kC + col];
    s += g;
    q = fmaf(g, (r[i * kC + col] - m) * rs, q);
  }
  if (half) { sh[0][col] = s; sh[1][col] = q; }
  __syncthreads();
  if (!half) {
    part[blockIdx.x * 2LL * kC + col] = s + sh[0][col];
    part[blockIdx.x * 2LL * kC + kC + col] = q + sh[1][col];
  }
}

// out[v] = sum of the partials, v < nv (dbeta | dgamma with nv = 256 and out2 = out + 128 elsewhere; the bias gradient with nv = 128)
__global__ void __launch_bounds__(kFinalThreads)
ss_colsum_finalize_kernel(const float* __restrict__ part, int nblk, int nv, float* __restrict__ out_lo, float* __restrict__ out_hi) {
  __shared__ double sh[kFinalThreads];
  const double t = reduce_partials(part, nblk, nv, sh);
  if (threadIdx.x < kC) out_lo[threadIdx.x] = static_cast<float>(t);
  else if (threadIdx.x < nv) out_hi[threadIdx.x - kC] = static_cast<float>(t);
}

// backward, pass 2: dr = gamma * rstd * (dy - mean(dy) - xhat * mean(dy * xhat)) * [r > 0]; part[blk][c] = sum dr (the conv's
// bias gradient).  r is the ReLU output the BatchNorm read, so [r > 0] is the ReLU's derivative.
__global__ void __launch_bounds__(kThreads)
ss_bn_relu_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ r, const float* __restrict__ mean,
                            const float* __restrict__ rstd, const float* __restrict__ gamma, const float* __restrict__ dbeta,
                            const float* __restrict__ dgamma, long long rows, float* __restrict__ dr, __nv_bfloat16* __restrict__ dr_hi,
                            __nv_bfloat16* __restrict__ dr_lo, float* __restrict__ part) {
  __shared__ float sh[kC];
  const int col = threadIdx.x & (kC - 1), half = threadIdx.x >> 7;
  const long long r0 = blockIdx.x * static_cast<long long>(kRows), r1 = min(rows, r0 + kRows);
  const float m = mean[col], rs = rstd[col], k = gamma[col] * rs;
  const float m1 = dbeta[col] / static_cast<float>(rows), m2 = dgamma[col] / static_cast<float>(rows);
  float s = 0.f;
  for (long long i = r0 + half; i < r1; i += 2) {
    const long long o = i * kC + col;
    const float rv = r[o];
    const float v = rv > 0.f ? k * (dy[o] - m1 - (rv - m) * rs * m2) : 0.f;
    s += v;
    if (dr) dr[o] = v;
    if (dr_hi) put_split(dr_hi, dr_lo, o, v);
  }
  if (half) sh[col] = s;
  __syncthreads();
  if (!half) part[blockIdx.x * static_cast<long long>(kC) + col] = s + sh[col];
}

// ---------------------------------------------------------------------------------------------------------------
// Losses.  SSIM: the 11 x 11 Gaussian window (sigma 1.5) is the outer product of a normalised 1-D window, so every filtered
// map is a pass along the mel axis (into shared memory) and a pass along time (out of it); zero padding 5 on every side.
// A block owns kTile frames of one utterance, all mel bins.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kWin = 11, kHalo = 5, kTile = 16, kMaxMel = 80;
constexpr float kC1 = 0.01f * 0.01f, kC2 = 0.03f * 0.03f;

__device__ __forceinline__ void gaussian_window(float* w) {
  if (threadIdx.x == 0) {
    double g[kWin], s = 0.0;
    for (int k = 0; k < kWin; ++k) { g[k] = exp(-static_cast<double>((k - kHalo) * (k - kHalo)) / (2.0 * 1.5 * 1.5)); s += g[k]; }
    for (int k = 0; k < kWin; ++k) w[k] = static_cast<float>(g[k] / s);
  }
}

// ssim map and its derivatives with respect to the three filtered maps that depend on the prediction (mu_x, E[x^2], E[xy]),
// scaled by gscale = d loss / d ssim_map = -1 / (batch * l * odim); per-block partial sums of the ssim map and of |d - y| * mask
__global__ void __launch_bounds__(256)
ss_ssim_fwd_kernel(const float* __restrict__ dec, const float* __restrict__ feats, const int32_t* __restrict__ num_frames, int l, int odim,
                   float gscale, float* __restrict__ gmaps, long long map_stride, float* __restrict__ part) {
  __shared__ float h[5][kTile + 2 * kHalo][kMaxMel];
  __shared__ float w[kWin];
  __shared__ double red[256];
  const int b = blockIdx.y, t0 = blockIdx.x * kTile;
  const int nf = min(num_frames[b], l);
  const long long base = static_cast<long long>(b) * l * odim;
  gaussian_window(w);
  __syncthreads();
  for (int idx = threadIdx.x; idx < (kTile + 2 * kHalo) * odim; idx += blockDim.x) {
    const int lr = idx / odim, col = idx % odim, t = t0 - kHalo + lr;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
    if (t >= 0 && t < nf) {                    // frames past the utterance are zeroed by the mask, frames outside [0, l) are padding
      const float* xr = dec + base + static_cast<long long>(t) * odim;
      const float* yr = feats + base + static_cast<long long>(t) * odim;
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const int cc = col + k - kHalo;
        if (cc >= 0 && cc < odim) {
          const float x = xr[cc], y = yr[cc], wk = w[k];
          a0 = fmaf(wk, x, a0);
          a1 = fmaf(wk, y, a1);
          a2 = fmaf(wk, x * x, a2);
          a3 = fmaf(wk, y * y, a3);
          a4 = fmaf(wk, x * y, a4);
        }
      }
    }
    h[0][lr][col] = a0; h[1][lr][col] = a1; h[2][lr][col] = a2; h[3][lr][col] = a3; h[4][lr][col] = a4;
  }
  __syncthreads();
  double s_ssim = 0.0, s_l1 = 0.0;
  for (int idx = threadIdx.x; idx < kTile * odim; idx += blockDim.x) {
    const int lr = idx / odim, col = idx % odim, t = t0 + lr;
    if (t >= l) continue;
    double mx = 0.0, my = 0.0, exx = 0.0, eyy = 0.0, exy = 0.0;
#pragma unroll
    for (int k = 0; k < kWin; ++k) {
      const double wk = w[k];
      mx += wk * h[0][lr + k][col];
      my += wk * h[1][lr + k][col];
      exx += wk * h[2][lr + k][col];
      eyy += wk * h[3][lr + k][col];
      exy += wk * h[4][lr + k][col];
    }
    const double a1 = 2.0 * mx * my + kC1, a2 = 2.0 * (exy - mx * my) + kC2;
    const double b1 = mx * mx + my * my + kC1, b2 = (exx - mx * mx) + (eyy - my * my) + kC2;
    const double s = a1 * a2 / (b1 * b2);
    s_ssim += s;
    const long long o = base + static_cast<long long>(t) * odim + col;
    if (gmaps) {
      gmaps[o] = static_cast<float>(gscale * (2.0 * my * (a2 - a1) / (b1 * b2) - 2.0 * mx * s / b1 + 2.0 * mx * s / b2));
      gmaps[map_stride + o] = static_cast<float>(gscale * (-s / b2));
      gmaps[2 * map_stride + o] = static_cast<float>(gscale * (2.0 * a1 / (b1 * b2)));
    }
    if (t < nf) s_l1 += fabs(static_cast<double>(dec[o]) - static_cast<double>(feats[o]));
  }
  const double t_ssim = block_sum_tree<256>(s_ssim, red);
  const double t_l1 = block_sum_tree<256>(s_l1, red);
  if (threadIdx.x == 0) {
    const long long blk = static_cast<long long>(b) * gridDim.x + blockIdx.x;
    part[2 * blk] = static_cast<float>(t_ssim);
    part[2 * blk + 1] = static_cast<float>(t_l1);
  }
}

// g_dec = mask * (F(G1) + 2 x F(G2) + y F(G3) + sign(d - y) / (frames * odim)): F is the same window (it is symmetric, so the
// adjoint of the filter is the filter), x / y the masked images
__global__ void __launch_bounds__(256)
ss_ssim_bwd_kernel(const float* __restrict__ dec, const float* __restrict__ feats, const int32_t* __restrict__ num_frames, int batch, int l,
                   int odim, const float* __restrict__ gmaps, long long map_stride, float* __restrict__ g_dec) {
  __shared__ float h[3][kTile + 2 * kHalo][kMaxMel];
  __shared__ float w[kWin];
  __shared__ float s_inv;
  const int b = blockIdx.y, t0 = blockIdx.x * kTile;
  const int nf = min(num_frames[b], l);
  const long long base = static_cast<long long>(b) * l * odim;
  gaussian_window(w);
  if (threadIdx.x == 32) {
    long long frames = 0;
    for (int i = 0; i < batch; ++i) frames += min(num_frames[i], l);
    s_inv = frames > 0 ? 1.f / (static_cast<float>(frames) * odim) : 0.f;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < (kTile + 2 * kHalo) * odim; idx += blockDim.x) {
    const int lr = idx / odim, col = idx % odim, t = t0 - kHalo + lr;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    if (t >= 0 && t < l) {
      const float* g = gmaps + base + static_cast<long long>(t) * odim;
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const int cc = col + k - kHalo;
        if (cc >= 0 && cc < odim) {
          const float wk = w[k];
          a0 = fmaf(wk, g[cc], a0);
          a1 = fmaf(wk, g[map_stride + cc], a1);
          a2 = fmaf(wk, g[2 * map_stride + cc], a2);
        }
      }
    }
    h[0][lr][col] = a0; h[1][lr][col] = a1; h[2][lr][col] = a2;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < kTile * odim; idx += blockDim.x) {
    const int lr = idx / odim, col = idx % odim, t = t0 + lr;
    if (t >= l) continue;
    const long long o = base + static_cast<long long>(t) * odim + col;
    float v = 0.f;
    if (t < nf) {
      float f1 = 0.f, f2 = 0.f, f3 = 0.f;
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        f1 = fmaf(w[k], h[0][lr + k][col], f1);
        f2 = fmaf(w[k], h[1][lr + k][col], f2);
        f3 = fmaf(w[k], h[2][lr + k][col], f3);
      }
      const float x = dec[o], y = feats[o], d = x - y;
      v = f1 + 2.f * x * f2 + y * f3 + (d > 0.f ? s_inv : (d < 0.f ? -s_inv : 0.f));
    }
    g_dec[o] = v;
  }
}

// the four scalars, and the duration loss with its gradient: weighted_mean(huber(pred, log(max(d, 1)), delta 1), token mask)
__global__ void __launch_bounds__(256)
ss_loss_finalize_kernel(const float* __restrict__ part, int nblk, const int32_t* __restrict__ num_frames, int batch, int l, int odim,
                        const float* __restrict__ pred, const int64_t* __restrict__ dur, const int32_t* __restrict__ num_phones, int t_max,
                        float* __restrict__ losses, float* __restrict__ g_dur) {
  __shared__ double red[256];
  __shared__ double s_tok;
  double s_ssim = 0.0, s_l1 = 0.0;
  for (int i = threadIdx.x; i < nblk; i += 256) { s_ssim += part[2 * i]; s_l1 += part[2 * i + 1]; }
  const double t_ssim = block_sum_tree<256>(s_ssim, red);
  const double t_l1 = block_sum_tree<256>(s_l1, red);
  if (threadIdx.x == 0) {
    long long toks = 0;
    for (int b = 0; b < batch; ++b) toks += max(min(num_phones[b], t_max), 0);
    s_tok = static_cast<double>(toks);
  }
  __syncthreads();
  const double inv_tok = s_tok > 0.0 ? 1.0 / s_tok : 0.0;
  double s_h = 0.0;
  for (int i = threadIdx.x; i < batch * t_max; i += 256) {
    const int b = i / t_max, t = i % t_max;
    float g = 0.f;
    if (t < num_phones[b]) {
      const float label = logf(fmaxf(static_cast<float>(dur[i]), 1.f));
      const float r = label - pred[i];
      if (fabsf(r) <= 1.f) { s_h += 0.5 * r * r; g = -r; }
      else { s_h += fabs(static_cast<double>(r)) - 0.5; g = r > 0.f ? -1.f : 1.f; }
    }
    if (g_dur) g_dur[i] = g * static_cast<float>(inv_tok);
  }
  const double t_h = block_sum_tree<256>(s_h, red);
  if (threadIdx.x == 0) {
    long long frames = 0;
    for (int b = 0; b < batch; ++b) frames += max(min(num_frames[b], l), 0);
    const double l1 = frames > 0 ? t_l1 / (static_cast<double>(frames) * odim) : 0.0;
    const double ssim = 1.0 - t_ssim / (static_cast<double>(batch) * l * odim);
    const double dl = t_h * inv_tok;
    losses[0] = static_cast<float>(l1 + ssim + dl);
    losses[1] = static_cast<float>(l1);
    losses[2] = static_cast<float>(dl);
    losses[3] = static_cast<float>(ssim);
  }
}

}  // namespace
}  // namespace pk

using namespace pk;

extern "C" int pk_ss_bn_train_fwd(const float* r, int64_t rows, int32_t c, const float* gamma, const float* beta, float eps, float momentum,
                                  float* run_mean, float* run_var, const float* residual, float* scratch, float* y, void* y_hi, void* y_lo,
                                  float* save_mean, float* save_rstd, pk_stream_t stream) {
  PK_CHECK_ARG(r && gamma && beta && scratch && save_mean && save_rstd, "NULL pointer");
  PK_CHECK_ARG(rows > 0 && rows < (1LL << 31) && eps > 0.f, "bad sizes");
  PK_CHECK_ARG((y || y_hi) && (y_hi == nullptr) == (y_lo == nullptr), "no output requested, or one split plane without the other");
  PK_CHECK_ARG((run_mean == nullptr) == (run_var == nullptr), "running mean and variance go together");
  if (c != kC) return fail(PK_ERR_UNSUPPORTED, "pk_ss_bn_train_fwd: channels must be %d (got %d)", kC, c);
  const int nblk = static_cast<int>((rows + kRows - 1) / kRows);
  ss_bn_stats_kernel<<<nblk, kThreads, 0, PK_STREAM>>>(r, rows, scratch);
  ss_bn_finalize_kernel<<<1, kFinalThreads, 0, PK_STREAM>>>(scratch, nblk, rows, eps, momentum, run_mean, run_var, save_mean, save_rstd);
  ss_bn_apply_kernel<<<nblk, kThreads, 0, PK_STREAM>>>(r, rows, save_mean, save_rstd, gamma, beta, residual, y,
                                                      static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo));
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch(3);
  return PK_OK;
}

extern "C" int pk_ss_bn_relu_bwd(const float* dy, const float* r, const float* mean, const float* rstd, const float* gamma, int64_t rows,
                                 int32_t c, float* scratch, float* dgamma, float* dbeta, float* dbias, float* dr, void* dr_hi, void* dr_lo,
                                 pk_stream_t stream) {
  PK_CHECK_ARG(dy && r && mean && rstd && gamma && scratch && dgamma && dbeta, "NULL pointer");
  PK_CHECK_ARG(rows > 0 && rows < (1LL << 31), "bad sizes");
  PK_CHECK_ARG((dr || dr_hi) && (dr_hi == nullptr) == (dr_lo == nullptr), "no output requested, or one split plane without the other");
  if (c != kC) return fail(PK_ERR_UNSUPPORTED, "pk_ss_bn_relu_bwd: channels must be %d (got %d)", kC, c);
  const int nblk = static_cast<int>((rows + kRows - 1) / kRows);
  ss_bn_bwd_stats_kernel<<<nblk, kThreads, 0, PK_STREAM>>>(dy, r, mean, rstd, rows, scratch);
  ss_colsum_finalize_kernel<<<1, kFinalThreads, 0, PK_STREAM>>>(scratch, nblk, 2 * kC, dbeta, dgamma);
  ss_bn_relu_bwd_apply_kernel<<<nblk, kThreads, 0, PK_STREAM>>>(dy, r, mean, rstd, gamma, dbeta, dgamma, rows, dr,
                                                               static_cast<__nv_bfloat16*>(dr_hi), static_cast<__nv_bfloat16*>(dr_lo), scratch);
  int launches = 3;
  if (dbias) {
    ss_colsum_finalize_kernel<<<1, kFinalThreads, 0, PK_STREAM>>>(scratch, nblk, kC, dbias, nullptr);
    ++launches;
  }
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch(launches);
  return PK_OK;
}

extern "C" int pk_ss_loss(const float* decoded, const float* feats, const int32_t* num_frames, int32_t batch, int32_t l, int32_t odim,
                          const float* pred_durations, const int64_t* durations, const int32_t* num_phones, int32_t t, float* scratch,
                          float* losses, float* g_decoded, float* g_durations, pk_stream_t stream) {
  PK_CHECK_ARG(decoded && feats && num_frames && pred_durations && durations && num_phones && scratch && losses, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && batch <= 65535 && l > 0 && t > 0, "bad sizes");
  PK_CHECK_ARG((g_decoded == nullptr) == (g_durations == nullptr), "the two gradients go together");
  if (odim < 1 || odim > kMaxMel) return fail(PK_ERR_UNSUPPORTED, "pk_ss_loss: odim must be in [1, %d] (got %d)", kMaxMel, odim);
  const long long n = static_cast<long long>(batch) * l * odim;
  dim3 grid((l + kTile - 1) / kTile, batch);
  const int nblk = static_cast<int>(grid.x) * batch;
  float* part = scratch;
  float* gmaps = g_decoded ? scratch + 2LL * nblk : nullptr;
  ss_ssim_fwd_kernel<<<grid, 256, 0, PK_STREAM>>>(decoded, feats, num_frames, l, odim, static_cast<float>(-1.0 / static_cast<double>(n)), gmaps, n,
                                                  part);
  ss_loss_finalize_kernel<<<1, 256, 0, PK_STREAM>>>(part, nblk, num_frames, batch, l, odim, pred_durations, durations, num_phones, t, losses,
                                                   g_durations);
  int launches = 2;
  if (g_decoded) {
    ss_ssim_bwd_kernel<<<grid, 256, 0, PK_STREAM>>>(decoded, feats, num_frames, batch, l, odim, gmaps, n, g_decoded);
    ++launches;
  }
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch(launches);
  return PK_OK;
}
