// Element-wise / reduction kernels of the Parallel WaveGAN training step (reference: PWGUpdater.update_core,
// parakeet/models/parallel_wavegan/parallel_wavegan_updater.py:76-153; SURVEY.md 8f.1).  The GEMM-shaped work of that step
// (every Conv1D forward, data gradient and weight gradient of generator and discriminator, the DFT of the STFT losses and its
// adjoint) runs through pk_conv_gemm on wgmma; this file holds what sits between the GEMMs:
//   gate (ResidualBlock :307-310) forward / backward, LeakyReLU forward / backward (PWGDiscriminator :579-582),
//   weight norm w = g v / ||v|| forward / backward (nn.utils.weight_norm, dim 0), MSE against a constant (criterion_mse),
//   the generator's residual / skip update, the upsampling stages (Stretch2D + FIR Conv2D, :48-63,119-138) one stage at a time
//   with their backward, the multi-resolution STFT loss gradient (modules/stft_loss.py:163-219) and the framing adjoint
//   (overlap-add through the reflect padding), the global gradient norm (ClipGradByGlobalNorm) that
//   pk_adam (train.cu) clips with.
#include <math.h>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace gan {

// block-wide sum -> one atomicAdd per block (double accumulator: the sums feed loss values and gradient norms)
__device__ __forceinline__ void block_accumulate(float v, double* out) {
  __shared__ float red[32];
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) atomicAdd(out, static_cast<double>(t));
  }
  __syncthreads();
}

// ---------------------------------------------------------------- gate
__global__ void gate_fwd_kernel(const float* __restrict__ h, long long rows, int c, float* __restrict__ z, __nv_bfloat16* __restrict__ z_hi,
                                __nv_bfloat16* __restrict__ z_lo) {
  PK_GRID_STRIDE(i, rows * c) {
    const long long r = i / c;
    const int k = static_cast<int>(i - r * c);
    const float a = h[r * 2 * c + k], g = h[r * 2 * c + c + k];
    const float v = tanhf(a) * (1.f / (1.f + expf(-g)));
    if (z) z[i] = v;
    if (z_hi) {
      __nv_bfloat16 hi, lo;
      split_bf16(v, hi, lo);
      z_hi[i] = hi; z_lo[i] = lo;
    }
  }
}
__global__ void gate_bwd_kernel(const float* __restrict__ h, const float* __restrict__ dz, long long rows, int c, float* __restrict__ dh) {
  PK_GRID_STRIDE(i, rows * c) {
    const long long r = i / c;
    const int k = static_cast<int>(i - r * c);
    const float a = h[r * 2 * c + k], g = h[r * 2 * c + c + k];
    const float t = tanhf(a), s = 1.f / (1.f + expf(-g)), d = dz[i];
    dh[r * 2 * c + k] = d * s * (1.f - t * t);
    dh[r * 2 * c + c + k] = d * t * s * (1.f - s);
  }
}

// ---------------------------------------------------------------- LeakyReLU
__global__ void leaky_fwd_kernel(const float* __restrict__ x, long long n, float slope, float* __restrict__ y, __nv_bfloat16* __restrict__ y_hi,
                                 __nv_bfloat16* __restrict__ y_lo) {
  PK_GRID_STRIDE(i, n) {
    const float v = x[i];
    const float o = v > 0.f ? v : v * slope;
    if (y) y[i] = o;
    if (y_hi) {
      __nv_bfloat16 hi, lo;
      split_bf16(o, hi, lo);
      y_hi[i] = hi; y_lo[i] = lo;
    }
  }
}
__global__ void leaky_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, long long n, float slope, float* __restrict__ dx) {
  PK_GRID_STRIDE(i, n) dx[i] = x[i] > 0.f ? dy[i] : dy[i] * slope;
}

// ---------------------------------------------------------------- weight norm (dim 0): one block per output channel
__global__ void weight_norm_fwd_kernel(const float* __restrict__ v, const float* __restrict__ g, int inner, float* __restrict__ w,
                                       float* __restrict__ norm_out) {
  const int r = blockIdx.x;
  __shared__ double s_norm;
  if (threadIdx.x == 0) s_norm = 0.0;
  __syncthreads();
  float acc = 0.f;
  for (int i = threadIdx.x; i < inner; i += blockDim.x) { const float t = v[static_cast<long long>(r) * inner + i]; acc = fmaf(t, t, acc); }
  block_accumulate(acc, &s_norm);
  const float nrm = sqrtf(static_cast<float>(s_norm));
  const float sc = g[r] / nrm;
  for (int i = threadIdx.x; i < inner; i += blockDim.x) w[static_cast<long long>(r) * inner + i] = v[static_cast<long long>(r) * inner + i] * sc;
  if (threadIdx.x == 0 && norm_out) norm_out[r] = nrm;
}
// dg = <dw, v> / ||v||;  dv = g / ||v|| * (dw - (<dw, v> / ||v||^2) v)
__global__ void weight_norm_bwd_kernel(const float* __restrict__ v, const float* __restrict__ g, const float* __restrict__ dw, int inner,
                                       float* __restrict__ dg, float* __restrict__ dv) {
  const int r = blockIdx.x;
  __shared__ double s_nn, s_dot;
  if (threadIdx.x == 0) { s_nn = 0.0; s_dot = 0.0; }
  __syncthreads();
  float nn = 0.f, dot = 0.f;
  for (int i = threadIdx.x; i < inner; i += blockDim.x) {
    const float t = v[static_cast<long long>(r) * inner + i];
    nn = fmaf(t, t, nn);
    dot = fmaf(t, dw[static_cast<long long>(r) * inner + i], dot);
  }
  block_accumulate(nn, &s_nn);
  block_accumulate(dot, &s_dot);
  const float n2 = static_cast<float>(s_nn), d = static_cast<float>(s_dot), nrm = sqrtf(n2);
  if (threadIdx.x == 0) dg[r] = d / nrm;
  const float gs = g[r] / nrm, proj = d / n2;
  for (int i = threadIdx.x; i < inner; i += blockDim.x)
    dv[static_cast<long long>(r) * inner + i] = gs * (dw[static_cast<long long>(r) * inner + i] - proj * v[static_cast<long long>(r) * inner + i]);
}

// ---------------------------------------------------------------- MSE against a constant: acc[0] += sum (x - t)^2; dx = coef (x - t)
__global__ void mse_const_kernel(const float* __restrict__ x, long long n, int ld, int col, float target, double* __restrict__ acc,
                                 float* __restrict__ dx, float coef) {
  float s = 0.f;
  PK_GRID_STRIDE(i, n) {
    const float d = x[i * ld + col] - target;
    s = fmaf(d, d, s);
    if (dx) dx[i * ld + col] = coef * d;
  }
  block_accumulate(s, acc);
}
__global__ void sq_sum_kernel(const float* __restrict__ x, long long n, double* __restrict__ acc) {
  float s = 0.f;
  PK_GRID_STRIDE(i, n) s = fmaf(x[i], x[i], s);
  block_accumulate(s, acc);
}
// ---------------------------------------------------------------- generator residual / skip update (parallel_wavegan.py:311-315, :466-468)
// so (rows, 128) = [skip | out] of conv1x1_skip / conv1x1_out (bias included); skips (=|+=) skip; x' = (out + x) * sqrt(1/2)
__global__ void pwg_res_update_kernel(const float* __restrict__ so, const float* __restrict__ x, long long rows, float* __restrict__ skips, int init,
                                      float* __restrict__ xo, __nv_bfloat16* __restrict__ xo_hi, __nv_bfloat16* __restrict__ xo_lo) {
  PK_GRID_STRIDE(i, rows * 64) {
    const long long r = i >> 6;
    const int k = static_cast<int>(i & 63);
    const float s = so[r * 128 + k];
    skips[i] = init ? s : skips[i] + s;
    const float o = (so[r * 128 + 64 + k] + x[i]) * 0.70710678118654752440f;
    xo[i] = o;
    __nv_bfloat16 hi, lo;
    split_bf16(o, hi, lo);
    xo_hi[i] = hi; xo_lo[i] = lo;
  }
}
// backward: dso = [dskips | dx' * sqrt(1/2)]; dx (+)= dx' * sqrt(1/2)   (dx accumulates: it already holds the conv's data gradient)
__global__ void pwg_res_update_bwd_kernel(const float* __restrict__ dskips, const float* __restrict__ dxo, long long rows, float* __restrict__ dso,
                                          float* __restrict__ dx_res) {
  PK_GRID_STRIDE(i, rows * 64) {
    const long long r = i >> 6;
    const int k = static_cast<int>(i & 63);
    const float d = dxo[i] * 0.70710678118654752440f;
    dso[r * 128 + k] = dskips[i];
    dso[r * 128 + 64 + k] = d;
    dx_res[i] = d;
  }
}

// ---------------------------------------------------------------- upsampling stage: Stretch2D (nearest, scale s) + FIR Conv2D(1,1,(1,2s+1), pad s)
// x (rows, tin) -> y (rows, tin * s):  y[t] = sum_q fir[q] * u[t + q - s],  u[j] = x[j / s] for 0 <= j < tin*s, else 0
__global__ void up_stage_fwd_kernel(const float* __restrict__ x, const float* __restrict__ fir, long long rows, int tin, int s, float* __restrict__ y) {
  const int tout = tin * s;
  PK_GRID_STRIDE(i, rows * tout) {
    const long long r = i / tout;
    const int t = static_cast<int>(i - r * tout);
    float acc = 0.f;
    for (int q = 0; q <= 2 * s; ++q) {
      const int j = t + q - s;
      if (j >= 0 && j < tout) acc = fmaf(fir[q], x[r * tin + j / s], acc);
    }
    y[i] = acc;
  }
}
// dx[j'] = sum_{t, q : (t + q - s) / s == j'} fir[q] dy[t]   (gather form: for each stretched position j of frame j', the taps that read it)
__global__ void up_stage_bwd_data_kernel(const float* __restrict__ dy, const float* __restrict__ fir, long long rows, int tin, int s,
                                         float* __restrict__ dx) {
  const int tout = tin * s;
  PK_GRID_STRIDE(i, rows * tin) {
    const long long r = i / tin;
    const int jf = static_cast<int>(i - r * tin);
    float acc = 0.f;
    for (int j = jf * s; j < (jf + 1) * s; ++j)
      for (int q = 0; q <= 2 * s; ++q) {
        const int t = j - q + s;
        if (t >= 0 && t < tout) acc = fmaf(fir[q], dy[r * tout + t], acc);
      }
    dx[i] = acc;
  }
}
// dfir[q] += sum_{r, t} dy[t] u[t + q - s]; one block per (q, slice of rows)
__global__ void up_stage_bwd_fir_kernel(const float* __restrict__ x, const float* __restrict__ dy, long long rows, int tin, int s,
                                        double* __restrict__ dfir) {
  const int q = blockIdx.y;
  const int tout = tin * s;
  float acc = 0.f;
  PK_GRID_STRIDE(i, rows * tout) {
    const long long r = i / tout;
    const int t = static_cast<int>(i - r * tout);
    const int j = t + q - s;
    if (j >= 0 && j < tout) acc = fmaf(dy[i], x[r * tin + j / s], acc);
  }
  block_accumulate(acc, dfir + q);
}

// ---------------------------------------------------------------- multi-resolution STFT loss gradient (modules/stft_loss.py:20-219)
// mag = sqrt(clip(re^2 + im^2, 1e-7));  sc = ||M_y - M_x||_F / ||M_y||_F;  lm = mean |log M_y - log M_x|   (x = generated, y = target)
// sums[0] = sum (M_y - M_x)^2, sums[1] = sum M_y^2 (device fp32, from pk_spectral_loss_sums).  Gradient w.r.t. re / im of X for weight w_res on both
// terms, written as a (B * frames, 2 * bins_p) row-major matrix [re | im] (bins padded to bins_p, zeros in the padding) for the adjoint DFT GEMM.
__global__ void stft_loss_grad_kernel(const float* __restrict__ xre, const float* __restrict__ xim, const float* __restrict__ yre,
                                      const float* __restrict__ yim, int batch, int bins, int frames, int bins_p, const float* __restrict__ sums,
                                      float w_res, float* __restrict__ g) {
  const long long n = static_cast<long long>(batch) * bins * frames;
  const float diff_norm = sqrtf(sums[0]), y_norm = sqrtf(sums[1]);
  const float c_sc = w_res / fmaxf(diff_norm * y_norm, 1e-30f);
  const float c_lm = w_res / static_cast<float>(n);
  PK_GRID_STRIDE(i, n) {
    const int f = static_cast<int>(i % frames);
    const int k = static_cast<int>((i / frames) % bins);
    const int b = static_cast<int>(i / (static_cast<long long>(frames) * bins));
    const float xr = xre[i], xi = xim[i], yr = yre[i], yi = yim[i];
    const float px = xr * xr + xi * xi, py = yr * yr + yi * yi;
    const float mx = sqrtf(fmaxf(px, 1e-7f)), my = sqrtf(fmaxf(py, 1e-7f));
    // d loss / d mx
    float dm = c_sc * (mx - my);
    const float dl = logf(my) - logf(mx);
    dm += c_lm * (dl > 0.f ? -1.f : (dl < 0.f ? 1.f : 0.f)) / mx;
    // mx = sqrt(clip(p, 1e-7)): zero gradient where the clip is active
    const float s = px > 1e-7f ? dm / mx : 0.f;
    float* row = g + (static_cast<long long>(b) * frames + f) * 2 * bins_p;
    row[k] = s * xr;
    row[bins_p + k] = s * xi;
  }
}
// frames_grad (B * frames, n_fft) (already multiplied by the DFT adjoint) -> dx (B, T): window, overlap-add, fold the reflect padding back
__global__ void frames_overlap_add_kernel(const float* __restrict__ fg, const float* __restrict__ win, int batch, int frames, int n_fft, int hop,
                                          int t, float* __restrict__ dx) {
  const long long n = static_cast<long long>(batch) * frames * n_fft;
  const int pad = n_fft / 2;
  PK_GRID_STRIDE(i, n) {
    const int k = static_cast<int>(i % n_fft);
    const int f = static_cast<int>((i / n_fft) % frames);
    const int b = static_cast<int>(i / (static_cast<long long>(n_fft) * frames));
    int pos = f * hop + k - pad;                 // position in the un-padded signal; reflect (no edge repeat) outside [0, t)
    if (pos < 0) pos = -pos;
    if (pos >= t) pos = 2 * (t - 1) - pos;
    if (pos >= 0 && pos < t) atomicAdd(dx + static_cast<long long>(b) * t + pos, fg[i] * win[k]);
  }
}

// y (rows, c) += column bias; used nowhere else: the conv GEMMs carry their biases themselves
}  // namespace gan
}  // namespace pk

extern "C" int pk_gate_fwd(const float* h, int64_t rows, int32_t c, float* z, void* z_hi, void* z_lo, pk_stream_t stream) {
  PK_CHECK_ARG(h && rows > 0 && c > 0 && (z || z_hi) && (z_hi == nullptr) == (z_lo == nullptr), "bad arguments");
  pk::gan::gate_fwd_kernel<<<pk::grid_stride_blocks(rows * c, 256), 256, 0, PK_STREAM>>>(h, rows, c, z, static_cast<__nv_bfloat16*>(z_hi), static_cast<__nv_bfloat16*>(z_lo));
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_gate_bwd(const float* h, const float* dz, int64_t rows, int32_t c, float* dh, pk_stream_t stream) {
  PK_CHECK_ARG(h && dz && dh && rows > 0 && c > 0, "bad arguments");
  pk::gan::gate_bwd_kernel<<<pk::grid_stride_blocks(rows * c, 256), 256, 0, PK_STREAM>>>(h, dz, rows, c, dh);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_leaky_relu(const float* x, int64_t n, float slope, float* y, void* y_hi, void* y_lo, pk_stream_t stream) {
  PK_CHECK_ARG(x && n > 0 && (y || y_hi) && (y_hi == nullptr) == (y_lo == nullptr), "bad arguments");
  pk::gan::leaky_fwd_kernel<<<pk::grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(x, n, slope, y, static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo));
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_leaky_relu_bwd(const float* x, const float* dy, int64_t n, float slope, float* dx, pk_stream_t stream) {
  PK_CHECK_ARG(x && dy && dx && n > 0, "bad arguments");
  pk::gan::leaky_bwd_kernel<<<pk::grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(x, dy, n, slope, dx);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_weight_norm_fwd(const float* v, const float* g, int32_t rows, int32_t inner, float* w, float* norm, pk_stream_t stream) {
  PK_CHECK_ARG(v && g && w && rows > 0 && inner > 0, "bad arguments");
  pk::gan::weight_norm_fwd_kernel<<<rows, 128, 0, PK_STREAM>>>(v, g, inner, w, norm);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_weight_norm_bwd(const float* v, const float* g, const float* dw, int32_t rows, int32_t inner, float* dg, float* dv,
                                  pk_stream_t stream) {
  PK_CHECK_ARG(v && g && dw && dg && dv && rows > 0 && inner > 0, "bad arguments");
  pk::gan::weight_norm_bwd_kernel<<<rows, 128, 0, PK_STREAM>>>(v, g, dw, inner, dg, dv);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_mse_const(const float* x, int64_t n, int32_t ld, int32_t col, float target, double* acc, float* dx, float coef,
                            pk_stream_t stream) {
  PK_CHECK_ARG(x && acc && n > 0 && ld > 0 && col >= 0 && col < ld, "bad arguments");
  pk::gan::mse_const_kernel<<<pk::grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(x, n, ld, col, target, acc, dx, coef);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_sq_sum(const float* x, int64_t n, double* acc, pk_stream_t stream) {
  PK_CHECK_ARG(x && acc && n > 0, "bad arguments");
  pk::gan::sq_sum_kernel<<<std::min(pk::grid_stride_blocks(n, 256), 2048), 256, 0, PK_STREAM>>>(x, n, acc);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_pwg_res_update(const float* so, const float* x, int64_t rows, float* skips, int32_t init, float* xo, void* xo_hi, void* xo_lo,
                                 pk_stream_t stream) {
  PK_CHECK_ARG(so && x && skips && xo && xo_hi && xo_lo && rows > 0, "bad arguments");
  pk::gan::pwg_res_update_kernel<<<pk::grid_stride_blocks(rows * 64, 256), 256, 0, PK_STREAM>>>(so, x, rows, skips, init, xo, static_cast<__nv_bfloat16*>(xo_hi),
                                                                                                static_cast<__nv_bfloat16*>(xo_lo));
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_pwg_res_update_bwd(const float* dskips, const float* dxo, int64_t rows, float* dso, float* dx_res, pk_stream_t stream) {
  PK_CHECK_ARG(dskips && dxo && dso && dx_res && rows > 0, "bad arguments");
  pk::gan::pwg_res_update_bwd_kernel<<<pk::grid_stride_blocks(rows * 64, 256), 256, 0, PK_STREAM>>>(dskips, dxo, rows, dso, dx_res);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_up_stage_fwd(const float* x, const float* fir, int64_t rows, int32_t tin, int32_t s, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(x && fir && y && rows > 0 && tin > 0 && s >= 1, "bad arguments");
  pk::gan::up_stage_fwd_kernel<<<pk::grid_stride_blocks(rows * tin * s, 256), 256, 0, PK_STREAM>>>(x, fir, rows, tin, s, y);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_up_stage_bwd(const float* x, const float* dy, const float* fir, int64_t rows, int32_t tin, int32_t s, float* dx, double* dfir,
                               pk_stream_t stream) {
  PK_CHECK_ARG(x && dy && fir && rows > 0 && tin > 0 && s >= 1 && (dx || dfir), "bad arguments");
  if (dx) pk::gan::up_stage_bwd_data_kernel<<<pk::grid_stride_blocks(rows * tin, 256), 256, 0, PK_STREAM>>>(dy, fir, rows, tin, s, dx);
  if (dfir) {
    dim3 grid(std::min(pk::grid_stride_blocks(rows * tin * s, 256), 512), 2 * s + 1);
    pk::gan::up_stage_bwd_fir_kernel<<<grid, 256, 0, PK_STREAM>>>(x, dy, rows, tin, s, dfir);
  }
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_stft_loss_grad(const float* xre, const float* xim, const float* yre, const float* yim, int32_t batch, int32_t bins,
                                 int32_t frames, int32_t bins_p, const float* sums, float weight, float* g, pk_stream_t stream) {
  PK_CHECK_ARG(xre && xim && yre && yim && sums && g && batch > 0 && bins > 0 && frames > 0 && bins_p >= bins, "bad arguments");
  pk::gan::stft_loss_grad_kernel<<<pk::grid_stride_blocks(static_cast<long long>(batch) * bins * frames, 256), 256, 0, PK_STREAM>>>(
      xre, xim, yre, yim, batch, bins, frames, bins_p, sums, weight, g);
  PK_LAUNCH_DONE(1);
}
extern "C" int pk_frames_overlap_add(const float* frames_grad, const float* window, int32_t batch, int32_t frames, int32_t n_fft, int32_t hop,
                                     int32_t t, float* dx, pk_stream_t stream) {
  PK_CHECK_ARG(frames_grad && window && dx && batch > 0 && frames > 0 && n_fft > 0 && hop > 0 && t > n_fft / 2, "bad arguments");
  pk::gan::frames_overlap_add_kernel<<<pk::grid_stride_blocks(static_cast<long long>(batch) * frames * n_fft, 256), 256, 0, PK_STREAM>>>(
      frames_grad, window, batch, frames, n_fft, hop, t, dx);
  PK_LAUNCH_DONE(1);
}
