// WaveFlow training step (reference: examples/waveflow/train.py:95-118 Experiment.train_batch - ConditionalWaveFlow.forward
// parakeet/models/waveflow.py:759-783, WaveFlowLoss :855-891, loss.backward(), Adam).  Every GEMM of the step (the 3x3 conv,
// condition_proj and out_proj of each ResidualBlock in both directions, the weight gradients) runs through pk_conv_gemm on
// wgmma; this file holds the pieces in between.
//
// Positions of one flow's residual net live in the "net layout" (batch * (n_group + 1), width, channels): utterance b owns rows
// b * (G + 1) + j, j < G - 1 are its net rows (the flow's heights 1 .. G-1) and the last two rows are zero.  The layer inputs
// are kept as split planes in the "input layout", the same allocation shifted by two rows (two zero rows BEFORE each
// utterance's net rows: the causal height padding), so that output row q of the 3x3 conv reads input rows q, q + 1, q + 2.
//
// No reduction here uses atomics: every sum over positions is a fixed-order per-block partial followed by a fixed-order sum
// of the partials, so a step is bit-for-bit reproducible.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace wft {

__device__ __forceinline__ void store_split(float v, __nv_bfloat16* hi, __nv_bfloat16* lo, long long i) {
  __nv_bfloat16 h, l;
  split_bf16(v, h, l);
  hi[i] = h;
  lo[i] = l;
}

__global__ void gather_split_kernel(const float* __restrict__ src, const int32_t* __restrict__ idx, long long n, __nv_bfloat16* hi,
                                    __nv_bfloat16* lo) {
  PK_GRID_STRIDE(i, n) {
    const int32_t j = idx[i];
    store_split(j >= 0 ? src[j] : 0.f, hi, lo, i);
  }
}

// input_proj (1x1 Conv2D 1 -> C) of the flow input rows 0 .. G-2
__global__ void input_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b, int G, int W, int C,
                                 long long n, float* __restrict__ h, __nv_bfloat16* x_hi, __nv_bfloat16* x_lo) {
  PK_GRID_STRIDE(i, n) {                                   // n = batch * (G + 1) * W * C, net layout
    const int c = static_cast<int>(i % C);
    const long long p = i / C;                              // position q * W + w
    const long long q = p / W;
    const int w_ = static_cast<int>(p - q * W);
    const int bb = static_cast<int>(q / (G + 1)), j = static_cast<int>(q - static_cast<long long>(bb) * (G + 1));
    float v = 0.f;
    if (j <= G - 2) {
      v = fmaf(w[c], x[(static_cast<long long>(bb) * G + j) * W + w_], b[c]);
      store_split(v, x_hi, x_lo, i + 2LL * W * C);         // input layout: two rows further
    }
    h[i] = v;
  }
}

// h += res, skip (= or +=) skip_part; next layer input planes <- h
__global__ void update_kernel(const float* __restrict__ out, int G, int W, int C, long long n, float* __restrict__ h, float* __restrict__ skip,
                              int skip_init, __nv_bfloat16* x_hi, __nv_bfloat16* x_lo) {
  PK_GRID_STRIDE(i, n) {
    const int c = static_cast<int>(i % C);
    const long long p = i / C;
    const float res = out[p * 2 * C + c], sk = out[p * 2 * C + C + c];
    const float v = h[i] + res;
    h[i] = v;
    skip[i] = skip_init ? sk : skip[i] + sk;
    if (x_hi) {
      const long long q = p / W;
      if (q % (G + 1) <= G - 2) store_split(v, x_hi, x_lo, i + 2LL * W * C);
    }
  }
}

// one warp per (b, h, w): output_proj of the skip sum, z = x exp(logs) + b, the height permutation
__global__ void tail_fwd_kernel(const float* __restrict__ skip, const float* __restrict__ out_w, const float* __restrict__ out_b,
                                const float* __restrict__ x, const int32_t* __restrict__ inv_perm, int B, int G, int W, int C,
                                float* __restrict__ x_next, float* __restrict__ logs_out) {
  const long long warps = static_cast<long long>(B) * G * W;
  const int lane = threadIdx.x & 31;
  for (long long t = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; t < warps;
       t += (static_cast<long long>(gridDim.x) * blockDim.x) >> 5) {
    const int w_ = static_cast<int>(t % W);
    const long long bh = t / W;
    const int hh = static_cast<int>(bh % G), bb = static_cast<int>(bh / G);
    const float xv = x[t];
    float zv = xv;
    if (hh > 0) {
      const float* s = skip + ((static_cast<long long>(bb) * (G + 1) + hh - 1) * W + w_) * C;
      float a0 = 0.f, a1 = 0.f;
      for (int c = lane; c < C; c += 32) {
        a0 = fmaf(out_w[c], s[c], a0);
        a1 = fmaf(out_w[C + c], s[c], a1);
      }
      const float logs = warp_sum(a0) + out_b[0], bias = warp_sum(a1) + out_b[1];
      zv = fmaf(xv, expf(logs), bias);
      if (lane == 0) logs_out[(static_cast<long long>(bb) * (G - 1) + hh - 1) * W + w_] = logs;
    }
    if (lane == 0) x_next[(static_cast<long long>(bb) * G + inv_perm[hh]) * W + w_] = zv;
  }
}

// backward of tail_fwd_kernel: dx (direct path, overwritten), d(logs, b) per position, dskip (fp32 and split planes)
__global__ void tail_bwd_kernel(const float* __restrict__ skip, const float* __restrict__ out_w, const float* __restrict__ out_b,
                                const float* __restrict__ x, const int32_t* __restrict__ inv_perm, const float* __restrict__ dy,
                                const float* __restrict__ y, float y_coef, float dlogs_const, int B, int G, int W, int C,
                                float* __restrict__ dx, float* __restrict__ dparams, float* __restrict__ dskip, __nv_bfloat16* ds_hi,
                                __nv_bfloat16* ds_lo, int ds_ld, int ds_col0) {
  const long long warps = static_cast<long long>(B) * G * W;
  const int lane = threadIdx.x & 31;
  for (long long t = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; t < warps;
       t += (static_cast<long long>(gridDim.x) * blockDim.x) >> 5) {
    const int w_ = static_cast<int>(t % W);
    const long long bh = t / W;
    const int hh = static_cast<int>(bh % G), bb = static_cast<int>(bh / G);
    const long long o = (static_cast<long long>(bb) * G + inv_perm[hh]) * W + w_;
    const float dz = dy ? dy[o] : y_coef * y[o];
    if (hh == 0) {
      if (lane == 0) dx[t] = dz;
      continue;
    }
    const long long p = (static_cast<long long>(bb) * (G + 1) + hh - 1) * W + w_;
    const float* s = skip + p * C;
    float a0 = 0.f;
    for (int c = lane; c < C; c += 32) a0 = fmaf(out_w[c], s[c], a0);
    const float logs = warp_sum(a0) + out_b[0];
    const float e = expf(logs), xv = x[t];
    const float dl = dz * xv * e + dlogs_const, db = dz;
    if (lane == 0) {
      dx[t] = dz * e;
      dparams[2 * p] = dl;
      dparams[2 * p + 1] = db;
    }
    for (int c = lane; c < C; c += 32) {
      const float v = fmaf(out_w[c], dl, out_w[C + c] * db);
      dskip[p * C + c] = v;
      store_split(v, ds_hi, ds_lo, p * ds_ld + ds_col0 + c);
    }
  }
}

// backward of input_fwd_kernel's data path: dx[b, j, w] += sum_c w[c] dh[q, w, c]; xcol[q * W + w] = x[b, j, w]
__global__ void input_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ x, const float* __restrict__ w, int B, int G, int W,
                                 int C, float* __restrict__ dx, float* __restrict__ xcol) {
  const long long warps = static_cast<long long>(B) * (G - 1) * W;
  const int lane = threadIdx.x & 31;
  for (long long t = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; t < warps;
       t += (static_cast<long long>(gridDim.x) * blockDim.x) >> 5) {
    const int w_ = static_cast<int>(t % W);
    const long long bj = t / W;
    const int j = static_cast<int>(bj % (G - 1)), bb = static_cast<int>(bj / (G - 1));
    const long long p = (static_cast<long long>(bb) * (G + 1) + j) * W + w_;
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a = fmaf(w[c], dh[p * C + c], a);
    a = warp_sum(a);
    if (lane == 0) {
      const long long xi = (static_cast<long long>(bb) * G + j) * W + w_;
      dx[xi] += a;
      xcol[p] = x[xi];
    }
  }
}

// partials[blk][i * kb + j] = sum over this block's rows of a[r * lda + i] * (b ? b[r * ldb + j] : 1)
__global__ void __launch_bounds__(256) outer_partial_kernel(const float* __restrict__ a, int lda, int ka, const float* __restrict__ b, int ldb,
                                                            int kb, long long rows, long long chunk, float* __restrict__ partials) {
  const int t = threadIdx.x;
  if (t >= ka * kb) return;
  const int i = t / kb, j = t - i * kb;
  const long long r0 = blockIdx.x * chunk, r1 = r0 + chunk < rows ? r0 + chunk : rows;
  float acc = 0.f;
  for (long long r = r0; r < r1; ++r) acc = fmaf(a[r * lda + i], b ? b[r * ldb + j] : 1.f, acc);
  partials[static_cast<long long>(blockIdx.x) * ka * kb + t] = acc;
}
__global__ void sum_partials_kernel(const float* __restrict__ partials, int nparts, int stride, int ka, int kb, float* __restrict__ out,
                                    long long os_i, long long os_j, int accumulate) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ka * kb) return;
  float acc = 0.f;
  for (int s = 0; s < nparts; ++s) acc += partials[static_cast<long long>(s) * stride + t];
  const int i = t / kb, j = t - i * kb;
  float* o = out + i * os_i + j * os_j;
  *o = accumulate ? *o + acc : acc;
}

// upsampler backward, leaky_relu part: dpre = dy * (y > 0 ? 1 : slope) (y the post-activation; slope > 0 keeps the sign)
__global__ void leaky_bwd_post_kernel(const float* __restrict__ y, const float* __restrict__ dy, long long n, float slope, float* __restrict__ dpre) {
  PK_GRID_STRIDE(i, n) dpre[i] = y[i] > 0.f ? dy[i] : slope * dy[i];
}
// dx[b, ih, iw] = sum_{kh, kw} w[kh, kw] dpre[b, ih - 1 + kh, iw f - f/2 + kw]
__global__ void upsample_dx_kernel(const float* __restrict__ dpre, const float* __restrict__ w, int M, int t_in, int f, int t_out, long long n,
                                   float* __restrict__ dx) {
  PK_GRID_STRIDE(i, n) {
    const int iw = static_cast<int>(i % t_in);
    const long long bm = i / t_in;
    const int m = static_cast<int>(bm % M);
    const long long base = (bm - m) * t_out;
    float acc = 0.f;
    for (int kh = 0; kh < 3; ++kh) {
      const int mo = m - 1 + kh;
      if (mo < 0 || mo >= M) continue;
      const float* row = dpre + base + static_cast<long long>(mo) * t_out;
      for (int kw = 0; kw < 2 * f; ++kw) {
        const int t = iw * f - f / 2 + kw;
        if (t >= 0 && t < t_out) acc = fmaf(w[kh * 2 * f + kw], row[t], acc);
      }
    }
    dx[i] = acc;
  }
}
// per block of `rows_per_block` input rows (b, ih): thread kh * 2f + kw accumulates x[b, ih, iw] * dpre[b, ih - 1 + kh, iw f - f/2 + kw],
// thread 6f the bias sum of dpre over the same rows (as output rows)
__global__ void upsample_dw_partial_kernel(const float* __restrict__ x, const float* __restrict__ dpre, int B, int M, int t_in, int f, int t_out,
                                           int rows_per_block, float* __restrict__ partials) {
  const int t = threadIdx.x, nw = 6 * f;
  if (t > nw) return;
  const long long r0 = static_cast<long long>(blockIdx.x) * rows_per_block, all = static_cast<long long>(B) * M;
  const long long r1 = r0 + rows_per_block < all ? r0 + rows_per_block : all;
  float acc = 0.f;
  if (t == nw) {
    for (long long r = r0; r < r1; ++r)
      for (int tt = 0; tt < t_out; ++tt) acc += dpre[r * t_out + tt];
  } else {
    const int kh = t / (2 * f), kw = t - kh * 2 * f;
    for (long long r = r0; r < r1; ++r) {
      const int m = static_cast<int>(r % M), mo = m - 1 + kh;
      if (mo < 0 || mo >= M) continue;
      const float* xr = x + r * t_in;
      const float* dr = dpre + (r - m + mo) * t_out;
      for (int iw = 0; iw < t_in; ++iw) {
        const int tt = iw * f - f / 2 + kw;
        if (tt >= 0 && tt < t_out) acc = fmaf(xr[iw], dr[tt], acc);
      }
    }
  }
  partials[static_cast<long long>(blockIdx.x) * (nw + 1) + t] = acc;
}

// condition of one flow, gathered into the net layout: row (b, j) <- condition height rows[j + 1]; (batch, n_mels, t_cond) -> split planes
__global__ void cond_gather_kernel(const float* __restrict__ cond, const int32_t* __restrict__ rows, int G, int W, int M, int t_cond, long long n,
                                   __nv_bfloat16* hi, __nv_bfloat16* lo) {
  PK_GRID_STRIDE(i, n) {
    const int m = static_cast<int>(i % M);
    const long long p = i / M, q = p / W;
    const int w_ = static_cast<int>(p - q * W);
    const int bb = static_cast<int>(q / (G + 1)), j = static_cast<int>(q - static_cast<long long>(bb) * (G + 1));
    const float v = j <= G - 2 ? cond[(static_cast<long long>(bb) * M + m) * t_cond + static_cast<long long>(w_) * G + rows[j + 1]] : 0.f;
    store_split(v, hi, lo, i);
  }
}
// its adjoint, accumulated: dcond[b, m, w G + rows[j + 1]] += dc[(q W + w) M + m]
__global__ void cond_scatter_kernel(const float* __restrict__ dc, const int32_t* __restrict__ rows, int B, int G, int W, int M, int t_cond,
                                    float* __restrict__ dcond) {
  const long long n = static_cast<long long>(B) * (G - 1) * W * M;
  PK_GRID_STRIDE(i, n) {
    const int m = static_cast<int>(i % M);
    const long long p = i / M;
    const int w_ = static_cast<int>(p % W);
    const long long bj = p / W;
    const int j = static_cast<int>(bj % (G - 1)), bb = static_cast<int>(bj / (G - 1));
    const long long src = ((static_cast<long long>(bb) * (G + 1) + j) * W + w_) * M + m;
    dcond[(static_cast<long long>(bb) * M + m) * t_cond + static_cast<long long>(w_) * G + rows[j + 1]] += dc[src];
  }
}

// WaveFlowLoss in one block: (sum z^2 / (2 sigma^2) - sum logs) / n + log(2 pi) / 2 + log(sigma); double, fixed order
__global__ void __launch_bounds__(1024) loss_kernel(const float* __restrict__ z, long long n, const float* __restrict__ logs, long long n_logs,
                                                    float sigma, float* __restrict__ loss) {
  __shared__ double s_z[1024], s_l[1024];
  double az = 0.0, al = 0.0;
  for (long long i = threadIdx.x; i < n; i += 1024) az += static_cast<double>(z[i]) * z[i];
  for (long long i = threadIdx.x; i < n_logs; i += 1024) al += logs[i];
  s_z[threadIdx.x] = az;
  s_l[threadIdx.x] = al;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      s_z[threadIdx.x] += s_z[threadIdx.x + s];
      s_l[threadIdx.x] += s_l[threadIdx.x + s];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double sg = sigma;
    loss[0] = static_cast<float>((s_z[0] / (2.0 * sg * sg) - s_l[0]) / static_cast<double>(n) + 0.5 * log(2.0 * M_PI) + log(sg));
  }
}

}  // namespace wft
}  // namespace pk

using namespace pk;
using namespace pk::wft;
#define BF(p) static_cast<__nv_bfloat16*>(p)

extern "C" int pk_waveflow_train_gather_split(const float* src, const int32_t* idx, int64_t n, void* dst_hi, void* dst_lo, pk_stream_t stream) {
  PK_CHECK_ARG(src && idx && dst_hi && dst_lo && n > 0, "bad arguments");
  gather_split_kernel<<<grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(src, idx, n, BF(dst_hi), BF(dst_lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_input_fwd(const float* x, const float* w, const float* bias, int32_t batch, int32_t n_group, int32_t width, int32_t c,
                                float* h, void* x_hi, void* x_lo, pk_stream_t stream) {
  PK_CHECK_ARG(x && w && bias && h && x_hi && x_lo && batch > 0 && n_group >= 2 && width > 0 && c > 0, "bad arguments");
  const long long n = static_cast<long long>(batch) * (n_group + 1) * width * c;
  input_fwd_kernel<<<grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(x, w, bias, n_group, width, c, n, h, BF(x_hi), BF(x_lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_update(const float* out, int32_t batch, int32_t n_group, int32_t width, int32_t c, float* h, float* skip, int32_t skip_init,
                             void* x_hi, void* x_lo, pk_stream_t stream) {
  PK_CHECK_ARG(out && h && skip && batch > 0 && n_group >= 2 && width > 0 && c > 0 && (x_hi == nullptr) == (x_lo == nullptr), "bad arguments");
  const long long n = static_cast<long long>(batch) * (n_group + 1) * width * c;
  update_kernel<<<grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(out, n_group, width, c, n, h, skip, skip_init, BF(x_hi), BF(x_lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_tail_fwd(const float* skip, const float* out_w, const float* out_b, const float* x, const int32_t* inv_perm, int32_t batch,
                               int32_t n_group, int32_t width, int32_t c, float* x_next, float* logs, pk_stream_t stream) {
  PK_CHECK_ARG(skip && out_w && out_b && x && inv_perm && x_next && logs && x != x_next && batch > 0 && n_group >= 2 && width > 0 && c > 0,
               "bad arguments");
  const long long warps = static_cast<long long>(batch) * n_group * width;
  tail_fwd_kernel<<<grid_stride_blocks(warps * 32, 256), 256, 0, PK_STREAM>>>(skip, out_w, out_b, x, inv_perm, batch, n_group, width, c, x_next, logs);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_forward_tail_bwd(const float* skip, const float* out_w, const float* out_b, const float* x, const int32_t* inv_perm, const float* dy,
                               const float* y, float y_coef, float dlogs, int32_t batch, int32_t n_group, int32_t width, int32_t c, float* dx,
                               float* dparams, float* dskip, void* ds_hi, void* ds_lo, int32_t ds_ld, int32_t ds_col0, pk_stream_t stream) {
  PK_CHECK_ARG(skip && out_w && out_b && x && inv_perm && (dy || y) && dx && dparams && dskip && ds_hi && ds_lo && batch > 0 && n_group >= 2 &&
               width > 0 && c > 0 && ds_col0 + c <= ds_ld, "bad arguments");
  const long long warps = static_cast<long long>(batch) * n_group * width;
  tail_bwd_kernel<<<grid_stride_blocks(warps * 32, 256), 256, 0, PK_STREAM>>>(skip, out_w, out_b, x, inv_perm, dy, y, y_coef, dlogs, batch, n_group, width, c, dx,
                                                                              dparams, dskip, BF(ds_hi), BF(ds_lo), ds_ld, ds_col0);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_input_bwd(const float* dh, const float* x, const float* w, int32_t batch, int32_t n_group, int32_t width, int32_t c, float* dx,
                                float* xcol, pk_stream_t stream) {
  PK_CHECK_ARG(dh && x && w && dx && xcol && batch > 0 && n_group >= 2 && width > 0 && c > 0, "bad arguments");
  const long long warps = static_cast<long long>(batch) * (n_group - 1) * width;
  input_bwd_kernel<<<grid_stride_blocks(warps * 32, 256), 256, 0, PK_STREAM>>>(dh, x, w, batch, n_group, width, c, dx, xcol);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_outer_sum(const float* a, int32_t lda, int32_t ka, const float* b, int32_t ldb, int32_t kb, int64_t rows, float* scratch,
                                int64_t scratch_len, float* out, int64_t os_i, int64_t os_j, int32_t accumulate, pk_stream_t stream) {
  PK_CHECK_ARG(a && scratch && out && ka > 0 && kb > 0 && ka * kb <= 256 && rows > 0 && lda >= ka && (b == nullptr || ldb >= kb),
               "bad arguments (ka * kb <= 256)");
  const int nparts = static_cast<int>(std::min<long long>(std::min<long long>(1024, (rows + 63) / 64), scratch_len / (ka * kb)));
  PK_CHECK_ARG(nparts >= 1, "scratch too small");
  const long long chunk = (rows + nparts - 1) / nparts;
  const int used = static_cast<int>((rows + chunk - 1) / chunk);
  outer_partial_kernel<<<used, 256, 0, PK_STREAM>>>(a, lda, ka, b, ldb, kb, rows, chunk, scratch);
  PK_CHECK_CUDA(cudaGetLastError());
  sum_partials_kernel<<<(ka * kb + 255) / 256, 256, 0, PK_STREAM>>>(scratch, used, ka * kb, ka, kb, out, os_i, os_j, accumulate);
  PK_LAUNCH_DONE(2);
}

extern "C" int pk_waveflow_upsample_bwd(const float* x, const float* y, const float* dy, const float* w, int32_t batch, int32_t c, int32_t t_in,
                                   int32_t factor, float slope, float* dpre, float* dx, float* scratch, int64_t scratch_len, float* dw, float* db,
                                   pk_stream_t stream) {
  PK_CHECK_ARG(x && y && dy && w && dpre && scratch && dw && db && batch > 0 && c > 0 && t_in > 0 && factor >= 2 && factor % 2 == 0 &&
               6 * factor + 1 <= 256 && slope > 0.f, "bad arguments");
  const int t_out = t_in * factor;
  const long long n_out = static_cast<long long>(batch) * c * t_out, rows = static_cast<long long>(batch) * c;
  const int per = 6 * factor + 1;
  const int rows_per_block = static_cast<int>(std::max<long long>(std::max<long long>(1, (rows + 1023) / 1024), (rows * per + scratch_len - 1) / scratch_len));
  const int nparts = static_cast<int>((rows + rows_per_block - 1) / rows_per_block);
  PK_CHECK_ARG(static_cast<long long>(nparts) * per <= scratch_len, "scratch too small");
  leaky_bwd_post_kernel<<<grid_stride_blocks(n_out, 256), 256, 0, PK_STREAM>>>(y, dy, n_out, slope, dpre);
  if (dx) upsample_dx_kernel<<<grid_stride_blocks(rows * t_in, 256), 256, 0, PK_STREAM>>>(dpre, w, c, t_in, factor, t_out, rows * t_in, dx);
  upsample_dw_partial_kernel<<<nparts, 128 * ((per + 127) / 128), 0, PK_STREAM>>>(x, dpre, batch, c, t_in, factor, t_out, rows_per_block, scratch);
  sum_partials_kernel<<<1, 256, 0, PK_STREAM>>>(scratch, nparts, per, per - 1, 1, dw, 1, 0, 0);
  sum_partials_kernel<<<1, 32, 0, PK_STREAM>>>(scratch + (per - 1), nparts, per, 1, 1, db, 0, 0, 0);
  PK_LAUNCH_DONE(dx ? 5 : 4);
}

extern "C" int pk_waveflow_train_cond_gather(const float* cond, const int32_t* rows, int32_t batch, int32_t n_group, int32_t width, int32_t n_mels, int32_t t_cond,
                                  void* hi, void* lo, pk_stream_t stream) {
  PK_CHECK_ARG(cond && rows && hi && lo && batch > 0 && n_group >= 2 && width > 0 && n_mels > 0 && t_cond >= width * n_group, "bad arguments");
  const long long n = static_cast<long long>(batch) * (n_group + 1) * width * n_mels;
  cond_gather_kernel<<<grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(cond, rows, n_group, width, n_mels, t_cond, n, BF(hi), BF(lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_cond_scatter(const float* dc, const int32_t* rows, int32_t batch, int32_t n_group, int32_t width, int32_t n_mels, int32_t t_cond,
                                   float* dcond, pk_stream_t stream) {
  PK_CHECK_ARG(dc && rows && dcond && batch > 0 && n_group >= 2 && width > 0 && n_mels > 0 && t_cond >= width * n_group, "bad arguments");
  const long long n = static_cast<long long>(batch) * (n_group - 1) * width * n_mels;
  cond_scatter_kernel<<<grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(dc, rows, batch, n_group, width, n_mels, t_cond, dcond);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_waveflow_train_loss(const float* z, int64_t n, const float* logs, int64_t n_logs, float sigma, float* loss, pk_stream_t stream) {
  PK_CHECK_ARG(z && logs && loss && n > 0 && n_logs > 0 && sigma > 0.f, "bad arguments");
  loss_kernel<<<1, 1024, 0, PK_STREAM>>>(z, n, logs, n_logs, sigma, loss);
  PK_LAUNCH_DONE(1);
}

// ------------------------------------------------------------------------------------------------------------------------
// pk_waveflow_backward_layer: one layer boundary of the residual net's backward, the mirror image of
// waveflow_forward_layer_kernel (waveflow_layer.cu).  Persistent CTAs over 128-position tiles of one (utterance, net row), a
// producer warpgroup whose TMA lane runs a 2-stage ring, two consumer warpgroups of 64 positions each:
//   GEMM1 (has_gemm1): dx_l = dx_{l+1} + conv^T(dh_l): 18 (C = 64) / 36 (C = 128) K-chunks = 3 kernel rows s x 3 width taps x
//         the 2C channels of dh_l in blocks of 64; kernel row s reads dh row q + s (the two zero rows after each utterance's
//         net rows are the anti-causal padding), tap t reads column w + (t - 1) 2^l (TMA's out-of-bounds fill is the width
//         padding).  Without GEMM1 (the boundary after the last layer) dx_l = 0.  dx_l is written fp32 and as split planes
//         into columns [0, C) of the [dx | dskip] planes.
//   GEMM2 (has_gemm2): dz = [dx_l | dskip] W2_{l-1} (K = 2C) with dx_l as the register A operand straight from GEMM1's
//         accumulators and dskip read from the planes' columns [C, 2C); then the gate backward on the accumulator with the
//         saved pre-gate a|g of layer l - 1 -> dh_{l-1} as split planes.
// ------------------------------------------------------------------------------------------------------------------------
namespace pk {
namespace wfb {

constexpr int kStages = 2;
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kATile = 128 * kSwizzleBytes;                  // 128 positions x 64 channels, one plane

template <int C>
struct Geo {
  static constexpr int kWBytes = 2 * C * kSwizzleBytes;      // hi | lo of one weight K-chunk (C rows)
  static constexpr int kStageBytes = 2 * kATile + kWBytes;
  static constexpr int kG1Chunks = 9 * (2 * C / 64);
  static constexpr int kG2Chunks = 2 * C / 64;
  static constexpr int kSmem = kStages * kStageBytes + 1024 + 256;
};

template <int C>
__device__ __forceinline__ void mma_ss(float (&d)[C / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (C == 64) wgmma_ss_n64(d, a, b, acc);
  else wgmma_ss_n128(d, a, b, acc);
}
template <int C>
__device__ __forceinline__ void mma_rs(float (&d)[C / 2], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
  if constexpr (C == 64) wgmma_rs_n64(d, a, b, acc);
  else wgmma_rs_n128(d, a, b, acc);
}

struct BwdArgs {
  int w, n_group, dil, tiles_per_row, total_tiles, has_gemm1, has_gemm2, dh_ld;
  float* dx;                          // (net layout, C) fp32: dx_{l+1} in, dx_l out
  __nv_bfloat16* a2_hi;               // (net layout, 2C) [dx | dskip] split planes
  __nv_bfloat16* a2_lo;
  const float* h;                     // (net layout, 2C) pre-gate a|g of layer l - 1
  __nv_bfloat16* dh_hi;               // dh_{l-1} planes: row pitch dh_ld
  __nv_bfloat16* dh_lo;
};

template <int C>
__global__ void __launch_bounds__(kThreads, 1)
waveflow_backward_layer_kernel(const __grid_constant__ CUtensorMap tm_dh,   // dh_l planes (batch * (n_group + 1) + 2, w, 2C)
                               const __grid_constant__ CUtensorMap tm_w1,   // conv^T weight planes (C, 9 * 2C)
                               const __grid_constant__ CUtensorMap tm_w2,   // out_proj^T weight planes (C, 2C)
                               const __grid_constant__ BwdArgs p) {
  using G = Geo<C>;
  constexpr int kIn = 2 * C / 64;                              // 64-channel blocks of dh
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full_bar = smem + kStages * G::kStageBytes;
  const uint32_t empty_bar = full_bar + 8 * kStages;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int rows = p.n_group - 1;
  const int n1 = p.has_gemm1 ? G::kG1Chunks : 0, n2 = p.has_gemm2 ? G::kG2Chunks : 0;

  if (threadIdx.x == kConsumerThreads) {
    if (p.has_gemm1) { tma_prefetch_desc(&tm_dh); tma_prefetch_desc(&tm_w1); }
    if (p.has_gemm2) tma_prefetch_desc(&tm_w2);
    for (int s = 0; s < kStages; ++s) { mbar_init_a(full_bar + 8 * s, 1); mbar_init_a(empty_bar + 8 * s, kConsumerThreads / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int br = tile / p.tiles_per_row, w0 = (tile - br * p.tiles_per_row) * 128;
        const int b = br / rows, r = br - b * rows;
        const int qrow = b * (p.n_group + 1) + r;
        for (int j = 0; j < n1 + n2; ++j, ++it) {
          const int s = it % kStages;
          mbar_wait_a(empty_bar + 8 * s, ((it / kStages) & 1) ^ 1);
          const uint32_t st = smem + s * G::kStageBytes;
          const uint32_t fb = full_bar + 8 * s;
          if (j < n1) {
            const int kr = j / (3 * kIn), rem = j - 3 * kIn * kr;
            const int tap = rem / kIn, hb = rem - kIn * tap;
            mbar_arrive_expect_tx_a(fb, G::kStageBytes);
            tma_load_4d_a(st, &tm_dh, fb, hb * 64, w0 + (tap - 1) * p.dil, qrow + kr, 0);
            tma_load_4d_a(st + 2 * kATile, &tm_w1, fb, j * kChunkK, 0, 0, 0);
          } else {
            mbar_arrive_expect_tx_a(fb, G::kWBytes);
            tma_load_4d_a(st + 2 * kATile, &tm_w2, fb, (j - n1) * kChunkK, 0, 0, 0);
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int rl = wg * 64 + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int br = tile / p.tiles_per_row, w0 = (tile - br * p.tiles_per_row) * 128;
      const int b = br / rows, r = br - b * rows;
      const long long prow = (static_cast<long long>(b) * (p.n_group + 1) + r) * p.w;      // first position of this net row
      uint32_t xh[C / 64][16], xl[C / 64][16];                   // dx_l as GEMM2's A fragments
      {
        float acc1[C / 2];
#pragma unroll
        for (int i = 0; i < C / 2; ++i) acc1[i] = 0.f;
        for (int j = 0; j < n1; ++j, ++it) {
          const int s = it % kStages;
          mbar_wait_a(full_bar + 8 * s, (it / kStages) & 1);
          const uint32_t st = smem + s * G::kStageBytes;
          const uint64_t a_hi = make_smem_desc_sw128(st + wg * 64 * kSwizzleBytes), a_lo = make_smem_desc_sw128(st + kATile + wg * 64 * kSwizzleBytes);
          const uint64_t b_hi = make_smem_desc_sw128(st + 2 * kATile), b_lo = make_smem_desc_sw128(st + 2 * kATile + C * kSwizzleBytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            mma_ss<C>(acc1, a_hi + desc_kstep(k), b_hi + desc_kstep(k), 1);
            mma_ss<C>(acc1, a_lo + desc_kstep(k), b_hi + desc_kstep(k), 1);
            mma_ss<C>(acc1, a_hi + desc_kstep(k), b_lo + desc_kstep(k), 1);
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(acc1);
          __syncwarp();
          if (lane == 0) mbar_arrive_a(empty_bar + 8 * s);
        }
        // dx_l = dx_{l+1} + acc1 (or 0): fp32 and split planes out, fragments kept for GEMM2
#pragma unroll
        for (int jj = 0; jj < C / 8; ++jj) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int col = w0 + rl + 8 * hh, c = 8 * jj + cq;
            float v0 = 0.f, v1 = 0.f;
            if (col < p.w) {
              const long long pos = prow + col;
              if (p.has_gemm1) {
                const float2 o = *reinterpret_cast<const float2*>(p.dx + pos * C + c);
                v0 = acc1[4 * jj + 2 * hh] + o.x;
                v1 = acc1[4 * jj + 2 * hh + 1] + o.y;
              }
              *reinterpret_cast<float2*>(p.dx + pos * C + c) = make_float2(v0, v1);
            }
            uint32_t hi, lo;
            split2(v0, v1, hi, lo);
            xh[jj / 8][2 * (jj % 8) + hh] = hi;
            xl[jj / 8][2 * (jj % 8) + hh] = lo;
            if (col < p.w) {
              const long long off = (prow + col) * 2 * C + c;
              *reinterpret_cast<uint32_t*>(p.a2_hi + off) = hi;
              *reinterpret_cast<uint32_t*>(p.a2_lo + off) = lo;
            }
          }
        }
      }
      if (!p.has_gemm2) continue;
      const uint32_t s0 = it % kStages;
      float acc2[C / 2];
#pragma unroll
      for (int kc = 0; kc < G::kG2Chunks; ++kc) {
        const int s = (s0 + kc) % kStages;
        mbar_wait_a(full_bar + 8 * s, ((it + kc) / kStages) & 1);
        const uint32_t st = smem + s * G::kStageBytes + 2 * kATile;
        const uint64_t b_hi = make_smem_desc_sw128(st), b_lo = make_smem_desc_sw128(st + C * kSwizzleBytes);
        uint32_t fh[16], fl[16];
        if (kc < C / 64) {
#pragma unroll
          for (int i = 0; i < 16; ++i) { fh[i] = xh[kc % (C / 64)][i]; fl[i] = xl[kc % (C / 64)][i]; }
        } else {                                                 // dskip: columns C + 64 (kc - C / 64) + ... of the planes
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int col = w0 + rl + 8 * hh;
              uint32_t hv = 0, lv = 0;
              if (col < p.w) {
                const long long off = (prow + col) * 2 * C + C + 64 * (kc - C / 64) + 8 * jj + cq;
                hv = *reinterpret_cast<const uint32_t*>(p.a2_hi + off);
                lv = *reinterpret_cast<const uint32_t*>(p.a2_lo + off);
              }
              fh[2 * jj + hh] = hv;
              fl[2 * jj + hh] = lv;
            }
          }
        }
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t ah[4] = {fh[4 * k], fh[4 * k + 1], fh[4 * k + 2], fh[4 * k + 3]};
          const uint32_t al[4] = {fl[4 * k], fl[4 * k + 1], fl[4 * k + 2], fl[4 * k + 3]};
          mma_rs<C>(acc2, ah, b_hi + desc_kstep(k), !(kc == 0 && k == 0));
          mma_rs<C>(acc2, al, b_hi + desc_kstep(k), 1);
          mma_rs<C>(acc2, ah, b_lo + desc_kstep(k), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(acc2);
        __syncwarp();
        if (lane == 0) mbar_arrive_a(empty_bar + 8 * s);
      }
      it += G::kG2Chunks;
      // gate backward: dh_a = dz s (1 - t^2), dh_g = dz t s (1 - s), t = tanh(a), s = sigmoid(g)
#pragma unroll
      for (int jj = 0; jj < C / 8; ++jj) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int col = w0 + rl + 8 * hh, c = 8 * jj + cq;
          if (col >= p.w) continue;
          const long long pos = prow + col;
          const float2 a = *reinterpret_cast<const float2*>(p.h + pos * 2 * C + c);
          const float2 g = *reinterpret_cast<const float2*>(p.h + pos * 2 * C + C + c);
          float da[2], dg[2];
          const float av[2] = {a.x, a.y}, gv[2] = {g.x, g.y};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float t = tanhf(av[e]), sg = 1.f / (1.f + expf(-gv[e])), d = acc2[4 * jj + 2 * hh + e];
            da[e] = d * sg * (1.f - t * t);
            dg[e] = d * t * sg * (1.f - sg);
          }
          const long long off = pos * p.dh_ld + c;
          uint32_t hi, lo;
          split2(da[0], da[1], hi, lo);
          *reinterpret_cast<uint32_t*>(p.dh_hi + off) = hi;
          *reinterpret_cast<uint32_t*>(p.dh_lo + off) = lo;
          split2(dg[0], dg[1], hi, lo);
          *reinterpret_cast<uint32_t*>(p.dh_hi + off + C) = hi;
          *reinterpret_cast<uint32_t*>(p.dh_lo + off + C) = lo;
        }
      }
    }
  }
}

}  // namespace wfb
}  // namespace pk

template <int C>
static int backward_layer_launch(const pk_waveflow_backward_layer_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::wfb;
  using G = Geo<C>;
  int resident = 0, rc;
  if ((rc = prepare_kernel(waveflow_backward_layer_kernel<C>, kThreads, G::kSmem, &resident))) return rc;
  const uint64_t W = a->width, Q = static_cast<uint64_t>(a->batch) * (a->n_group + 1);
  CUtensorMap tdh, tw1, tw2;                                   // a map the launch does not use stays zero and is never read
  memset(&tdh, 0, sizeof(tdh));
  memset(&tw1, 0, sizeof(tw1));
  memset(&tw2, 0, sizeof(tw2));
  if (a->has_gemm1) {
    if ((rc = encode_tmap_bf16_planes(&tdh, a->dh_in_hi, a->dh_in_lo, 2 * C, W, Q + 2, a->dh_ld, W * a->dh_ld, 128))) return rc;
    if ((rc = encode_tmap_bf16_planes(&tw1, a->w1_hi, a->w1_lo, 18 * C, C, 1, 18 * C, 0, C))) return rc;
  }
  if (a->has_gemm2) {
    if ((rc = encode_tmap_bf16_planes(&tw2, a->w2_hi, a->w2_lo, 2 * C, C, 1, 2 * C, 0, C))) return rc;
  }
  BwdArgs p;
  p.w = a->width; p.n_group = a->n_group; p.dil = a->dilation; p.has_gemm1 = a->has_gemm1; p.has_gemm2 = a->has_gemm2;
  p.dh_ld = a->dh_ld;
  p.tiles_per_row = (a->width + 127) / 128;
  const long long total = static_cast<long long>(p.tiles_per_row) * a->batch * (a->n_group - 1);
  PK_CHECK_ARG(total < (1ll << 31), "too many tiles (%lld)", total);
  p.total_tiles = static_cast<int>(total);
  p.dx = a->dx;
  p.a2_hi = static_cast<__nv_bfloat16*>(a->a2_hi); p.a2_lo = static_cast<__nv_bfloat16*>(a->a2_lo);
  p.h = a->h;
  p.dh_hi = static_cast<__nv_bfloat16*>(a->dh_out_hi); p.dh_lo = static_cast<__nv_bfloat16*>(a->dh_out_lo);
  const int grid = std::min(p.total_tiles, resident);
  waveflow_backward_layer_kernel<C><<<grid, kThreads, G::kSmem, PK_STREAM>>>(tdh, tw1, tw2, p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_backward_layer(const pk_waveflow_backward_layer_args* a, pk_stream_t stream) {
  PK_CHECK_ARG(a && a->batch > 0 && a->width > 0 && a->n_group >= 2 && a->n_group <= 16 && a->dx && a->a2_hi && a->a2_lo,
               "bad arguments");
  PK_CHECK_ARG(a->channels == 64 || a->channels == 128, "channels must be 64 or 128");
  PK_CHECK_ARG(a->has_gemm1 || a->has_gemm2, "nothing to do");
  PK_CHECK_ARG(!a->has_gemm1 || (a->dh_in_hi && a->dh_in_lo && a->w1_hi && a->w1_lo && a->dilation >= 1 && a->dh_ld >= 2 * a->channels &&
                                 a->dh_ld % 8 == 0), "GEMM1 operands");
  PK_CHECK_ARG(!a->has_gemm2 || (a->w2_hi && a->w2_lo && a->h && a->dh_out_hi && a->dh_out_lo && a->dh_ld >= 2 * a->channels), "GEMM2 operands");
  return a->channels == 64 ? backward_layer_launch<64>(a, stream) : backward_layer_launch<128>(a, stream);
}
