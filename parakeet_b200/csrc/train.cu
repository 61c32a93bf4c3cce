// Backward / optimiser kernels of the FastSpeech2 training step (reference: FastSpeech2Updater.update_core,
// parakeet/models/fastspeech2/fastspeech2_updater.py:51-99 = forward, FastSpeech2Loss, loss.backward(), Adam.step()).
// GEMM-shaped gradients (dgrad = conv with flipped taps, wgrad = dY^T X over the flattened batch*time axis, attention
// dQ/dK/dV/dP) reuse pk_conv_gemm on transposed split planes; everything here is row-wise / reduction glue.
#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {

// ---------------------------------------------------------------------------------------------------------------
// dst[z*dst_zstride + c*ld_dst + r] = src[z, r + shift, c0 + c]  (0 where r + shift is outside [0, rows)), split planes.
// 32x32 tiles through shared memory.  grid = (ceil(r_out/32), ceil(cols/32), Z)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
transpose_planes_kernel(const __nv_bfloat16* __restrict__ src_hi, const __nv_bfloat16* __restrict__ src_lo, int rows, long long src_zstride,
                        int ld_src, int c0, int cols, int shift, int r_out, __nv_bfloat16* __restrict__ dst_hi,
                        __nv_bfloat16* __restrict__ dst_lo, long long dst_zstride, long long ld_dst) {
  __shared__ __nv_bfloat16 th[32][34], tl[32][34];
  const int z = blockIdx.z;
  const int r0 = blockIdx.x * 32, cc0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i + shift, c = cc0 + tx;
    __nv_bfloat16 vh = __float2bfloat16(0.f), vl = vh;
    if (r >= 0 && r < rows && c < cols && (r0 + i) < r_out) {
      const long long o = z * src_zstride + static_cast<long long>(r) * ld_src + c0 + c;
      vh = src_hi[o];
      vl = src_lo[o];
    }
    th[i][tx] = vh;
    tl[i][tx] = vl;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = cc0 + i, r = r0 + tx;
    if (c < cols && r < r_out) {
      const long long o = z * dst_zstride + c * ld_dst + r;
      dst_hi[o] = th[tx][i];
      dst_lo[o] = tl[tx][i];
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LayerNorm backward, one warp per row; dgamma / dbeta accumulated per block in smem then atomically.
//   xhat = (x - mean) * rstd; g = dy * gamma; dx (+)= rstd * (g - mean(g) - xhat * mean(g * xhat))
// ---------------------------------------------------------------------------------------------------------------
template <int MAX_PER_LANE>
__global__ void __launch_bounds__(256)
layer_norm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ dy, float eps,
                      long long rows, int d, float* __restrict__ dx, int accumulate, float* __restrict__ dgamma,
                      float* __restrict__ dbeta) {
  extern __shared__ float ln_smem[];  // [2][d]
  float* sg = ln_smem;
  float* sb = ln_smem + d;
  for (int c = threadIdx.x; c < 2 * d; c += blockDim.x) ln_smem[c] = 0.f;
  __syncthreads();
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row < rows) {
    const float* xr = x + row * d;
    const float* dr = dy + row * d;
    float v[MAX_PER_LANE], g[MAX_PER_LANE];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < MAX_PER_LANE; ++i) {
      const int c = lane + 32 * i;
      v[i] = c < d ? xr[c] : 0.f;
      s += v[i];
    }
    const float mean = warp_sum(s) / d;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < MAX_PER_LANE; ++i) {
      const int c = lane + 32 * i;
      const float dv = c < d ? v[i] - mean : 0.f;
      q += dv * dv;
    }
    const float rstd = rsqrtf(warp_sum(q) / d + eps);
    float sg1 = 0.f, sg2 = 0.f;
#pragma unroll
    for (int i = 0; i < MAX_PER_LANE; ++i) {
      const int c = lane + 32 * i;
      if (c < d) {
        const float xh = (v[i] - mean) * rstd;
        const float dyv = dr[c];
        g[i] = dyv * __ldg(gamma + c);
        sg1 += g[i];
        sg2 += g[i] * xh;
        atomicAdd(sg + c, dyv * xh);
        atomicAdd(sb + c, dyv);
        v[i] = xh;
      } else {
        g[i] = 0.f;
      }
    }
    const float m1 = warp_sum(sg1) / d, m2 = warp_sum(sg2) / d;
#pragma unroll
    for (int i = 0; i < MAX_PER_LANE; ++i) {
      const int c = lane + 32 * i;
      if (c < d) {
        const float o = rstd * (g[i] - m1 - v[i] * m2);
        dx[row * d + c] = accumulate ? dx[row * d + c] + o : o;
      }
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    atomicAdd(dgamma + c, sg[c]);
    atomicAdd(dbeta + c, sb[c]);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Softmax backward of the attention probabilities P (batch * heads, rows, ld):
//   dS = scale * P * (dP - sum_k P dP) over the first `keys` columns, 0 in the padding columns.  One warp per row.
// The TransformerTTS guided attention loss (GuidedMultiHeadAttentionLoss, transformer_tts.py:874-1075) is folded into dP of the
// heads h < guided_heads (none for guided_heads = 0): for query row i < olen_b and key j < ilen_b,
//   dP[i, j] += coef * G[i, j],  G = 1 - exp(-(j / ilen_b - i / olen_b)^2 / (2 sigma^2)),
// coef = lambda / (guided_heads * guided_layers * sum_b ilen_b olen_b) (the mean over the selected elements of every guided
// layer), and partials[(b * guided_heads + h) * rows + i] = sum_j G[i, j] P[i, j] (0 for rows i >= olen_b).
// kGuided = false (guided_heads = 0) compiles the guided terms away: the plain backward keeps its unrolled, load-bound loops.
// ---------------------------------------------------------------------------------------------------------------
template <bool kGuided>
__global__ void __launch_bounds__(256)
softmax_bwd_kernel(const __nv_bfloat16* __restrict__ p_hi, const __nv_bfloat16* __restrict__ p_lo, const float* __restrict__ dp,
                   int batch, int heads, int rows_per_z, int keys, int ld, float scale, int guided_heads, int guided_layers,
                   const int32_t* __restrict__ ilens, const int32_t* __restrict__ olens, float inv_two_sigma2, float lambda,
                   float* __restrict__ partials, __nv_bfloat16* __restrict__ ds_hi, __nv_bfloat16* __restrict__ ds_lo) {
  const long long rows = static_cast<long long>(batch) * heads * rows_per_z;
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const int z = static_cast<int>(row / rows_per_z), i = static_cast<int>(row % rows_per_z);
  const int b = z / heads, h = z % heads;
  const bool guided_head = kGuided && h < guided_heads;
  int il = 0, ol = 0;
  float coef = 0.f;
  if (guided_head) {
    long long n = 0;
    for (int q = 0; q < batch; ++q) n += static_cast<long long>(min(__ldg(ilens + q), keys)) * min(__ldg(olens + q), rows_per_z);
    coef = n > 0 ? lambda / (static_cast<float>(guided_heads) * guided_layers * static_cast<float>(n)) : 0.f;
    il = min(__ldg(ilens + b), keys);
    ol = min(__ldg(olens + b), rows_per_z);
  }
  const bool live = guided_head && i < ol && il > 0;
  const float fi = live ? static_cast<float>(i) / static_cast<float>(ol) : 0.f;
  const float inv_il = live ? 1.f / static_cast<float>(il) : 0.f;
  const float* dr = dp + row * ld;
  float dot = 0.f, gp = 0.f;
  for (int c = lane; c < keys; c += 32) {
    const float pv = ld_split(p_hi, p_lo, row * ld + c);
    float d = dr[c];
    if (live && c < il) {
      const float x = static_cast<float>(c) * inv_il - fi;
      const float g = 1.f - expf(-(x * x) * inv_two_sigma2);
      d = fmaf(coef, g, d);
      gp = fmaf(g, pv, gp);
    }
    dot = fmaf(pv, d, dot);
  }
  dot = warp_sum(dot);
  if (guided_head) {
    gp = warp_sum(gp);
    if (lane == 0) partials[(static_cast<long long>(b) * guided_heads + h) * rows_per_z + i] = gp;
  }
  for (int c = lane; c < ld; c += 32) {
    float v = 0.f;
    if (c < keys) {
      float d = dr[c];
      if (live && c < il) {
        const float x = static_cast<float>(c) * inv_il - fi;
        d = fmaf(coef, 1.f - expf(-(x * x) * inv_two_sigma2), d);
      }
      v = scale * ld_split(p_hi, p_lo, row * ld + c) * (d - dot);
    }
    __nv_bfloat16 hh, ll;
    split_bf16(v, hh, ll);
    ds_hi[row * ld + c] = hh;
    ds_lo[row * ld + c] = ll;
  }
}

// out[c] += sum_rows x[row, c]  (bias gradients); block = 256 threads handles a 64-row x 64-col patch
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, long long rows, int c, float* __restrict__ out) {
  __shared__ float part[4][64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int col = blockIdx.y * 64 + tx;
  float s = 0.f;
  if (col < c)
    for (long long r = blockIdx.x * 64LL + ty; r < rows && r < (blockIdx.x + 1) * 64LL; r += 4) s += x[r * c + col];
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && col < c) atomicAdd(out + col, part[0][tx] + part[1][tx] + part[2][tx] + part[3][tx]);
}

// the same for split planes (rows, ld): out[c] += sum_rows (hi + lo)[row, c], c < cols
__global__ void __launch_bounds__(256) colsum_split_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                                                           long long rows, int cols, int ld, float* __restrict__ out) {
  __shared__ float part[4][64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int col = blockIdx.y * 64 + tx;
  float s = 0.f;
  if (col < cols)
    for (long long r = blockIdx.x * 64LL + ty; r < rows && r < (blockIdx.x + 1) * 64LL; r += 4)
      s += __bfloat162float(hi[r * ld + col]) + __bfloat162float(lo[r * ld + col]);
  part[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && col < cols) atomicAdd(out + col, part[0][tx] + part[1][tx] + part[2][tx] + part[3][tx]);
}

// out[i] = sum_s part[s][i]: the reduction of split-K partial products (overwrites: no zero fill, no copy afterwards)
__global__ void __launch_bounds__(256) sum_slices_kernel(const float* __restrict__ part, int s, long long n, float* __restrict__ out,
                                                         int vec) {
  const long long i = (blockIdx.x * 256LL + threadIdx.x) * 4;
  if (i >= n) return;
  if (vec) {                     // n % 4 == 0 and both pointers 16-byte aligned
    float4 a = *reinterpret_cast<const float4*>(part + i);
    for (int k = 1; k < s; ++k) {
      const float4 b = *reinterpret_cast<const float4*>(part + k * n + i);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    *reinterpret_cast<float4*>(out + i) = a;
  } else {
    for (long long j = i; j < n && j < i + 4; ++j) {
      float a = part[j];
      for (int k = 1; k < s; ++k) a += part[k * n + j];
      out[j] = a;
    }
  }
}

// BatchNorm batch statistics, second pass: sums[C + c] += sum (x - mean)^2 with mean = sums[c] / rows from the first pass (colsum_kernel).
// Two passes rather than E[x^2] - mean^2: for a column whose mean is large against its spread (30 + N(0, 1)) the single-pass
// difference cancels in fp32 and loses three decimal digits of the variance.
__global__ void __launch_bounds__(256) col_centered_sq_kernel(const float* __restrict__ x, long long rows, int c, float* __restrict__ sums) {
  __shared__ float p2[4][64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int col = blockIdx.y * 64 + tx;
  float q = 0.f;
  if (col < c) {
    const float m = sums[col] / rows;
    for (long long r = blockIdx.x * 64LL + ty; r < rows && r < (blockIdx.x + 1) * 64LL; r += 4) {
      const float d = x[r * c + col] - m;
      q = fmaf(d, d, q);
    }
  }
  p2[ty][tx] = q;
  __syncthreads();
  if (ty == 0 && col < c) atomicAdd(sums + c + col, p2[0][tx] + p2[1][tx] + p2[2][tx] + p2[3][tx]);
}

// BatchNorm1D training forward (given sum x and sum (x - mean)^2 per column): y = act(gamma * (x - mean) * rstd + beta); running stats updated by
// thread block 0 (paddle momentum 0.9: running = 0.9 * running + 0.1 * batch, biased variance).  act: 0 none, 2 tanh.
__global__ void bn_train_fwd_kernel(const float* __restrict__ x, const float* __restrict__ sums, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, float eps, int act, long long rows, int c, float momentum,
                                    float* __restrict__ run_mean, float* __restrict__ run_var, float* __restrict__ y,
                                    __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo, float* __restrict__ save_mean,
                                    float* __restrict__ save_rstd) {
  const long long n = rows * c;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (blockIdx.x == 0) {
    for (int col = threadIdx.x; col < c; col += blockDim.x) {
      const float mean = sums[col] / rows;
      const float var = sums[c + col] / rows;
      save_mean[col] = mean;
      save_rstd[col] = rsqrtf(var + eps);
      if (run_mean) {
        run_mean[col] = momentum * run_mean[col] + (1.f - momentum) * mean;
        run_var[col] = momentum * run_var[col] + (1.f - momentum) * var;
      }
    }
  }
  if (i >= n) return;
  const int col = i % c;
  const float mean = sums[col] / rows;
  const float var = sums[c + col] / rows;
  float v = (x[i] - mean) * rsqrtf(var + eps) * __ldg(gamma + col) + __ldg(beta + col);
  if (act == PK_ACT_TANH) v = tanhf(v);
  if (y) y[i] = v;
  if (y_hi) {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    y_hi[i] = h;
    y_lo[i] = l;
  }
}

// BatchNorm backward, pass 1: sums[c] += sum dyp, sums[C+c] += sum dyp * xhat, with dyp = dy * (act == tanh ? 1 - y^2 : 1)
__global__ void __launch_bounds__(256)
bn_bwd_stats_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ y_act,
                    const float* __restrict__ mean, const float* __restrict__ rstd, int act, long long rows, int c,
                    float* __restrict__ sums) {
  __shared__ float p1[4][64], p2[4][64];
  const int tx = threadIdx.x & 63, ty = threadIdx.x >> 6;
  const int col = blockIdx.y * 64 + tx;
  float s = 0.f, q = 0.f;
  if (col < c) {
    const float m = mean[col], rs = rstd[col];
    for (long long r = blockIdx.x * 64LL + ty; r < rows && r < (blockIdx.x + 1) * 64LL; r += 4) {
      float g = dy[r * c + col];
      if (act == PK_ACT_TANH) { const float yv = y_act[r * c + col]; g *= 1.f - yv * yv; }
      s += g;
      q += g * (x[r * c + col] - m) * rs;
    }
  }
  p1[ty][tx] = s;
  p2[ty][tx] = q;
  __syncthreads();
  if (ty == 0 && col < c) {
    atomicAdd(sums + col, p1[0][tx] + p1[1][tx] + p1[2][tx] + p1[3][tx]);
    atomicAdd(sums + c + col, p2[0][tx] + p2[1][tx] + p2[2][tx] + p2[3][tx]);
  }
}
// pass 2: dx = gamma * rstd / N * (N * dyp - sum dyp - xhat * sum(dyp * xhat)); dgamma = sums[C+c], dbeta = sums[c]
__global__ void bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ y_act,
                                    const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                                    const float* __restrict__ sums, int act, long long rows, int c, float* __restrict__ dx) {
  const long long n = rows * c;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const int col = i % c;
  float g = dy[i];
  if (act == PK_ACT_TANH) { const float yv = y_act[i]; g *= 1.f - yv * yv; }
  const float xh = (x[i] - mean[col]) * rstd[col];
  const float N = static_cast<float>(rows);
  dx[i] = __ldg(gamma + col) * rstd[col] / N * (N * g - sums[col] - xh * sums[c + col]);
}

// dx = dy * (y > 0) with y given as split planes; output fp32 and split
__global__ void relu_bwd_kernel(const float* __restrict__ dy, const __nv_bfloat16* __restrict__ y_hi, long long n,
                                float* __restrict__ dx, __nv_bfloat16* __restrict__ dx_hi, __nv_bfloat16* __restrict__ dx_lo) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= n) return;
  const float v = __bfloat162float(y_hi[i]) > 0.f ? dy[i] : 0.f;   // relu output > 0 <=> its bf16 hi part > 0
  if (dx) dx[i] = v;
  if (dx_hi) {
    __nv_bfloat16 h, l;
    split_bf16(v, h, l);
    dx_hi[i] = h;
    dx_lo[i] = l;
  }
}

__global__ void axpy_kernel(float a, const float* __restrict__ x, long long n, float* __restrict__ y) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) y[i] = fmaf(a, x[i], y[i]);
}

// gradients of FastSpeech2Loss (use_masking=True) w.r.t. before, after, d_outs, p_outs, e_outs; loss = l1 + dur + pitch + energy
__global__ void fs2_loss_bwd_kernel(const float* __restrict__ before, const float* __restrict__ after, const float* __restrict__ ys,
                                    const int32_t* __restrict__ olens, int l_max, int odim, const float* __restrict__ d_outs,
                                    const int64_t* __restrict__ ds, const float* __restrict__ p_outs, const float* __restrict__ ps,
                                    const float* __restrict__ e_outs, const float* __restrict__ es, const int32_t* __restrict__ ilens,
                                    int t_max, int batch, float* __restrict__ g_before, float* __restrict__ g_after,
                                    float* __restrict__ g_d, float* __restrict__ g_p, float* __restrict__ g_e) {
  long long frames = 0, toks = 0;
  for (int b = 0; b < batch; ++b) { frames += min(olens[b], l_max); toks += min(ilens[b], t_max); }
  const float inv_m = 1.f / (static_cast<float>(frames) * odim), inv_t = 1.f / static_cast<float>(toks);
  const long long n_mel = static_cast<long long>(batch) * l_max * odim;
  const long long n_tok = static_cast<long long>(batch) * t_max;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n_mel) {
    const long long row = i / odim;
    const int b = row / l_max, t = row % l_max;
    float gb = 0.f, ga = 0.f;
    if (t < olens[b]) {
      const float y = ys[i];
      const float db = before[i] - y, da = after[i] - y;
      gb = db > 0.f ? inv_m : (db < 0.f ? -inv_m : 0.f);
      ga = da > 0.f ? inv_m : (da < 0.f ? -inv_m : 0.f);
    }
    g_before[i] = gb;
    g_after[i] = ga;
  }
  if (i < n_tok) {
    const int b = i / t_max, t = i % t_max;
    float gd = 0.f, gp = 0.f, ge = 0.f;
    if (t < ilens[b]) {
      gd = 2.f * (d_outs[i] - logf(static_cast<float>(ds[i]) + 1.0f)) * inv_t;
      gp = 2.f * (p_outs[i] - ps[i]) * inv_t;
      ge = 2.f * (e_outs[i] - es[i]) * inv_t;
    }
    g_d[i] = gd;
    g_p[i] = gp;
    g_e[i] = ge;
  }
}

// embedding backward (scatter-add, padding_idx rows get nothing) and alpha gradient of the scaled positional encoding
__global__ void __launch_bounds__(256)
embed_pe_bwd_kernel(const int64_t* __restrict__ ids, const float* __restrict__ dx, int vocab, int padding_idx, int rows_per_b,
                    long long rows, int d, float* __restrict__ dtable, float* __restrict__ dalpha) {
  const long long row = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  if (row < rows) {
    const int t = row % rows_per_b;
    const long long id = ids ? ids[row] : -1;
    const bool scatter = ids && id != padding_idx && id >= 0 && id < vocab;
    const float neg = -(logf(10000.0f) / static_cast<float>(d));
    for (int c = lane; c < d; c += 32) {
      const float g = dx[row * d + c];
      if (scatter) atomicAdd(dtable + id * d + c, g);
      const float ang = static_cast<float>(t) * expf(static_cast<float>(c & ~1) * neg);
      acc += g * ((c & 1) ? cosf(ang) : sinf(ang));
    }
  }
  acc = warp_sum(acc);
  __shared__ float red[8];
  if (lane == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[w];
    atomicAdd(dalpha, s);
  }
}

// length regulator backward: dx[b, j, :] = sum_{frames of token j} dy[b, frame, :]
__global__ void __launch_bounds__(128)
lr_bwd_kernel(const float* __restrict__ dy, const int64_t* __restrict__ dur, int t_in, int c, int t_out, float* __restrict__ dx) {
  const int b = blockIdx.y, j = blockIdx.x;
  __shared__ int s_start, s_d;
  if (threadIdx.x == 0) {
    int k = 0;
    for (int q = 0; q < j; ++q) { const long long d = dur[static_cast<long long>(b) * t_in + q]; k += d > 0 ? static_cast<int>(d) : 0; }
    const long long d = dur[static_cast<long long>(b) * t_in + j];
    s_start = k;
    s_d = d > 0 ? static_cast<int>(d) : 0;
  }
  __syncthreads();
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    float s = 0.f;
    for (int f = s_start; f < s_start + s_d && f < t_out; ++f) s += dy[(static_cast<long long>(b) * t_out + f) * c + ch];
    dx[(static_cast<long long>(b) * t_in + j) * c + ch] = s;
  }
}

// gradients of Conv1D(1 -> C, k) on a scalar track: dW[c][q] += sum_{b,t} dhs[b,t,c] * track[b, t + q - pad]; db[c] += sum dhs
__global__ void __launch_bounds__(256)
scalar_conv_wgrad_kernel(const float* __restrict__ dhs, const float* __restrict__ track, int t_len, int c, int k, long long rows,
                         float* __restrict__ dw, float* __restrict__ db) {
  // block handles 64 rows for all channels (strided), accumulates privately then atomics
  const long long r0 = blockIdx.x * 64LL;
  for (int ch = threadIdx.x; ch < c; ch += blockDim.x) {
    float sb = 0.f;
    float sw[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) sw[q] = 0.f;
    for (long long r = r0; r < rows && r < r0 + 64; ++r) {
      const float g = dhs[r * c + ch];
      sb += g;
      const int b = r / t_len, t = r % t_len;
      for (int q = 0; q < k; ++q) {
        const int tt = t + q - (k - 1) / 2;
        if (tt >= 0 && tt < t_len) sw[q] = fmaf(g, track[static_cast<long long>(b) * t_len + tt], sw[q]);
      }
    }
    atomicAdd(db + ch, sb);
    for (int q = 0; q < k; ++q) atomicAdd(dw + ch * k + q, sw[q]);
  }
}

// Adam (paddle.optimizer.Adam semantics) with ClipGradByGlobalNorm folded in:
//   g' = g * grad_scale * sc, sc = clip / max(sqrt(*sqnorm), clip) (1 without sqnorm or for clip <= 0);
//   m = b1 m + (1-b1) g'; v = b2 v + (1-b2) g'^2; lr_t = lr * sqrt(1 - b2^t) / (1 - b1^t);
//   p -= lr_t * m / (sqrt(v) + eps * sqrt(1 - b2^t)).
__global__ void adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                            long long n, float lr_t, float beta1, float beta2, float eps_t, float grad_scale,
                            const double* __restrict__ sqnorm, float clip) {
  float sc = 1.f;
  if (sqnorm != nullptr && clip > 0.f) sc = clip / fmaxf(sqrtf(static_cast<float>(*sqnorm)), clip);
#pragma unroll 1  // each thread takes one element at the steps' flat sizes; the unrolled loop is slower there
  PK_GRID_STRIDE(i, n) {
    const float gi = g[i] * grad_scale * sc;
    const float mi = beta1 * m[i] + (1.f - beta1) * gi;
    const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] -= lr_t * mi / (sqrtf(vi) + eps_t);
  }
}

}  // namespace pk

using namespace pk;

extern "C" int pk_transpose_planes(const void* src_hi, const void* src_lo, int32_t z, int32_t rows, int64_t src_zstride, int32_t ld_src,
                                   int32_t c0, int32_t cols, int32_t shift, int32_t r_out, void* dst_hi, void* dst_lo,
                                   int64_t dst_zstride, int64_t ld_dst, pk_stream_t stream) {
  PK_CHECK_ARG(src_hi && src_lo && dst_hi && dst_lo && z > 0 && rows > 0 && cols > 0 && r_out > 0, "bad arguments");
  dim3 grid((r_out + 31) / 32, (cols + 31) / 32, z);
  transpose_planes_kernel<<<grid, 256, 0, PK_STREAM>>>(static_cast<const __nv_bfloat16*>(src_hi), static_cast<const __nv_bfloat16*>(src_lo),
                                                       rows, src_zstride, ld_src, c0, cols, shift, r_out, static_cast<__nv_bfloat16*>(dst_hi),
                                                       static_cast<__nv_bfloat16*>(dst_lo), dst_zstride, ld_dst);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_layer_norm_bwd(const float* x, const float* gamma, const float* dy, float eps, int64_t rows, int32_t d, float* dx,
                                 int32_t accumulate, float* dgamma, float* dbeta, pk_stream_t stream) {
  PK_CHECK_ARG(x && gamma && dy && dx && dgamma && dbeta && rows > 0 && d > 0 && d <= 512, "bad arguments (d <= 512)");
  const int blocks = nblk(rows * 32, 256);
  const size_t smem = 2 * d * sizeof(float);
  if (d <= 256) layer_norm_bwd_kernel<8><<<blocks, 256, smem, PK_STREAM>>>(x, gamma, dy, eps, rows, d, dx, accumulate, dgamma, dbeta);
  else layer_norm_bwd_kernel<16><<<blocks, 256, smem, PK_STREAM>>>(x, gamma, dy, eps, rows, d, dx, accumulate, dgamma, dbeta);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_softmax_bwd(const void* p_hi, const void* p_lo, const float* dp, int32_t batch, int32_t heads, int32_t rows,
                              int32_t keys, int32_t ld, float scale, int32_t guided_heads, int32_t guided_layers,
                              const int32_t* ilens, const int32_t* olens, float sigma, float lambda, float* partials, void* ds_hi,
                              void* ds_lo, pk_stream_t stream) {
  PK_CHECK_ARG(p_hi && p_lo && dp && ds_hi && ds_lo && batch > 0 && heads > 0 && rows > 0 && keys > 0 && ld >= keys,
               "bad arguments to pk_softmax_bwd");
  PK_CHECK_ARG(guided_heads >= 0 && guided_heads <= heads && guided_layers >= 1 && sigma > 0.f, "bad guided-loss arguments");
  PK_CHECK_ARG(guided_heads == 0 || (ilens && olens && partials), "the guided heads need ilens, olens and partials");
  const long long total = static_cast<long long>(batch) * heads * rows;
  const float inv_two_sigma2 = static_cast<float>(1.0 / (2.0 * static_cast<double>(sigma) * sigma));
  (guided_heads > 0 ? softmax_bwd_kernel<true> : softmax_bwd_kernel<false>)<<<nblk(total * 32, 256), 256, 0, PK_STREAM>>>(
      static_cast<const __nv_bfloat16*>(p_hi), static_cast<const __nv_bfloat16*>(p_lo), dp, batch, heads, rows, keys, ld, scale, guided_heads,
      guided_layers, ilens, olens, inv_two_sigma2, lambda, partials, static_cast<__nv_bfloat16*>(ds_hi), static_cast<__nv_bfloat16*>(ds_lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_colsum(const float* x, int64_t rows, int32_t c, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(x && out && rows > 0 && c > 0, "bad arguments");
  dim3 grid(static_cast<unsigned>((rows + 63) / 64), (c + 63) / 64);
  colsum_kernel<<<grid, 256, 0, PK_STREAM>>>(x, rows, c, out);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_colsum_split(const void* x_hi, const void* x_lo, int64_t rows, int32_t cols, int32_t ld, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(x_hi && x_lo && out && rows > 0 && cols > 0 && ld >= cols, "bad arguments");
  dim3 grid(static_cast<unsigned>((rows + 63) / 64), (cols + 63) / 64);
  colsum_split_kernel<<<grid, 256, 0, PK_STREAM>>>(static_cast<const __nv_bfloat16*>(x_hi), static_cast<const __nv_bfloat16*>(x_lo), rows, cols,
                                                   ld, out);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_sum_slices(const float* part, int32_t slices, int64_t n, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(part && out && slices > 0 && n > 0, "bad arguments");
  const int vec = (n & 3) == 0 && (reinterpret_cast<uintptr_t>(part) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  sum_slices_kernel<<<nblk((n + 3) / 4, 256), 256, 0, PK_STREAM>>>(part, slices, n, out, vec);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_batch_norm_train(const float* x, int64_t rows, int32_t c, const float* gamma, const float* beta, float eps,
                                   int32_t act, float momentum, float* run_mean, float* run_var, float* sums2c, float* y, void* y_hi,
                                   void* y_lo, float* save_mean, float* save_rstd, pk_stream_t stream) {
  PK_CHECK_ARG(x && gamma && beta && sums2c && save_mean && save_rstd && rows > 0 && c > 0, "bad arguments");
  PK_CHECK_ARG(y || y_hi, "no output requested");
  PK_CHECK_CUDA(cudaMemsetAsync(sums2c, 0, 2 * c * sizeof(float), PK_STREAM));
  dim3 grid(static_cast<unsigned>((rows + 63) / 64), (c + 63) / 64);
  colsum_kernel<<<grid, 256, 0, PK_STREAM>>>(x, rows, c, sums2c);
  col_centered_sq_kernel<<<grid, 256, 0, PK_STREAM>>>(x, rows, c, sums2c);
  bn_train_fwd_kernel<<<nblk(rows * c, 256), 256, 0, PK_STREAM>>>(x, sums2c, gamma, beta, eps, act, rows, c, momentum, run_mean, run_var, y,
                                                                  static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo),
                                                                  save_mean, save_rstd);
  PK_LAUNCH_DONE(3);
}

extern "C" int pk_batch_norm_bwd(const float* x, const float* dy, const float* y_act, const float* mean, const float* rstd,
                                 const float* gamma, int32_t act, int64_t rows, int32_t c, float* sums2c, float* dx, pk_stream_t stream) {
  PK_CHECK_ARG(x && dy && mean && rstd && gamma && sums2c && dx && rows > 0 && c > 0, "bad arguments");
  PK_CHECK_ARG(act != PK_ACT_TANH || y_act != nullptr, "tanh backward needs the activation output");
  PK_CHECK_CUDA(cudaMemsetAsync(sums2c, 0, 2 * c * sizeof(float), PK_STREAM));
  dim3 grid(static_cast<unsigned>((rows + 63) / 64), (c + 63) / 64);
  bn_bwd_stats_kernel<<<grid, 256, 0, PK_STREAM>>>(x, dy, y_act, mean, rstd, act, rows, c, sums2c);
  bn_bwd_apply_kernel<<<nblk(rows * c, 256), 256, 0, PK_STREAM>>>(x, dy, y_act, mean, rstd, gamma, sums2c, act, rows, c, dx);
  PK_LAUNCH_DONE(2);
}

extern "C" int pk_relu_bwd(const float* dy, const void* y_hi, int64_t n, float* dx, void* dx_hi, void* dx_lo, pk_stream_t stream) {
  PK_CHECK_ARG(dy && y_hi && n > 0 && (dx || dx_hi), "bad arguments");
  relu_bwd_kernel<<<nblk(n, 256), 256, 0, PK_STREAM>>>(dy, static_cast<const __nv_bfloat16*>(y_hi), n, dx,
                                                       static_cast<__nv_bfloat16*>(dx_hi), static_cast<__nv_bfloat16*>(dx_lo));
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_axpy(float a, const float* x, int64_t n, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(x && y && n > 0, "bad arguments");
  axpy_kernel<<<nblk(n, 256), 256, 0, PK_STREAM>>>(a, x, n, y);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_fs2_loss_bwd(const float* before, const float* after, const float* ys, const int32_t* olens, int32_t l_max,
                               int32_t odim, const float* d_outs, const int64_t* ds, const float* p_outs, const float* ps,
                               const float* e_outs, const float* es, const int32_t* ilens, int32_t t_max, int32_t batch,
                               float* g_before, float* g_after, float* g_d, float* g_p, float* g_e, pk_stream_t stream) {
  PK_CHECK_ARG(before && after && ys && olens && d_outs && ds && p_outs && ps && e_outs && es && ilens && g_before && g_after && g_d &&
               g_p && g_e, "NULL pointer");
  const long long n = std::max(static_cast<long long>(batch) * l_max * odim, static_cast<long long>(batch) * t_max);
  fs2_loss_bwd_kernel<<<nblk(n, 256), 256, 0, PK_STREAM>>>(before, after, ys, olens, l_max, odim, d_outs, ds, p_outs, ps, e_outs, es, ilens,
                                                          t_max, batch, g_before, g_after, g_d, g_p, g_e);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_embed_pe_bwd(const int64_t* ids, const float* dx, int32_t vocab, int32_t padding_idx, int32_t batch, int32_t t,
                               int32_t d, float* dtable, float* dalpha, pk_stream_t stream) {
  PK_CHECK_ARG(dx && dalpha && batch > 0 && t > 0 && d > 0 && (ids == nullptr || dtable != nullptr), "bad arguments");
  const long long rows = static_cast<long long>(batch) * t;
  embed_pe_bwd_kernel<<<nblk(rows * 32, 256), 256, 0, PK_STREAM>>>(ids, dx, vocab, padding_idx, t, rows, d, dtable, dalpha);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_length_regulate_bwd(const float* dy, const int64_t* dur, int32_t batch, int32_t t_in, int32_t c, int32_t t_out,
                                      float* dx, pk_stream_t stream) {
  PK_CHECK_ARG(dy && dur && dx && batch > 0 && t_in > 0 && c > 0 && t_out > 0, "bad arguments");
  dim3 grid(t_in, batch);
  lr_bwd_kernel<<<grid, 128, 0, PK_STREAM>>>(dy, dur, t_in, c, t_out, dx);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_scalar_conv_wgrad(const float* dhs, const float* track, int32_t batch, int32_t t, int32_t c, int32_t k, float* dw,
                                    float* db, pk_stream_t stream) {
  PK_CHECK_ARG(dhs && track && dw && db && batch > 0 && t > 0 && c > 0 && k >= 1 && k <= 16, "bad arguments (k <= 16)");
  const long long rows = static_cast<long long>(batch) * t;
  scalar_conv_wgrad_kernel<<<nblk(rows, 64), 256, 0, PK_STREAM>>>(dhs, track, t, c, k, rows, dw, db);
  PK_LAUNCH_DONE(1);
}

extern "C" int pk_adam(float* params, const float* grads, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                       int32_t step, float grad_scale, const double* sqnorm, float clip_norm, pk_stream_t stream) {
  PK_CHECK_ARG(params && grads && m && v && n > 0 && step >= 1, "bad arguments");
  const double c1 = 1.0 - pow(static_cast<double>(beta1), step), c2 = sqrt(1.0 - pow(static_cast<double>(beta2), step));
  adam_kernel<<<grid_stride_blocks(n, 256), 256, 0, PK_STREAM>>>(params, grads, m, v, n, static_cast<float>(lr * c2 / c1), beta1, beta2,
                                                                 static_cast<float>(eps * c2), grad_scale, sqnorm, clip_norm);
  PK_LAUNCH_DONE(1);
}

// ----------------------------------------------------------------------------------------------------------------
// Dropout (paddle.nn.Dropout, mode "upscale_in_train": y = x * mask / (1 - p) while training; the reference's FastSpeech2
// applies it after the positional encodings, on the attention probabilities, after both sub-layers of every FFT block,
// inside the position-wise feed-forward, in the predictors and in the postnet - SURVEY.md 8a).
// The mask is never stored: element i keeps iff word (i & 3) of Philox4x32-10(counter = {i >> 2 (64 bit), site, step},
// key = seed) is >= p * 2^32, so the backward pass regenerates it from (seed, step, site) with the same kernel applied
// to the gradient (philox4x32_10: pk_sm90.cuh).  oracle/fastspeech2.py restates the generator in numpy for the parity tests.
// ----------------------------------------------------------------------------------------------------------------
namespace pk {

__global__ void dropout_kernel(const float* __restrict__ x, const __nv_bfloat16* __restrict__ x_hi, const __nv_bfloat16* __restrict__ x_lo,
                               long long n, uint32_t thresh, float scale, uint32_t seed_lo, uint32_t seed_hi, uint32_t site, uint32_t step,
                               const uint32_t* __restrict__ step_dev, float* __restrict__ y, __nv_bfloat16* __restrict__ y_hi, __nv_bfloat16* __restrict__ y_lo) {
  const long long blk = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;     // one Philox block = 4 elements
  const long long i0 = blk * 4;
  if (i0 >= n) return;
  uint32_t r[4];
  if (step_dev) step += __ldg(step_dev);      // device-resident step counter: a captured CUDA graph draws fresh masks on every replay
  philox4x32_10(static_cast<uint32_t>(blk), static_cast<uint32_t>(blk >> 32), site, step, seed_lo, seed_hi, r);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const long long i = i0 + e;
    if (i >= n) break;
    const float v = x ? x[i] : __bfloat162float(x_hi[i]) + __bfloat162float(x_lo[i]);
    const float o = r[e] >= thresh ? v * scale : 0.f;
    if (y) y[i] = o;
    if (y_hi) {
      __nv_bfloat16 h, l;
      split_bf16(o, h, l);
      y_hi[i] = h; y_lo[i] = l;
    }
  }
}

}  // namespace pk

extern "C" int pk_dropout(const float* x, const void* x_hi, const void* x_lo, int64_t n, float p, uint64_t seed, uint32_t site,
                          uint32_t step, const uint32_t* step_dev, float* y, void* y_hi, void* y_lo, pk_stream_t stream) {
  using namespace pk;
  PK_CHECK_ARG((x != nullptr) != (x_hi != nullptr) && (x_hi == nullptr) == (x_lo == nullptr), "give x (fp32) or x_hi + x_lo");
  PK_CHECK_ARG((y || y_hi) && (y_hi == nullptr) == (y_lo == nullptr) && n > 0, "bad outputs / size");
  PK_CHECK_ARG(p >= 0.f && p < 1.f, "dropout probability must be in [0, 1)");
  const double t = static_cast<double>(p) * 4294967296.0;
  const uint32_t thresh = t >= 4294967295.0 ? 0xFFFFFFFFu : static_cast<uint32_t>(t);
  const long long blocks4 = (n + 3) / 4;
  dropout_kernel<<<nblk(blocks4, 256), 256, 0, PK_STREAM>>>(x, static_cast<const __nv_bfloat16*>(x_hi), static_cast<const __nv_bfloat16*>(x_lo), n,
                                                            thresh, 1.f / (1.f - p), static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32),
                                                            site, step, step_dev, y, static_cast<__nv_bfloat16*>(y_hi), static_cast<__nv_bfloat16*>(y_lo));
  PK_LAUNCH_DONE(1);
}
