// Losses of the TransformerTTS training step (reference: TransformerTTSUpdater.update_core, parakeet/models/transformer_tts/
// transformer_tts_updater.py:73-170): the guided source-attention loss (GuidedMultiHeadAttentionLoss, transformer_tts.py:874-1075)
// from the row partials that pk_softmax_bwd (train.cu) writes while it folds the loss's gradient into the softmax backward, and
// TransformerTTSLoss (transformer_tts.py:770-872) with its gradients.  The causal self-attention mask is pk_masked_softmax's
// (fs2.cu).  No atomics: every reduction runs in a fixed order.
#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace {

// Sum of v over a 256-thread block in a fixed order (warp trees, then the 8 warp sums in order); every thread gets the result.
__device__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += red[w];
  return s;
}

// guided loss = lambda * sum(partials) / (heads_layers * sum_b ilen_b olen_b) -> losses[4], added to losses[0].  One block.
__global__ void __launch_bounds__(256)
guided_loss_kernel(const float* __restrict__ partials, long long n, const int32_t* __restrict__ ilens, const int32_t* __restrict__ olens,
                   int batch, int rows, int keys, int heads_layers, float lambda, float* __restrict__ losses) {
  __shared__ float red[8];
  float s = 0.f;
  for (long long k = threadIdx.x; k < n; k += 256) s += partials[k];
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) {
    long long cnt = 0;
    for (int q = 0; q < batch; ++q) cnt += static_cast<long long>(min(ilens[q], keys)) * min(olens[q], rows);
    const float g = cnt > 0 ? lambda * s / (static_cast<float>(heads_layers) * static_cast<float>(cnt)) : 0.f;
    losses[4] = g;
    losses[0] += g;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// TransformerTTSLoss (use_masking=True): over the frames t < olens[b],
//   l1 = mean|after - ys| + mean|before - ys|,  l2 = mean (after - ys)^2 + mean (before - ys)^2,
//   bce = mean [pw y softplus(-x) + (1 - y) softplus(x)]  (BCEWithLogitsLoss with pos_weight pw on the stop logits x),
// loss = l1 + bce (loss_type 0, "L1"), l2 + bce (1, "L2"), l1 + l2 + bce (2, "L1+L2").
// Pass 1: one block per TTS_LOSS_FRAMES frames writes its three partial sums; pass 2 (one block) sums them in block order.
// ---------------------------------------------------------------------------------------------------------------
constexpr int TTS_LOSS_FRAMES = 32;

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

__global__ void __launch_bounds__(256)
tts_loss_partial_kernel(const float* __restrict__ before, const float* __restrict__ after, const float* __restrict__ ys,
                        const float* __restrict__ logits, const float* __restrict__ labels, const int32_t* __restrict__ olens, int batch,
                        int l_max, int odim, float pos_weight, float* __restrict__ part) {
  __shared__ float red[8];
  const long long f0 = static_cast<long long>(blockIdx.x) * TTS_LOSS_FRAMES;
  const long long frames = static_cast<long long>(batch) * l_max;
  const long long f1 = min(f0 + TTS_LOSS_FRAMES, frames);
  float s1 = 0.f, s2 = 0.f, sb = 0.f;
  for (long long e = f0 * odim + threadIdx.x; e < f1 * odim; e += 256) {
    const long long f = e / odim;
    if (static_cast<int>(f % l_max) < __ldg(olens + f / l_max)) {
      const float y = ys[e], da = after[e] - y, db = before[e] - y;
      s1 += fabsf(da) + fabsf(db);
      s2 += da * da + db * db;
    }
  }
  if (threadIdx.x < TTS_LOSS_FRAMES) {
    const long long f = f0 + threadIdx.x;
    if (f < f1 && static_cast<int>(f % l_max) < __ldg(olens + f / l_max)) {
      const float x = logits[f], y = labels[f];
      sb = pos_weight * y * softplus(-x) + (1.f - y) * softplus(x);
    }
  }
  s1 = block_sum_256(s1, red);
  s2 = block_sum_256(s2, red);
  sb = block_sum_256(sb, red);
  if (threadIdx.x == 0) {
    part[3 * blockIdx.x] = s1;
    part[3 * blockIdx.x + 1] = s2;
    part[3 * blockIdx.x + 2] = sb;
  }
}

__global__ void __launch_bounds__(256)
tts_loss_final_kernel(const float* __restrict__ part, int nparts, const int32_t* __restrict__ olens, int batch, int l_max, int odim,
                      int loss_type, float* __restrict__ losses) {
  __shared__ float red[8];
  float s1 = 0.f, s2 = 0.f, sb = 0.f;
  for (int k = threadIdx.x; k < nparts; k += 256) {
    s1 += part[3 * k];
    s2 += part[3 * k + 1];
    sb += part[3 * k + 2];
  }
  s1 = block_sum_256(s1, red);
  s2 = block_sum_256(s2, red);
  sb = block_sum_256(sb, red);
  if (threadIdx.x == 0) {
    long long frames = 0;
    for (int b = 0; b < batch; ++b) frames += max(0, min(olens[b], l_max));
    const float inv_f = frames > 0 ? 1.f / static_cast<float>(frames) : 0.f;
    const float inv_e = frames > 0 ? 1.f / (static_cast<float>(frames) * odim) : 0.f;
    const float l1 = s1 * inv_e, l2 = s2 * inv_e, bce = sb * inv_f;
    losses[0] = (loss_type == 1 ? l2 : loss_type == 2 ? l1 + l2 : l1) + bce;
    losses[1] = l1;
    losses[2] = l2;
    losses[3] = bce;
  }
}

// gradients of the loss above w.r.t. before, after (B, l_max, odim) and the stop logits (B, l_max); 0 on the padded frames
__global__ void __launch_bounds__(256)
tts_loss_bwd_kernel(const float* __restrict__ before, const float* __restrict__ after, const float* __restrict__ ys,
                    const float* __restrict__ logits, const float* __restrict__ labels, const int32_t* __restrict__ olens, int batch, int l_max,
                    int odim, float pos_weight, int loss_type, float* __restrict__ g_before, float* __restrict__ g_after,
                    float* __restrict__ g_logits) {
  long long frames = 0;
  for (int b = 0; b < batch; ++b) frames += max(0, min(__ldg(olens + b), l_max));
  const float inv_f = frames > 0 ? 1.f / static_cast<float>(frames) : 0.f;
  const float inv_e = frames > 0 ? 1.f / (static_cast<float>(frames) * odim) : 0.f;
  const float w1 = loss_type == 1 ? 0.f : inv_e, w2 = loss_type == 0 ? 0.f : 2.f * inv_e;
  const long long n = static_cast<long long>(batch) * l_max * odim;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i < n) {
    const long long f = i / odim;
    float gb = 0.f, ga = 0.f;
    if (static_cast<int>(f % l_max) < __ldg(olens + f / l_max)) {
      const float y = ys[i], da = after[i] - y, db = before[i] - y;
      ga = w1 * (da > 0.f ? 1.f : (da < 0.f ? -1.f : 0.f)) + w2 * da;
      gb = w1 * (db > 0.f ? 1.f : (db < 0.f ? -1.f : 0.f)) + w2 * db;
    }
    g_before[i] = gb;
    g_after[i] = ga;
  }
  if (i < static_cast<long long>(batch) * l_max) {
    float g = 0.f;
    if (static_cast<int>(i % l_max) < __ldg(olens + i / l_max)) {
      const float x = logits[i], y = labels[i];
      const float sig = 1.f / (1.f + expf(-x));
      g = (sig * (pos_weight * y + 1.f - y) - pos_weight * y) * inv_f;
    }
    g_logits[i] = g;
  }
}

}  // namespace
}  // namespace pk

using namespace pk;

extern "C" int pk_tts_guided_loss(const float* partials, int64_t n, const int32_t* ilens, const int32_t* olens, int32_t batch, int32_t rows,
                                  int32_t keys, int32_t heads_layers, float lambda, float* losses, pk_stream_t stream) {
  PK_CHECK_ARG(partials && ilens && olens && losses && n > 0 && batch > 0 && rows > 0 && keys > 0 && heads_layers > 0,
               "bad arguments to pk_tts_guided_loss");
  guided_loss_kernel<<<1, 256, 0, PK_STREAM>>>(partials, n, ilens, olens, batch, rows, keys, heads_layers, lambda, losses);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int64_t pk_tts_loss_workspace(int32_t batch, int32_t l_max) {
  return 3 * ((static_cast<int64_t>(batch) * l_max + TTS_LOSS_FRAMES - 1) / TTS_LOSS_FRAMES);
}

extern "C" int pk_tts_loss(const float* before, const float* after, const float* ys, const float* logits, const float* labels,
                           const int32_t* olens, int32_t batch, int32_t l_max, int32_t odim, float pos_weight, int32_t loss_type,
                           float* workspace, float* losses, pk_stream_t stream) {
  PK_CHECK_ARG(before && after && ys && logits && labels && olens && workspace && losses && batch > 0 && l_max > 0 && odim > 0,
               "bad arguments to pk_tts_loss");
  PK_CHECK_ARG(loss_type >= 0 && loss_type <= 2, "loss_type must be 0 (L1), 1 (L2) or 2 (L1+L2)");
  const int parts = static_cast<int>(pk_tts_loss_workspace(batch, l_max) / 3);
  tts_loss_partial_kernel<<<parts, 256, 0, PK_STREAM>>>(before, after, ys, logits, labels, olens, batch, l_max, odim, pos_weight, workspace);
  tts_loss_final_kernel<<<1, 256, 0, PK_STREAM>>>(workspace, parts, olens, batch, l_max, odim, loss_type, losses);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch(2);
  return PK_OK;
}

extern "C" int pk_tts_loss_bwd(const float* before, const float* after, const float* ys, const float* logits, const float* labels,
                               const int32_t* olens, int32_t batch, int32_t l_max, int32_t odim, float pos_weight, int32_t loss_type,
                               float* g_before, float* g_after, float* g_logits, pk_stream_t stream) {
  PK_CHECK_ARG(before && after && ys && logits && labels && olens && g_before && g_after && g_logits && batch > 0 && l_max > 0 && odim > 0,
               "bad arguments to pk_tts_loss_bwd");
  PK_CHECK_ARG(loss_type >= 0 && loss_type <= 2, "loss_type must be 0 (L1), 1 (L2) or 2 (L1+L2)");
  const long long n = static_cast<long long>(batch) * l_max * odim;
  tts_loss_bwd_kernel<<<nblk(n, 256), 256, 0, PK_STREAM>>>(before, after, ys, logits, labels, olens, batch, l_max, odim, pos_weight,
                                                          loss_type, g_before, g_after, g_logits);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
