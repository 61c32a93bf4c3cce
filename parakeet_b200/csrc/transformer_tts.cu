// TransformerTTS (reference: parakeet/models/transformer_tts/transformer_tts.py `inference`, modules/fastspeech2_transformer/
// decoder.py `forward_one_step`, decoder_layer.py with a cache): the autoregressive decoder as one persistent launch, B = 1.
//
// Step s feeds the last of the r frames of step s - 1 (zeros at s = 0) through the decoder prenet (ReLU, then the always-on
// dropout keyed by frame position: site i for prenet layer i, Philox step s, element j), the input Linear and + alpha pe[s]
// (rows precomputed by pk_embed_pe, so the decoder adds the very values the teacher-forced path adds).
// Then, per decoder layer (pre-LN, concat_after = False), for the new row only:
//   QKV   LN1 -> q, k, v; k and v appended to the layer's cache at row s
//   SA    softmax(q k^T / sqrt(d_k)) v over cache rows 0..s             one CTA per head
//   O1    x += linear_out(ctx)
//   CQ    LN2 -> cross q
//   CA    softmax(q K_mem^T / sqrt(d_k)) V_mem over the encoder rows    one CTA per head; the weights go to att_ws[l, h, s, :]
//   O2    x += linear_out(ctx)
//   F1    LN3 -> relu(w_1 x + b_1)                                       the decoder's PositionwiseFeedForward is two Linears
//   F2    x += w_2 u + b_2
// and last after_norm -> [prob_out | feat_out]; CTA 0 applies the stop rule.  Each arrow is a grid hand-off; LayerNorm statistics
// of the 1 x adim row are recomputed by every CTA that needs them, so the hand-offs sit only after the matrix-vector phases.
// Caching K / V is exact: layer l >= 1 reads earlier rows from the reference's own cache, and layer 0's re-embedded earlier
// frames are the same rows every step because the prenet masks are keyed by frame position, not by step.
// The cross-attention K / V of every layer come from one pk_conv_gemm over the encoder output before the launch.
// All math is fp32 FFMA; every dot product is one warp in a fixed order and nothing uses atomics: a seed gives bit-identical output.
#include <cuda_runtime.h>
#include <stdint.h>

#include "pk_decode.cuh"
#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace tts {

using namespace pdec;

struct Ws {
  long long x, q, ctx, h, u, kc, vc, total;
};
__host__ __device__ inline long long up4(long long n) { return (n + 3) / 4 * 4; }
__host__ __device__ inline Ws ws_layout(int A, int U, int Up, int L, int steps) {
  Ws s;
  long long o = 4;                          // [0] grid counter, [1] frame count at the stop
  s.x = o; o += up4(A);
  s.q = o; o += up4(A);
  s.ctx = o; o += up4(A);
  s.h = o; o += 2 * up4(Up);
  s.u = o; o += up4(U);
  s.kc = o; o += static_cast<long long>(L) * steps * A;
  s.vc = o; o += static_cast<long long>(L) * steps * A;
  s.total = o;
  return s;
}

// one decoder layer's fp32 weights, [out][in] rows: wqkv, bqkv, wo_s, bo_s, wq_c, bq_c, wo_c, bo_c, w1, b1, w2, b2, then the
// three LayerNorms (gamma, beta) -- the order models/transformer_tts.py packs them in
struct LayerOff {
  long long wqkv, bqkv, wo_s, bo_s, wq_c, bq_c, wo_c, bo_c, w1, b1, w2, b2, ln, total;
};
__host__ __device__ inline LayerOff layer_off(int A, int U) {
  LayerOff f;
  long long o = 0;
  f.wqkv = o; o += 3ll * A * A;
  f.bqkv = o; o += 3ll * A;
  f.wo_s = o; o += 1ll * A * A;
  f.bo_s = o; o += A;
  f.wq_c = o; o += 1ll * A * A;
  f.bq_c = o; o += A;
  f.wo_c = o; o += 1ll * A * A;
  f.bo_c = o; o += A;
  f.w1 = o; o += 1ll * U * A;
  f.b1 = o; o += U;
  f.w2 = o; o += 1ll * A * U;
  f.b2 = o; o += A;
  f.ln = o; o += 6ll * A;
  f.total = o;
  return f;
}

struct Params {
  int t_enc, A, H, dk, U, odim, r, n_pre, Up, L, steps, minlen, maxlen, grid, kmax;
  float threshold, scale, p_prenet, drop_scale;
  uint32_t drop_thresh, seed_lo, seed_hi;
  const float* mem_kv;      // (t_enc, L * 2A): [K_0 | V_0 | K_1 | V_1 | ...]
  const float* pre_w; const float* pre_b; const float* in_w; const float* in_b; const float* pe;
  const float* lw; const float* norm; const float* out_w; const float* out_b;
  float* ws; Ws W; LayerOff F;
  float* outs; float* probs; float* att_ws; int32_t* frames;
};

struct Smem {
  float* xs;     // [kmax] staged input vector
  float* sc;     // [max(steps, t_enc)] attention scores / weights
  float* part;   // [kThreads] context partial sums
  float* qs;     // [dk]
  float* red;    // [2 * kWarps]
};

// xs[0..K) = src (written by other CTAs of this launch: L2 loads)
__device__ __forceinline__ void stage(const float* src, int K, float* xs) {
  for (int i = threadIdx.x; i < K; i += kThreads) xs[i] = __ldcg(src + i);
  __syncthreads();
}

// xs = LayerNorm(x) (eps 1e-5 inside the square root), statistics in a fixed order so that every CTA gets the same row
__device__ __forceinline__ void stage_ln(const float* x, const float* g, const float* b, int A, float* xs, float* red) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  float s = 0.f;
  for (int i = threadIdx.x; i < A; i += kThreads) { const float v = __ldcg(x + i); xs[i] = v; s += v; }
  s = warp_sum(s);
  if (lane == 0) red[warp] = s;
  __syncthreads();
  float mean = 0.f;
  for (int i = 0; i < kWarps; ++i) mean += red[i];
  mean /= static_cast<float>(A);
  float v2 = 0.f;
  for (int i = threadIdx.x; i < A; i += kThreads) { const float d = xs[i] - mean; v2 = fmaf(d, d, v2); }
  v2 = warp_sum(v2);
  if (lane == 0) red[kWarps + warp] = v2;
  __syncthreads();
  float var = 0.f;
  for (int i = 0; i < kWarps; ++i) var += red[kWarps + i];
  const float rstd = rsqrtf(var / static_cast<float>(A) + 1e-5f);
  for (int i = threadIdx.x; i < A; i += kThreads) xs[i] = (xs[i] - mean) * rstd * __ldg(g + i) + __ldg(b + i);
  __syncthreads();
}

// sink(row, W_row . xs) for the rows of an n-row matrix this CTA owns: blocks of kWarps rows, block k on CTA k mod grid
template <class RowPtr, class Sink>
__device__ __forceinline__ void rows_phase(const Params& p, int K, int n, RowPtr row_ptr, Sink sink, const float* xs) {
  const int G = p.grid, cta = blockIdx.x;
  const int nb = (n + kWarps - 1) / kWarps;
  const int mine = cta < nb ? (nb - cta + G - 1) / G : 0;
  auto row_of = [&](int rl) { return ((rl / kWarps) * G + cta) * kWarps + rl % kWarps; };
  matvec_rows<1>(
      K, mine * kWarps, [&](int rl) { return row_ptr(min(row_of(rl), n - 1)); },
      [&](int rl, int, float y) {
        const int row = row_of(rl);
        if (row < n) sink(row, y);
      },
      xs);
  __syncthreads();
}

// one head: ctx[0..dk) = softmax(scale q K^T) V over n keys (rows of K / V ld floats apart); the weights also go to att (or not)
__device__ __forceinline__ void attend(const Params& p, const float* q, const float* K, const float* V, long long ld, int n, float* ctx, float* att,
                       const Smem s) {
  const int warp = threadIdx.x / 32, lane = threadIdx.x & 31, dk = p.dk;
  for (int d = threadIdx.x; d < dk; d += kThreads) s.qs[d] = __ldcg(q + d);
  __syncthreads();
  for (int j = warp; j < n; j += kWarps) {
    const float* k = K + static_cast<long long>(j) * ld;
    float acc = 0.f;
    for (int d = lane; d < dk; d += 32) acc = fmaf(s.qs[d], __ldcg(k + d), acc);
    acc = warp_sum(acc);
    if (lane == 0) s.sc[j] = acc * p.scale;
  }
  __syncthreads();
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n; i += kThreads) m = fmaxf(m, s.sc[i]);
  m = warp_max(m);
  if (lane == 0) s.red[warp] = m;
  __syncthreads();
  m = s.red[0];
  for (int i = 1; i < kWarps; ++i) m = fmaxf(m, s.red[i]);
  float sum = 0.f;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const float e = expf(s.sc[i] - m);
    s.sc[i] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) s.red[kWarps + warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < kWarps; ++i) sum += s.red[kWarps + i];
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const float a = s.sc[i] / sum;
    s.sc[i] = a;
    if (att) att[i] = a;
  }
  __syncthreads();
  // context: thread t sums column t % dk over its contiguous chunk of keys, then the chunks in order
  const int nch = kThreads / dk, t = threadIdx.x;
  if (t < nch * dk) {
    const int d = t % dk, c = t / dk, per = (n + nch - 1) / nch, j0 = c * per, j1 = min(n, j0 + per);
    float acc = 0.f;
    for (int j = j0; j < j1; ++j) acc = fmaf(s.sc[j], __ldcg(V + static_cast<long long>(j) * ld + d), acc);
    s.part[t] = acc;
  }
  __syncthreads();
  for (int d = threadIdx.x; d < dk; d += kThreads) {
    float acc = 0.f;
    for (int c = 0; c < nch; ++c) acc += s.part[c * dk + d];
    ctx[d] = acc;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads, 1) tts_decode_kernel(const __grid_constant__ Params p) {
  extern __shared__ float4 smem4[];
  float* smem = reinterpret_cast<float*>(smem4);
  Smem s;
  s.xs = smem;
  s.sc = s.xs + up4(p.kmax);
  s.part = s.sc + up4(p.steps > p.t_enc ? p.steps : p.t_enc);
  s.qs = s.part + kThreads;
  s.red = s.qs + up4(p.dk);
  unsigned* ctr = reinterpret_cast<unsigned*>(p.ws);
  unsigned* done = ctr + 1;
  unsigned target = 0;
  const int G = p.grid, cta = blockIdx.x, A = p.A, dk = p.dk, fr = p.r * p.odim;
  float* x = p.ws + p.W.x;
  float* q = p.ws + p.W.q;
  float* ctx = p.ws + p.W.ctx;
  float* u = p.ws + p.W.u;
  const long long mld = 2ll * A * p.L;
  int frames = p.steps;
  for (int t = 0; t < p.steps; ++t) {
    // decoder prenet on frame t - 1's last frame (zeros at t = 0): Linear -> ReLU -> dropout, site = layer, step = position t
    for (int i = 0; i < p.n_pre; ++i) {
      const int kin = i == 0 ? p.odim : p.Up;
      const float* w = p.pre_w + (i == 0 ? 0ll : static_cast<long long>(p.Up) * p.odim + static_cast<long long>(i - 1) * p.Up * p.Up);
      float* h = p.ws + p.W.h + (i & 1) * up4(p.Up);
      if (i == 0) {
        if (t == 0) {
          for (int k = threadIdx.x; k < kin; k += kThreads) s.xs[k] = 0.f;
          __syncthreads();
        } else {
          stage(p.outs + static_cast<long long>(t - 1) * fr + (p.r - 1) * p.odim, kin, s.xs);
        }
      } else {
        stage(p.ws + p.W.h + ((i - 1) & 1) * up4(p.Up), kin, s.xs);
      }
      rows_phase(
          p, kin, p.Up, [&](int row) { return w + static_cast<long long>(row) * kin; },
          [&](int j, float y) {
            float v = fmaxf(y + __ldg(p.pre_b + i * p.Up + j), 0.f);
            if (p.p_prenet > 0.f) {
              uint32_t rr[4];
              philox4x32_10(static_cast<uint32_t>(j) >> 2, 0u, static_cast<uint32_t>(i), static_cast<uint32_t>(t), p.seed_lo, p.seed_hi, rr);
              const uint32_t rj = (j & 2) ? ((j & 1) ? rr[3] : rr[2]) : ((j & 1) ? rr[1] : rr[0]);   // no local-memory index
              v = rj >= p.drop_thresh ? v * p.drop_scale : 0.f;
            }
            h[j] = v;
          },
          s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
    }
    // input Linear + alpha pe[t] (ScaledPositionalEncoding; pe holds alpha pe rows from pk_embed_pe)
    stage(p.ws + p.W.h + ((p.n_pre - 1) & 1) * up4(p.Up), p.Up, s.xs);
    rows_phase(
        p, p.Up, A, [&](int row) { return p.in_w + static_cast<long long>(row) * p.Up; },
        [&](int c, float y) { x[c] = (y + __ldg(p.in_b + c)) + __ldg(p.pe + static_cast<long long>(t) * A + c); },
        s.xs);
    grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
    for (int l = 0; l < p.L; ++l) {
      const float* lw = p.lw + static_cast<long long>(l) * p.F.total;
      const float* ln = lw + p.F.ln;
      float* kc = p.ws + p.W.kc + static_cast<long long>(l) * p.steps * A;
      float* vc = p.ws + p.W.vc + static_cast<long long>(l) * p.steps * A;
      // QKV of the new row; k, v appended to the cache
      stage_ln(x, ln, ln + A, A, s.xs, s.red);
      rows_phase(
          p, A, 3 * A, [&](int row) { return lw + p.F.wqkv + static_cast<long long>(row) * A; },
          [&](int row, float y) {
            const float v = y + __ldg(lw + p.F.bqkv + row);
            if (row < A) q[row] = v;
            else if (row < 2 * A) kc[static_cast<long long>(t) * A + row - A] = v;
            else vc[static_cast<long long>(t) * A + row - 2 * A] = v;
          },
          s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      for (int h = cta; h < p.H; h += G) attend(p, q + h * dk, kc + h * dk, vc + h * dk, A, t + 1, ctx + h * dk, nullptr, s);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      stage(ctx, A, s.xs);
      rows_phase(
          p, A, A, [&](int row) { return lw + p.F.wo_s + static_cast<long long>(row) * A; },
          [&](int c, float y) { x[c] = __ldcg(x + c) + (y + __ldg(lw + p.F.bo_s + c)); }, s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      // source attention over the encoder output
      stage_ln(x, ln + 2 * A, ln + 3 * A, A, s.xs, s.red);
      rows_phase(
          p, A, A, [&](int row) { return lw + p.F.wq_c + static_cast<long long>(row) * A; },
          [&](int c, float y) { q[c] = y + __ldg(lw + p.F.bq_c + c); }, s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      for (int h = cta; h < p.H; h += G) {
        const float* km = p.mem_kv + 2ll * A * l + h * dk;
        float* att = p.att_ws + ((static_cast<long long>(l) * p.H + h) * p.steps + t) * p.t_enc;
        attend(p, q + h * dk, km, km + A, mld, p.t_enc, ctx + h * dk, att, s);
      }
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      stage(ctx, A, s.xs);
      rows_phase(
          p, A, A, [&](int row) { return lw + p.F.wo_c + static_cast<long long>(row) * A; },
          [&](int c, float y) { x[c] = __ldcg(x + c) + (y + __ldg(lw + p.F.bo_c + c)); }, s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      // position-wise feed-forward on the one row
      stage_ln(x, ln + 4 * A, ln + 5 * A, A, s.xs, s.red);
      rows_phase(
          p, A, p.U, [&](int row) { return lw + p.F.w1 + static_cast<long long>(row) * A; },
          [&](int j, float y) { u[j] = fmaxf(y + __ldg(lw + p.F.b1 + j), 0.f); }, s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
      stage(u, p.U, s.xs);
      rows_phase(
          p, p.U, A, [&](int row) { return lw + p.F.w2 + static_cast<long long>(row) * p.U; },
          [&](int c, float y) { x[c] = __ldcg(x + c) + (y + __ldg(lw + p.F.b2 + c)); }, s.xs);
      grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
    }
    // after_norm -> [prob_out (r rows, CTA 0) | feat_out (r odim rows)]
    stage_ln(x, p.norm, p.norm + A, A, s.xs, s.red);
    rows_phase(
        p, A, p.r + fr, [&](int row) { return p.out_w + static_cast<long long>(row) * A; },
        [&](int row, float y) {
          const float v = y + __ldg(p.out_b + row);
          if (row < p.r) p.probs[static_cast<long long>(t) * p.r + row] = sigmoidf_(v);
          else p.outs[static_cast<long long>(t) * fr + row - p.r] = v;
        },
        s.xs);
    if (cta == 0 && threadIdx.x == 0) {
      // inference's loop exit after step idx = t + 1: (any prob >= threshold or idx >= maxlen) and idx >= minlen
      const int idx = t + 1;
      bool hit = idx >= p.maxlen;
      for (int j = 0; j < p.r; ++j) hit |= p.probs[static_cast<long long>(t) * p.r + j] >= p.threshold;
      if ((hit && idx >= p.minlen) || idx == p.steps) *reinterpret_cast<volatile unsigned*>(done) = static_cast<unsigned>(idx);
    }
    grid_sync(ctr, target, G, nullptr, 0, 0, nullptr);
    const unsigned d = ld_acquire_gpu(done);
    if (d) { frames = static_cast<int>(d); break; }
  }
  if (cta == 0 && threadIdx.x == 0) p.frames[0] = frames;
}

// ---------------------------------------------------------------------------------------------------------------
// glue of the teacher-forced forward (TransformerTTS.forward / _forward)
// ---------------------------------------------------------------------------------------------------------------
// xs[b] = [text[b, :lens[b]], eos, 0 ...] (width T + 1), ilens = lens + 1
__global__ void text_eos_kernel(const int64_t* __restrict__ text, const int32_t* __restrict__ lens, int B, int T, long long eos,
                                int64_t* __restrict__ xs, int32_t* __restrict__ ilens) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(B) * (T + 1)) return;
  const int b = static_cast<int>(i / (T + 1)), t = static_cast<int>(i % (T + 1));
  const int len = lens[b];
  xs[i] = t < len ? text[static_cast<long long>(b) * T + t] : (t == len ? eos : 0);
  if (t == 0) ilens[b] = len + 1;
}

// out[b, 0] = 0, out[b, t] = ys[b, t r - 1]: ys[:, r-1::r] with a zero first frame and the last frame dropped
__global__ void shift_frames_kernel(const float* __restrict__ ys, int B, int L, int odim, int r, float* __restrict__ out) {
  const int Lr = L / r;
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(B) * Lr * odim) return;
  const int c = static_cast<int>(i % odim);
  const long long bt = i / odim;
  const int t = static_cast<int>(bt % Lr), b = static_cast<int>(bt / Lr);
  out[i] = t == 0 ? 0.f : ys[(static_cast<long long>(b) * L + static_cast<long long>(t) * r - 1) * odim + c];
}

// the decoder prenet's dropout on (B, L, U), keyed by frame position: site, Philox step t, element b U + j (pk_tts_decode's masks)
__global__ void prenet_dropout_kernel(float* __restrict__ x, int B, int L, int U, uint32_t thresh, float scale, uint32_t seed_lo,
                                      uint32_t seed_hi, uint32_t site) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(B) * L * U) return;
  const int j = static_cast<int>(i % U);
  const long long bt = i / U;
  const int t = static_cast<int>(bt % L), b = static_cast<int>(bt / L);
  const uint32_t e = static_cast<uint32_t>(b * U + j);
  uint32_t rr[4];
  philox4x32_10(e >> 2, 0u, site, static_cast<uint32_t>(t), seed_lo, seed_hi, rr);
  const uint32_t re = (e & 2) ? ((e & 1) ? rr[3] : rr[2]) : ((e & 1) ? rr[1] : rr[0]);
  x[i] = re >= thresh ? x[i] * scale : 0.f;
}

// stop labels: pad(make_pad_mask(olens - 1), 1 column of ones); the last column is 1 for every utterance
__global__ void stop_labels_kernel(const int32_t* __restrict__ olens, int B, int W, float* __restrict__ out) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(B) * W) return;
  const int b = static_cast<int>(i / W), t = static_cast<int>(i % W);
  out[i] = (t >= olens[b] - 1 || t == W - 1) ? 1.f : 0.f;
}

size_t smem_bytes(int kmax, int steps, int t_enc, int dk) {
  return sizeof(float) * (up4(kmax) + up4(steps > t_enc ? steps : t_enc) + kThreads + up4(dk) + 2 * kWarps);
}

}  // namespace tts
}  // namespace pk

using namespace pk;
using namespace pk::tts;

extern "C" int64_t pk_tts_layer_floats(int32_t adim, int32_t units) { return layer_off(adim, units).total; }

extern "C" int64_t pk_tts_workspace(int32_t adim, int32_t units, int32_t prenet_units, int32_t layers, int32_t steps) {
  return ws_layout(adim, units, prenet_units, layers, steps).total;
}

extern "C" int pk_tts_decode(const PkTtsDecodeArgs* a, pk_stream_t stream) {
  PK_CHECK_ARG(a != nullptr, "NULL arguments");
  PK_CHECK_ARG(a->t_enc >= 1 && a->steps >= 1 && a->layers >= 1 && a->heads >= 1 && a->prenet_layers >= 1 && a->r >= 1 &&
                   a->minlen >= 0 && a->maxlen >= 0, "t_enc, steps, layers, heads, prenet_layers and r must be >= 1");
  PK_CHECK_ARG(a->steps >= a->minlen && a->steps >= a->maxlen, "steps must hold max(minlen, maxlen) decoder steps");
  const int A = a->adim, H = a->heads;
  // head widths: the ones TransformerTTS can build (its teacher-forced path runs pk_fused_attention_ex, which takes 64, 128, 192)
  const int dk = A % H == 0 ? A / H : 0;
  if ((dk != 64 && dk != 128 && dk != 192) || a->units % 4 || a->prenet_units % 4 || a->odim % 4 || a->r > kWarps)
    return fail(PK_ERR_UNSUPPORTED, "pk_tts_decode supports head widths 64, 128 and 192, units, prenet units and odim multiples of 4 "
                                    "and r <= %d (got adim %d, heads %d, units %d, prenet %d, odim %d, r %d)",
                kWarps, A, H, a->units, a->prenet_units, a->odim, a->r);
  PK_CHECK_ARG(a->mem_kv && a->pre_w && a->pre_b && a->in_w && a->in_b && a->pe && a->layer_w && a->norm && a->out_w && a->out_b &&
                   a->workspace && a->outs && a->probs && a->att_ws && a->frames, "NULL pointer in pk_tts_decode");
  PK_CHECK_ARG(a->p_prenet >= 0.f && a->p_prenet < 1.f, "prenet dropout must be in [0, 1)");
  PK_CHECK_ARG(aligned16(a->pre_w) && aligned16(a->in_w) && aligned16(a->layer_w) && aligned16(a->out_w) && aligned16(a->workspace) &&
                   aligned16(a->outs), "weights, outs and the workspace must be 16-byte aligned");
  const Ws W = ws_layout(A, a->units, a->prenet_units, a->layers, a->steps);
  PK_CHECK_ARG(a->workspace_len >= W.total, "workspace must hold pk_tts_workspace() = %lld floats", W.total);
  Params p;
  p.t_enc = a->t_enc; p.A = A; p.H = H; p.dk = A / H; p.U = a->units; p.odim = a->odim; p.r = a->r;
  p.n_pre = a->prenet_layers; p.Up = a->prenet_units; p.L = a->layers; p.steps = a->steps; p.minlen = a->minlen; p.maxlen = a->maxlen;
  int kmax = A > p.U ? A : p.U;
  kmax = kmax > p.Up ? kmax : p.Up;
  p.kmax = kmax > p.odim ? kmax : p.odim;
  p.threshold = a->threshold;
  p.scale = 1.f / sqrtf(static_cast<float>(p.dk));
  p.p_prenet = a->p_prenet;
  p.drop_scale = a->p_prenet > 0.f ? 1.f / (1.f - a->p_prenet) : 1.f;
  const double th = static_cast<double>(a->p_prenet) * 4294967296.0;
  p.drop_thresh = th >= 4294967295.0 ? 0xFFFFFFFFu : static_cast<uint32_t>(th);
  p.seed_lo = static_cast<uint32_t>(a->seed); p.seed_hi = static_cast<uint32_t>(a->seed >> 32);
  p.mem_kv = a->mem_kv; p.pre_w = a->pre_w; p.pre_b = a->pre_b; p.in_w = a->in_w; p.in_b = a->in_b; p.pe = a->pe;
  p.lw = a->layer_w; p.norm = a->norm; p.out_w = a->out_w; p.out_b = a->out_b;
  p.ws = a->workspace; p.W = W; p.F = layer_off(A, p.U);
  p.outs = a->outs; p.probs = a->probs; p.att_ws = a->att_ws; p.frames = a->frames;
  const size_t smem = smem_bytes(p.kmax, p.steps, p.t_enc, p.dk);
  if (smem > 200 * 1024)
    return fail(PK_ERR_UNSUPPORTED, "pk_tts_decode: max(steps, t_enc) = %d does not fit the attention scores in shared memory",
                p.steps > p.t_enc ? p.steps : p.t_enc);
  if (int rc = prepare_kernel(tts_decode_kernel, kThreads, smem, &p.grid)) return rc;
  if (p.grid < H)
    return fail(PK_ERR_UNSUPPORTED, "pk_tts_decode: only %d CTAs can be co-resident (needs one per head, %d)", p.grid, H);
  auto st = static_cast<cudaStream_t>(stream);
  // zero the counters and the outputs (rows past the stop stay zero); the K / V caches are written before they are read
  PK_CHECK_CUDA(cudaMemsetAsync(a->workspace, 0, 4 * sizeof(float), st));
  PK_CHECK_CUDA(cudaMemsetAsync(a->outs, 0, static_cast<size_t>(a->steps) * a->r * a->odim * sizeof(float), st));
  PK_CHECK_CUDA(cudaMemsetAsync(a->probs, 0, static_cast<size_t>(a->steps) * a->r * sizeof(float), st));
  PK_CHECK_CUDA(cudaMemsetAsync(a->att_ws, 0, static_cast<size_t>(a->layers) * H * a->steps * a->t_enc * sizeof(float), st));
  tts_decode_kernel<<<p.grid, kThreads, smem, st>>>(p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_tts_text_eos(const int64_t* text, const int32_t* lens, int32_t batch, int32_t t, int64_t eos, int64_t* xs, int32_t* ilens,
                               pk_stream_t stream) {
  // text may be NULL when t == 0 (an empty tensor has no storage): every row is then [eos] and text is never read
  PK_CHECK_ARG((text || t == 0) && lens && xs && ilens && batch > 0 && t >= 0, "bad arguments to pk_tts_text_eos");
  text_eos_kernel<<<nblk(static_cast<long long>(batch) * (t + 1), 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(text, lens, batch, t,
                                                                                                                     eos, xs, ilens);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_tts_shift_frames(const float* ys, int32_t batch, int32_t l, int32_t odim, int32_t r, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(ys && out && batch > 0 && l >= r && odim > 0 && r >= 1, "bad arguments to pk_tts_shift_frames");
  shift_frames_kernel<<<nblk(static_cast<long long>(batch) * (l / r) * odim, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(ys, batch, l,
                                                                                                                                odim, r, out);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_tts_prenet_dropout(float* x, int32_t batch, int32_t l, int32_t units, float p, uint64_t seed, int32_t site,
                                     pk_stream_t stream) {
  PK_CHECK_ARG(x && batch > 0 && l > 0 && units > 0 && p >= 0.f && p < 1.f && site >= 0, "bad arguments to pk_tts_prenet_dropout");
  const double th = static_cast<double>(p) * 4294967296.0;
  const uint32_t thresh = th >= 4294967295.0 ? 0xFFFFFFFFu : static_cast<uint32_t>(th);
  prenet_dropout_kernel<<<nblk(static_cast<long long>(batch) * l * units, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, batch, l, units, thresh, p > 0.f ? 1.f / (1.f - p) : 1.f, static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32),
      static_cast<uint32_t>(site));
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_tts_stop_labels(const int32_t* olens, int32_t batch, int32_t width, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(olens && out && batch > 0 && width > 0, "bad arguments to pk_tts_stop_labels");
  stop_labels_kernel<<<nblk(static_cast<long long>(batch) * width, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(olens, batch, width, out);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
