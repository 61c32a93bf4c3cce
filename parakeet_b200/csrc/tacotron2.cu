// Tacotron2 (reference: parakeet/models/tacotron2.py, parakeet/modules/attention.py LocationSensitiveAttention,
// parakeet/modules/losses.py guided_attention_loss): the autoregressive decoder as one persistent launch, the encoder's
// embedding / bidirectional-LSTM glue and the validation loss.
//
// pk_taco2_decode runs every decoder step of Tacotron2Decoder.infer (prenet input = the previous projection, stop rule on the
// device) or of Tacotron2Decoder.forward (teacher-forced: prenet input = frame t-1 of the given mels, energies masked with
// text_lens) in one launch of a co-resident grid.  A step is six phases separated by grid-wide hand-offs (a release add on
// one counter, acquired by every CTA):
//   P1  prenet layer 1 (256 rows x 80 r) + ReLU + dropout     rows spread over the grid, one warp per row
//   P2  prenet layer 2 (256 x 256) + ReLU + dropout           rows spread over the grid
//   A   attention LSTMCell on [prenet, context_{t-1}, h_att] CTA c owns units c, c + G, ... with all four gates each
//   B   location-sensitive attention                          CTA b owns batch item b (query layer, energies, softmax,
//                                                            context, w_cum), so the softmax needs no hand-off
//   C   decoder LSTMCell on [h_att, context, h_dec]           as A
//   D   projection + stop layer on [h_dec, context]           rows spread over the grid; CTA 0 evaluates the stop rule
// All math is fp32 FFMA.  Every dot product is one warp: each lane accumulates a fixed stride of K, then a xor butterfly;
// softmax and context sums run in a fixed order inside one CTA.  Nothing uses atomics, so a fixed seed gives bit-identical
// results, and both modes run the same arithmetic (infer fed its own frames reproduces infer).
#include <cuda_runtime.h>
#include <stdint.h>

#include "pk_host.h"
#include "pk_decode.cuh"
#include "pk_sm90.cuh"

namespace pk {
namespace taco2 {

using pdec::kThreads;
using pdec::kWarps;
using namespace pdec;
constexpr int kH = 1024;          // d_attention_rnn = d_decoder_rnn
constexpr int kPre = 256;         // d_prenet
constexpr int kAtt = 128;         // d_attention
constexpr int kMinGrid = 32;      // the gate staging below holds ceil(1024 / grid) units per CTA
constexpr int kGateRows = 4 * (kH / kMinGrid);
constexpr uint32_t kSitePrenet1 = 0, kSitePrenet2 = 1;   // Philox sites of the two prenet dropouts

// workspace (fp32 slots): [0] grid counter, [1] done flag, then the recurrent state, each part 16-byte aligned
struct Ws {
  long long h_att, c_att, h_dec, c_dec, ctx, w, wc, e, pre1, pre2, total;
};
__host__ __device__ inline long long up4(long long n) { return (n + 3) / 4 * 4; }
__host__ __device__ inline Ws ws_layout(int B, int t_enc, int d_enc) {
  Ws s;
  long long o = 4;
  s.h_att = o; o += up4(2ll * B * kH);
  s.c_att = o; o += up4(1ll * B * kH);
  s.h_dec = o; o += up4(2ll * B * kH);
  s.c_dec = o; o += up4(1ll * B * kH);
  s.ctx = o; o += up4(1ll * B * d_enc);
  s.w = o; o += up4(1ll * B * t_enc);
  s.wc = o; o += up4(1ll * B * t_enc);
  s.e = o; o += up4(1ll * B * t_enc);
  s.pre1 = o; o += up4(1ll * B * kPre);
  s.pre2 = o; o += up4(1ll * B * kPre);
  s.total = o;
  return s;
}

struct Params {
  int B, t_enc, d_enc, dmr, steps, teacher, loc_k, grid;
  float p_prenet, drop_scale;
  uint32_t drop_thresh, seed_lo, seed_hi;
  const float* keys; const float* pkeys; const int32_t* text_lens; const float* mels;
  const float* pre_w1; const float* pre_w2;
  const float* att_w; const float* att_b_ih; const float* att_b_hh;
  const float* q_w; const float* loc_w; const float* v_w;
  const float* dec_w; const float* dec_b_ih; const float* dec_b_hh;
  const float* proj_w; const float* proj_b; const float* stop_w; const float* stop_b;
  float* ws; Ws L;
  float* mel_out; float* align_out; float* stop_out; int32_t* frames;
  unsigned long long* prof;
};

constexpr int kPhases = 6;

// ReLU then the prenet's always-on dropout: element b * 256 + j of site `site` at decoder step `step` (pk_dropout's convention)
__device__ __forceinline__ float prenet_act(const Params& p, float v, int b, int j, uint32_t site, int step) {
  v = fmaxf(v, 0.f);
  if (p.p_prenet > 0.f) {
    const uint32_t i = static_cast<uint32_t>(b * kPre + j);
    uint32_t r[4];
    philox4x32_10(i >> 2, 0u, site, static_cast<uint32_t>(step), p.seed_lo, p.seed_hi, r);
    v = r[i & 3] >= p.drop_thresh ? v * p.drop_scale : 0.f;
  }
  return v;
}

// one LSTMCell (gate order i, f, g, o; two biases) for the units this CTA owns
template <int BC>
__device__ void lstm_phase(const Params& p, const float* W, const float* b_ih, const float* b_hh, const Seg (&seg)[3], float* c_state,
                           float* h_out, float* xs, float* gates) {
  const int G = p.grid, cta = blockIdx.x;
  const int nu = (kH - cta + G - 1) / G;
  const int K = seg[0].n + seg[1].n + seg[2].n;
  matvec<BC>(
      K, seg, p.B, 4 * nu,
      [&](int rl) { return W + static_cast<long long>((rl & 3) * kH + cta + G * (rl >> 2)) * K; },
      [&](int rl, int b, float y) { gates[rl * BC + (b % BC)] = y; },
      [&](int b0) {
        for (int idx = threadIdx.x; idx < nu * BC; idx += kThreads) {
          const int i = idx / BC, bb = idx - i * BC, b = b0 + bb, u = cta + G * i;
          if (b >= p.B) continue;
          const float* g = gates + 4 * i * BC + bb;
          const float ig = sigmoidf_(g[0] + b_ih[u] + b_hh[u]);
          const float fg = sigmoidf_(g[BC] + b_ih[kH + u] + b_hh[kH + u]);
          const float gg = tanhf(g[2 * BC] + b_ih[2 * kH + u] + b_hh[2 * kH + u]);
          const float og = sigmoidf_(g[3 * BC] + b_ih[3 * kH + u] + b_hh[3 * kH + u]);
          const float c = fg * c_state[b * kH + u] + ig * gg;
          c_state[b * kH + u] = c;
          h_out[b * kH + u] = og * tanhf(c);
        }
      },
      xs);
}

struct AttnSmem {
  float* locw;   // [128][2][loc_k], location_layer o location_conv folded
  float* v;      // [128]
  float* pq;     // [128]
  float* red;    // [2 * kWarps]
  int* ired;     // [kWarps]
};

// LocationSensitiveAttention for batch item b: energies over T_enc, softmax, context; w_cum += w.  -> argmax of w (first on ties)
template <int BC>
__device__ int attention_phase(const Params& p, int b, int t, const float* h_att, const AttnSmem& s, float* xs) {
  const int T = p.t_enc, warp = threadIdx.x / 32, lane = threadIdx.x & 31, half = p.loc_k / 2;
  float* w = p.ws + p.L.w + static_cast<long long>(b) * T;
  float* wc = p.ws + p.L.wc + static_cast<long long>(b) * T;
  float* e = p.ws + p.L.e + static_cast<long long>(b) * T;
  const Seg q[3] = {{h_att + static_cast<long long>(b) * kH, kH, 0}, {nullptr, 0, 0}, {nullptr, 0, 0}};
  matvec<1>(
      kH, q, 1, kAtt, [&](int rl) { return p.q_w + static_cast<long long>(rl) * kH; }, [&](int rl, int, float y) { s.pq[rl] = y; },
      [](int) {}, xs);
  const int lens = p.text_lens ? p.text_lens[b] : T;
  const float* pk = p.pkeys + static_cast<long long>(b) * T * kAtt;
  for (int tt = warp; tt < T; tt += kWarps) {
    float loc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < p.loc_k; ++k) {
      const int src = tt + k - half;
      if (src < 0 || src >= T) continue;
      const float a0 = __ldcg(w + src), a1 = __ldcg(wc + src);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* f = s.locw + (lane + 32 * j) * 2 * p.loc_k;
        loc[j] = fmaf(f[k], a0, loc[j]);
        loc[j] = fmaf(f[p.loc_k + k], a1, loc[j]);
      }
    }
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int d = lane + 32 * j;
      acc = fmaf(s.v[d], tanhf(loc[j] + __ldg(pk + static_cast<long long>(tt) * kAtt + d) + s.pq[d]), acc);
    }
    acc = warp_sum(acc);
    if (lane == 0) e[tt] = tt < lens ? acc : acc + -1e9f;
  }
  __syncthreads();
  // softmax over T (fixed-order block reductions)
  float m = -INFINITY;
  for (int i = threadIdx.x; i < T; i += kThreads) m = fmaxf(m, __ldcg(e + i));
  m = warp_max(m);
  if (lane == 0) s.red[warp] = m;
  __syncthreads();
  m = s.red[0];
  for (int i = 1; i < kWarps; ++i) m = fmaxf(m, s.red[i]);
  float sum = 0.f;
  for (int i = threadIdx.x; i < T; i += kThreads) sum += expf(__ldcg(e + i) - m);
  sum = warp_sum(sum);
  if (lane == 0) s.red[kWarps + warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < kWarps; ++i) sum += s.red[kWarps + i];
  float best = -1.f;
  int arg = 0x7fffffff;
  float* al = p.align_out + (static_cast<long long>(b) * p.steps + t) * T;
  for (int i = threadIdx.x; i < T; i += kThreads) {
    const float a = expf(__ldcg(e + i) - m) / sum;
    w[i] = a;
    wc[i] = __ldcg(wc + i) + a;
    al[i] = a;
    if (a > best) { best = a; arg = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  __syncthreads();                         // every thread is done with s.red
  if (lane == 0) { s.red[warp] = best; s.ired[warp] = arg; }
  __syncthreads();
  best = s.red[0];
  arg = s.ired[0];
  for (int i = 1; i < kWarps; ++i)
    if (s.red[i] > best || (s.red[i] == best && s.ired[i] < arg)) { best = s.red[i]; arg = s.ired[i]; }
  // context = sum_t w_t key_t, sequential in t
  const float* key = p.keys + static_cast<long long>(b) * T * p.d_enc;
  float* ctx = p.ws + p.L.ctx + static_cast<long long>(b) * p.d_enc;
  for (int c = threadIdx.x; c < p.d_enc; c += kThreads) {
    float acc = 0.f;
    for (int i = 0; i < T; ++i) acc = fmaf(__ldcg(w + i), __ldg(key + static_cast<long long>(i) * p.d_enc + c), acc);
    ctx[c] = acc;
  }
  __syncthreads();
  return arg;
}

template <int BC>
__global__ void __launch_bounds__(kThreads, 1) taco2_decode_kernel(const __grid_constant__ Params p) {
  extern __shared__ float4 smem4[];
  float* smem = reinterpret_cast<float*>(smem4);
  const int kx = 2 * kH + p.d_enc > p.dmr ? 2 * kH + p.d_enc : p.dmr;
  float* xs = smem;
  float* gates = xs + BC * kx;
  AttnSmem as;
  as.locw = gates + kGateRows * BC;
  as.v = as.locw + kAtt * 2 * p.loc_k;
  as.pq = as.v + kAtt;
  as.red = as.pq + kAtt;
  as.ired = reinterpret_cast<int*>(as.red + 2 * kWarps);
  __shared__ int s_arg0, s_first_hit;
  for (int i = threadIdx.x; i < kAtt * 2 * p.loc_k; i += kThreads) as.locw[i] = p.loc_w[i];
  for (int i = threadIdx.x; i < kAtt; i += kThreads) as.v[i] = p.v_w[i];
  if (threadIdx.x == 0) { s_arg0 = 0; s_first_hit = -1; }
  __syncthreads();

  unsigned* ctr = reinterpret_cast<unsigned*>(p.ws);
  unsigned* done = ctr + 1;
  unsigned target = 0;
  __shared__ unsigned long long s_last;     // thread 0's previous release time (phase timers only)
  if (threadIdx.x == 0 && p.prof) s_last = globaltimer();
  const int G = p.grid, cta = blockIdx.x, B = p.B, dmr = p.dmr;
  const long long fstride = static_cast<long long>(p.steps) * dmr;     // mel_out / mels: (B, steps, dmr)
  const float* feed = p.teacher ? p.mels : p.mel_out;
  float* pre1 = p.ws + p.L.pre1;
  float* pre2 = p.ws + p.L.pre2;
  float* ctx = p.ws + p.L.ctx;
  const int use_stop = p.stop_w != nullptr;
  const int n_out = dmr + use_stop;
  int frames = p.steps;
  for (int t = 0; t < p.steps; ++t) {
    float* h_att_prev = p.ws + p.L.h_att + static_cast<long long>(t & 1) * B * kH;
    float* h_att = p.ws + p.L.h_att + static_cast<long long>((t + 1) & 1) * B * kH;
    float* h_dec_prev = p.ws + p.L.h_dec + static_cast<long long>(t & 1) * B * kH;
    float* h_dec = p.ws + p.L.h_dec + static_cast<long long>((t + 1) & 1) * B * kH;
    // P1: prenet layer 1 on frame t - 1 (zeros at t = 0)
    for (int r0 = cta * kWarps; r0 < kPre; r0 += G * kWarps) {
      const Seg sg[3] = {{t > 0 ? feed + static_cast<long long>(t - 1) * dmr : nullptr, dmr, fstride}, {nullptr, 0, 0}, {nullptr, 0, 0}};
      matvec<BC>(
          dmr, sg, B, min(kWarps, kPre - r0), [&](int rl) { return p.pre_w1 + static_cast<long long>(r0 + rl) * dmr; },
          [&](int rl, int b, float y) { pre1[b * kPre + r0 + rl] = prenet_act(p, y, b, r0 + rl, kSitePrenet1, t); }, [](int) {}, xs);
    }
    grid_sync(ctr, target, G, p.prof, kPhases, 0, &s_last);
    // P2: prenet layer 2
    for (int r0 = cta * kWarps; r0 < kPre; r0 += G * kWarps) {
      const Seg sg[3] = {{pre1, kPre, kPre}, {nullptr, 0, 0}, {nullptr, 0, 0}};
      matvec<BC>(
          kPre, sg, B, min(kWarps, kPre - r0), [&](int rl) { return p.pre_w2 + static_cast<long long>(r0 + rl) * kPre; },
          [&](int rl, int b, float y) { pre2[b * kPre + r0 + rl] = prenet_act(p, y, b, r0 + rl, kSitePrenet2, t); }, [](int) {}, xs);
    }
    grid_sync(ctr, target, G, p.prof, kPhases, 1, &s_last);
    // A: attention LSTMCell
    {
      const Seg sg[3] = {{pre2, kPre, kPre}, {ctx, p.d_enc, p.d_enc}, {h_att_prev, kH, kH}};
      lstm_phase<BC>(p, p.att_w, p.att_b_ih, p.att_b_hh, sg, p.ws + p.L.c_att, h_att, xs, gates);
    }
    grid_sync(ctr, target, G, p.prof, kPhases, 2, &s_last);
    // B: attention, one CTA per batch item
    for (int b = cta; b < B; b += G) {
      const int a = attention_phase<BC>(p, b, t, h_att, as, xs);
      if (b == 0 && threadIdx.x == 0) s_arg0 = a;
    }
    grid_sync(ctr, target, G, p.prof, kPhases, 3, &s_last);
    // C: decoder LSTMCell
    {
      const Seg sg[3] = {{h_att, kH, kH}, {ctx, p.d_enc, p.d_enc}, {h_dec_prev, kH, kH}};
      lstm_phase<BC>(p, p.dec_w, p.dec_b_ih, p.dec_b_hh, sg, p.ws + p.L.c_dec, h_dec, xs, gates);
    }
    grid_sync(ctr, target, G, p.prof, kPhases, 4, &s_last);
    // D: projection (and stop logit, output row 0 when present: CTA 0 evaluates the rule)
    for (int r0 = cta * kWarps; r0 < n_out; r0 += G * kWarps) {    // any dmr: row blocks of 16 strided over the grid
      const Seg sg[3] = {{h_dec, kH, kH}, {ctx, p.d_enc, p.d_enc}, {nullptr, 0, 0}};
      const int K = kH + p.d_enc;
      matvec<BC>(
          K, sg, B, min(kWarps, n_out - r0),
          [&](int rl) {
            const int j = r0 + rl - use_stop;
            return j < 0 ? p.stop_w : p.proj_w + static_cast<long long>(j) * K;
          },
          [&](int rl, int b, float y) {
            const int j = r0 + rl - use_stop;
            if (j < 0) p.stop_out[static_cast<long long>(b) * p.steps + t] = y + p.stop_b[0];
            else p.mel_out[b * fstride + static_cast<long long>(t) * dmr + j] = y + p.proj_b[j];
          },
          [](int) {}, xs);
    }
    if (!p.teacher && cta == 0 && threadIdx.x == 0) {
      // Tacotron2Decoder.infer's loop exit after appending frame t (item 0 only)
      bool stop = t + 1 == p.steps;
      if (use_stop) {
        stop |= sigmoidf_(p.stop_out[t]) > 0.5f;
      } else if (s_arg0 == p.t_enc - 1) {
        if (s_first_hit < 0) s_first_hit = t;
        else if (t > s_first_hit + 20) stop = true;
      }
      if (stop) *reinterpret_cast<volatile unsigned*>(done) = static_cast<unsigned>(t + 1);
    }
    grid_sync(ctr, target, G, p.prof, kPhases, 5, &s_last);
    if (!p.teacher) {
      const unsigned d = ld_acquire_gpu(done);
      if (d) { frames = static_cast<int>(d); break; }
    }
  }
  if (cta == 0)
    for (int b = threadIdx.x; b < B; b += kThreads) p.frames[b] = frames;
}

size_t smem_bytes(int bc, int d_enc, int dmr, int loc_k) {
  const int kx = 2 * kH + d_enc > dmr ? 2 * kH + d_enc : dmr;
  return sizeof(float) * (static_cast<size_t>(bc) * kx + kGateRows * bc + kAtt * 2 * loc_k + 2 * kAtt + 3 * kWarps);
}

template <int BC>
int decode_launch(Params& p, cudaStream_t st) {
  const size_t smem = smem_bytes(BC, p.d_enc, p.dmr, p.loc_k);
  if (int rc = prepare_kernel(taco2_decode_kernel<BC>, kThreads, smem, &p.grid)) return rc;
  if (p.prof && p.grid > 1024) return fail(PK_ERR_UNSUPPORTED, "pk_taco2_decode: phase timers hold 1024 CTAs (grid %d)", p.grid);
  if (p.grid < kMinGrid)
    return fail(PK_ERR_UNSUPPORTED, "pk_taco2_decode: only %d CTAs can be co-resident (needs %d)", p.grid, kMinGrid);
  taco2_decode_kernel<BC><<<p.grid, kThreads, smem, st>>>(p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// encoder glue
// ---------------------------------------------------------------------------------------------------------------
// y[b, t] = table[ids[b, t]] + (tone_ids ? tone_table[tone] (zero for tone 0, padding_idx) : 0)
__global__ void embed_kernel(const int64_t* __restrict__ ids, const float* __restrict__ table, const int64_t* __restrict__ tones,
                             const float* __restrict__ tone_table, long long rows, int C, float* __restrict__ y) {
  const long long row = blockIdx.x;
  if (row >= rows) return;
  const float* e = table + ids[row] * C;
  const long long tn = tones ? tones[row] : 0;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float v = e[c];
    if (tones) v += tn != 0 ? tone_table[tn * C + c] : 0.f;
    y[row * C + c] = v;
  }
}

// dst (T, B, C) time-major from src (B, T, C); with reverse, each sequence reversed within its own length (lens or T)
__global__ void time_major_kernel(const float* __restrict__ src, const int32_t* __restrict__ lens, int reverse, int B, int T, int C,
                                  float* __restrict__ dst) {
  const int t = blockIdx.x / B, b = blockIdx.x % B;
  const int len = lens ? lens[b] : T;
  const int s = reverse && t < len ? len - 1 - t : t;
  const float* x = src + (static_cast<long long>(b) * T + s) * C;
  float* y = dst + (static_cast<long long>(t) * B + b) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) y[c] = x[c];
}

// out (B, T, 2H + Gc) = [h_fwd_t | h_bwd at its own position | global condition], rows t >= len zero
__global__ void bilstm_merge_kernel(const float* __restrict__ hf, const float* __restrict__ hb, const int32_t* __restrict__ lens,
                                    const float* __restrict__ gc, int B, int T, int H, int Gc, float* __restrict__ out) {
  const int b = blockIdx.x / T, t = blockIdx.x % T;
  const int len = lens ? lens[b] : T;
  const int W = 2 * H + Gc;
  float* y = out + (static_cast<long long>(b) * T + t) * W;
  const float* f = hf + (static_cast<long long>(t) * B + b) * H;
  const float* r = hb + (static_cast<long long>(len - 1 - t) * B + b) * H;
  for (int c = threadIdx.x; c < W; c += blockDim.x) {
    float v = 0.f;
    if (t < len) v = c < H ? f[c] : (c < 2 * H ? r[c - H] : gc[static_cast<long long>(b) * Gc + c - 2 * H]);
    y[c] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Tacotron2Loss (forward): out = {loss, mel_loss, post_mel_loss, guided_attn_loss, stop_loss}, one block in double
// ---------------------------------------------------------------------------------------------------------------
constexpr int kLossThreads = 1024;

__global__ void __launch_bounds__(kLossThreads, 1)
loss_kernel(const float* __restrict__ mel, const float* __restrict__ post, const float* __restrict__ tgt, int B, int T, int C,
            const float* __restrict__ align, int t_enc, const int32_t* __restrict__ slens, const int32_t* __restrict__ plens, double sigma,
            const float* __restrict__ stop, float* __restrict__ out) {
  __shared__ double red[kLossThreads];
  const long long n = static_cast<long long>(B) * T * C;
  double a = 0.0, c = 0.0;
  for (long long i = threadIdx.x; i < n; i += kLossThreads) {
    const double d1 = static_cast<double>(mel[i]) - tgt[i], d2 = static_cast<double>(post[i]) - tgt[i];
    a += d1 * d1;
    c += d2 * d2;
  }
  const double mel_loss = block_sum_tree<kLossThreads>(a, red) / n, post_loss = block_sum_tree<kLossThreads>(c, red) / n;
  double total = mel_loss + post_loss, gal = 0.0, st = 0.0;
  if (align) {
    for (int b = 0; b < B; ++b) {
      const int dl = slens[b], el = plens[b];
      double s = 0.0;
      for (long long i = threadIdx.x; i < static_cast<long long>(T) * t_enc; i += kLossThreads) {
        const int nn = static_cast<int>(i / t_enc), tt = static_cast<int>(i % t_enc);
        if (nn >= dl || tt >= el) continue;
        const double d = static_cast<double>(nn) / dl - static_cast<double>(tt) / el;
        s += (1.0 - exp(-d * d / (2.0 * sigma * sigma))) * align[static_cast<long long>(b) * T * t_enc + i];
      }
      gal += block_sum_tree<kLossThreads>(s, red) / (static_cast<double>(dl) * el);
    }
    gal /= B;
    total += gal;
  }
  if (stop) {
    double s = 0.0;
    for (long long i = threadIdx.x; i < static_cast<long long>(B) * T; i += kLossThreads) {
      const int b = static_cast<int>(i / T), nn = static_cast<int>(i % T);
      const double x = stop[i], y = nn == slens[b] - 1 ? 1.0 : 0.0;
      s += fmax(x, 0.0) - x * y + log1p(exp(-fabs(x)));
    }
    st = block_sum_tree<kLossThreads>(s, red) / (static_cast<double>(B) * T);
    total += st;
  }
  if (threadIdx.x == 0) {
    out[0] = static_cast<float>(total); out[1] = static_cast<float>(mel_loss); out[2] = static_cast<float>(post_loss);
    out[3] = static_cast<float>(gal); out[4] = static_cast<float>(st);
  }
}

}  // namespace taco2
}  // namespace pk

using namespace pk;
using namespace pk::taco2;

extern "C" int64_t pk_taco2_workspace(int32_t batch, int32_t t_enc, int32_t d_enc) { return ws_layout(batch, t_enc, d_enc).total; }

extern "C" int64_t pk_taco2_prof_len() { return 2ll * kPhases * 1024; }   // 2 x 6 counters for each of up to 1024 CTAs

extern "C" int pk_taco2_decode(const PkTaco2DecodeArgs* a, pk_stream_t stream) {
  PK_CHECK_ARG(a != nullptr, "NULL arguments");
  PK_CHECK_ARG(a->batch >= 1 && a->t_enc >= 1 && a->steps >= 1 && a->dmr >= 4, "batch, t_enc, steps must be >= 1 and dmr >= 4");
  if (a->batch > 32 || (a->d_enc != 512 && a->d_enc != 768) || a->dmr % 4 != 0 || a->loc_k < 1 || a->loc_k > 63 || a->loc_k % 2 == 0)
    return fail(PK_ERR_UNSUPPORTED, "pk_taco2_decode supports batch <= 32, d_encoder 512 or 768, d_mels * r a multiple of 4 and an "
                                    "odd location kernel <= 63 (got %d, %d, %d, %d)", a->batch, a->d_enc, a->dmr, a->loc_k);
  PK_CHECK_ARG(a->keys && a->pkeys && a->pre_w1 && a->pre_w2 && a->att_w && a->att_b_ih && a->att_b_hh && a->q_w && a->loc_w && a->v_w &&
               a->dec_w && a->dec_b_ih && a->dec_b_hh && a->proj_w && a->proj_b && a->workspace && a->mel_out && a->align_out && a->frames,
               "NULL pointer in pk_taco2_decode");
  PK_CHECK_ARG((a->stop_w == nullptr) == (a->stop_b == nullptr) && (a->stop_w == nullptr) == (a->stop_out == nullptr),
               "stop_w, stop_b and stop_out come together");
  PK_CHECK_ARG(!a->teacher || a->mels, "teacher-forced decoding needs mels");
  PK_CHECK_ARG(a->teacher || a->stop_w == nullptr || a->batch == 1, "the stop-token rule of infer is defined for batch 1");
  PK_CHECK_ARG(a->p_prenet >= 0.f && a->p_prenet < 1.f, "prenet dropout must be in [0, 1)");
  PK_CHECK_ARG(aligned16(a->pre_w1) && aligned16(a->pre_w2) && aligned16(a->att_w) && aligned16(a->q_w) && aligned16(a->dec_w) &&
               aligned16(a->proj_w) && (a->stop_w == nullptr || aligned16(a->stop_w)) && aligned16(a->workspace) && aligned16(a->mel_out) &&
               (a->mels == nullptr || aligned16(a->mels)), "weights, mels, mel_out and the workspace must be 16-byte aligned");
  const Ws L = ws_layout(a->batch, a->t_enc, a->d_enc);
  PK_CHECK_ARG(a->workspace_len >= L.total, "workspace must hold pk_taco2_workspace() = %lld floats", L.total);
  Params p;
  p.B = a->batch; p.t_enc = a->t_enc; p.d_enc = a->d_enc; p.dmr = a->dmr; p.steps = a->steps; p.teacher = a->teacher;
  p.loc_k = a->loc_k; p.grid = 0;
  p.p_prenet = a->p_prenet;
  p.drop_scale = a->p_prenet > 0.f ? 1.f / (1.f - a->p_prenet) : 1.f;
  const double th = static_cast<double>(a->p_prenet) * 4294967296.0;
  p.drop_thresh = th >= 4294967295.0 ? 0xFFFFFFFFu : static_cast<uint32_t>(th);
  p.seed_lo = static_cast<uint32_t>(a->seed); p.seed_hi = static_cast<uint32_t>(a->seed >> 32);
  p.keys = a->keys; p.pkeys = a->pkeys; p.text_lens = a->teacher ? a->text_lens : nullptr; p.mels = a->mels;
  p.pre_w1 = a->pre_w1; p.pre_w2 = a->pre_w2; p.att_w = a->att_w; p.att_b_ih = a->att_b_ih; p.att_b_hh = a->att_b_hh;
  p.q_w = a->q_w; p.loc_w = a->loc_w; p.v_w = a->v_w; p.dec_w = a->dec_w; p.dec_b_ih = a->dec_b_ih; p.dec_b_hh = a->dec_b_hh;
  p.proj_w = a->proj_w; p.proj_b = a->proj_b; p.stop_w = a->stop_w; p.stop_b = a->stop_b;
  p.ws = a->workspace; p.L = L;
  p.mel_out = a->mel_out; p.align_out = a->align_out; p.stop_out = a->stop_out; p.frames = a->frames;
  p.prof = reinterpret_cast<unsigned long long*>(a->prof);
  auto st = static_cast<cudaStream_t>(stream);
  const long long out_rows = static_cast<long long>(a->batch) * a->steps;
  // zero the counters, the recurrent state (h, c, w, w_cum, context) and the outputs (rows past the stop stay zero for the postnet)
  PK_CHECK_CUDA(cudaMemsetAsync(a->workspace, 0, L.total * sizeof(float), st));
  PK_CHECK_CUDA(cudaMemsetAsync(a->mel_out, 0, out_rows * a->dmr * sizeof(float), st));
  PK_CHECK_CUDA(cudaMemsetAsync(a->align_out, 0, out_rows * a->t_enc * sizeof(float), st));
  if (a->stop_out) PK_CHECK_CUDA(cudaMemsetAsync(a->stop_out, 0, out_rows * sizeof(float), st));
  if (a->prof) PK_CHECK_ARG(a->prof_len >= pk_taco2_prof_len(), "prof must hold pk_taco2_prof_len() = %lld counters", pk_taco2_prof_len());
  if (a->prof) PK_CHECK_CUDA(cudaMemsetAsync(a->prof, 0, pk_taco2_prof_len() * sizeof(uint64_t), st));
  return a->batch == 1 ? decode_launch<1>(p, st) : decode_launch<8>(p, st);
}

extern "C" int pk_taco2_embed(const int64_t* ids, const float* table, const int64_t* tones, const float* tone_table, int32_t batch,
                              int32_t t, int32_t channels, float* y, pk_stream_t stream) {
  PK_CHECK_ARG(batch > 0 && t > 0 && channels > 0 && ids && table && y && (tones == nullptr) == (tone_table == nullptr),
               "bad arguments to pk_taco2_embed");
  embed_kernel<<<batch * t, 128, 0, static_cast<cudaStream_t>(stream)>>>(ids, table, tones, tone_table, static_cast<long long>(batch) * t,
                                                                         channels, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_taco2_time_major(const float* src, const int32_t* lens, int32_t reverse, int32_t batch, int32_t t, int32_t channels,
                                   float* dst, pk_stream_t stream) {
  PK_CHECK_ARG(batch > 0 && t > 0 && channels > 0 && src && dst, "bad arguments to pk_taco2_time_major");
  time_major_kernel<<<batch * t, 256, 0, static_cast<cudaStream_t>(stream)>>>(src, lens, reverse, batch, t, channels, dst);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_taco2_bilstm_merge(const float* h_fwd, const float* h_bwd, const int32_t* lens, const float* gc, int32_t batch, int32_t t,
                                     int32_t hidden, int32_t gc_dim, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(batch > 0 && t > 0 && hidden > 0 && gc_dim >= 0 && h_fwd && h_bwd && out && (gc_dim == 0 || gc),
               "bad arguments to pk_taco2_bilstm_merge");
  bilstm_merge_kernel<<<batch * t, 256, 0, static_cast<cudaStream_t>(stream)>>>(h_fwd, h_bwd, lens, gc, batch, t, hidden, gc_dim, out);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_taco2_loss(const float* mel, const float* post, const float* target, int32_t batch, int32_t t, int32_t channels,
                             const float* align, int32_t t_enc, const int32_t* slens, const int32_t* plens, float sigma,
                             const float* stop_logits, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(batch > 0 && t > 0 && channels > 0 && mel && post && target && out, "bad arguments to pk_taco2_loss");
  PK_CHECK_ARG(align == nullptr || (t_enc > 0 && slens && plens), "the guided attention loss needs t_enc, slens and plens");
  PK_CHECK_ARG(stop_logits == nullptr || slens, "the stop loss needs slens");
  loss_kernel<<<1, kLossThreads, 0, static_cast<cudaStream_t>(stream)>>>(mel, post, target, batch, t, channels, align, t_enc, slens, plens,
                                                                          static_cast<double>(sigma), stop_logits, out);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
