// Parallel WaveGAN generator kernels (reference: parakeet/models/parallel_wavegan/parallel_wavegan.py).
//
//   pk_pwg_residual_layer : one fused ResidualBlock (:284-315) over the whole batch, channels-last, wgmma:
//        GEMM1  h[128 t x 128]  = sum_{tap} x[t + (tap-1) d, 0:64] W_conv[tap] + c[t, 0:80] W_aux      (K = 272)
//        gate   z[128 x 64]     = tanh(h[:, :64] + b) * sigmoid(h[:, 64:] + b)       (in registers, never memory)
//        GEMM2  [skip | out]    = [0 | x] + z W_so                                    (K = 64, z as register A operand)
//        epi    skip_acc += skip (its bias is summed into the tail);  x_out = (out + b_out + x) * sqrt(0.5)
//     persistent CTAs over 128-sample tiles: a producer warpgroup (one TMA lane) streams A and W1 chunks through a 2-deep
//     ring, W2 stays resident, two consumer warpgroups (64 samples each) run both GEMMs, the gate and the stores.
//   pk_pwg_upsample       : ConvInUpsampleNet (:201-216) conv_in + [nearest stretch + FIR] x scales, fused per frame.
//   pk_pwg_first_conv     : first_conv 1 -> R channels (:464).
//   pk_pwg_tail           : skips * sqrt(1/L) -> ReLU -> 1x1 -> ReLU -> 1x1 (:469-471).
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {

// ---------------------------------------------------------------------------------------------------------------
// fused residual layer
// ---------------------------------------------------------------------------------------------------------------
constexpr int kPwgR = 64;        // residual channels
constexpr int kPwgG = 128;       // gate channels
constexpr int kPwgS = 64;        // skip channels
constexpr int kPwgStages = 2;
constexpr int kPwgTile = 128 * kSwizzleBytes;                 // 16 KB: one plane of a 128-row K-chunk
constexpr int kPwgStageBytes = 4 * kPwgTile;                  // A hi, A lo, B hi, B lo
constexpr int kPwgW2Bytes = 2 * kPwgTile;                     // resident W2: 128 outputs (skip | out) x 64, both planes
constexpr int kPwgSmem = kPwgStages * kPwgStageBytes + kPwgW2Bytes + 1024 + 256;
static_assert(kPwgSmem <= 227 * 1024, "shared memory budget");
constexpr int kPwgConsumerThreads = 256;
constexpr int kPwgThreads = kPwgConsumerThreads + 128;
constexpr int kPwgG1Chunks = 5;                               // 3 taps + 2 aux chunks (64 + 16 channels)

struct PwgLayerArgs {
  int batch, t, dil, aux_ch;
  int tiles_per_b, total_tiles;
  const int32_t* lens;          // valid samples per utterance or NULL
  float gate_c[128];            // constant bank: [0,64) -2*log2e*bias_a, [64,128) -log2e*bias_g (conv bias, pre-scaled)
  float out_b[64];              // constant bank: conv1x1_out bias (the skip biases are summed into the tail)
  float k_a, k_g;               // -2*log2e, -log2e
  float* skip;                  // fp32 (B, T, 64) accumulator
  int skip_init;                // 1: write, 0: accumulate
  __nv_bfloat16* y_hi;          // layer output planes
  __nv_bfloat16* y_lo;
};

struct PwgTileIter {
  int idx, step, tiles_per_b, total, t;
  const int32_t* lens;
  __device__ PwgTileIter(const PwgLayerArgs& p) : idx(static_cast<int>(blockIdx.x) - static_cast<int>(gridDim.x)),
      step(gridDim.x), tiles_per_b(p.tiles_per_b), total(p.total_tiles), t(p.t), lens(p.lens) {}
  // advance to the next tile that holds at least one valid sample
  __device__ bool next(int& b, int& m0) {
    for (;;) {
      idx += step;
      if (idx >= total) return false;
      b = idx / tiles_per_b;
      m0 = (idx % tiles_per_b) * 128;
      const int len = lens ? min(__ldg(lens + b), t) : t;
      if (m0 < len) return true;
    }
  }
};

__global__ void __launch_bounds__(kPwgThreads, 1)
pwg_layer_kernel(const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                 const __grid_constant__ CUtensorMap tm_c_hi, const __grid_constant__ CUtensorMap tm_c_lo,
                 const __grid_constant__ CUtensorMap tm_w1_hi, const __grid_constant__ CUtensorMap tm_w1_lo,
                 const __grid_constant__ CUtensorMap tm_w2_hi, const __grid_constant__ CUtensorMap tm_w2_lo,
                 const PwgLayerArgs p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;      // 1024-B aligned for SWIZZLE_128B
  const uint32_t w2 = smem + kPwgStages * kPwgStageBytes;
  const uint32_t bars = w2 + kPwgW2Bytes;
  const uint32_t full_bar = bars;                       // [stages]
  const uint32_t empty_bar = full_bar + 8 * kPwgStages; // [stages]
  const uint32_t w_bar = empty_bar + 8 * kPwgStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == kPwgConsumerThreads) {
    tma_prefetch_desc(&tm_x_hi); tma_prefetch_desc(&tm_x_lo); tma_prefetch_desc(&tm_c_hi); tma_prefetch_desc(&tm_c_lo);
    tma_prefetch_desc(&tm_w1_hi); tma_prefetch_desc(&tm_w1_lo); tma_prefetch_desc(&tm_w2_hi); tma_prefetch_desc(&tm_w2_lo);
    for (int s = 0; s < kPwgStages; ++s) { mbar_init_a(full_bar + 8 * s, 1); mbar_init_a(empty_bar + 8 * s, kPwgConsumerThreads / 32); }
    mbar_init_a(w_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kPwgConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kPwgConsumerThreads / 32 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      mbar_arrive_expect_tx_a(w_bar, kPwgW2Bytes);
      tma_load_3d_a(w2, &tm_w2_hi, w_bar, 0, 0, 0);
      tma_load_3d_a(w2 + kPwgTile, &tm_w2_lo, w_bar, 0, 0, 0);
      uint32_t it = 0;
      PwgTileIter ti(p);
      int b, m0;
      while (ti.next(b, m0)) {
        for (int j = 0; j < kPwgG1Chunks; ++j, ++it) {
          const int s = it % kPwgStages;
          mbar_wait_a(empty_bar + 8 * s, ((it / kPwgStages) & 1) ^ 1);
          const uint32_t st = smem + s * kPwgStageBytes;
          const uint32_t fb = full_bar + 8 * s;
          mbar_arrive_expect_tx_a(fb, kPwgStageBytes);
          // chunk order: tap -d, tap +d, aux[0:64], aux[64:], centre tap (last: it also supplies the residual x)
          const int wj = j == 0 ? 0 : j == 1 ? 2 : j == 2 ? 3 : j == 3 ? 4 : 1;   // K-chunk of the packed weight
          if (wj < 3) {
            const int row = m0 + (wj - 1) * p.dil;
            tma_load_3d_a(st, &tm_x_hi, fb, 0, row, b);
            tma_load_3d_a(st + kPwgTile, &tm_x_lo, fb, 0, row, b);
          } else {
            tma_load_3d_a(st, &tm_c_hi, fb, (wj - 3) * kChunkK, m0, b);
            tma_load_3d_a(st + kPwgTile, &tm_c_lo, fb, (wj - 3) * kChunkK, m0, b);
          }
          tma_load_3d_a(st + 2 * kPwgTile, &tm_w1_hi, fb, wj * kChunkK, 0, 0);
          tma_load_3d_a(st + 3 * kPwgTile, &tm_w1_lo, fb, wj * kChunkK, 0, 0);
        }
      }
    }
  } else {
    // ------------------------------ consumers: 64 samples per warpgroup ------------------------------
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int rl = 16 * (warp & 3) + (lane >> 2);              // this thread's rows: rl and rl + 8 of the warpgroup's 64
    const int cq = 2 * (lane & 3);                             // and columns 8 j + cq, + 1
    const int aux_tail_ksteps = ((p.aux_ch - kChunkK) + kWgmmaK - 1) / kWgmmaK;  // k-steps in the 2nd aux chunk
    const float kSqrtHalf = 0.70710678118654752440f;
    mbar_wait_a(w_bar, 0);
    uint32_t it = 0;
    PwgTileIter ti(p);
    int b, m0;
    while (ti.next(b, m0)) {
      float acc1[64], acc2[64];
      for (int j = 0; j < kPwgG1Chunks; ++j, ++it) {
        const int s = it % kPwgStages;
        mbar_wait_a(full_bar + 8 * s, (it / kPwgStages) & 1);
        const uint32_t st = smem + s * kPwgStageBytes;
        const uint32_t sa = st + wg * 64 * kSwizzleBytes;
        const uint64_t a_hi = make_smem_desc_sw128(sa), a_lo = make_smem_desc_sw128(sa + kPwgTile);
        const uint64_t b_hi = make_smem_desc_sw128(st + 2 * kPwgTile), b_lo = make_smem_desc_sw128(st + 3 * kPwgTile);
        const int ksteps = j == 3 ? aux_tail_ksteps : 4;
        wgmma_fence();
        for (int k = 0; k < ksteps; ++k) {
          wgmma_ss_n128(acc1, a_hi + desc_kstep(k), b_hi + desc_kstep(k), !(j == 0 && k == 0));
          wgmma_ss_n128(acc1, a_lo + desc_kstep(k), b_hi + desc_kstep(k), 1);
          wgmma_ss_n128(acc1, a_hi + desc_kstep(k), b_lo + desc_kstep(k), 1);
        }
        wgmma_commit();
        if (j == kPwgG1Chunks - 1) {
          // GEMM2's accumulator starts as [0 | x]: x = hi + lo of this tile's own rows, from the centre-tap chunk
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int r = rl + 8 * hh;
              const uint32_t off = r * kSwizzleBytes + ((((8 * jj + cq) >> 3) ^ (r & 7)) << 4) + (cq & 7) * 2;
              const uint32_t xh = lds_u32(sa + off), xl = lds_u32(sa + kPwgTile + off);
              acc2[4 * jj + 2 * hh] = 0.f;
              acc2[4 * jj + 2 * hh + 1] = 0.f;
              acc2[32 + 4 * jj + 2 * hh] = __uint_as_float(xh << 16) + __uint_as_float(xl << 16);
              acc2[32 + 4 * jj + 2 * hh + 1] = __uint_as_float(xh & 0xffff0000u) + __uint_as_float(xl & 0xffff0000u);
            }
          }
        }
        wgmma_wait<0>();
        reg_fence(acc1);
        __syncwarp();
        if (lane == 0) mbar_arrive_a(empty_bar + 8 * s);
      }
      // gate: z = tanh(a + ba) * sigmoid(g + bg) = (1 - e1) / ((1 + e1)(1 + e2)), e1 = exp(-2(a+ba)), e2 = exp(-(g+bg))
      // (one reciprocal; the exp2 argument of e1 is clamped at 60 so that the product cannot overflow where z != 0).
      // a column c and its g column 64 + c sit in the same thread (fragments j and j + 8).
      uint32_t zh[16], zl[16];
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float z[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int c = 8 * jj + cq + (e & 1);
          const float e1 = ex2_approx(fminf(fmaf(acc1[4 * jj + e], p.k_a, p.gate_c[c]), 60.f));
          const float e2 = ex2_approx(fmaf(acc1[32 + 4 * jj + e], p.k_g, p.gate_c[64 + c]));
          const float t1 = 1.f + e1;
          z[e] = (1.f - e1) * rcp_approx(fmaf(t1, e2, t1));
        }
        split2(z[0], z[1], zh[2 * jj], zl[2 * jj]);            // row rl
        split2(z[2], z[3], zh[2 * jj + 1], zl[2 * jj + 1]);    // row rl + 8
      }
      // GEMM2: [skip | out] += z W2, K = 64 = 4 K-steps; A fragment of K-step k = z column groups 2k, 2k + 1
      const uint64_t b2_hi = make_smem_desc_sw128(w2), b2_lo = make_smem_desc_sw128(w2 + kPwgTile);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t ah[4] = {zh[4 * k], zh[4 * k + 1], zh[4 * k + 2], zh[4 * k + 3]};
        const uint32_t al[4] = {zl[4 * k], zl[4 * k + 1], zl[4 * k + 2], zl[4 * k + 3]};
        wgmma_rs_n128(acc2, ah, b2_hi + desc_kstep(k), 1);
        wgmma_rs_n128(acc2, al, b2_hi + desc_kstep(k), 1);
        wgmma_rs_n128(acc2, ah, b2_lo + desc_kstep(k), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc2);
      // stores: skip half -> fp32 skip sum (write or red.add), out half -> (out + b_out) * sqrt(1/2) as split planes
      const int len = p.lens ? min(__ldg(p.lens + b), p.t) : p.t;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int trow = m0 + wg * 64 + rl + 8 * hh;
        if (trow < p.t) {
          const long long row_off = (static_cast<long long>(b) * p.t + trow) * 64;
          const bool live = trow < len;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int c = 8 * jj + cq;
            float* d2 = p.skip + row_off + c;
            const float s0 = acc2[4 * jj + 2 * hh], s1 = acc2[4 * jj + 2 * hh + 1];
            if (p.skip_init) *reinterpret_cast<float2*>(d2) = make_float2(s0, s1);
            else asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(d2), "f"(s0), "f"(s1) : "memory");
            const float y0 = live ? (acc2[32 + 4 * jj + 2 * hh] + p.out_b[c]) * kSqrtHalf : 0.f;
            const float y1 = live ? (acc2[32 + 4 * jj + 2 * hh + 1] + p.out_b[c + 1]) * kSqrtHalf : 0.f;
            uint32_t oh, ol;
            split2(y0, y1, oh, ol);
            *reinterpret_cast<uint32_t*>(p.y_hi + row_off + c) = oh;
            *reinterpret_cast<uint32_t*>(p.y_lo + row_off + c) = ol;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ConvInUpsampleNet: conv_in (no padding) then up to 4 x [nearest stretch by s, FIR of 2s+1 taps, zero padded]
// grid = (frames, batch); one CTA produces the hop = prod(scales) output samples of one frame for all channels.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kUpMaxStages = 4;
constexpr int kUpMaxScale = 16;
struct UpsampleArgs {
  int n_stages;
  int scale[kUpMaxStages];
  // polyphase form of "nearest stretch by s, then FIR w[0..2s] with zero padding s":
  //   out[s*m + r] = sum_{k=0..2} poly[k][r] * in[m - 1 + k],  poly[k][r] = sum_{q : floor((r+q)/s) == k} w[q]
  float poly[kUpMaxStages][3][kUpMaxScale];
  int aux, frames, window;       // channels, T' (after conv_in), aux_context_window
  int hop;
};

__device__ __forceinline__ int floordiv(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// conv_in (Conv1D aux -> aux, k = 2*window + 1, no padding, no bias) once per frame:
//   m[b, f, ch] = sum_{ci, q} w[ch][ci][q] * mel[b, ci, f + q],  f in [0, frames)          (channels-last fp32 workspace)
// grid = (ceil(frames / 16), batch), 320 threads = 80-channel lanes x 4 groups of 4 frames (aux <= 80 per pass);
// the weight is staged once per CTA, transposed to [ci*k + q][ch] (pitch aux + 1: conflict-free both ways).
constexpr int kCinFrames = 16;
__global__ void __launch_bounds__(320)
pwg_conv_in_kernel(const float* __restrict__ mel, const float* __restrict__ w_in, int aux, int frames, int window,
                   float* __restrict__ m_out) {
  extern __shared__ float cin_smem[];
  const int kin = 2 * window + 1;
  const int wrow = aux * kin;                 // taps per output channel
  const int pitch = aux + 1;
  float* sw = cin_smem;                       // [wrow][pitch]
  float* sm = sw + wrow * pitch;              // [aux][kCinFrames + kin - 1]
  const int span = kCinFrames + kin - 1;
  const int f0 = blockIdx.x * kCinFrames, b = blockIdx.y;
  const int mel_len = frames + 2 * window;
  for (int idx = threadIdx.x; idx < aux * wrow; idx += blockDim.x) {
    const int ch = idx / wrow, r = idx - ch * wrow;
    sw[r * pitch + ch] = __ldg(w_in + idx);
  }
  for (int idx = threadIdx.x; idx < aux * span; idx += blockDim.x) {
    const int ci = idx / span, i = idx - ci * span;
    const int f = f0 + i;
    sm[idx] = f < mel_len ? __ldg(mel + (static_cast<long long>(b) * aux + ci) * mel_len + f) : 0.f;
  }
  __syncthreads();
  const int fg = threadIdx.x / 80, lane_ch = threadIdx.x - fg * 80;   // 4 frame groups x 80 channel lanes
  for (int ch = lane_ch; ch < aux; ch += 80) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int ci = 0; ci < aux; ++ci) {
      const float* mp = sm + ci * span + fg * 4;
      const float* wp = sw + (ci * kin) * pitch + ch;
      for (int q = 0; q < kin; ++q) {
        const float wv = wp[q * pitch];
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] = fmaf(wv, mp[q + i], acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = f0 + fg * 4 + i;
      if (f < frames) m_out[(static_cast<long long>(b) * frames + f) * aux + ch] = acc[i];
    }
  }
}

// grid = (frames, batch): one CTA produces the hop = prod(scales) output samples of frame j for all channels from the
// conv_in frames j-2 .. j+2 (workspace m), every intermediate stage in shared memory.
__global__ void __launch_bounds__(256)
pwg_upsample_kernel(const float* __restrict__ m,          // (B, frames, aux) conv_in output, channels-last
                    const int32_t* __restrict__ frame_lens, // valid frames per utterance or NULL
                    const UpsampleArgs a, float* __restrict__ c_f32 /* (B, aux, T) or NULL */,
                    __nv_bfloat16* __restrict__ c_hi, __nv_bfloat16* __restrict__ c_lo /* (B, T, aux) or NULL */) {
  extern __shared__ float up_smem[];
  __shared__ float s_poly[kUpMaxStages][3][kUpMaxScale];
  const int j = blockIdx.x, b = blockIdx.y;
  const int aux = a.aux;
  const int n_frames = frame_lens ? min(__ldg(frame_lens + b), a.frames) : a.frames;
  for (int i = threadIdx.x; i < kUpMaxStages * 3 * kUpMaxScale; i += blockDim.x) (&s_poly[0][0][0])[i] = (&a.poly[0][0][0])[i];
  // stage k output index range [lo[k], hi[k]) needed for outputs [j*hop, (j+1)*hop) of the last stage
  int lo[kUpMaxStages + 1], hi[kUpMaxStages + 1], len[kUpMaxStages + 1];
  len[0] = n_frames;
#pragma unroll
  for (int k = 0; k < kUpMaxStages; ++k) len[k + 1] = k < a.n_stages ? len[k] * a.scale[k] : 0;
#pragma unroll
  for (int k = kUpMaxStages; k >= 0; --k) {
    if (k == a.n_stages) { lo[k] = j * a.hop; hi[k] = (j + 1) * a.hop; }
    else if (k < a.n_stages) {
      const int s = a.scale[k];
      lo[k] = floordiv(lo[k + 1], s) - 1;
      hi[k] = floordiv(hi[k + 1] - 1, s) + 2;
    } else { lo[k] = 0; hi[k] = 0; }
  }
  // Every stage buffer is [pos][ch] (pitch aux): threads run over channels fastest, so stage reads / writes are
  // conflict-free and the final stage reads 8 consecutive channels with two LDS.128 per tap.
  float* buf[kUpMaxStages + 1];
  int width[kUpMaxStages + 1];
  {
    float* ptr = up_smem;
#pragma unroll
    for (int k = 0; k <= kUpMaxStages; ++k) {
      width[k] = hi[k] - lo[k];
      buf[k] = ptr;
      if (k < a.n_stages) ptr += aux * width[k];
    }
  }
  const int last = a.n_stages - 1;                // index of the last stage (its input buffer is buf[last])
  // stage 0: conv_in frames f in [lo[0], hi[0]) (zero outside [0, n_frames)); coalesced read, channel fastest
  for (int idx = threadIdx.x; idx < aux * width[0]; idx += blockDim.x) {
    const int i = idx / aux, ch = idx - i * aux;
    const int f = lo[0] + i;
    const float v = (f >= 0 && f < n_frames) ? __ldg(m + (static_cast<long long>(b) * a.frames + f) * aux + ch) : 0.f;
    buf[0][idx] = v;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k + 1 < kUpMaxStages; ++k) {   // intermediate stages stay in shared memory
    if (k + 1 < a.n_stages) {
      const int s = a.scale[k];
      for (int idx = threadIdx.x; idx < aux * width[k + 1]; idx += blockDim.x) {
        const int tt = idx / aux, ch = idx - tt * aux;
        const int t = lo[k + 1] + tt;
        float acc = 0.f;
        if (t >= 0 && t < len[k + 1]) {
          const int mm = t / s, r = t - mm * s;
          const float* in = buf[k] + (mm - 1 - lo[k]) * aux + ch;   // taps mm-1, mm, mm+1 are all inside the buffer
          acc = s_poly[k][0][r] * in[0];
          acc = fmaf(s_poly[k][1][r], in[aux], acc);
          acc = fmaf(s_poly[k][2][r], in[2 * aux], acc);
        }
        buf[k + 1][idx] = acc;
      }
      __syncthreads();
    }
  }
  {
    // last stage: one thread per (sample, group of 8 channels) so the channels-last store is 16-byte vectorised
    const int k = last;
    const int s = a.scale[k];
    const long long T = static_cast<long long>(a.frames) * a.hop;  // row pitch of the (padded) batch
    const int groups = aux / 8;                                     // aux % 8 == 0 (host check)
    const float* src = buf[k];                                      // [pos][aux]
    for (int idx = threadIdx.x; idx < a.hop * groups; idx += blockDim.x) {
      const int tt = idx / groups, g = idx - tt * groups;
      const int t = lo[k + 1] + tt;
      const bool live = t < len[k + 1];
      const int mm = t / s, r = t - mm * s;
      const float p0 = s_poly[k][0][r], p1 = s_poly[k][1][r], p2 = s_poly[k][2][r];
      float v[8];
      if (live) {
        const float4* in = reinterpret_cast<const float4*>(src + (mm - 1 - lo[k]) * aux + g * 8);
        const int pitch4 = aux / 4;
        const float4 a0 = in[0], a1 = in[1], b0 = in[pitch4], b1 = in[pitch4 + 1], c0 = in[2 * pitch4], c1 = in[2 * pitch4 + 1];
        v[0] = fmaf(p2, c0.x, fmaf(p1, b0.x, p0 * a0.x)); v[1] = fmaf(p2, c0.y, fmaf(p1, b0.y, p0 * a0.y));
        v[2] = fmaf(p2, c0.z, fmaf(p1, b0.z, p0 * a0.z)); v[3] = fmaf(p2, c0.w, fmaf(p1, b0.w, p0 * a0.w));
        v[4] = fmaf(p2, c1.x, fmaf(p1, b1.x, p0 * a1.x)); v[5] = fmaf(p2, c1.y, fmaf(p1, b1.y, p0 * a1.y));
        v[6] = fmaf(p2, c1.z, fmaf(p1, b1.z, p0 * a1.z)); v[7] = fmaf(p2, c1.w, fmaf(p1, b1.w, p0 * a1.w));
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = 0.f;
      }
      if (c_f32) {
#pragma unroll
        for (int e = 0; e < 8; ++e) c_f32[(static_cast<long long>(b) * aux + g * 8 + e) * T + t] = v[e];
      }
      if (c_hi) {
        uint4 h, l;
        split8(v, h, l);
        const long long o = (static_cast<long long>(b) * T + t) * aux + g * 8;
        *reinterpret_cast<uint4*>(c_hi + o) = h;
        *reinterpret_cast<uint4*>(c_lo + o) = l;
      }
    }
  }
}

// first_conv: x[b, t, r] = w[r] * noise[b, t] + bias[r]  (in_channels = 1), written as split planes, masked by lens
__global__ void pwg_first_conv_kernel(const float* __restrict__ noise, const float* __restrict__ w, const float* __restrict__ bias,
                                      const int32_t* __restrict__ lens, int t_len, long long total_rows,
                                      __nv_bfloat16* __restrict__ x_hi, __nv_bfloat16* __restrict__ x_lo) {
  // one thread per (row, 8-channel group): 8 groups per row
  const long long n = total_rows * 8;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < n;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = idx >> 3;
    const int g = idx & 7;
    const int b = row / t_len, t = row % t_len;
    const bool live = lens == nullptr || t < __ldg(lens + b);
    const float xv = __ldg(noise + row);
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = live ? fmaf(__ldg(w + g * 8 + e), xv, __ldg(bias + g * 8 + e)) : 0.f;
    uint4 h, l;
    split8(v, h, l);
    reinterpret_cast<uint4*>(x_hi)[idx] = h;
    reinterpret_cast<uint4*>(x_lo)[idx] = l;
  }
}

// tail: y = W2 relu(W1 relu(skips * scale) + b1) + b2, skip channels = 64, out channels = 1
// Two rows per thread share every (broadcast) weight load: 64 x 2 accumulators in registers, the skip rows streamed in
// chunks of 16 channels; weights in shared memory as [k/4][o] float4 (4 consecutive inputs of one output channel).
__global__ void __launch_bounds__(128)
pwg_tail_kernel(const float* __restrict__ skip, const float* __restrict__ skip_bias /*[64] or NULL*/,
                const float* __restrict__ w1 /*[64][64] out,in*/, const float* __restrict__ b1,
                const float* __restrict__ w2 /*[64]*/, const float* __restrict__ b2, float scale, long long rows,
                float* __restrict__ out) {
  __shared__ float4 sw1[16 * 64];             // [kq][o] = w1[o][4*kq .. 4*kq+3]
  __shared__ float sb1[64], sw2[64], ssb[64];
  for (int i = threadIdx.x; i < 64 * 16; i += blockDim.x) {
    const int o = i >> 4, kq = i & 15;
    sw1[kq * 64 + o] = reinterpret_cast<const float4*>(w1)[i];
  }
  if (threadIdx.x < 64) {
    sb1[threadIdx.x] = b1[threadIdx.x];
    sw2[threadIdx.x] = w2[threadIdx.x];
    ssb[threadIdx.x] = skip_bias ? skip_bias[threadIdx.x] : 0.f;
  }
  __syncthreads();
  const float bias2 = __ldg(b2);
  const long long pairs = (rows + 1) >> 1;
  for (long long pr = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; pr < pairs;
       pr += static_cast<long long>(gridDim.x) * blockDim.x) {
    // rows r0 = pr and r1 = pr + pairs: consecutive threads read consecutive rows in both halves
    const long long r0 = pr, r1 = pr + pairs;
    const bool has1 = r1 < rows;
    const float4* p0 = reinterpret_cast<const float4*>(skip + r0 * 64);
    const float4* p1 = reinterpret_cast<const float4*>(skip + (has1 ? r1 : r0) * 64);
    float h0[64], h1[64];
#pragma unroll
    for (int o = 0; o < 64; ++o) { h0[o] = sb1[o]; h1[o] = sb1[o]; }
#pragma unroll 1
    for (int kc = 0; kc < 4; ++kc) {            // 16 input channels per chunk
      float s0[16], s1[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 u = __ldg(p0 + kc * 4 + q), v = __ldg(p1 + kc * 4 + q);
        const float* sbp = ssb + kc * 16 + q * 4;
        s0[4 * q] = fmaxf((u.x + sbp[0]) * scale, 0.f); s0[4 * q + 1] = fmaxf((u.y + sbp[1]) * scale, 0.f);
        s0[4 * q + 2] = fmaxf((u.z + sbp[2]) * scale, 0.f); s0[4 * q + 3] = fmaxf((u.w + sbp[3]) * scale, 0.f);
        s1[4 * q] = fmaxf((v.x + sbp[0]) * scale, 0.f); s1[4 * q + 1] = fmaxf((v.y + sbp[1]) * scale, 0.f);
        s1[4 * q + 2] = fmaxf((v.z + sbp[2]) * scale, 0.f); s1[4 * q + 3] = fmaxf((v.w + sbp[3]) * scale, 0.f);
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int o = 0; o < 64; ++o) {
          const float4 w = sw1[(kc * 4 + q) * 64 + o];   // warp-uniform address: broadcast
          h0[o] = fmaf(w.x, s0[4 * q], h0[o]); h0[o] = fmaf(w.y, s0[4 * q + 1], h0[o]);
          h0[o] = fmaf(w.z, s0[4 * q + 2], h0[o]); h0[o] = fmaf(w.w, s0[4 * q + 3], h0[o]);
          h1[o] = fmaf(w.x, s1[4 * q], h1[o]); h1[o] = fmaf(w.y, s1[4 * q + 1], h1[o]);
          h1[o] = fmaf(w.z, s1[4 * q + 2], h1[o]); h1[o] = fmaf(w.w, s1[4 * q + 3], h1[o]);
        }
      }
    }
    float y0 = bias2, y1 = bias2;
#pragma unroll
    for (int o = 0; o < 64; ++o) {
      y0 = fmaf(sw2[o], fmaxf(h0[o], 0.f), y0);
      y1 = fmaf(sw2[o], fmaxf(h1[o], 0.f), y1);
    }
    out[r0] = y0;
    if (has1) out[r1] = y1;
  }
}

}  // namespace pk

// ===============================================================================================================
// C-ABI
// ===============================================================================================================
extern "C" int pk_pwg_residual_layer(const pk_pwg_layer_args* a, pk_stream_t stream) {
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  PK_CHECK_ARG(a->batch > 0 && a->t > 0 && a->dilation >= 1, "bad batch/t/dilation");
  PK_CHECK_ARG(a->aux_channels > 64 && a->aux_channels <= 128 && (a->aux_channels % 8) == 0,
               "aux_channels must be in (64,128] and a multiple of 8 (got %d)", a->aux_channels);
  PK_CHECK_ARG(a->x_hi && a->x_lo && a->y_hi && a->y_lo && a->c_hi && a->c_lo && a->w1_hi && a->w1_lo && a->w2_hi && a->w2_lo &&
               a->bias1 && a->bias2 && a->skip, "NULL pointer in pk_pwg_layer_args");
  PK_CHECK_ARG(a->x_hi != a->y_hi, "layer output must not alias its input (neighbouring tiles read the input halo)");
  using namespace pk;
  CUtensorMap tx_hi, tx_lo, tc_hi, tc_lo, tw1_hi, tw1_lo, tw2_hi, tw2_lo;
  int rc;
  const uint64_t T = a->t, B = a->batch;
  const uint32_t w_box_rows = 128;
  if ((rc = encode_tmap_bf16_3d(&tx_hi, a->x_hi, kPwgR, T, B, kPwgR, T * kPwgR, 128))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tx_lo, a->x_lo, kPwgR, T, B, kPwgR, T * kPwgR, 128))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tc_hi, a->c_hi, a->aux_channels, T, B, a->aux_channels, T * a->aux_channels, 128))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tc_lo, a->c_lo, a->aux_channels, T, B, a->aux_channels, T * a->aux_channels, 128))) return rc;
  const uint64_t k1 = kPwgG1Chunks * kChunkK;  // 320: row pitch of the packed W1 (3 taps x 64 + aux padded to 128)
  const uint64_t k1_valid = 3 * kChunkK + a->aux_channels;   // columns past the aux weights are never fetched (TMA zero fill)
  if ((rc = encode_tmap_bf16_3d(&tw1_hi, a->w1_hi, k1_valid, kPwgG, 1, k1, k1 * kPwgG, w_box_rows))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tw1_lo, a->w1_lo, k1_valid, kPwgG, 1, k1, k1 * kPwgG, w_box_rows))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tw2_hi, a->w2_hi, 64, 128, 1, 64, 0, w_box_rows))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tw2_lo, a->w2_lo, 64, 128, 1, 64, 0, w_box_rows))) return rc;
  int resident = 0;
  if ((rc = prepare_kernel(pwg_layer_kernel, kPwgThreads, kPwgSmem, &resident))) return rc;
  PwgLayerArgs p;
  p.batch = a->batch; p.t = a->t; p.dil = a->dilation; p.aux_ch = a->aux_channels;
  p.tiles_per_b = (a->t + 127) / 128;
  p.total_tiles = p.tiles_per_b * a->batch;
  p.lens = a->lens; p.skip = a->skip; p.skip_init = a->skip_init;
  p.k_a = kGateKa; p.k_g = kGateKg;
  fold_gate_bias(p.gate_c, a->bias1, 64);   // host pointers: the biases travel in the kernel's parameter block
  for (int i = 0; i < 64; ++i) p.out_b[i] = a->bias2[64 + i];
  p.y_hi = static_cast<__nv_bfloat16*>(a->y_hi); p.y_lo = static_cast<__nv_bfloat16*>(a->y_lo);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = std::min(p.total_tiles, resident);
  pwg_layer_kernel<<<grid, kPwgThreads, kPwgSmem, st>>>(tx_hi, tx_lo, tc_hi, tc_lo, tw1_hi, tw1_lo, tw2_hi, tw2_lo, p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_pwg_upsample(const float* mel, const float* conv_in_w, const float* fir, const int32_t* scales,
                               int32_t n_stages, int32_t batch, int32_t aux, int32_t frames, int32_t window,
                               const int32_t* frame_lens, float* conv_in_ws, float* c_f32, void* c_hi, void* c_lo,
                               pk_stream_t stream) {
  using namespace pk;
  PK_CHECK_ARG(mel && conv_in_w && fir && scales && conv_in_ws, "NULL pointer");
  PK_CHECK_ARG(n_stages >= 1 && n_stages <= kUpMaxStages, "n_stages must be in [1,%d]", kUpMaxStages);
  PK_CHECK_ARG(batch > 0 && aux > 0 && frames > 0 && window >= 0, "bad sizes");
  // c_f32 == c_hi == NULL: conv_in only (frame-rate conditioning, pk_pwg_residual_layer_fc, needs no sample-rate tensor)
  PK_CHECK_ARG((c_hi == nullptr) == (c_lo == nullptr), "c_hi and c_lo must both be set or both NULL");
  PK_CHECK_ARG((aux % 8) == 0, "aux must be a multiple of 8 (got %d)", aux);
  UpsampleArgs a;
  memset(&a, 0, sizeof(a));
  a.n_stages = n_stages; a.aux = aux; a.frames = frames; a.window = window; a.hop = 1;
  for (int k = 0; k < n_stages; ++k) {
    const int s = scales[k];
    PK_CHECK_ARG(s >= 1 && s <= kUpMaxScale, "upsample scale %d unsupported (max %d)", s, kUpMaxScale);
    a.scale[k] = s;
    a.hop *= s;
    for (int r = 0; r < s; ++r)
      for (int q = 0; q < 2 * s + 1; ++q) a.poly[k][(r + q) / s][r] += fir[q];  // host pointer (tiny FIRs, concatenated)
    fir += 2 * s + 1;
  }
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  {
    // conv_in once per frame into the caller's workspace
    const int kin = 2 * window + 1;
    const size_t cin_smem = (static_cast<size_t>(aux) * kin * (aux + 1) + static_cast<size_t>(aux) * (kCinFrames + kin - 1)) * sizeof(float);
    PK_CHECK_ARG(cin_smem <= 220 * 1024, "conv_in weight does not fit shared memory (%zu bytes)", cin_smem);
    if (int rc = prepare_kernel(pwg_conv_in_kernel, 320, cin_smem)) return rc;
    dim3 cgrid((frames + kCinFrames - 1) / kCinFrames, batch);
    pwg_conv_in_kernel<<<cgrid, 320, cin_smem, st>>>(mel, conv_in_w, aux, frames, window, conv_in_ws);
    PK_CHECK_CUDA(cudaGetLastError());
    count_launch();
  }
  if (c_f32 == nullptr && c_hi == nullptr) return PK_OK;
  size_t floats = 0;
  {
    int w = a.hop;
    for (int k = n_stages - 1; k >= 0; --k) {
      w = (w - 1) / a.scale[k] + 4;          // upper bound of hi[k] - lo[k]
      floats += static_cast<size_t>(aux) * w;
    }
  }
  const size_t smem = floats * sizeof(float);
  PK_CHECK_ARG(smem <= 200 * 1024, "upsample tile does not fit shared memory (%zu bytes)", smem);
  if (int rc = prepare_kernel(pwg_upsample_kernel, 256, smem)) return rc;
  dim3 grid(frames, batch);
  pwg_upsample_kernel<<<grid, 256, smem, st>>>(conv_in_ws, frame_lens, a, c_f32, static_cast<__nv_bfloat16*>(c_hi),
                                               static_cast<__nv_bfloat16*>(c_lo));
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_pwg_first_conv(const float* noise, const float* w, const float* bias, const int32_t* lens, int32_t batch,
                                 int32_t t, void* x_hi, void* x_lo, pk_stream_t stream) {
  PK_CHECK_ARG(noise && w && bias && x_hi && x_lo, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && t > 0, "bad sizes");
  const long long rows = static_cast<long long>(batch) * t;
  const int threads = 256;
  const int blocks = static_cast<int>(std::min<long long>((rows * 8 + threads - 1) / threads, pk::sm_count() * 16LL));
  pk::pwg_first_conv_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(
      noise, w, bias, lens, t, rows, static_cast<__nv_bfloat16*>(x_hi), static_cast<__nv_bfloat16*>(x_lo));
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}

extern "C" int pk_pwg_tail(const float* skip, const float* skip_bias, const float* w1, const float* b1, const float* w2,
                           const float* b2, float scale, int64_t rows, float* out, pk_stream_t stream) {
  PK_CHECK_ARG(skip && w1 && b1 && w2 && b2 && out, "NULL pointer");
  PK_CHECK_ARG(rows > 0, "bad sizes");
  const int threads = 128;
  const long long pairs = (rows + 1) / 2;
  const int blocks = static_cast<int>(std::min<long long>((pairs + threads - 1) / threads, pk::sm_count() * 12LL));
  pk::pwg_tail_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(skip, skip_bias, w1, b1, w2, b2, scale, rows, out);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}
