// The fused WaveFlow residual blocks (reference parakeet/models/waveflow.py) for 64 or 128 residual channels:
// pk_waveflow_flow runs all row steps x layers of one Flow.inverse in one persistent launch, pk_waveflow_forward_layer one
// ResidualBlock.forward of Flow.forward over all net rows.  Both compute, per 128-position tile, in consume_tile:
//
//   a | g   = conv2d(3 rows, dilation 2^l along the width) + condition_proj(condition row) + biases
//   z       = tanh(a) * sigmoid(g)
//   res|skip= out_proj(z);   new row = row + res  -> the next layer's input (split planes);   skip (=|+=) skip
//
// Structure:
//   * persistent CTAs over 128-position tiles, 384 threads: a producer warpgroup (one TMA lane) and two consumer warpgroups
//     of 64 positions each;
//   * GEMM1 has 9 C/64 + 2 K-chunks: 3 width taps x 3 rows x C/64 channel blocks + the n_mels condition channels (64 + 64);
//     every stage of a 2-deep ring carries the A chunk (32 KB: hi | lo) and the weight chunk for all 2C gate channels, and
//     out_proj follows as C/64 weight-only chunks;
//   * the accumulators live in registers (wgmma), the gate runs on them in place and z is GEMM2's register A operand;
//   * the residual add reads the input row (hi + lo, 16 mantissa bits, re-split after every layer);
//   * out_proj's rows are ordered [skip | res] per 64-channel block so that the accumulator halves line up with the two
//     kinds of stores.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace wf {

constexpr int kATile = 128 * kSwizzleBytes;                  // 16 KB: 128 positions x one 64-channel chunk of one plane
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kStages = 2;

// ring geometry for C residual channels: N = 2C gate channels (a | g per 64-channel block)
template <int C>
struct Geo {
  static constexpr int kN = 2 * C;
  static constexpr int kWBytes = 2 * kN * kSwizzleBytes;     // hi | lo of one weight chunk, all kN rows
  static constexpr int kStageBytes = 2 * kATile + kWBytes;
  static constexpr int kG1Chunks = 9 * (C / 64) + 2;
  static constexpr int kG2Chunks = C / 64;
  static constexpr int kSmem = kStages * kStageBytes + 1024 + 256;
  static_assert(kSmem <= 227 * 1024, "shared memory budget");
};

__device__ __forceinline__ uint32_t ld_cg_u32(const void* ptr) {
  uint32_t v;
  asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(ptr) : "memory");
  return v;
}
__device__ __forceinline__ float2 ld_cg_f2(const float* ptr) {
  float2 v;
  asm volatile("ld.global.cg.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(ptr) : "memory");
  return v;
}
// hi + lo of two consecutive bf16 split-plane elements
__device__ __forceinline__ float2 ld_split2(const __nv_bfloat16* hi, const __nv_bfloat16* lo, long long off) {
  const uint32_t h = ld_cg_u32(hi + off), l = ld_cg_u32(lo + off);
  return make_float2(__uint_as_float(h << 16) + __uint_as_float(l << 16),
                     __uint_as_float(h & 0xffff0000u) + __uint_as_float(l & 0xffff0000u));
}

template <int N>
__device__ __forceinline__ void mma_ss(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (N == 128) wgmma_ss_n128(d, a, b, acc);
  else wgmma_ss_n256(d, a, b, acc);
}

// Consumer side of one 128-position tile: GEMM1 over the G1 chunks of the ring, the gate in registers, then GEMM2 with z as
// the register A operand, one 128-column output block [skip_blk | res_blk] at a time (64 accumulator registers), each block
// handed to epi(blk, acc) without biases / residual.  The C / 64 out_proj K-chunks stay in their stages until the last block.
// gc: pre-scaled gate biases in accumulator order; `it` is the running ring counter of this consumer.
template <int C, class Epi>
__device__ __forceinline__ void consume_tile(uint32_t smem, uint32_t full_bar, uint32_t empty_bar, uint32_t& it, int wg, int lane,
                                             const float* gc, float k_a, float k_g, int cond_ksteps_last, Epi&& epi) {
  using G = Geo<C>;
  constexpr int N = G::kN;
  const int cq = 2 * (lane & 3);
  uint32_t zh[C / 64][16], zl[C / 64][16];
  {
    float acc1[C];
    for (int j = 0; j < G::kG1Chunks; ++j, ++it) {
      const int s = it % kStages;
      mbar_wait_a(full_bar + 8 * s, (it / kStages) & 1);
      const uint32_t st = smem + s * G::kStageBytes;
      const uint64_t a_hi = make_smem_desc_sw128(st + wg * 64 * kSwizzleBytes), a_lo = make_smem_desc_sw128(st + kATile + wg * 64 * kSwizzleBytes);
      const uint64_t b_hi = make_smem_desc_sw128(st + 2 * kATile), b_lo = make_smem_desc_sw128(st + 2 * kATile + N * kSwizzleBytes);
      const int ksteps = j == G::kG1Chunks - 1 ? cond_ksteps_last : 4;
      wgmma_fence();
      for (int k = 0; k < ksteps; ++k) {
        mma_ss<N>(acc1, a_hi + desc_kstep(k), b_hi + desc_kstep(k), !(j == 0 && k == 0));
        mma_ss<N>(acc1, a_lo + desc_kstep(k), b_hi + desc_kstep(k), 1);
        mma_ss<N>(acc1, a_hi + desc_kstep(k), b_lo + desc_kstep(k), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc1);
      __syncwarp();
      if (lane == 0) mbar_arrive_a(empty_bar + 8 * s);
    }
    // tanh(a) sigmoid(g) = (1 - e1) / ((1 + e1) (1 + e2)), e1 = exp(-2a) (clamped: e1 * e2 must stay finite), e2 = exp(-g);
    // channel c of block blk: a in fragment 16 blk + c / 8, g in 16 blk + 8 + c / 8 (same thread)
#pragma unroll
    for (int blk = 0; blk < C / 64; ++blk) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float z[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int c = 128 * blk + 8 * jj + cq + (e & 1);
          const float e1 = ex2_approx(fminf(fmaf(acc1[4 * (16 * blk + jj) + e], k_a, gc[c]), 60.f));
          const float e2 = ex2_approx(fminf(fmaf(acc1[4 * (16 * blk + 8 + jj) + e], k_g, gc[c + 64]), 60.f));
          const float t1 = 1.f + e1;
          z[e] = (1.f - e1) * rcp_approx(fmaf(t1, e2, t1));
        }
        split2(z[0], z[1], zh[blk][2 * jj], zl[blk][2 * jj]);
        split2(z[2], z[3], zh[blk][2 * jj + 1], zl[blk][2 * jj + 1]);
      }
    }
  }
  const uint32_t s0 = it % kStages;                            // out_proj K-chunk kc (= z of channel block kc) is in stage
  for (int kc = 0; kc < G::kG2Chunks; ++kc)                    // (it + kc) % kStages
    mbar_wait_a(full_bar + 8 * ((s0 + kc) % kStages), ((it + kc) / kStages) & 1);
#pragma unroll
  for (int blk = 0; blk < C / 64; ++blk) {
    float acc2[64];
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < G::kG2Chunks; ++kc) {
      const uint32_t st = smem + ((s0 + kc) % kStages) * G::kStageBytes + 2 * kATile + blk * 128 * kSwizzleBytes;
      const uint64_t b_hi = make_smem_desc_sw128(st), b_lo = make_smem_desc_sw128(st + N * kSwizzleBytes);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t ah[4] = {zh[kc][4 * k], zh[kc][4 * k + 1], zh[kc][4 * k + 2], zh[kc][4 * k + 3]};
        const uint32_t al[4] = {zl[kc][4 * k], zl[kc][4 * k + 1], zl[kc][4 * k + 2], zl[kc][4 * k + 3]};
        wgmma_rs_n128(acc2, ah, b_hi + desc_kstep(k), !(kc == 0 && k == 0));
        wgmma_rs_n128(acc2, al, b_hi + desc_kstep(k), 1);
        wgmma_rs_n128(acc2, ah, b_lo + desc_kstep(k), 1);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc2);
    if (blk == C / 64 - 1) {
      __syncwarp();
      if (lane == 0)
        for (int kc = 0; kc < G::kG2Chunks; ++kc) mbar_arrive_a(empty_bar + 8 * ((s0 + kc) % kStages));
    }
    epi(blk, acc2);
  }
  it += G::kG2Chunks;
}

// ------------------------------------------------------------------------------------------------------------------------
// pk_waveflow_flow: ALL row steps x layers of one Flow.inverse (:515-556) in ONE persistent launch, for 64 or 128 residual
// channels (the reference's shipped config, examples/waveflow/config.py, has 128: gate channels a0 | g0 | a1 | g1, out_proj
// rows skip0 | res0 | skip1 | res1, 64 each, so that every 64-channel block runs the 64-channel code).
//
// Layer-step s = (row step, layer) touches, for a 256-position tile, only the tiles m-1, m, m+1 of step s-1 (width dilation
// <= 128, the row boundary - output_proj, inverse transform, input_proj - is pointwise), so the (G-1) x L steps run as a
// DATAFLOW over tiles instead of (G-1) x (L+2) grid-wide launches: tile T = s * tiles_per_step + (b, m) is processed by CTA
// T mod grid (as two 128-position halves); its TMA producer first acquires the completion counters of the (up to) three
// tiles it reads from; each consumer warp publishes its rows of a half with a gpu-scope release.  All CTAs are co-resident
// (the grid is sized by the occupancy query) and every CTA walks its tiles in increasing T, so the lowest unfinished tile
// can always run; a tile may wait for the CTA's own previous tile, which needs nothing more from the producer.  The last
// layer's skip stores finish the row in registers (output_proj, inverse transform, next row's input_proj).
// ------------------------------------------------------------------------------------------------------------------------
constexpr int kMaxLayers = 8;
constexpr int kMaxGroup = 16;
constexpr unsigned kTileDone = 2 * kConsumerThreads / 32;    // arrivals on a tile's counter: every consumer warp, per half

template <int C>
struct FlowArgs {
  CUtensorMap tm_x[kMaxLayers];          // ring planes of each layer (batch, w, 3C)
  CUtensorMap tm_w1[kMaxLayers][3];      // GEMM1 weight planes per layer and row-step variant, box = all 2C rows
  CUtensorMap tm_w2[kMaxLayers];         // out_proj planes (2C, C): [skip | res] per block
  CUtensorMap tm_c;                      // condition planes as (batch * n_group, w, n_mels): one row of one utterance per index
  int batch, w, n_layers, n_rows, n_group, tiles_per_b, tiles_per_step, total_tiles, cond_ksteps_last;
  int cmap[kMaxGroup];                   // condition row (after the flows' permutations) of row step i
  float gate_c[kMaxLayers][2 * C];       // accumulator order, pre-scaled
  float out_b[kMaxLayers][2 * C];
  float in_w[C], in_b[C];                // input_proj (1 -> C)
  float po_w[2 * C], po_b[2];            // output_proj (C -> logs, b)
  float k_a, k_g;
  float* skip;                           // (batch, w, C)
  const float* z;                        // (batch, n_group, w) rows of this flow's input
  float* x;                              // (batch, n_group, w) rows of its output; row 0 is filled by the caller
  __nv_bfloat16* ring_hi[kMaxLayers];
  __nv_bfloat16* ring_lo[kMaxLayers];
  unsigned* flags;                       // [total_tiles] completion counters, zeroed by the caller
};

struct FlowTile {
  int s, l, r, b, m0, mt;
  template <class A>
  __device__ void decode(const A& p, int t) {
    s = t / p.tiles_per_step;
    const int rem = t - s * p.tiles_per_step;
    r = s / p.n_layers;
    l = s - r * p.n_layers;
    b = rem / p.tiles_per_b;
    mt = rem - b * p.tiles_per_b;
    m0 = mt * 256;
  }
};

__device__ __forceinline__ void wait_tile_done(const unsigned* flag) {
  const long long t0 = clock64();
  while (ld_acquire_gpu(flag) < kTileDone) {
    __nanosleep(64);
    if (clock64() - t0 > (1ll << 33)) {   // ~4 s: a dependency that never completes is a scheduling bug - fail loudly, do not hang
      printf("pk_waveflow_flow: tile dependency timed out (block %d)\n", static_cast<int>(blockIdx.x));
      __trap();
    }
  }
}

template <int C>
__global__ void __launch_bounds__(kThreads, 1)
waveflow_flow_kernel(const __grid_constant__ FlowArgs<C> p) {
  using G = Geo<C>;
  constexpr int kPer = C / 64;                                 // 64-channel blocks
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full_bar = smem + kStages * G::kStageBytes;   // [stages]
  const uint32_t empty_bar = full_bar + 8 * kStages;           // [stages]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == kConsumerThreads) {
    for (int s = 0; s < kStages; ++s) { mbar_init_a(full_bar + 8 * s, 1); mbar_init_a(empty_bar + 8 * s, kConsumerThreads / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      uint32_t it = 0;
      FlowTile t;
      for (int T = blockIdx.x; T < p.total_tiles; T += gridDim.x) {
        t.decode(p, T);
        if (t.s > 0) {
          // the rows this tile reads were written by tiles mt-1 .. mt+1 of the previous step (generic-proxy stores) ...
          const unsigned* f = p.flags + (T - p.tiles_per_step);
          if (t.mt > 0) wait_tile_done(f - 1);
          wait_tile_done(f);
          if (t.mt + 1 < p.tiles_per_b) wait_tile_done(f + 1);
          fence_proxy_async_all();       // ... and are read here through the async proxy
        }
        const int variant = (t.r + 1) % 3;                     // row step i = r + 1
        const int crow = t.b * p.n_group + p.cmap[t.r + 1];
        for (int half = 0; half < 2; ++half) {
          const int row0 = t.m0 + 128 * half;
          for (int j = 0; j < G::kG1Chunks + G::kG2Chunks; ++j, ++it) {
            const int s = it % kStages;
            mbar_wait_a(empty_bar + 8 * s, ((it / kStages) & 1) ^ 1);
            const uint32_t st = smem + s * G::kStageBytes;
            const uint32_t fb = full_bar + 8 * s;
            if (j < 9 * kPer) {
              // (tap, ring slot, channel block); the centre tap comes last among the taps
              const int t3 = j / (3 * kPer), rem = j - 3 * kPer * t3;
              const int tap = t3 == 0 ? 0 : t3 == 1 ? 2 : 1, slot = rem / kPer, hb = rem % kPer;
              mbar_arrive_expect_tx_a(fb, G::kStageBytes);
              tma_load_4d_a(st, &p.tm_x[t.l], fb, slot * C + hb * 64, row0 + (tap - 1) * (1 << t.l), t.b, 0);
              tma_load_4d_a(st + 2 * kATile, &p.tm_w1[t.l][variant], fb, ((3 * tap + slot) * kPer + hb) * kChunkK, 0, 0, 0);
            } else if (j < G::kG1Chunks) {
              mbar_arrive_expect_tx_a(fb, G::kStageBytes);
              tma_load_4d_a(st, &p.tm_c, fb, (j - 9 * kPer) * kChunkK, row0, crow, 0);
              tma_load_4d_a(st + 2 * kATile, &p.tm_w1[t.l][variant], fb, j * kChunkK, 0, 0, 0);
            } else {
              mbar_arrive_expect_tx_a(fb, G::kWBytes);                                   // out_proj K-chunk: weights only
              tma_load_4d_a(st + 2 * kATile, &p.tm_w2[t.l], fb, (j - G::kG1Chunks) * kChunkK, 0, 0, 0);
            }
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers ------------------------------
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int rl = wg * 64 + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
    uint32_t it = 0;
    FlowTile t;
    for (int T = blockIdx.x; T < p.total_tiles; T += gridDim.x) {
      t.decode(p, T);
      const bool last_layer = t.l == p.n_layers - 1;
      const float* ob = p.out_b[t.l];
      for (int half = 0; half < 2; ++half) {
        float s0[2] = {0.f, 0.f}, s1[2] = {0.f, 0.f};          // output_proj partial sums (last layer)
        consume_tile<C>(smem, full_bar, empty_bar, it, wg, lane, p.gate_c[t.l], p.k_a, p.k_g, p.cond_ksteps_last,
                        [&](int blk, const float (&acc2)[64]) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int row = t.m0 + 128 * half + rl + 8 * hh;
            if (row >= p.w) continue;                          // positions past the end of the row: nothing to store
            const long long pos = static_cast<long long>(t.b) * p.w + row;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int c = 64 * blk + 8 * jj + cq;            // channel inside C
              const int ca = 128 * blk + 8 * jj + cq;          // accumulator column of its skip value
              float o0 = acc2[4 * jj + 2 * hh] + ob[ca], o1 = acc2[4 * jj + 2 * hh + 1] + ob[ca + 1];
              float* dst = p.skip + pos * C + c;
              if (last_layer) {
                // the sum of the skips is complete here: output_proj in registers instead of a last read-modify-write
                if (p.n_layers > 1) {
                  const float2 a = ld_cg_f2(dst);
                  o0 += a.x; o1 += a.y;
                }
                s0[hh] = fmaf(p.po_w[c], o0, fmaf(p.po_w[c + 1], o1, s0[hh]));
                s1[hh] = fmaf(p.po_w[C + c], o0, fmaf(p.po_w[C + c + 1], o1, s1[hh]));
              } else {
                if (t.l == 0) *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
                else asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(o0), "f"(o1) : "memory");
                // new row = newest row + res -> the next layer's ring, same slot
                const long long off = pos * (3 * C) + (t.r % 3) * C + c;
                const float2 x = ld_split2(p.ring_hi[t.l], p.ring_lo[t.l], off);
                uint32_t oh, ol;
                split2(acc2[4 * (8 + jj) + 2 * hh] + ob[ca + 64] + x.x, acc2[4 * (8 + jj) + 2 * hh + 1] + ob[ca + 65] + x.y, oh, ol);
                *reinterpret_cast<uint32_t*>(p.ring_hi[t.l + 1] + off) = oh;
                *reinterpret_cast<uint32_t*>(p.ring_lo[t.l + 1] + off) = ol;
              }
            }
          }
        });
        if (last_layer) {
          // Flow._inverse_transform_row (:505-510) and, for the next row step, Flow.input_proj (:437-442) into layer 0's ring
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            s0[hh] += __shfl_xor_sync(0xffffffffu, s0[hh], 1);
            s0[hh] += __shfl_xor_sync(0xffffffffu, s0[hh], 2);
            s1[hh] += __shfl_xor_sync(0xffffffffu, s1[hh], 1);
            s1[hh] += __shfl_xor_sync(0xffffffffu, s1[hh], 2);
            const int row = t.m0 + 128 * half + rl + 8 * hh;
            if (row >= p.w) continue;
            const long long pos = static_cast<long long>(t.b) * p.w + row;
            const int irow = t.r + 1;
            const long long xi = (static_cast<long long>(t.b) * p.n_group + irow) * p.w + row;
            const float logs = s0[hh] + p.po_b[0], bb = s1[hh] + p.po_b[1];
            const float xn = (__ldg(p.z + xi) - bb) * expf(-logs);
            if ((lane & 3) == 0) p.x[xi] = xn;
            if (irow + 1 < p.n_group) {
              const long long off = pos * (3 * C) + (irow % 3) * C;
#pragma unroll
              for (int jj = 0; jj < C / 8; ++jj) {
                const int c = 8 * jj + cq;
                uint32_t oh, ol;
                split2(fmaf(p.in_w[c], xn, p.in_b[c]), fmaf(p.in_w[c + 1], xn, p.in_b[c + 1]), oh, ol);
                *reinterpret_cast<uint32_t*>(p.ring_hi[0] + off + c) = oh;
                *reinterpret_cast<uint32_t*>(p.ring_lo[0] + off + c) = ol;
              }
            }
          }
        }
        // publish: this warp's rows of the half are written (generic proxy) -> visible to the async-proxy reads of the consumers
        __syncwarp();
        if (lane == 0) {
          fence_proxy_async_all();
          __threadfence();
          red_release_gpu_inc(p.flags + T);
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------------------------------------
// pk_waveflow_forward_layer: one ResidualBlock.forward (:197-226) of Flow.forward (:465-494) over ALL n_group - 1 net rows
// of all utterances in one launch - no row dependency, so it is a plain 2-D gated convolution over 128-position tiles along
// the width of one (utterance, net row).  Input / output are (batch * (n_group + 1), w, C) split planes: two zero rows per
// utterance, then its net rows, so that kernel row kh of net row r reads buffer row r + kh (= net row r - 2 + kh, the causal
// padding [2, 0]) and never the previous utterance; the width taps read columns w + (tap - 1) 2^l, and TMA's out-of-bounds
// fill is the "same" padding.  GEMM1 chunk j = (tap, kh, channel block) reads weight columns [64 j, 64 j + 64) of the row
// step variant 0 of the inverse's packed weight (slot s = kernel row s).  Consumer side and epilogue as pk_waveflow_flow.
// ------------------------------------------------------------------------------------------------------------------------
template <int C>
struct FwdLayerArgs {
  int w, n_group, dil, tiles_per_row, total_tiles, cond_ksteps_last, skip_init;
  int cmap[kMaxGroup];                   // condition row (after the previous flows' permutations) of height h
  float gate_c[2 * C];                   // accumulator order, pre-scaled
  float out_b[2 * C];
  float k_a, k_g;
  float* skip;                           // (batch, n_group - 1, w, C)
  const __nv_bfloat16* x_hi;             // (batch * (n_group + 1), w, C): the residual reads the net row itself
  const __nv_bfloat16* x_lo;
  __nv_bfloat16* y_hi;                   // same layout; NULL on the last layer
  __nv_bfloat16* y_lo;
};

template <int C>
__global__ void __launch_bounds__(kThreads, 1)
waveflow_forward_layer_kernel(const __grid_constant__ CUtensorMap tm_x,    // input planes (batch * (n_group + 1), w, C)
                              const __grid_constant__ CUtensorMap tm_c,    // condition planes (batch * n_group, w, n_mels)
                              const __grid_constant__ CUtensorMap tm_w1,   // GEMM1 weight planes (2C, 64 G1), box = all rows
                              const __grid_constant__ CUtensorMap tm_w2,   // out_proj planes (2C, C)
                              const __grid_constant__ FwdLayerArgs<C> p) {
  using G = Geo<C>;
  constexpr int kPer = C / 64;                                 // 64-channel blocks
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full_bar = smem + kStages * G::kStageBytes;   // [stages]
  const uint32_t empty_bar = full_bar + 8 * kStages;           // [stages]
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int rows = p.n_group - 1;

  if (threadIdx.x == kConsumerThreads) {
    tma_prefetch_desc(&tm_x); tma_prefetch_desc(&tm_c); tma_prefetch_desc(&tm_w1); tma_prefetch_desc(&tm_w2);
    for (int s = 0; s < kStages; ++s) { mbar_init_a(full_bar + 8 * s, 1); mbar_init_a(empty_bar + 8 * s, kConsumerThreads / 32); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const int br = tile / p.tiles_per_row, w0 = (tile - br * p.tiles_per_row) * 128;
        const int b = br / rows, r = br - b * rows;
        const int xrow = b * (p.n_group + 1) + r;              // + kh: net row r - 2 + kh
        const int crow = b * p.n_group + p.cmap[r + 1];        // Flow.forward conditions net row r on height r + 1
        for (int j = 0; j < G::kG1Chunks + G::kG2Chunks; ++j, ++it) {
          const int s = it % kStages;
          mbar_wait_a(empty_bar + 8 * s, ((it / kStages) & 1) ^ 1);
          const uint32_t st = smem + s * G::kStageBytes;
          const uint32_t fb = full_bar + 8 * s;
          if (j < 9 * kPer) {
            const int tap = j / (3 * kPer), rem = j - 3 * kPer * tap;
            const int kh = rem / kPer, hb = rem - kPer * kh;
            mbar_arrive_expect_tx_a(fb, G::kStageBytes);
            tma_load_4d_a(st, &tm_x, fb, hb * 64, w0 + (tap - 1) * p.dil, xrow + kh, 0);   // columns outside [0, w) read as zero
            tma_load_4d_a(st + 2 * kATile, &tm_w1, fb, j * kChunkK, 0, 0, 0);
          } else if (j < G::kG1Chunks) {
            mbar_arrive_expect_tx_a(fb, G::kStageBytes);
            tma_load_4d_a(st, &tm_c, fb, (j - 9 * kPer) * kChunkK, w0, crow, 0);              // channels >= n_mels read as zero
            tma_load_4d_a(st + 2 * kATile, &tm_w1, fb, j * kChunkK, 0, 0, 0);
          } else {
            mbar_arrive_expect_tx_a(fb, G::kWBytes);                                         // out_proj K-chunk: weights only
            tma_load_4d_a(st + 2 * kATile, &tm_w2, fb, (j - G::kG1Chunks) * kChunkK, 0, 0, 0);
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers ------------------------------
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int rl = wg * 64 + 16 * (warp & 3) + (lane >> 2);
    const int cq = 2 * (lane & 3);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const int br = tile / p.tiles_per_row, w0 = (tile - br * p.tiles_per_row) * 128;
      const int b = br / rows, r = br - b * rows;
      const long long srow = static_cast<long long>(br) * p.w;                             // skip row (b, r)
      const long long xrow = (static_cast<long long>(b) * (p.n_group + 1) + 2 + r) * p.w;  // buffer row of net row r
      consume_tile<C>(smem, full_bar, empty_bar, it, wg, lane, p.gate_c, p.k_a, p.k_g, p.cond_ksteps_last,
                      [&](int blk, const float (&acc2)[64]) {
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int col = w0 + rl + 8 * hh;
          if (col >= p.w) continue;                            // positions past the end of the row: nothing to store
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int c = 64 * blk + 8 * jj + cq;              // channel inside C
            const int ca = 128 * blk + 8 * jj + cq;            // accumulator column of its skip value
            float* dst = p.skip + (srow + col) * C + c;
            const float o0 = acc2[4 * jj + 2 * hh] + p.out_b[ca], o1 = acc2[4 * jj + 2 * hh + 1] + p.out_b[ca + 1];
            if (p.skip_init) *reinterpret_cast<float2*>(dst) = make_float2(o0, o1);
            else asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(o0), "f"(o1) : "memory");
            if (p.y_hi != nullptr) {
              // ResidualBlock.forward: res = x_in + res, into the other buffer (neighbouring tiles still read this one)
              const long long off = (xrow + col) * C + c;
              const float2 x = ld_split2(p.x_hi, p.x_lo, off);
              uint32_t oh, ol;
              split2(acc2[4 * (8 + jj) + 2 * hh] + p.out_b[ca + 64] + x.x, acc2[4 * (8 + jj) + 2 * hh + 1] + p.out_b[ca + 65] + x.y, oh, ol);
              *reinterpret_cast<uint32_t*>(p.y_hi + off) = oh;
              *reinterpret_cast<uint32_t*>(p.y_lo + off) = ol;
            }
          }
        }
      });
    }
  }
}

}  // namespace wf
}  // namespace pk

template <int C>
static int flow_launch(const pk_waveflow_flow_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::wf;
  using G = Geo<C>;
  // every CTA must be resident at once (tiles wait for tiles of other CTAs): ask the driver how many fit
  int max_ctas = 0, rc;
  if ((rc = prepare_kernel(waveflow_flow_kernel<C>, kThreads, G::kSmem, &max_ctas))) return rc;
  PK_CHECK_ARG(max_ctas >= 1, "no resident CTA available for pk_waveflow_flow");
  static std::mutex mu;
  std::lock_guard<std::mutex> lock(mu);
  static FlowArgs<C> p;    // up to 22 KB of kernel parameters, built in place under `mu`; the launch copies them
  const uint64_t W = a->width, B = a->batch;
  for (int l = 0; l < a->n_layers; ++l) {
    PK_CHECK_ARG(a->ring_hi[l] && a->ring_lo[l] && a->w2_hi[l] && a->w2_lo[l] && a->bias1[l] && a->bias2[l], "NULL entry for layer %d", l);
    if ((rc = encode_tmap_bf16_planes(&p.tm_x[l], a->ring_hi[l], a->ring_lo[l], 3 * C, W, B, 3 * C, W * 3 * C, 128))) return rc;
    for (int v = 0; v < 3; ++v) {
      PK_CHECK_ARG(a->w1_hi[3 * l + v] && a->w1_lo[3 * l + v], "NULL GEMM1 weight for layer %d variant %d", l, v);
      if ((rc = encode_tmap_bf16_planes(&p.tm_w1[l][v], a->w1_hi[3 * l + v], a->w1_lo[3 * l + v], G::kG1Chunks * kChunkK, 2 * C, 1,
                                        G::kG1Chunks * kChunkK, 0, 2 * C)))
        return rc;
    }
    if ((rc = encode_tmap_bf16_planes(&p.tm_w2[l], a->w2_hi[l], a->w2_lo[l], C, 2 * C, 1, C, 0, 2 * C))) return rc;
    fold_gate_bias(p.gate_c[l], a->bias1[l], C);
    for (int i = 0; i < 2 * C; ++i) p.out_b[l][i] = a->bias2[l][i];
    p.ring_hi[l] = static_cast<__nv_bfloat16*>(a->ring_hi[l]);
    p.ring_lo[l] = static_cast<__nv_bfloat16*>(a->ring_lo[l]);
  }
  if ((rc = encode_tmap_bf16_planes(&p.tm_c, a->cond_hi, a->cond_lo, a->n_mels, W, B * a->n_group, a->n_mels, W * a->n_mels, 128)))
    return rc;
  p.batch = a->batch; p.w = a->width; p.n_layers = a->n_layers; p.n_group = a->n_group; p.n_rows = a->n_group - 1;
  p.tiles_per_b = (a->width + 255) / 256;
  p.tiles_per_step = p.tiles_per_b * a->batch;
  const long long total = static_cast<long long>(p.tiles_per_step) * p.n_rows * p.n_layers;
  PK_CHECK_ARG(total < (1ll << 30) && a->flags_len >= total, "flags must hold one counter per tile (%lld)", total);
  p.total_tiles = static_cast<int>(total);
  p.cond_ksteps_last = (a->n_mels - 64 + kWgmmaK - 1) / kWgmmaK;
  for (int i = 0; i < a->n_group; ++i) {
    PK_CHECK_ARG(a->cond_rows[i] >= 0 && a->cond_rows[i] < a->n_group, "cond_rows[%d] out of range", i);
    p.cmap[i] = a->cond_rows[i];
  }
  for (int i = 0; i < C; ++i) { p.in_w[i] = a->in_w[i]; p.in_b[i] = a->in_b[i]; p.po_w[i] = a->out_w[i]; p.po_w[C + i] = a->out_w[C + i]; }
  p.po_b[0] = a->out_b[0]; p.po_b[1] = a->out_b[1];
  p.k_a = kGateKa; p.k_g = kGateKg;
  p.skip = a->skip; p.z = a->z; p.x = a->x; p.flags = a->flags;
  const int grid = std::max(1, std::min(max_ctas, p.total_tiles));
  waveflow_flow_kernel<C><<<grid, kThreads, G::kSmem, static_cast<cudaStream_t>(stream)>>>(p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_flow(const pk_waveflow_flow_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::wf;
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  PK_CHECK_ARG(a->batch > 0 && a->width > 0, "bad batch/width");
  PK_CHECK_ARG(a->channels == 64 || a->channels == 128, "the fused WaveFlow flow is built for 64 or 128 residual channels (got %d)",
               a->channels);
  PK_CHECK_ARG(a->n_mels > 64 && a->n_mels <= 128 && (a->n_mels % 8) == 0, "n_mels must be in (64, 128], a multiple of 8");
  // One layer is refused: the last layer's epilogue writes the next row's input_proj into layer 0's ring slot (r + 1) % 3, which
  // layer 0 of the same layer-step still reads through its +-1 width taps in the neighbouring tiles, and nothing orders them.
  PK_CHECK_ARG(a->n_layers >= 2, "n_layers must be at least 2: with one layer the next row's input_proj overwrites layer 0's "
               "ring slot in the same layer-step whose neighbouring tiles still read it (got %d)", a->n_layers);
  PK_CHECK_ARG(a->n_layers <= kMaxLayers && a->n_group >= 2 && a->n_group <= kMaxGroup,
               "n_layers must be 2..8 (width dilation 2^l <= 128) and n_group 2..16");
  PK_CHECK_ARG(a->cond_rows && a->ring_hi && a->ring_lo && a->cond_hi && a->cond_lo && a->w1_hi && a->w1_lo && a->w2_hi && a->w2_lo &&
               a->bias1 && a->bias2 && a->in_w && a->in_b && a->out_w && a->out_b && a->z && a->x && a->skip && a->flags,
               "NULL pointer in pk_waveflow_flow_args");
  return a->channels == 128 ? flow_launch<128>(a, stream) : flow_launch<64>(a, stream);
}

template <int C>
static int forward_layer_launch(const pk_waveflow_forward_layer_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::wf;
  using G = Geo<C>;
  int resident = 0, rc;
  if ((rc = prepare_kernel(waveflow_forward_layer_kernel<C>, kThreads, G::kSmem, &resident))) return rc;
  const uint64_t W = a->width, B = a->batch, NG = a->n_group;
  CUtensorMap tx, tc, tw1, tw2;
  if ((rc = encode_tmap_bf16_planes(&tx, a->x_hi, a->x_lo, C, W, B * (NG + 1), C, W * C, 128))) return rc;
  if ((rc = encode_tmap_bf16_planes(&tc, a->cond_hi, a->cond_lo, a->n_mels, W, B * NG, a->n_mels, W * a->n_mels, 128))) return rc;
  if ((rc = encode_tmap_bf16_planes(&tw1, a->w1_hi, a->w1_lo, G::kG1Chunks * kChunkK, 2 * C, 1, G::kG1Chunks * kChunkK, 0, 2 * C)))
    return rc;
  if ((rc = encode_tmap_bf16_planes(&tw2, a->w2_hi, a->w2_lo, C, 2 * C, 1, C, 0, 2 * C))) return rc;
  FwdLayerArgs<C> p;
  p.w = a->width; p.n_group = a->n_group; p.dil = a->dilation; p.skip_init = a->skip_init;
  p.tiles_per_row = (a->width + 127) / 128;
  const long long total = static_cast<long long>(p.tiles_per_row) * a->batch * (a->n_group - 1);
  PK_CHECK_ARG(total < (1ll << 31), "too many tiles (%lld)", total);
  p.total_tiles = static_cast<int>(total);
  p.cond_ksteps_last = (a->n_mels - 64 + kWgmmaK - 1) / kWgmmaK;
  for (int i = 0; i < a->n_group; ++i) {
    PK_CHECK_ARG(a->cond_rows[i] >= 0 && a->cond_rows[i] < a->n_group, "cond_rows[%d] out of range", i);
    p.cmap[i] = a->cond_rows[i];
  }
  p.k_a = kGateKa; p.k_g = kGateKg;
  fold_gate_bias(p.gate_c, a->bias1, C);
  for (int i = 0; i < 2 * C; ++i) p.out_b[i] = a->bias2[i];
  p.skip = a->skip;
  p.x_hi = static_cast<const __nv_bfloat16*>(a->x_hi); p.x_lo = static_cast<const __nv_bfloat16*>(a->x_lo);
  p.y_hi = static_cast<__nv_bfloat16*>(a->y_hi); p.y_lo = static_cast<__nv_bfloat16*>(a->y_lo);
  const int grid = std::min(p.total_tiles, resident);
  waveflow_forward_layer_kernel<C><<<grid, kThreads, G::kSmem, static_cast<cudaStream_t>(stream)>>>(tx, tc, tw1, tw2, p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_waveflow_forward_layer(const pk_waveflow_forward_layer_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::wf;
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  PK_CHECK_ARG(a->batch > 0 && a->width > 0 && a->dilation >= 1 && a->dilation <= 128, "bad batch/width/dilation");
  PK_CHECK_ARG(a->channels == 64 || a->channels == 128,
               "the WaveFlow forward layer is built for 64 or 128 residual channels (got %d)", a->channels);
  PK_CHECK_ARG(a->n_mels > 64 && a->n_mels <= 128 && (a->n_mels % 8) == 0, "n_mels must be in (64, 128], a multiple of 8");
  PK_CHECK_ARG(a->n_group >= 2 && a->n_group <= kMaxGroup, "n_group must be 2..16");
  PK_CHECK_ARG(a->cond_rows && a->x_hi && a->x_lo && a->cond_hi && a->cond_lo && a->w1_hi && a->w1_lo && a->w2_hi && a->w2_lo &&
               a->bias1 && a->bias2 && a->skip, "NULL pointer in pk_waveflow_forward_layer_args");
  PK_CHECK_ARG((a->y_hi == nullptr) == (a->y_lo == nullptr), "y_hi / y_lo: both or neither");
  PK_CHECK_ARG(a->y_hi == nullptr || (a->y_hi != a->x_hi && a->y_lo != a->x_lo), "the layer cannot write its input in place");
  return a->channels == 128 ? forward_layer_launch<128>(a, stream) : forward_layer_launch<64>(a, stream);
}
