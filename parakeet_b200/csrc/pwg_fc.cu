// pk_pwg_residual_layer_fc: the fused Parallel WaveGAN residual layer (pwg.cu) with FRAME-RATE CONDITIONING (the default
// residual-stack path of the Python model - DESIGN.md 5).
//
// The upsampling network is linear and per channel, so conv1x1_aux(upsample(m'))[t, n] = sum_j U[t, j] (W_aux m')[j, n].
// GEMM1's two conditioning K-chunks (80 channels of the 1.23 GB sample-rate conditioning tensor, 5 K-steps, 32 KB of
// resident W_aux) become ONE K-step: A = the tile-relative band table of U (constants of the model,
// models/_pwg_frame_cond.py), B = the 16-frame window of P = W_aux m' that the tile touches (frame rate, L2 resident).
//
// Hopper structure: persistent CTAs over 128-sample half tiles of the 256-sample windows that one band-table / P-window pair
// describes; each half tile is two 64-row tiles, one per consumer warpgroup ("ping-pong": while one warpgroup gates and
// stores, the other keeps the tensor cores busy).  384 threads:
//   * warps 8-11 (producer warpgroup, one TMA lane): per 64-row tile 4 A chunks (tap -d, tap +d, conditioning, centre tap)
//     through one 4-deep ring of 16 KB stages, the two warpgroups' tiles alternating; the conditioning stage holds a
//     16-column box of the band table and the 16-frame P window of the tile (32-byte swizzle).  W1 (three tap chunks) and
//     W2 stay resident (128 KB);
//   * warps 0-7 (two consumer warpgroups, one 64-row tile each): GEMM1 (wgmma, accumulator in registers, one commit group
//     in flight), the gate in registers, z as the register A operand of GEMM2 - z never touches shared memory.  The residual
//     add `+ x` is folded in by starting GEMM2's accumulator at [0 | x], read from the centre-tap chunk while it is in
//     shared memory; every stage goes back to the producer during GEMM1.  An ordering barrier alternates the warpgroups'
//     GEMM1s, so their epilogues alternate too and share one 32 KB staging area: y (split planes) and the fp32 skip tile,
//     written by one TMA store and one TMA reduce-add.
//
// The two ends of the stack are instantiations of the same kernel (FcMode), so that neither x0 nor the final skip sum makes
// a round trip through HBM:
//   * first layer: x0 = first_conv(noise) = w n + b is never stored.  The dilated conv of x0 is rank one per tap,
//     sum_tap valid(t') (n[t'] u_tap + v_tap) with u_tap = W1_tap w, v_tap = W1_tap b (t' = t + (tap - 1) d; a tap outside
//     [0, len) is the conv's zero padding and adds nothing): the consumers start GEMM1's accumulator from these fp32 FMAs and
//     add only the conditioning K-step on the tensor cores; GEMM2 starts at [0 | w n + b].  No x chunks, no resident W1 (u_tap
//     and v_tap sit in its place);
//   * last layer: the tile's fp32 skip sum comes in through the ring ahead of GEMM1's chunks and starts GEMM2's skip half;
//     the epilogue runs last_conv_layers on it (relu, a K = 64 wgmma chain against the tail weights, which take the skip staging
//     area, relu, a dot product) and stores one sample per row.  Nothing is written to the skip buffer; y still is.
#include <stdlib.h>
#include <string.h>

#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace fc {

constexpr int kPwgR = 64;
constexpr int kPwgG = 128;
constexpr int kATile = 128 * kSwizzleBytes;                  // 16 KB: one plane of a resident 128-row weight chunk
constexpr int kQTile = 64 * kSwizzleBytes;                   // 8 KB: one plane of a 64-row K-chunk of x
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kFcStages = 4;
constexpr int kFcStageBytes = 2 * kQTile;                    // A hi, A lo
constexpr int kFcUBytes = 2 * 64 * 32;                       // 4 KB: hi | lo of 16 band-table columns x 64 rows
constexpr int kFcPBytes = 2 * 128 * 32;                      // 8 KB: hi | lo of 16 P frames x 128 output channels
constexpr int kFcW1Bytes = 3 * 2 * kATile;                   // 96 KB: three tap chunks x 128 output channels
constexpr int kFcW2Bytes = 2 * kATile;                       // 32 KB: 128 outputs (skip | out) x 64
constexpr int kFcYBytes = 2 * kQTile;                        // 16 KB: y staging, hi | lo planes of 64 rows
constexpr int kFcSkipBytes = 64 * 64 * 4;                    // 16 KB: skip staging, 64 rows x 64 fp32 channels
constexpr int kFcSmem = kFcW1Bytes + kFcW2Bytes + kFcStages * kFcStageBytes + kFcYBytes + kFcSkipBytes + 1024 + 256;
static_assert(kFcUBytes + kFcPBytes <= kFcStageBytes, "the conditioning operands share one ring stage");
static_assert(kFcSmem <= 227 * 1024, "shared memory budget");

struct FcLayerArgs {
  int batch, t, dil, hop;
  int u_period, u_start_row, u_end_base;   // compact band table layout (include/parakeet_b200.h)
  int p_row0;                   // first row of this layer's 128 output channels in the P planes
  const int32_t* lens;
  float gate_c[128];
  float out_b[64];
  float k_a, k_g;
  float* skip;
  int skip_init;
};

enum FcMode { kFcFirst, kFcMiddle, kFcLast };
constexpr int kFirstPair = 80;                               // bytes of first_conv vectors per column pair in the first layer

// ring chunks of a 64-row tile, in load order: in the last layer the tile's skip sum (read and handed back before GEMM1, so
// that it does not hold a stage through it), then GEMM1's: tap -d, tap +d, conditioning, centre tap (it also supplies the
// residual x); the first layer loads the conditioning chunk only
template <int M>
struct FcChunks {
  static constexpr int kG1 = M == kFcFirst ? 1 : 4;          // read by GEMM1
  static constexpr int kG1Base = M == kFcLast ? 1 : 0;       // position of GEMM1's first chunk
  static constexpr int kCond = M == kFcFirst ? 0 : 2;        // among GEMM1's
  static constexpr int kAll = kG1Base + kG1;
};

// what the first and the last layer read beyond FcLayerArgs (the middle layers: nothing)
template <int M>
struct FcEnds {};
template <>
struct FcEnds<kFcFirst> {
  const float* noise;                                        // (batch, t)
  float w[64], b[64];                                        // first_conv
  float u[3][128], v[3][128];                                // per tap: W1_tap w, W1_tap b
};
template <>
struct FcEnds<kFcLast> {
  const uint4* w1_hi;                                        // last_conv_layers.1 [64 out][64 in], split planes
  const uint4* w1_lo;
  float* out;                                                // (batch, t)
  float skip_b[64];                                          // the sum of the 30 conv1x1_skip biases
  float b1[64], w2[64];                                      // last_conv_layers.1 bias, last_conv_layers.3 weight
  float b2, scale;                                           // last_conv_layers.3 bias, sqrt(1 / layers)
};

struct FcTileIter {   // 128-sample tiles = halves of the 256-sample windows; live windows only
  int idx, step, tiles_per_b, total, t;
  const int32_t* lens;
  __device__ FcTileIter(const FcLayerArgs& p)
      : idx(static_cast<int>(blockIdx.x) - static_cast<int>(gridDim.x)), step(gridDim.x),
        tiles_per_b((p.t + 255) >> 8), total(((p.t + 255) >> 8) * p.batch * 2), t(p.t), lens(p.lens) {}
  // b, m0 (first row of the 256-sample window), half (which 128 rows of it)
  __device__ bool next(int& b, int& m0, int& half) {
    for (;;) {
      idx += step;
      if (idx >= total) return false;
      const int w = idx >> 1;
      half = idx & 1;
      b = w / tiles_per_b;
      m0 = (w % tiles_per_b) * 256;
      const int len = lens ? min(__ldg(lens + b), t) : t;
      if (m0 < len) return true;
    }
  }
};

template <int kMode>
__global__ void __launch_bounds__(kThreads, 1)
pwg_layer_fc_kernel(const __grid_constant__ CUtensorMap tm_x, const __grid_constant__ CUtensorMap tm_u,
                    const __grid_constant__ CUtensorMap tm_p,          // 4-D maps: both planes of a tile in one TMA box
                    const __grid_constant__ CUtensorMap tm_w1_hi, const __grid_constant__ CUtensorMap tm_w1_lo,
                    const __grid_constant__ CUtensorMap tm_w2_hi, const __grid_constant__ CUtensorMap tm_w2_lo,
                    const __grid_constant__ CUtensorMap tm_y, const __grid_constant__ CUtensorMap tm_skip,
                    const FcLayerArgs p, const FcEnds<kMode> ends) {
  using Ch = FcChunks<kMode>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w1 = smem;                                    // [tap chunk][hi | lo] 128-row tiles, resident
  const uint32_t w2 = w1 + kFcW1Bytes;                         // [hi | lo]
  const uint32_t ring = w2 + kFcW2Bytes;                       // [stages] 64-row chunks [hi | lo]
  // epilogue staging, used by the two consumer warpgroups in turn
  const uint32_t ystage = ring + kFcStages * kFcStageBytes;    // y: [hi | lo] 64 rows, the layout of x in a ring stage
  const uint32_t sstage = ystage + kFcYBytes;                  // skip: 64 rows x 2 lines of 32 fp32, 128B-swizzled
  const uint32_t bars = sstage + kFcSkipBytes;
  const uint32_t full_bar = bars;                              // [stages]
  const uint32_t empty_bar = full_bar + 8 * kFcStages;         // [stages]
  const uint32_t w_bar = empty_bar + 8 * kFcStages;
  const uint32_t free_bar = w_bar + 8;                         // [warpgroup]: the staging area is free for it

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if constexpr (kMode == kFcLast) {
    // the tail weights take the skip staging area, which this layer does not use: 128B-swizzled K-major planes, as wgmma reads
    // them, written here and handed to the async proxy before the barrier below
    for (int i = threadIdx.x; i < 2 * 64 * 8; i += kThreads) {
      const int plane = i >> 9, n = (i >> 3) & 63, q = i & 7;
      const uint4 v = __ldg((plane ? ends.w1_lo : ends.w1_hi) + 8 * n + q);
      const uint32_t dst = sstage + plane * (kFcSkipBytes / 2) + n * kSwizzleBytes + ((q ^ (n & 7)) << 4);
      sts_u32(dst, v.x); sts_u32(dst + 4, v.y); sts_u32(dst + 8, v.z); sts_u32(dst + 12, v.w);
    }
    fence_proxy_async_shared();
  }
  if constexpr (kMode == kFcFirst) {
    // the first_conv vectors go to the W1 area, which this layer does not use: per column pair (c, c + 1) five 16-byte
    // entries (kFirstPair bytes) {u0, u1}, {u2, v0 + v1 + v2}, {v0, v1}, {v2, 0}, {w, b} - a broadcast load per fragment
    // column pair instead of lane-divergent parameter loads
    for (int c = threadIdx.x; c < 128; c += kThreads) {
      const uint32_t dst = w1 + kFirstPair * (c >> 1) + 4 * (c & 1);
      const float vs = ends.v[0][c] + ends.v[1][c] + ends.v[2][c];
      const float e[5][2] = {{ends.u[0][c], ends.u[1][c]}, {ends.u[2][c], vs}, {ends.v[0][c], ends.v[1][c]}, {ends.v[2][c], 0.f},
                             {c < 64 ? ends.w[c] : 0.f, c < 64 ? ends.b[c] : 0.f}};
#pragma unroll
      for (int k = 0; k < 5; ++k) { sts_u32(dst + 16 * k, __float_as_uint(e[k][0])); sts_u32(dst + 16 * k + 8, __float_as_uint(e[k][1])); }
    }
  }
  if (threadIdx.x == kConsumerThreads) {
    if constexpr (kMode != kFcFirst) tma_prefetch_desc(&tm_x);
    tma_prefetch_desc(&tm_u); tma_prefetch_desc(&tm_p);
    if constexpr (kMode != kFcFirst) { tma_prefetch_desc(&tm_w1_hi); tma_prefetch_desc(&tm_w1_lo); }
    tma_prefetch_desc(&tm_w2_hi); tma_prefetch_desc(&tm_w2_lo);
    tma_prefetch_desc(&tm_y); tma_prefetch_desc(&tm_skip);
    // a stage is read by one consumer warpgroup: one arrival per warp
    for (int s = 0; s < kFcStages; ++s) { mbar_init_a(full_bar + 8 * s, 1); mbar_init_a(empty_bar + 8 * s, 4); }
    mbar_init_a(w_bar, 1);
    mbar_init_a(free_bar, 1); mbar_init_a(free_bar + 8, 1);    // arrived on by the other warpgroup's store lane
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      // resident weights: all 128 output channels of the three tap chunks of W1 (not in the first layer) and of W2, both planes
      mbar_arrive_expect_tx_a(w_bar, (kMode == kFcFirst ? 0 : kFcW1Bytes) + kFcW2Bytes);
      if constexpr (kMode != kFcFirst) {
        for (int j = 0; j < 3; ++j) {
          tma_load_3d_a(w1 + j * 2 * kATile, &tm_w1_hi, w_bar, j * kChunkK, 0, 0);
          tma_load_3d_a(w1 + j * 2 * kATile + kATile, &tm_w1_lo, w_bar, j * kChunkK, 0, 0);
        }
      }
      tma_load_3d_a(w2, &tm_w2_hi, w_bar, 0, 0, 0);
      tma_load_3d_a(w2 + kATile, &tm_w2_lo, w_bar, 0, 0, 0);
      uint32_t it = 0;
      FcTileIter ti(p);
      int b, m0, half;
      while (ti.next(b, m0, half)) {
        const int mh = m0 + 128 * half;
        // band rows of this half tile: first 128 rows of an utterance, the half tiles touching its last 128 rows
        // (per-utterance block; 2 * 128 clamps halves lying wholly past the end onto the zero block), else interior
        const int len = p.lens ? min(__ldg(p.lens + b), p.t) : p.t;
        const int m1 = ((len - 128) >> 7) << 7;
        const int urow = mh == 0 ? p.u_start_row
                         : (mh + 128 > len - 128) ? p.u_end_base + 384 * b + min(mh - m1, 256)
                                                  : mh % p.u_period;
        // one K window per 256-sample window: it starts at the frame of the window's first row, aligned down to
        // 8 frames (16 B) - TMA faults on an unaligned innermost coordinate
        const int j0 = (m0 / p.hop - 2) & ~7;
        for (int wg = 0; wg < 2; ++wg) {                       // the 64-row tiles of consumer warpgroups 0 and 1
          for (int j = 0; j < Ch::kAll; ++j, ++it) {
            const int s = it % kFcStages;
            mbar_wait_a(empty_bar + 8 * s, ((it / kFcStages) & 1) ^ 1);
            const uint32_t st = ring + s * kFcStageBytes;
            const uint32_t fb = full_bar + 8 * s;
            // chunk order: [skip sum,] tap -d, tap +d, conditioning, centre tap (it also supplies the residual x) (FcChunks)
            if (kMode == kFcLast && j == 0) {
              // the tile's fp32 skip sum, in the layout the middle layers' epilogue stages it in (rows past t read as zero)
              mbar_arrive_expect_tx_a(fb, kFcSkipBytes);
              tma_load_3d_a(st, &tm_skip, fb, 0, 2 * (mh + 64 * wg), b);
            } else if (j - Ch::kG1Base == Ch::kCond) {
              // conditioning as U (W_aux m'): A = the tile's 64 band-table rows (K window = columns 0..15), B = the same 16
              // frames of P for the 128 output channels; frames outside the utterance are out of bounds of the tensor map
              // and read as zero
              mbar_arrive_expect_tx_a(fb, kFcUBytes + kFcPBytes);
              tma_load_4d_a(st, &tm_u, fb, 0, urow + 64 * wg, 0, 0);
              tma_load_4d_a(st + kFcUBytes, &tm_p, fb, j0, p.p_row0, b, 0);
            } else if constexpr (kMode != kFcFirst) {
              mbar_arrive_expect_tx_a(fb, kFcStageBytes);
              const int jg = j - Ch::kG1Base;
              const int wj = jg == 0 ? 0 : jg == 1 ? 2 : 1;
              tma_load_4d_a(st, &tm_x, fb, 0, mh + 64 * wg + (wj - 1) * p.dil, b, 0);
            }
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers: one 64-row tile per warpgroup ------------------------------
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int rl = 16 * (warp & 3) + (lane >> 2);              // this thread's rows: rl and rl + 8 of the warpgroup's 64
    const int cq = 2 * (lane & 3);                             // and columns 8 j + cq, + 1
    const float kSqrtHalf = 0.70710678118654752440f;
    mbar_wait_a(w_bar, 0);
    uint32_t it = wg * Ch::kAll;                               // ring position of this warpgroup's first chunk
    FcTileIter ti(p);
    int b, m0, half;
    bool more = ti.next(b, m0, half);
    bool first = true;
    // Both warpgroups take one 64-row tile of every half tile, and their epilogues alternate (0, 1, 0, 1, ...): warpgroup 1's
    // k-th epilogue waits for the k-th release by warpgroup 0, warpgroup 0's k-th for the (k - 1)-th release by warpgroup 1
    // (its first passes on the fresh barrier's parity).  A warpgroup cannot get two releases ahead of the other's waits, so a
    // parity bit per warpgroup is enough.
    uint32_t free_phase = wg ^ 1;
    while (more) {
      const int mh = m0 + 128 * half;
      float acc1[64], acc2[64];
      if constexpr (kMode == kFcFirst) {
        // GEMM1's taps as fp32 FMAs on the noise (file comment), and GEMM2's accumulator at [0 | x0], x0 zero past len;
        // done before the ordering barrier, while the other warpgroup's GEMM1 has the tensor cores
        const int len = p.lens ? min(__ldg(p.lens + b), p.t) : p.t;
        const float* noise = ends.noise + static_cast<size_t>(b) * p.t;
        float nv[3][2], mv[3][2];                              // noise at t' of each tap and row, and valid(t')
#pragma unroll
        for (int tap = 0; tap < 3; ++tap) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int t = mh + 64 * wg + rl + 8 * hh + (tap - 1) * p.dil;
            const bool valid = t >= 0 && t < len;
            nv[tap][hh] = valid ? __ldg(noise + t) : 0.f;
            mv[tap][hh] = valid ? 1.f : 0.f;
          }
        }
        // a warp whose rows see all three taps inside the utterance (all but the edge tiles) adds the summed v directly
        const bool inner = __all_sync(0xffffffffu, mv[0][0] * mv[0][1] * mv[2][0] * mv[2][1] != 0.f);
        if (inner) {
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const uint32_t e = w1 + kFirstPair * (4 * jj + (cq >> 1));
            const float4 u01 = lds_f4(e), u2s = lds_f4(e + 16);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int hh = q >> 1, o = q & 1;
              acc1[4 * jj + q] = fmaf(nv[0][hh], o ? u01.y : u01.x, fmaf(nv[1][hh], o ? u01.w : u01.z,
                                      fmaf(nv[2][hh], o ? u2s.y : u2s.x, o ? u2s.w : u2s.z)));
            }
          }
        } else {
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const uint32_t e = w1 + kFirstPair * (4 * jj + (cq >> 1));
            const float4 u01 = lds_f4(e), u2s = lds_f4(e + 16), v01 = lds_f4(e + 32), v2 = lds_f4(e + 48);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const int hh = q >> 1, o = q & 1;
              float a = mv[0][hh] * (o ? v01.y : v01.x);
              a = fmaf(nv[0][hh], o ? u01.y : u01.x, a);
              a = fmaf(mv[1][hh], o ? v01.w : v01.z, a);
              a = fmaf(nv[1][hh], o ? u01.w : u01.z, a);
              a = fmaf(mv[2][hh], o ? v2.y : v2.x, a);
              acc1[4 * jj + q] = fmaf(nv[2][hh], o ? u2s.y : u2s.x, a);
            }
          }
        }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const float4 wb = lds_f4(w1 + kFirstPair * (4 * jj + (cq >> 1)) + 64);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int hh = q >> 1, o = q & 1;
            acc2[4 * jj + q] = 0.f;
            acc2[32 + 4 * jj + q] = mv[1][hh] != 0.f ? fmaf(o ? wb.y : wb.x, nv[1][hh], o ? wb.w : wb.z) : 0.f;
          }
        }
      }
      // ordering barrier: the warpgroups take turns at GEMM1 (warpgroup 0 first), so that one of them gates and stores while
      // the other's GEMM1 has the tensor cores
      if (wg == 1 || !first) named_bar_sync(1 + wg, kConsumerThreads);
      first = false;
      if constexpr (kMode == kFcLast) {
        // GEMM2's skip half starts at the tile's running skip sum plus the sum of the skip biases; the stage goes straight
        // back to the producer.  Not before the ordering barrier: only behind it is every earlier use of the stage complete,
        // so that the parity wait cannot pass on the phase before
        mbar_wait_a(full_bar + 8 * (it % kFcStages), (it / kFcStages) & 1);
        const uint32_t st = ring + (it % kFcStages) * kFcStageBytes;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int c = 8 * jj + cq, line = 2 * (rl + 8 * hh) + (c >> 5);
            const float2 v = lds_f2(st + line * 128 + ((((c & 31) >> 2) ^ (line & 7)) << 4) + (c & 3) * 4);
            acc2[4 * jj + 2 * hh] = v.x + ends.skip_b[c];
            acc2[4 * jj + 2 * hh + 1] = v.y + ends.skip_b[c + 1];
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive_a(empty_bar + 8 * (it % kFcStages));
      }
      // fully unrolled: the chunk kind is a compile-time case, so the wgmma chains of consecutive chunks stay asynchronous
      // (one commit group in flight; the stage of chunk j - 1 goes back to the producer once chunk j has been issued)
#pragma unroll
      for (int j = 0; j < Ch::kG1; ++j) {
        const int s = (it + Ch::kG1Base + j) % kFcStages;
        mbar_wait_a(full_bar + 8 * s, ((it + Ch::kG1Base + j) / kFcStages) & 1);
        const uint32_t st = ring + s * kFcStageBytes;
        wgmma_fence();
        if (j == Ch::kCond) {                                  // one K-step: 16 frames of band table x P window
          const uint64_t a_hi = make_smem_desc_sw32(st), a_lo = make_smem_desc_sw32(st + kFcUBytes / 2);
          const uint64_t b_hi = make_smem_desc_sw32(st + kFcUBytes), b_lo = make_smem_desc_sw32(st + kFcUBytes + kFcPBytes / 2);
          wgmma_ss_n128(acc1, a_hi, b_hi, 1);
          wgmma_ss_n128(acc1, a_lo, b_hi, 1);
          wgmma_ss_n128(acc1, a_hi, b_lo, 1);
        } else if constexpr (kMode != kFcFirst) {
          const int wj = j == 0 ? 0 : j == 1 ? 2 : 1;
          const uint64_t a_hi = make_smem_desc_sw128(st), a_lo = make_smem_desc_sw128(st + kQTile);
          const uint64_t b_hi = make_smem_desc_sw128(w1 + wj * 2 * kATile), b_lo = make_smem_desc_sw128(w1 + wj * 2 * kATile + kATile);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            wgmma_ss_n128(acc1, a_hi + desc_kstep(k), b_hi + desc_kstep(k), !(j == 0 && k == 0));
            wgmma_ss_n128(acc1, a_lo + desc_kstep(k), b_hi + desc_kstep(k), 1);
            wgmma_ss_n128(acc1, a_hi + desc_kstep(k), b_lo + desc_kstep(k), 1);
          }
        }
        wgmma_commit();
        if (kMode != kFcFirst && j == Ch::kG1 - 1) {
          // GEMM2's accumulator starts as [0 | x]: x = hi + lo of this tile's own rows, from the centre-tap chunk
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const int r = rl + 8 * hh;
              const uint32_t off = r * kSwizzleBytes + ((((8 * jj + cq) >> 3) ^ (r & 7)) << 4) + (cq & 7) * 2;
              const uint32_t xh = lds_u32(st + off), xl = lds_u32(st + kQTile + off);
              if constexpr (kMode != kFcLast) {
                acc2[4 * jj + 2 * hh] = 0.f;
                acc2[4 * jj + 2 * hh + 1] = 0.f;
              }
              acc2[32 + 4 * jj + 2 * hh] = __uint_as_float(xh << 16) + __uint_as_float(xl << 16);
              acc2[32 + 4 * jj + 2 * hh + 1] = __uint_as_float(xh & 0xffff0000u) + __uint_as_float(xl & 0xffff0000u);
            }
          }
        }
        if (j > 0) {
          wgmma_wait<1>();
          __syncwarp();
          if (lane == 0) mbar_arrive_a(empty_bar + 8 * ((it + Ch::kG1Base + j - 1) % kFcStages));
        }
      }
      wgmma_wait<0>();
      reg_fence(acc1);
      // the centre-tap stage has been read by its wgmmas and for [0 | x]: back to the producer
      __syncwarp();
      if (lane == 0) mbar_arrive_a(empty_bar + 8 * ((it + Ch::kAll - 1) % kFcStages));
      it += 2 * Ch::kAll;                                      // the other warpgroup's tile sits in between
      // hand GEMM1 to the other warpgroup (warpgroup 1 skips this after its last tile: warpgroup 0 waits for no more turns)
      int nb, nm0, nhalf;
      const bool next = ti.next(nb, nm0, nhalf);
      if (wg == 0 || next) named_bar_arrive(2 - wg, kConsumerThreads);
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
      const uint64_t b2_hi = make_smem_desc_sw128(w2), b2_lo = make_smem_desc_sw128(w2 + kATile);
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
      if constexpr (kMode == kFcLast) {
        // the tail on the scaled skip sum s = relu(acc2's skip half * scale): h = tail W1 s (split-bf16, K = 64 = 4 K-steps,
        // A from registers as z in GEMM2), then out = w2 . relu(h + b1) + b2, the dot product reduced over the quad of lanes
        // that holds a row; rows past len get zero (the tiles wholly past it are not visited at all)
        uint32_t sh[16], sl[16];
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            split2(fmaxf(acc2[4 * jj + 2 * hh] * ends.scale, 0.f), fmaxf(acc2[4 * jj + 2 * hh + 1] * ends.scale, 0.f),
                   sh[2 * jj + hh], sl[2 * jj + hh]);
          }
        }
        float h[32];
        const uint64_t bt_hi = make_smem_desc_sw128(sstage), bt_lo = make_smem_desc_sw128(sstage + kFcSkipBytes / 2);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint32_t ah[4] = {sh[4 * k], sh[4 * k + 1], sh[4 * k + 2], sh[4 * k + 3]};
          const uint32_t al[4] = {sl[4 * k], sl[4 * k + 1], sl[4 * k + 2], sl[4 * k + 3]};
          wgmma_rs_n64(h, ah, bt_hi + desc_kstep(k), k > 0);
          wgmma_rs_n64(h, al, bt_hi + desc_kstep(k), 1);
          wgmma_rs_n64(h, ah, bt_lo + desc_kstep(k), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(h);
        float o[2] = {0.f, 0.f};
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int c = 8 * jj + cq + (q & 1);
            o[q >> 1] = fmaf(fmaxf(h[4 * jj + q] + ends.b1[c], 0.f), ends.w2[c], o[q >> 1]);
          }
        }
        const int len = p.lens ? min(__ldg(p.lens + b), p.t) : p.t;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          o[hh] += __shfl_xor_sync(0xffffffffu, o[hh], 1);
          o[hh] += __shfl_xor_sync(0xffffffffu, o[hh], 2);
          const int t = mh + wg * 64 + rl + 8 * hh;
          if ((lane & 3) == 0 && t < p.t) ends.out[static_cast<size_t>(b) * p.t + t] = t < len ? o[hh] + ends.b2 : 0.f;
        }
      }
      // stores: out half -> (out + b_out) * sqrt(1/2) as split planes into the y staging tile, skip half -> the fp32 skip
      // staging tile (not in the last layer); then one TMA store of y and one TMA reduce-add (store at skip_init) of the skip
      // tile.  Rows past t lie outside both tensor maps and are not written; rows in [len, t) get a zero y and their skip
      // contribution.
      mbar_wait_a(free_bar + 8 * wg, free_phase);
      free_phase ^= 1;
      const int len = p.lens ? min(__ldg(p.lens + b), p.t) : p.t;
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int r = rl + 8 * hh;
        const bool live = mh + wg * 64 + r < len;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int c = 8 * jj + cq;
          const float y0 = live ? (acc2[32 + 4 * jj + 2 * hh] + p.out_b[c]) * kSqrtHalf : 0.f;
          const float y1 = live ? (acc2[32 + 4 * jj + 2 * hh + 1] + p.out_b[c + 1]) * kSqrtHalf : 0.f;
          uint32_t oh, ol;
          split2(y0, y1, oh, ol);
          const uint32_t off = r * kSwizzleBytes + (((c >> 3) ^ (r & 7)) << 4) + (cq & 7) * 2;   // where x was read
          sts_u32(ystage + off, oh);
          sts_u32(ystage + kQTile + off, ol);
          // skip row r = 128-byte lines 2 r (channels 0..31) and 2 r + 1; the 16-byte chunk XOR (line & 7) keeps each
          // half warp's 8-byte writes on 32 distinct banks
          if constexpr (kMode != kFcLast) {
            const int line = 2 * r + (c >> 5);
            sts_f2(sstage + line * 128 + ((((c & 31) >> 2) ^ (line & 7)) << 4) + (c & 3) * 4, acc2[4 * jj + 2 * hh],
                   acc2[4 * jj + 2 * hh + 1]);
          }
        }
      }
      fence_proxy_async_shared();
      named_bar_sync(3 + wg, 128);
      if ((threadIdx.x & 127) == 0) {
        tma_store_4d_a(&tm_y, ystage, 0, mh + wg * 64, b, 0);
        if constexpr (kMode != kFcLast) {
          if (p.skip_init) tma_store_3d_a(&tm_skip, sstage, 0, 2 * (mh + wg * 64), b);
          else tma_reduce_add_3d_a(&tm_skip, sstage, 0, 2 * (mh + wg * 64), b);
        }
        bulk_commit();
        bulk_wait_read<0>();                                   // the staging tiles have been read
        mbar_arrive_a(free_bar + 8 * (wg ^ 1));
      }
      b = nb; m0 = nm0; half = nhalf; more = next;
    }
  }
}

template <int M>
int launch_layer(const CUtensorMap (&tm)[9], const FcLayerArgs& p, const FcEnds<M>& ends, int batch, int t, cudaStream_t st) {
  int resident = 0;
  if (int rc = prepare_kernel(pwg_layer_fc_kernel<M>, kThreads, kFcSmem, &resident)) return rc;
  const int tiles = ((t + 255) / 256) * 2 * batch;
  const int grid = std::min(tiles, resident);
  pwg_layer_fc_kernel<M><<<grid, kThreads, kFcSmem, st>>>(tm[0], tm[1], tm[2], tm[3], tm[4], tm[5], tm[6], tm[7], tm[8], p, ends);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

}  // namespace fc
}  // namespace pk

extern "C" int pk_pwg_residual_layer_fc(const pk_pwg_layer_fc_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::fc;
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  PK_CHECK_ARG(a->batch > 0 && a->t > 0 && a->dilation >= 1 && a->hop >= 256, "bad batch/t/dilation/hop (hop must be >= 256)");
  const bool first = a->noise != nullptr, last = a->out != nullptr;
  PK_CHECK_ARG(!(first && last), "noise (first layer) and out (last layer) are exclusive");
  PK_CHECK_ARG(!first || (a->x_hi == nullptr && a->x_lo == nullptr), "the first layer reads no x planes: x_hi / x_lo must be NULL");
  PK_CHECK_ARG(first || (a->x_hi && a->x_lo), "NULL x planes");
  PK_CHECK_ARG(a->y_hi && a->y_lo && a->u_hi && a->u_lo && a->p_hi && a->p_lo && a->w1_hi && a->w1_lo &&
               a->w2_hi && a->w2_lo && a->bias1 && a->bias2 && a->skip, "NULL pointer in pk_pwg_layer_fc_args");
  PK_CHECK_ARG(!first || (a->first_w && a->first_b && a->first_u && a->first_v), "NULL first_conv vector");
  PK_CHECK_ARG(!last || (a->tail_w1_hi && a->tail_w1_lo && a->tail_b1 && a->tail_w2 && a->tail_b2 && a->skip_bias),
               "NULL tail operand");
  PK_CHECK_ARG(!last || a->skip_init == 0, "the last layer reads the running skip sum: skip_init must be 0");
  PK_CHECK_ARG(!last || (aligned16(a->tail_w1_hi) && aligned16(a->tail_w1_lo)), "tail weight planes must be 16-byte aligned");
  PK_CHECK_ARG(first || a->x_hi != a->y_hi, "layer output must not alias its input");
  PK_CHECK_ARG(a->u_period > 0 && (a->u_period % 128) == 0 && a->u_start_row >= a->u_period && a->u_end_base >= a->u_start_row + 128 &&
               a->u_rows >= a->u_end_base + 384 * a->batch, "bad compact band table layout");
  PK_CHECK_ARG(a->p_rows > 0 && a->p_row0 >= 0 && a->p_row0 + 128 <= a->p_rows && (a->p_ld % 8) == 0 && a->p_ld >= 64 && a->p_frames > 0 &&
               a->p_frames <= a->p_ld, "bad P plane geometry");
  // x, u, p, w1 hi / lo, w2 hi / lo, y, skip (the first layer's x map is never read and stays zero)
  CUtensorMap tm[9];
  memset(tm, 0, sizeof(tm));
  int rc;
  const uint64_t T = a->t, B = a->batch;
  if (!first && (rc = encode_tmap_bf16_planes(&tm[0], a->x_hi, a->x_lo, kPwgR, T, B, kPwgR, T * kPwgR, 64))) return rc;
  if ((rc = encode_tmap_bf16_planes(&tm[7], a->y_hi, a->y_lo, kPwgR, T, B, kPwgR, T * kPwgR, 64))) return rc;
  // skip sum (B, T, 64) fp32: each 256-byte row is two 128-byte lines, a 64-row tile one box of 128 lines
  if ((rc = encode_tmap_f32_3d(&tm[8], a->skip, 2 * T, B, 0, 128))) return rc;
  // compact band table planes (u_rows, 64): the K window sits in columns 0..15, a 16-column box of 64 rows
  if ((rc = encode_tmap_bf16_planes(&tm[1], a->u_hi, a->u_lo, 64, a->u_rows, 1, 64, 0, 64, 16))) return rc;
  // P planes (batch, p_rows, p_ld): frames are the K axis; columns >= p_frames (and < 0) read as zero
  const uint64_t prow = a->p_rows, pld = a->p_ld;
  // (the extent is the padded row length p_ld >= 64: columns [p_frames, p_ld) hold zeros in memory, frames < 0 are out of bounds)
  // (16-frame box of the 128 output channels of the layer)
  if ((rc = encode_tmap_bf16_planes(&tm[2], a->p_hi, a->p_lo, pld, prow, B, pld, prow * pld, 128, 16))) return rc;
  const uint64_t k1 = 5 * kChunkK;     // row pitch of the packed W1 (pk_pwg_residual_layer layout); only the 3 tap chunks are read
  if ((rc = encode_tmap_bf16_3d(&tm[3], a->w1_hi, 3 * kChunkK, kPwgG, 1, k1, k1 * kPwgG, 128))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tm[4], a->w1_lo, 3 * kChunkK, kPwgG, 1, k1, k1 * kPwgG, 128))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tm[5], a->w2_hi, 64, 128, 1, 64, 0, 128))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tm[6], a->w2_lo, 64, 128, 1, 64, 0, 128))) return rc;
  FcLayerArgs p;
  p.batch = a->batch; p.t = a->t; p.dil = a->dilation; p.hop = a->hop;
  p.u_period = a->u_period; p.u_start_row = a->u_start_row; p.u_end_base = a->u_end_base;
  p.p_row0 = a->p_row0;
  p.lens = a->lens; p.skip = a->skip; p.skip_init = a->skip_init;
  p.k_a = kGateKa; p.k_g = kGateKg;
  fold_gate_bias(p.gate_c, a->bias1, 64);
  for (int i = 0; i < 64; ++i) p.out_b[i] = a->bias2[64 + i];
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (first) {
    FcEnds<kFcFirst> e;
    e.noise = a->noise;
    memcpy(e.w, a->first_w, sizeof(e.w));
    memcpy(e.b, a->first_b, sizeof(e.b));
    memcpy(e.u, a->first_u, sizeof(e.u));
    memcpy(e.v, a->first_v, sizeof(e.v));
    return launch_layer(tm, p, e, a->batch, a->t, st);
  }
  if (last) {
    FcEnds<kFcLast> e;
    e.w1_hi = static_cast<const uint4*>(a->tail_w1_hi);
    e.w1_lo = static_cast<const uint4*>(a->tail_w1_lo);
    e.out = a->out;
    memcpy(e.skip_b, a->skip_bias, sizeof(e.skip_b));
    memcpy(e.b1, a->tail_b1, sizeof(e.b1));
    memcpy(e.w2, a->tail_w2, sizeof(e.w2));
    e.b2 = a->tail_b2[0];
    e.scale = a->tail_scale;
    return launch_layer(tm, p, e, a->batch, a->t, st);
  }
  return launch_layer(tm, p, FcEnds<kFcMiddle>{}, a->batch, a->t, st);
}
