// pk_conv_gemm: channels-last Conv1D / Linear / batched matmul as an im2col-free tiled GEMM on wgmma.
//
//   - persistent CTAs (one per SM) walking 128(time) x BLOCK_N(channel) output tiles; 384 threads:
//       warps 0-7: two consumer warpgroups, each accumulating 64 rows x BLOCK_N in registers (wgmma) and then running the
//                  epilogue (registers -> shared-memory staging -> bias/act/residual/mask -> global), one output row per thread
//       warps 8-11: producer warpgroup: one TMA lane running ahead of the consumers through a ring of shared-memory stages;
//                  it drops to 40 registers so that the consumers can hold a 64 x 256 fp32 accumulator (232 registers)
//   - K loop over (tap, 64-channel chunk): each conv tap is just the same A tensor read `(tap - pad) * dil` rows
//     further along; TMA zero-fills rows outside the utterance, which is the conv's zero padding (no im2col).
//   - split-bf16 operands, 3 wgmma per K-step (hi*hi + lo*hi + hi*lo), fp32 accumulation.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {

constexpr int kBlockM = 128;
constexpr int kConsumerThreads = 256;                            // two warpgroups of 64 rows each
constexpr int kGemmThreads = kConsumerThreads + 128;             // + the producer warpgroup (one TMA lane; registers handed over)

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int kABytes = kBlockM * kSwizzleBytes;       // one plane of one A chunk (16 KB)
  static constexpr int kBBytes = BLOCK_N * kSwizzleBytes;       // one plane of one B chunk
  static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;  // hi + lo
  static constexpr int kStages = (BLOCK_N >= 256) ? 2 : (BLOCK_N >= 128 ? 3 : 4);
  static constexpr int kStagingBytes = 2 * 2 * kStageSlotBytes;  // two epilogue slots per warpgroup
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
};

struct GemmKernelArgs {
  int m, n, k_chunks, taps, dil, pad, heads, batch;
  int tiles_m, total_tiles;       // persistent schedule (set by launch<>)
  int a_bmul, a_hmul, a_col0, a_colh;
  int b_bmul, b_hmul, b_col0, b_colh, b_tap_stride;
  float scale;
  const float* bias;
  int act;
  const float* residual;
  const int32_t* lens;
  float* y_f32;
  __nv_bfloat16* y_hi;
  __nv_bfloat16* y_lo;
  long long y_batch_stride, y_head_stride;
  int y_ld;
  int passes;
  // fused pair epilogues (pk_conv_gemm_ex): the tile covers n = 2 * epi_c columns, column c is paired with column epi_c + c
  int epi, epi_c;
  const float* e_res;            // GATE: fp32 (batch, m, e_res_ld) added before the gate, or NULL
  long long e_res_bs;
  int e_res_ld;
  float* e_state;                // WF_UPDATE: fp32 (batch, m, epi_c) running state / skip sum
  float* e_skip;
  int e_skip_init;
  __nv_bfloat16* e_buf_hi;       // WF_UPDATE: optional split planes (batch, m, e_buf_ld) receiving the new state at e_buf_col0
  __nv_bfloat16* e_buf_lo;
  int e_buf_ld, e_buf_col0;
};

// bias / activation / residual / row mask / stores for one 32-column chunk of one output row (v: the accumulators)
__device__ __forceinline__ void gemm_epilogue_chunk(const GemmKernelArgs& p, float (&v)[32], const int nb, const bool row_ok,
                                                    const bool row_live, const long long y_off) {
  if (row_ok && nb < p.n) {
    // bias: one batch of independent loads per 32-column chunk (a dependent load per element would serialise the
    // epilogue on global-memory latency), activation selected outside the element loops
    float bv[32];
    if (p.bias == nullptr) {
#pragma unroll
      for (int j = 0; j < 32; ++j) bv[j] = 0.f;
    } else if (nb + 32 <= p.n && (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0) {
      const float4* b4 = reinterpret_cast<const float4*>(p.bias + nb);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 b = __ldg(b4 + j);
        bv[4 * j] = b.x; bv[4 * j + 1] = b.y; bv[4 * j + 2] = b.z; bv[4 * j + 3] = b.w;
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) bv[j] = nb + j < p.n ? __ldg(p.bias + nb + j) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] = fmaf(v[j], p.scale, bv[j]);
    if (p.act == PK_ACT_RELU) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
    } else if (p.act == PK_ACT_TANH) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = tanhf(v[j]);
    }
    const bool full = (nb + 32 <= p.n) && ((p.y_ld & 7) == 0) && (((y_off + nb) & 7) == 0);
    if (p.residual != nullptr) {
      if (full) {
        const float4* r4 = reinterpret_cast<const float4*>(p.residual + y_off + nb);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float4 r = __ldg(r4 + j);
          v[4 * j + 0] += r.x; v[4 * j + 1] += r.y; v[4 * j + 2] += r.z; v[4 * j + 3] += r.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (nb + j < p.n) v[j] += __ldg(p.residual + y_off + nb + j);
      }
    }
    if (!row_live) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = 0.f;
    }
    if (full) {
      if (p.y_f32 != nullptr) {
        float4* o4 = reinterpret_cast<float4*>(p.y_f32 + y_off + nb);
#pragma unroll
        for (int j = 0; j < 8; ++j) o4[j] = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
      }
      if (p.y_hi != nullptr) {
        uint4* oh = reinterpret_cast<uint4*>(p.y_hi + y_off + nb);
        uint4* ol = reinterpret_cast<uint4*>(p.y_lo + y_off + nb);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          uint4 h, l;
          split8(v + 8 * j, h, l);
          oh[j] = h;
          ol[j] = l;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (nb + j < p.n) {
          if (p.y_f32 != nullptr) p.y_f32[y_off + nb + j] = v[j];
          if (p.y_hi != nullptr) {
            __nv_bfloat16 h, l;
            split_bf16(v[j], h, l);
            p.y_hi[y_off + nb + j] = h;
            p.y_lo[y_off + nb + j] = l;
          }
        }
      }
    }
  }
}

// Fused pair epilogues: one 32-column chunk of the first half (va: columns [nb, nb+32) of [0, C)) together with the
// matching chunk of the second half (vg: columns C + [nb, nb+32)); bias / scale applied to both.
//   PK_EPI_GATE      z = tanh(a + res_a) * sigmoid(g + res_g) -> split planes (batch, m, y_ld) at column nb
//                    (ResidualBlock gate of waveflow.py:277-281 fused into the dilated-conv GEMM)
//   PK_EPI_WF_UPDATE state += a; skip (=|+=) g; new state -> optional split planes
//                    (waveflow.py:282-294 `res, skip = split(out_proj(z))`, ResidualNet.add_input :386-392)
__device__ __forceinline__ void gemm_epilogue_pair(const GemmKernelArgs& p, float (&va)[32], float (&vg)[32], const int nb,
                                                   const int bz, const int row, const bool row_ok) {
  if (!row_ok) return;
  const int C = p.epi_c;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float4 ba = make_float4(0.f, 0.f, 0.f, 0.f), bg = ba;
    if (p.bias != nullptr) {
      ba = __ldg(reinterpret_cast<const float4*>(p.bias + nb) + j);
      bg = __ldg(reinterpret_cast<const float4*>(p.bias + C + nb) + j);
    }
    va[4 * j] = fmaf(va[4 * j], p.scale, ba.x); va[4 * j + 1] = fmaf(va[4 * j + 1], p.scale, ba.y);
    va[4 * j + 2] = fmaf(va[4 * j + 2], p.scale, ba.z); va[4 * j + 3] = fmaf(va[4 * j + 3], p.scale, ba.w);
    vg[4 * j] = fmaf(vg[4 * j], p.scale, bg.x); vg[4 * j + 1] = fmaf(vg[4 * j + 1], p.scale, bg.y);
    vg[4 * j + 2] = fmaf(vg[4 * j + 2], p.scale, bg.z); vg[4 * j + 3] = fmaf(vg[4 * j + 3], p.scale, bg.w);
  }
  const long long grow = static_cast<long long>(bz) * p.m + row;       // row index in (batch, m, .) tensors
  if (p.epi == PK_EPI_GATE) {
    if (p.e_res != nullptr) {
      const float4* ra = reinterpret_cast<const float4*>(p.e_res + bz * p.e_res_bs + static_cast<long long>(row) * p.e_res_ld + nb);
      const float4* rg = reinterpret_cast<const float4*>(p.e_res + bz * p.e_res_bs + static_cast<long long>(row) * p.e_res_ld + C + nb);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 x = __ldg(ra + j), y = __ldg(rg + j);
        va[4 * j] += x.x; va[4 * j + 1] += x.y; va[4 * j + 2] += x.z; va[4 * j + 3] += x.w;
        vg[4 * j] += y.x; vg[4 * j + 1] += y.y; vg[4 * j + 2] += y.z; vg[4 * j + 3] += y.w;
      }
    }
#pragma unroll
    for (int j = 0; j < 32; ++j) va[j] = tanhf(va[j]) * (1.f / (1.f + expf(-vg[j])));
    uint4* oh = reinterpret_cast<uint4*>(p.y_hi + grow * p.y_ld + nb);
    uint4* ol = reinterpret_cast<uint4*>(p.y_lo + grow * p.y_ld + nb);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      uint4 h, l;
      split8(va + 8 * j, h, l);
      oh[j] = h;
      ol[j] = l;
    }
  } else {   // PK_EPI_WF_UPDATE
    float4* st4 = reinterpret_cast<float4*>(p.e_state + grow * C + nb);
    float4* sk4 = reinterpret_cast<float4*>(p.e_skip + grow * C + nb);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 s = st4[j];
      va[4 * j] += s.x; va[4 * j + 1] += s.y; va[4 * j + 2] += s.z; va[4 * j + 3] += s.w;
      st4[j] = make_float4(va[4 * j], va[4 * j + 1], va[4 * j + 2], va[4 * j + 3]);
      float4 k = make_float4(vg[4 * j], vg[4 * j + 1], vg[4 * j + 2], vg[4 * j + 3]);
      if (!p.e_skip_init) {
        const float4 o = sk4[j];
        k.x += o.x; k.y += o.y; k.z += o.z; k.w += o.w;
      }
      sk4[j] = k;
    }
    if (p.e_buf_hi != nullptr) {
      uint4* oh = reinterpret_cast<uint4*>(p.e_buf_hi + grow * p.e_buf_ld + p.e_buf_col0 + nb);
      uint4* ol = reinterpret_cast<uint4*>(p.e_buf_lo + grow * p.e_buf_ld + p.e_buf_col0 + nb);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        uint4 h, l;
        split8(va + 8 * j, h, l);
        oh[j] = h;
        ol[j] = l;
      }
    }
  }
}

struct GemmTile {     // persistent tile schedule: (batch, head) fastest, then m-tile, then n-tile, so that the CTAs running
  int m0, n0, bz, hz; // at the same time share one n-tile of B (the weights stay hot in L2) AND the dead tiles of a ragged
};                    // batch (all utterances' m-tile k for large k) are consecutive indices, i.e. spread evenly over the
                      // grid-strided CTAs (with m fastest and 132 % tiles_m == 0 some CTAs would own only dead tiles)
__device__ __forceinline__ GemmTile gemm_tile(int tile, int tiles_m, int zdim, int heads, int block_n) {
  GemmTile t;
  const int z = tile % zdim;
  const int r = tile / zdim;
  const int mt = r % tiles_m;
  t.m0 = mt * kBlockM;
  t.n0 = (r / tiles_m) * block_n;
  t.bz = z / heads;
  t.hz = z % heads;
  return t;
}

// Ragged batches (`lens`): an m-tile that starts at or past its utterance's length holds no live row.  Every role skips it
// with the same test - no loads, no MMAs, no accumulator hand-over - and the epilogue warps just write its zero rows (the rows
// are the utterance's own zero padding for the next conv).  On LJSpeech-shaped batches (T ~ U{60..140}, padded to the longest)
// a third of the m-tiles are dead.
__device__ __forceinline__ bool gemm_tile_live(const GemmKernelArgs& p, int m0, int bz) {
  return p.lens == nullptr || m0 < __ldg(p.lens + bz);
}

template <int BLOCK_N>
__device__ __forceinline__ void wgmma_ss(float (&d)[BLOCK_N / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (BLOCK_N == 64) wgmma_ss_n64(d, a, b, acc);
  else if constexpr (BLOCK_N == 128) wgmma_ss_n128(d, a, b, acc);
  else wgmma_ss_n256(d, a, b, acc);
}

template <int BLOCK_N>
__global__ void __launch_bounds__(kGemmThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                 const __grid_constant__ CUtensorMap tm_b_hi, const __grid_constant__ CUtensorMap tm_b_lo,
                 const GemmKernelArgs p) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int kChunks = BLOCK_N / 32;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;     // 1024-B alignment for SWIZZLE_128B tiles
  const uint32_t staging = smem + Cfg::kStages * Cfg::kStageBytes;
  const uint32_t full_bar = staging + Cfg::kStagingBytes;         // [stages] TMA bytes landed
  const uint32_t empty_bar = full_bar + 8 * Cfg::kStages;         // [stages] both warpgroups have read the stage

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_chunks = p.taps * p.k_chunks;
  const int zdim = p.batch * p.heads;

  if (threadIdx.x == kConsumerThreads) {
    tma_prefetch_desc(&tm_a_hi);
    tma_prefetch_desc(&tm_a_lo);
    tma_prefetch_desc(&tm_b_hi);
    tma_prefetch_desc(&tm_b_lo);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init_a(full_bar + 8 * s, 1);
      mbar_init_a(empty_bar + 8 * s, kConsumerThreads / 32);       // one elected lane per consumer warp
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      // ------------------------------ TMA producer ------------------------------
      const uint32_t tx_bytes = (p.passes == 3) ? Cfg::kStageBytes : (Cfg::kABytes + Cfg::kBBytes);
      uint32_t it = 0;                                 // running stage counter across tiles
      for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        const GemmTile t = gemm_tile(tile, p.tiles_m, zdim, p.heads, BLOCK_N);
        if (!gemm_tile_live(p, t.m0, t.bz)) continue;
        const int a_batch = t.bz * p.a_bmul + t.hz * p.a_hmul;
        const int b_batch = t.bz * p.b_bmul + t.hz * p.b_hmul;
        const int a_col = p.a_col0 + t.hz * p.a_colh;
        const int b_col = p.b_col0 + t.hz * p.b_colh;
        for (int i = 0; i < num_chunks; ++i, ++it) {
          const int s = it % Cfg::kStages;
          const uint32_t ph = (it / Cfg::kStages) & 1;
          const int tap = i / p.k_chunks;
          const int kc = i % p.k_chunks;
          mbar_wait_a(empty_bar + 8 * s, ph ^ 1);
          const uint32_t st = smem + s * Cfg::kStageBytes;
          const uint32_t fb = full_bar + 8 * s;
          mbar_arrive_expect_tx_a(fb, tx_bytes);
          const int a_row = t.m0 + (tap - p.pad) * p.dil;
          const int bc = b_col + tap * p.b_tap_stride + kc * kChunkK;
          tma_load_3d_a(st, &tm_a_hi, fb, a_col + kc * kChunkK, a_row, a_batch);
          tma_load_3d_a(st + 2 * Cfg::kABytes, &tm_b_hi, fb, bc, t.n0, b_batch);
          if (p.passes == 3) {
            tma_load_3d_a(st + Cfg::kABytes, &tm_a_lo, fb, a_col + kc * kChunkK, a_row, a_batch);
            tma_load_3d_a(st + 2 * Cfg::kABytes + Cfg::kBBytes, &tm_b_lo, fb, bc, t.n0, b_batch);
          }
        }
      }
    }
  } else {
    // ------------------------------ consumers: wgmma main loop + epilogue ------------------------------
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;                        // rows [64 wg, 64 wg + 64) of the tile
    const int wt = threadIdx.x & 127;                // thread inside the warpgroup
    const int er = wt & 63;                          // epilogue: the row this thread owns ...
    const int eh = wt >> 6;                          // ... and which of the two staged chunks
    const uint32_t slots = staging + wg * 2 * kStageSlotBytes;
    uint32_t it = 0;
    float acc[BLOCK_N / 2];
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const GemmTile t = gemm_tile(tile, p.tiles_m, zdim, p.heads, BLOCK_N);
      const int row = t.m0 + wg * 64 + er;           // output time step
      const bool row_ok = row < p.m;
      const bool row_live = row_ok && (p.lens == nullptr || row < __ldg(p.lens + t.bz));
      const long long y_off = t.bz * p.y_batch_stride + t.hz * p.y_head_stride + static_cast<long long>(row) * p.y_ld;
      if (!gemm_tile_live(p, t.m0, t.bz)) {        // dead tile: zero rows, nothing to wait for
#pragma unroll 1
        for (int c = eh; c < kChunks; c += 2) {
          float v[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = 0.f;
          gemm_epilogue_chunk(p, v, t.n0 + c * 32, row_ok, false, y_off);
        }
        continue;
      }
      for (int i = 0; i < num_chunks; ++i, ++it) {
        const int s = it % Cfg::kStages;
        mbar_wait_a(full_bar + 8 * s, (it / Cfg::kStages) & 1);
        const uint32_t st = smem + s * Cfg::kStageBytes;
        const uint64_t a_hi = make_smem_desc_sw128(st + wg * 64 * kSwizzleBytes);
        const uint64_t a_lo = make_smem_desc_sw128(st + Cfg::kABytes + wg * 64 * kSwizzleBytes);
        const uint64_t b_hi = make_smem_desc_sw128(st + 2 * Cfg::kABytes);
        const uint64_t b_lo = make_smem_desc_sw128(st + 2 * Cfg::kABytes + Cfg::kBBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kChunkK / kWgmmaK; ++k) {
          wgmma_ss<BLOCK_N>(acc, a_hi + desc_kstep(k), b_hi + desc_kstep(k), (i | k) != 0);
          if (p.passes == 3) {
            wgmma_ss<BLOCK_N>(acc, a_lo + desc_kstep(k), b_hi + desc_kstep(k), 1);
            wgmma_ss<BLOCK_N>(acc, a_hi + desc_kstep(k), b_lo + desc_kstep(k), 1);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive_a(empty_bar + 8 * s);   // this warp is done reading the stage
      }
      if (p.epi == PK_EPI_NONE) {
#pragma unroll
        for (int c = 0; c < kChunks; c += 2) {
          stage_store(slots, acc, c, wt);
          if (c + 1 < kChunks) stage_store(slots + kStageSlotBytes, acc, c + 1, wt);
          named_bar_sync(1 + wg, 128);
          if (c + eh < kChunks) {
            float v[32];
            stage_load_row(slots + eh * kStageSlotBytes, er, v);
            gemm_epilogue_chunk(p, v, t.n0 + (c + eh) * 32, row_ok, row_live, y_off);
          }
          named_bar_sync(1 + wg, 128);
        }
      } else {
        // fused pair epilogues: the tile holds columns [0, 2C); chunk c of the first half with chunk c of the second half
        const int hc = p.epi_c / 32;
#pragma unroll
        for (int c = 0; c < kChunks / 2; ++c) {
          if (c < hc) {
            stage_store(slots, acc, c, wt);
#pragma unroll
            for (int g = 1; g < kChunks; ++g)
              if (g == c + hc) stage_store(slots + kStageSlotBytes, acc, g, wt);
            named_bar_sync(1 + wg, 128);
            if (eh == 0) {
              float va[32], vg[32];
              stage_load_row(slots, er, va);
              stage_load_row(slots + kStageSlotBytes, er, vg);
              gemm_epilogue_pair(p, va, vg, c * 32, t.bz, row, row_ok);
            }
            named_bar_sync(1 + wg, 128);
          }
        }
      }
    }
  }
}

// fp32 SIMT evaluation of the same contract (debug / cross-check).
__global__ void conv_gemm_simt_kernel(const __nv_bfloat16* a_hi, const __nv_bfloat16* a_lo, const __nv_bfloat16* b_hi,
                                      const __nv_bfloat16* b_lo, pk_operand oa, pk_operand ob, GemmKernelArgs p, int k,
                                      int batch) {
  const long long total = static_cast<long long>(batch) * p.heads * p.m * p.n;
  for (long long idx = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int n = idx % p.n;
    const int t = (idx / p.n) % p.m;
    const int z = idx / (static_cast<long long>(p.n) * p.m);
    const int b = z / p.heads, h = z % p.heads;
    const long long ab = (b * p.a_bmul + h * p.a_hmul) * oa.batch_stride;
    const long long bb = (b * p.b_bmul + h * p.b_hmul) * ob.batch_stride;
    const int ac = p.a_col0 + h * p.a_colh, bc = p.b_col0 + h * p.b_colh;
    float acc = 0.f;
    for (int tap = 0; tap < p.taps; ++tap) {
      const int r = t + (tap - p.pad) * p.dil;
      if (r < 0 || r >= oa.rows) continue;
      for (int kk = 0; kk < k; ++kk) {
        if (ac + kk >= oa.cols) break;
        const long long ai = ab + static_cast<long long>(r) * oa.ld + ac + kk;
        const int bcol = bc + tap * p.b_tap_stride + kk;
        if (bcol >= ob.cols || n >= ob.rows) continue;
        const long long bi = bb + static_cast<long long>(n) * ob.ld + bcol;
        float av = __bfloat162float(a_hi[ai]);
        float bv = __bfloat162float(b_hi[bi]);
        if (p.passes == 3) {
          av += __bfloat162float(a_lo[ai]);
          bv += __bfloat162float(b_lo[bi]);
        }
        acc = fmaf(av, bv, acc);
      }
    }
    float x = acc * p.scale;
    if (p.bias) x += p.bias[n];
    if (p.act == PK_ACT_RELU) x = fmaxf(x, 0.f);
    else if (p.act == PK_ACT_TANH) x = tanhf(x);
    const long long yo = b * p.y_batch_stride + h * p.y_head_stride + static_cast<long long>(t) * p.y_ld + n;
    if (p.residual) x += p.residual[yo];
    if (p.lens && t >= p.lens[b]) x = 0.f;
    if (p.y_f32) p.y_f32[yo] = x;
    if (p.y_hi) {
      __nv_bfloat16 hh, ll;
      split_bf16(x, hh, ll);
      p.y_hi[yo] = hh;
      p.y_lo[yo] = ll;
    }
  }
}

static int validate_common(const pk_conv_gemm_args* a) {
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  PK_CHECK_ARG(a->a.hi && a->b.hi, "operand hi planes must be non-NULL");
  PK_CHECK_ARG(a->passes == 1 || a->passes == 3, "passes must be 1 or 3 (got %d)", a->passes);
  PK_CHECK_ARG(a->passes == 1 || (a->a.lo && a->b.lo), "passes=3 needs lo planes");
  PK_CHECK_ARG(a->batch > 0 && a->heads > 0 && a->m > 0 && a->n > 0 && a->k > 0, "batch/heads/m/n/k must be > 0");
  PK_CHECK_ARG(a->taps >= 1 && a->dil >= 1 && a->pad >= 0, "bad taps/dil/pad");
  PK_CHECK_ARG((a->a.ld % 8) == 0 && (a->b.ld % 8) == 0, "operand row strides must be multiples of 8 elements (16 B)");
  PK_CHECK_ARG((a->a.batch_stride % 8) == 0 && (a->b.batch_stride % 8) == 0, "operand batch strides must be multiples of 8");
  PK_CHECK_ARG((reinterpret_cast<uintptr_t>(a->a.hi) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->b.hi) & 15) == 0,
               "operand planes must be 16-byte aligned");
  PK_CHECK_ARG((a->y_hi == nullptr) == (a->y_lo == nullptr), "y_hi and y_lo must both be set or both NULL");
  PK_CHECK_ARG(a->act >= PK_ACT_NONE && a->act <= PK_ACT_TANH, "unknown activation %d", a->act);
  return PK_OK;
}

static int validate(const pk_conv_gemm_args* a) {
  int rc = validate_common(a);
  if (rc) return rc;
  PK_CHECK_ARG((a->y_f32 != nullptr) || (a->y_hi != nullptr), "no output requested");
  return PK_OK;
}

static int validate_epilogue(const pk_conv_gemm_args* a, const pk_gemm_epilogue* e) {
  int rc = validate_common(a);
  if (rc) return rc;
  PK_CHECK_ARG(e->mode == PK_EPI_GATE || e->mode == PK_EPI_WF_UPDATE, "unknown epilogue mode %d", e->mode);
  PK_CHECK_ARG(e->channels > 0 && (e->channels % 32) == 0 && a->n == 2 * e->channels && a->n <= 256,
               "fused epilogues need n == 2 * channels, channels %% 32 == 0, n <= 256 (n=%d channels=%d)", a->n, e->channels);
  PK_CHECK_ARG(a->heads == 1 && a->act == PK_ACT_NONE && a->residual == nullptr && a->lens == nullptr,
               "fused epilogues take heads == 1, no activation / residual / lens in the base arguments");
  PK_CHECK_ARG(a->bias == nullptr || (reinterpret_cast<uintptr_t>(a->bias) & 15) == 0, "bias must be 16-byte aligned");
  if (e->mode == PK_EPI_GATE) {
    PK_CHECK_ARG(a->y_hi && a->y_lo && (a->y_ld % 8) == 0, "GATE writes split planes (y_hi / y_lo), y_ld %% 8 == 0");
    PK_CHECK_ARG(e->residual == nullptr || ((e->residual_ld % 4) == 0 && (e->residual_batch_stride % 4) == 0 &&
                                            (reinterpret_cast<uintptr_t>(e->residual) & 15) == 0),
                 "GATE residual must be 16-byte aligned with strides %% 4 == 0");
  } else {
    PK_CHECK_ARG(e->state && e->skip, "WF_UPDATE needs state and skip");
    PK_CHECK_ARG((e->buf_hi == nullptr) == (e->buf_lo == nullptr), "buf_hi and buf_lo must both be set or both NULL");
    PK_CHECK_ARG(e->buf_hi == nullptr || ((e->buf_ld % 8) == 0 && (e->buf_col0 % 8) == 0), "buf_ld / buf_col0 must be multiples of 8");
  }
  return PK_OK;
}

static GemmKernelArgs to_kernel_args(const pk_conv_gemm_args* a) {
  GemmKernelArgs p;
  p.m = a->m; p.n = a->n; p.k_chunks = (a->k + kChunkK - 1) / kChunkK; p.taps = a->taps; p.dil = a->dil; p.pad = a->pad;
  p.heads = a->heads; p.batch = a->batch; p.tiles_m = 0; p.total_tiles = 0;
  p.a_bmul = a->a.bmul; p.a_hmul = a->a.hmul; p.a_col0 = a->a.col0; p.a_colh = a->a.colh;
  p.b_bmul = a->b.bmul; p.b_hmul = a->b.hmul; p.b_col0 = a->b.col0; p.b_colh = a->b.colh;
  p.b_tap_stride = p.k_chunks * kChunkK;
  p.scale = a->scale; p.bias = a->bias; p.act = a->act; p.residual = a->residual; p.lens = a->lens;
  p.y_f32 = a->y_f32; p.y_hi = static_cast<__nv_bfloat16*>(a->y_hi); p.y_lo = static_cast<__nv_bfloat16*>(a->y_lo);
  p.y_batch_stride = a->y_batch_stride; p.y_head_stride = a->y_head_stride; p.y_ld = a->y_ld;
  p.passes = a->passes;
  p.epi = PK_EPI_NONE; p.epi_c = 0; p.e_res = nullptr; p.e_res_bs = 0; p.e_res_ld = 0; p.e_state = nullptr; p.e_skip = nullptr;
  p.e_skip_init = 0; p.e_buf_hi = nullptr; p.e_buf_lo = nullptr; p.e_buf_ld = 0; p.e_buf_col0 = 0;
  return p;
}

template <int BLOCK_N>
static int launch(const pk_conv_gemm_args* a, cudaStream_t stream, const pk_gemm_epilogue* e = nullptr) {
  using Cfg = GemmCfg<BLOCK_N>;
  CUtensorMap ta_hi, ta_lo, tb_hi, tb_lo;
  int rc;
  if ((rc = encode_tmap_bf16_3d(&ta_hi, a->a.hi, a->a.cols, a->a.rows, a->a.batches, a->a.ld, a->a.batch_stride, kBlockM))) return rc;
  if ((rc = encode_tmap_bf16_3d(&tb_hi, a->b.hi, a->b.cols, a->b.rows, a->b.batches, a->b.ld, a->b.batch_stride, BLOCK_N))) return rc;
  if (a->passes == 3) {
    if ((rc = encode_tmap_bf16_3d(&ta_lo, a->a.lo, a->a.cols, a->a.rows, a->a.batches, a->a.ld, a->a.batch_stride, kBlockM))) return rc;
    if ((rc = encode_tmap_bf16_3d(&tb_lo, a->b.lo, a->b.cols, a->b.rows, a->b.batches, a->b.ld, a->b.batch_stride, BLOCK_N))) return rc;
  } else {
    ta_lo = ta_hi;
    tb_lo = tb_hi;
  }
  int resident = 0;
  if ((rc = prepare_kernel(conv_gemm_kernel<BLOCK_N>, kGemmThreads, Cfg::kSmemBytes, &resident))) return rc;
  GemmKernelArgs p = to_kernel_args(a);
  if (e != nullptr) {
    p.epi = e->mode; p.epi_c = e->channels; p.e_res = e->residual; p.e_res_bs = e->residual_batch_stride; p.e_res_ld = e->residual_ld;
    p.e_state = e->state; p.e_skip = e->skip; p.e_skip_init = e->skip_init;
    p.e_buf_hi = static_cast<__nv_bfloat16*>(e->buf_hi); p.e_buf_lo = static_cast<__nv_bfloat16*>(e->buf_lo);
    p.e_buf_ld = e->buf_ld; p.e_buf_col0 = e->buf_col0;
  }
  p.tiles_m = (a->m + kBlockM - 1) / kBlockM;
  const long long total = static_cast<long long>(p.tiles_m) * ((a->n + BLOCK_N - 1) / BLOCK_N) * a->batch * a->heads;
  PK_CHECK_ARG(total < (1LL << 31), "too many output tiles");
  p.total_tiles = static_cast<int>(total);
  const int grid = static_cast<int>(std::min<long long>(total, resident));   // persistent: every CTA resident (one per SM)
  conv_gemm_kernel<BLOCK_N><<<grid, kGemmThreads, Cfg::kSmemBytes, stream>>>(ta_hi, ta_lo, tb_hi, tb_lo, p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

}  // namespace pk

extern "C" int pk_conv_gemm(const pk_conv_gemm_args* args, pk_stream_t stream) {
  int rc = pk::validate(args);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // tile width with the fewest padded columns (ties -> wider tile)
  const int n = args->n;
  auto waste = [n](int bn) { return (n + bn - 1) / bn * bn - n; };
  if (n <= 64) return pk::launch<64>(args, s);
  if (waste(256) <= waste(128) && n > 128) return pk::launch<256>(args, s);
  return pk::launch<128>(args, s);
}

extern "C" int pk_conv_gemm_ex(const pk_conv_gemm_args* args, const pk_gemm_epilogue* epi, pk_stream_t stream) {
  if (epi == nullptr || epi->mode == PK_EPI_NONE) return pk_conv_gemm(args, stream);
  int rc = pk::validate_epilogue(args, epi);
  if (rc) return rc;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // the whole 2C-wide row must sit in one tile of the single-CTA kernel
  return args->n <= 128 ? pk::launch<128>(args, s, epi) : pk::launch<256>(args, s, epi);
}

extern "C" int pk_conv_gemm_simt(const pk_conv_gemm_args* args, pk_stream_t stream) {
  int rc = pk::validate(args);
  if (rc) return rc;
  const pk::GemmKernelArgs p = pk::to_kernel_args(args);
  const long long total = static_cast<long long>(args->batch) * args->heads * args->m * args->n;
  const int threads = 256;
  const int blocks = static_cast<int>(std::min<long long>((total + threads - 1) / threads, 132LL * 16));
  pk::conv_gemm_simt_kernel<<<blocks, threads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const __nv_bfloat16*>(args->a.hi), static_cast<const __nv_bfloat16*>(args->a.lo),
      static_cast<const __nv_bfloat16*>(args->b.hi), static_cast<const __nv_bfloat16*>(args->b.lo), args->a, args->b, p,
      args->k, args->batch);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}
