// Building blocks of the persistent autoregressive decoders (tacotron2.cu, transformer_tts.cu): one co-resident grid runs every
// decoder step, phases separated by a release/acquire grid hand-off, every dot product one warp in a fixed order (no atomics, so
// a fixed seed gives bit-identical results).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "pk_sm90.cuh"

namespace pk {
namespace pdec {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// every CTA of the (co-resident) grid arrives; `target` advances by the grid size per hand-off (thread 0 keeps it).  With prof
// (n_phases x 2 ns counters of this CTA), hand-off `phase` adds this CTA's time since the previous release (`last`) and its wait
// from arrival to release: the smallest wait over the CTAs is the hand-off's own latency (the last CTA to arrive waits only for it).
__device__ __forceinline__ void grid_sync(unsigned* ctr, unsigned& target, int grid, unsigned long long* prof_all, int n_phases,
                                          int phase, unsigned long long* last) {
  unsigned long long* prof = prof_all ? prof_all + static_cast<long long>(blockIdx.x) * 2 * n_phases : nullptr;
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned long long t_arrive = prof ? globaltimer() : 0ull;
    target += grid;
    __threadfence();
    red_release_gpu_inc(ctr);
    const long long t0 = clock64();
    while (ld_acquire_gpu(ctr) < target) {
      __nanosleep(20);
      if (clock64() - t0 > (1ll << 33)) __trap();   // ~4 s: a CTA that never arrives is a scheduling bug - fail, do not hang
    }
    if (prof) {
      const unsigned long long t_release = globaltimer();
      prof[phase] += t_release - *last;
      prof[n_phases + phase] += t_release - t_arrive;
      *last = t_release;
    }
  }
  __syncthreads();
}

struct Seg {
  const float* p;   // row b at p + b * ld
  int n;            // columns (multiple of 4)
  long long ld;
};

// y[row][bb] = W_row . xs[bb] for nrows rows and BC staged inputs xs (BC x K floats in shared memory, K a multiple of 4):
// warp w takes rows w, w + kWarps, ...; each lane accumulates a fixed stride of K, then a xor butterfly.  sink(rl, bb, y) gets
// each result (lane 0 of the row's warp).
template <int BC, class RowPtr, class Sink>
__device__ __forceinline__ void matvec_rows(int K, int nrows, RowPtr row_ptr, Sink sink, const float* xs) {
  const int K4 = K / 4, warp = threadIdx.x / 32, lane = threadIdx.x & 31;
  const float4* xs4 = reinterpret_cast<const float4*>(xs);
  for (int rl = warp; rl < nrows; rl += kWarps) {
    const float4* w4 = reinterpret_cast<const float4*>(row_ptr(rl));
    float acc[BC];
#pragma unroll
    for (int bb = 0; bb < BC; ++bb) acc[bb] = 0.f;
#pragma unroll (BC == 1 ? 4 : 2)
    for (int k4 = lane; k4 < K4; k4 += 32) {
      const float4 w = __ldg(w4 + k4);
#pragma unroll
      for (int bb = 0; bb < BC; ++bb) {
        const float4 x = xs4[bb * K4 + k4];
        acc[bb] = fmaf(w.x, x.x, acc[bb]);
        acc[bb] = fmaf(w.y, x.y, acc[bb]);
        acc[bb] = fmaf(w.z, x.z, acc[bb]);
        acc[bb] = fmaf(w.w, x.w, acc[bb]);
      }
    }
#pragma unroll
    for (int bb = 0; bb < BC; ++bb) acc[bb] = warp_sum(acc[bb]);
    if (lane == 0) {
#pragma unroll
      for (int bb = 0; bb < BC; ++bb) sink(rl, bb, acc[bb]);
    }
  }
}

// y[row][b] = W_row . [seg0 | seg1 | seg2][b] for the CTA's nrows rows and every b < B, in chunks of BC items staged in shared
// memory (xs).  sink(rl, b, y) gets each result (lane 0 of the row's warp); after(b0) runs once per chunk after all its rows.
template <int BC, class RowPtr, class Sink, class After>
__device__ void matvec(int K, const Seg (&seg)[3], int B, int nrows, RowPtr row_ptr, Sink sink, After after, float* xs) {
  const int K4 = K / 4;
  float4* xs4 = reinterpret_cast<float4*>(xs);
  for (int b0 = 0; b0 < B; b0 += BC) {
    for (int idx = threadIdx.x; idx < BC * K4; idx += kThreads) {
      const int bb = idx / K4, k = 4 * (idx - bb * K4), b = b0 + bb;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b < B) {
        const float* src;                 // constant indices only: seg stays in registers
        if (k < seg[0].n) src = seg[0].p ? seg[0].p + b * seg[0].ld + k : nullptr;
        else if (k < seg[0].n + seg[1].n) src = seg[1].p + b * seg[1].ld + (k - seg[0].n);
        else src = seg[2].p + b * seg[2].ld + (k - seg[0].n - seg[1].n);
        if (src) v = __ldcg(reinterpret_cast<const float4*>(src));
      }
      xs4[idx] = v;
    }
    __syncthreads();
    matvec_rows<BC>(K, nrows, row_ptr, [&](int rl, int bb, float y) { if (b0 + bb < B) sink(rl, b0 + bb, y); }, xs);
    __syncthreads();
    after(b0);
    __syncthreads();
  }
}

}  // namespace pdec
}  // namespace pk
