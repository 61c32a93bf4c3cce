// LSTM recurrence (forward and backward through time) as persistent launches, and the GE2E loss of the speaker encoder
// (reference: parakeet/models/lstm_speaker_encoder.py; Paddle's nn.LSTM, gate order i, f, g, o).
//
// Recurrence layout: sequences are time-major, row r of step t at t * rows + r.  The input half of the gates,
// G_in = x W_ih^T + b_ih for every step, is one pk_conv_gemm before the launch; the kernels only carry the h_{t-1} W_hh^T half.
// The hidden axis is cut into slices of kSlice units; CTA (slice, group) keeps W_hh's rows (forward) or columns (backward) of
// its slice resident in shared memory as split-bf16 for all steps and walks the row tiles g, g + groups, ... of every step.  The
// per-step GEMM is wgmma in the bf16x3 format; h_{t-1} (forward) and dgates_{t+1} (backward) are read as split planes by TMA.
// A step of a row tile needs the previous step's h (forward) or dgates (backward) of ALL slices of that tile: each CTA publishes
// its part with a gpu-scope release on the (step, tile) counter, and readers acquire it until it equals the slice count.
// Every CTA of the grid is co-resident (the host sizes the grid by the occupancy query and refuses otherwise) and a CTA only
// ever waits on the previous step, which every CTA finishes before its own next step: no wait can be on a CTA that cannot run.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <cstdio>
#include <stdint.h>

#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace lstm {

constexpr int kSlice = 32;      // hidden units per CTA
constexpr int kRows = 64;       // rows per tile (the wgmma M)
constexpr int kThreads = 128;   // one warpgroup
constexpr int kGroupChunks = 4; // K-chunks of 64 of the backward's dgates tile staged at a time

__device__ __forceinline__ void wait_count(const unsigned* flag, unsigned target) {
  const long long t0 = clock64();
  while (ld_acquire_gpu(flag) < target) {
    __nanosleep(32);
    // ~4 s: a dependency that never completes is a scheduling bug - fail loudly (launch error), do not hang.  No printf here: a
    // call inside the kernel would serialize its wgmma pipeline.
    if (clock64() - t0 > (1ll << 33)) __trap();
  }
}

__device__ __forceinline__ void wgmma_ss_n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
               "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, "
               "p, 1, 1, 0, 0;\n}\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
                 "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
               : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

template <int H>
struct Geo {
  static constexpr int kSlices = H / kSlice;
  static constexpr int kChunks = H / kChunkK;                 // K-chunks of the forward (K = H)
  static constexpr int kWChunk = 2 * 4 * kSlice * 128;        // forward: [hi | lo] of 128 gate rows x 64 K = 32 KB
  static constexpr int kHChunk = 2 * kRows * 128;             // [hi | lo] of 64 rows x 64 K = 16 KB
  static constexpr int kFwdSmem = 1024 + kChunks * (kWChunk + kHChunk) + 64;
  static constexpr int kBChunks = 4 * H / kChunkK;            // K-chunks of the backward (K = 4H)
  static constexpr int kBWChunk = 2 * kSlice * 128;           // backward: [hi | lo] of 32 unit rows x 64 K = 8 KB
  static constexpr int kBwdSmem = 1024 + kBChunks * kBWChunk + kGroupChunks * kHChunk + 64;
};

template <int H>
struct FwdArgs {
  CUtensorMap tm_w;            // packed W_hh planes [4H rows (gate-permuted, see pk_lstm_fwd), H]
  CUtensorMap tm_h;            // h planes {H, rows, T + 1}
  const float* g_in;
  const float* b_hh;
  float* h_all;
  __nv_bfloat16* h_hi;
  __nv_bfloat16* h_lo;
  float* c;
  long long c_step;
  float* gates;
  unsigned* counters;
  int rows, T, groups;
};

// Forward: gates_t = G_in[t] + b_hh + h_{t-1} W_hh^T as wgmma m64n128 in bf16x3 (h_hi W_hi + h_lo W_hi + h_hi W_lo), W_hh's 128
// gate rows of the slice resident in shared memory, h_{t-1}'s tile fetched by TMA.  The gate rows are packed so that accumulator
// columns 8 (2p + jj) + 2q + e hold gate 2 jj + e of local unit 4p + q: every thread holds all four gates of its units.
template <int H>
__global__ void __launch_bounds__(kThreads, 1) lstm_fwd_kernel(const __grid_constant__ FwdArgs<H> p) {
  using G = Geo<H>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_s = base, h_s = base + G::kChunks * G::kWChunk;
  const uint32_t bar_w = h_s + G::kChunks * G::kHChunk, bar_h = bar_w + 8;
  const int slice = blockIdx.x % G::kSlices, group = blockIdx.x / G::kSlices;
  const int u_base = slice * kSlice;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  const int n_tiles = (p.rows + kRows - 1) / kRows;
  const int rows = p.rows;
  if (tid == 0) {
    mbar_init_a(bar_w, 1);
    mbar_init_a(bar_h, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx_a(bar_w, G::kChunks * G::kWChunk);
    for (int kc = 0; kc < G::kChunks; ++kc) tma_load_4d_a(w_s + kc * G::kWChunk, &p.tm_w, bar_w, kc * kChunkK, slice * 4 * kSlice, 0, 0);
  }
  float bh[8][4];
#pragma unroll
  for (int pp = 0; pp < 8; ++pp)
#pragma unroll
    for (int g = 0; g < 4; ++g) bh[pp][g] = p.b_hh ? p.b_hh[g * H + u_base + 4 * pp + q] : 0.f;
  __syncthreads();
  mbar_wait_a(bar_w, 0);
  uint32_t phase = 0;
  for (int t = 0; t < p.T; ++t) {
    for (int m = group; m < n_tiles; m += p.groups) {
      const int r0 = m * kRows;
      if (tid == 0) {
        if (t > 0) wait_count(p.counters + static_cast<long long>(t - 1) * n_tiles + m, G::kSlices);
        fence_proxy_async_all();         // h_{t-1} was written by generic stores; TMA reads it through the async proxy
        mbar_arrive_expect_tx_a(bar_h, G::kChunks * G::kHChunk);
        for (int kc = 0; kc < G::kChunks; ++kc) tma_load_4d_a(h_s + kc * G::kHChunk, &p.tm_h, bar_h, kc * kChunkK, r0, t, 0);
      }
      mbar_wait_a(bar_h, phase);
      phase ^= 1;
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      wgmma_fence();
#pragma unroll
      for (int kc = 0; kc < G::kChunks; ++kc) {
        const uint32_t ah = h_s + kc * G::kHChunk, bh_ = w_s + kc * G::kWChunk;
#pragma unroll
        for (int ks = 0; ks < kChunkK / kWgmmaK; ++ks) {
          const uint64_t a_hi = make_smem_desc_sw128(ah) + desc_kstep(ks), a_lo = make_smem_desc_sw128(ah + kRows * 128) + desc_kstep(ks);
          const uint64_t b_hi = make_smem_desc_sw128(bh_) + desc_kstep(ks), b_lo = make_smem_desc_sw128(bh_ + 4 * kSlice * 128) + desc_kstep(ks);
          wgmma_ss_n128(d, a_hi, b_hi, 1);
          wgmma_ss_n128(d, a_lo, b_hi, 1);
          wgmma_ss_n128(d, a_hi, b_lo, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(d);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = r0 + 16 * warp + (lane >> 2) + 8 * half;
        if (row < rows) {
          const float* gi = p.g_in + (static_cast<long long>(t) * rows + row) * 4 * H;
#pragma unroll
          for (int pp = 0; pp < 8; ++pp) {
            const int u = u_base + 4 * pp + q;
            const float ig = sigmoidf_(d[8 * pp + 2 * half] + gi[u] + bh[pp][0]);
            const float fg = sigmoidf_(d[8 * pp + 2 * half + 1] + gi[H + u] + bh[pp][1]);
            const float gg = tanhf(d[8 * pp + 4 + 2 * half] + gi[2 * H + u] + bh[pp][2]);
            const float og = sigmoidf_(d[8 * pp + 4 + 2 * half + 1] + gi[3 * H + u] + bh[pp][3]);
            const long long cu = static_cast<long long>(row) * H + u;
            const float cn = fg * p.c[t * p.c_step + cu] + ig * gg;
            p.c[(t + 1) * p.c_step + cu] = cn;
            const float hn = og * tanhf(cn);
            const long long ho = static_cast<long long>(t + 1) * rows * H + cu;
            p.h_all[ho] = hn;
            split_bf16(hn, p.h_hi[ho], p.h_lo[ho]);
            if (p.gates) {
              float* gp = p.gates + (static_cast<long long>(t) * rows + row) * 4 * H;
              gp[u] = ig; gp[H + u] = fg; gp[2 * H + u] = gg; gp[3 * H + u] = og;
            }
          }
        }
      }
      __syncthreads();                   // every thread's h is written and every wgmma has read the h tile
      if (tid == 0) {
        __threadfence();
        red_release_gpu_inc(p.counters + static_cast<long long>(t) * n_tiles + m);
      }
    }
  }
}

template <int H>
struct BwdArgs {
  CUtensorMap tm_w;            // W_hh^T planes [H rows (units), 4H]
  CUtensorMap tm_d;            // dgates planes {4H, rows, T}
  const float* gates;
  const float* c_all;
  const float* dh_in;
  const float* dh_last;
  float* dc;
  float* dgates;
  __nv_bfloat16* dg_hi;
  __nv_bfloat16* dg_lo;
  unsigned* counters;
  int rows, T, groups;
};

// Backward through time, t = T-1 .. 0: dh_t = dh_in[t] (+ dh_last at T-1) + dgates_{t+1} W_hh[:, slice] as wgmma m64n32 in bf16x3
// (K = 4H staged through shared memory kGroupChunks chunks at a time), then the cell backward with dc carried in `dc` (each
// element only ever touched by the thread that owns it).  Accumulator column 8 j + 2q + e is local unit 8 j + 2q + e.
template <int H>
__global__ void __launch_bounds__(kThreads, 1) lstm_bwd_kernel(const __grid_constant__ BwdArgs<H> p) {
  using G = Geo<H>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t w_s = base, a_s = base + G::kBChunks * G::kBWChunk;
  const uint32_t bar_w = a_s + kGroupChunks * G::kHChunk, bar_a = bar_w + 8;
  const int slice = blockIdx.x % G::kSlices, group = blockIdx.x / G::kSlices;
  const int u_base = slice * kSlice;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  const int n_tiles = (p.rows + kRows - 1) / kRows;
  const int rows = p.rows, T = p.T;
  if (tid == 0) {
    mbar_init_a(bar_w, 1);
    mbar_init_a(bar_a, 1);
    fence_barrier_init();
    mbar_arrive_expect_tx_a(bar_w, G::kBChunks * G::kBWChunk);
    for (int kc = 0; kc < G::kBChunks; ++kc) tma_load_4d_a(w_s + kc * G::kBWChunk, &p.tm_w, bar_w, kc * kChunkK, u_base, 0, 0);
  }
  __syncthreads();
  mbar_wait_a(bar_w, 0);
  uint32_t phase = 0;
  for (int t = T - 1; t >= 0; --t) {
    for (int m = group; m < n_tiles; m += p.groups) {
      const int r0 = m * kRows;
      float d[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) d[i] = 0.f;
      if (t < T - 1) {
        if (tid == 0) {
          wait_count(p.counters + static_cast<long long>(t + 1) * n_tiles + m, G::kSlices);
          fence_proxy_async_all();
        }
#pragma unroll 1
        for (int k0 = 0; k0 < G::kBChunks; k0 += kGroupChunks) {
          if (tid == 0) {
            mbar_arrive_expect_tx_a(bar_a, kGroupChunks * G::kHChunk);
            for (int kc = 0; kc < kGroupChunks; ++kc)
              tma_load_4d_a(a_s + kc * G::kHChunk, &p.tm_d, bar_a, (k0 + kc) * kChunkK, r0, t + 1, 0);
          }
          mbar_wait_a(bar_a, phase);
          phase ^= 1;
          wgmma_fence();
#pragma unroll
          for (int kc = 0; kc < kGroupChunks; ++kc) {
            const uint32_t ah = a_s + kc * G::kHChunk, bw = w_s + (k0 + kc) * G::kBWChunk;
#pragma unroll
            for (int ks = 0; ks < kChunkK / kWgmmaK; ++ks) {
              const uint64_t a_hi = make_smem_desc_sw128(ah) + desc_kstep(ks), a_lo = make_smem_desc_sw128(ah + kRows * 128) + desc_kstep(ks);
              const uint64_t b_hi = make_smem_desc_sw128(bw) + desc_kstep(ks), b_lo = make_smem_desc_sw128(bw + kSlice * 128) + desc_kstep(ks);
              wgmma_ss_n32(d, a_hi, b_hi, 1);
              wgmma_ss_n32(d, a_lo, b_hi, 1);
              wgmma_ss_n32(d, a_hi, b_lo, 1);
            }
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(d);
          __syncthreads();               // every wgmma has read the staged chunks before the next TMA overwrites them
        }
      }
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int row = r0 + 16 * warp + (lane >> 2) + 8 * half;
        if (row >= rows) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int u = u_base + 8 * j + 2 * q + e;
            const long long cu = static_cast<long long>(row) * H + u;
            float dh = d[4 * j + 2 * half + e];
            if (p.dh_in) dh += p.dh_in[static_cast<long long>(t) * rows * H + cu];
            if (p.dh_last && t == T - 1) dh += p.dh_last[cu];
            const long long gb = (static_cast<long long>(t) * rows + row) * 4 * H;
            const float ig = p.gates[gb + u], fg = p.gates[gb + H + u], gg = p.gates[gb + 2 * H + u], og = p.gates[gb + 3 * H + u];
            const float ct = p.c_all[static_cast<long long>(t + 1) * rows * H + cu];
            const float cp = p.c_all[static_cast<long long>(t) * rows * H + cu];
            const float th = tanhf(ct);
            const float dct = (t < T - 1 ? p.dc[cu] : 0.f) + dh * og * (1.f - th * th);
            const float dg[4] = {dct * gg * ig * (1.f - ig), dct * cp * fg * (1.f - fg), dct * ig * (1.f - gg * gg), dh * th * og * (1.f - og)};
            p.dc[cu] = dct * fg;
#pragma unroll
            for (int g = 0; g < 4; ++g) {
              p.dgates[gb + g * H + u] = dg[g];
              split_bf16(dg[g], p.dg_hi[gb + g * H + u], p.dg_lo[gb + g * H + u]);
            }
          }
        }
      }
      __syncthreads();
      if (tid == 0) {
        __threadfence();
        red_release_gpu_inc(p.counters + static_cast<long long>(t) * n_tiles + m);
      }
    }
  }
}

// GE2E softmax loss on embeds (n, m, c), one block in double (lstm_speaker_encoder.py similarity_matrix / loss; phases below).
constexpr int kLossThreads = 512;

__global__ void __launch_bounds__(kLossThreads, 1)
ge2e_loss_kernel(const float* __restrict__ e, int N, int M, int C, const float* __restrict__ wp, const float* __restrict__ bp,
                 double* ws, float* loss, float* sim, float* de, float* dw, float* db) {
  __shared__ double red[kLossThreads];
  const int NM = N * M, tid = threadIdx.x;
  double* S = ws;                    // [N][C] sums per speaker
  double* ci = S + N * C;            // [N][C] normalised inclusive centroids
  double* nin = ci + N * C;          // [N]
  double* ce = nin + N;              // [NM][C] normalised exclusive centroids
  double* nex = ce + NM * C;         // [NM]
  double* p = nex + NM;              // [NM][N] raw similarities (own speaker: exclusive)
  double* dsm = p + NM * N;          // [NM][N] dL/ds
  double* ded = dsm + NM * N;        // [NM][C] de through the dot products
  double* dci = ded + NM * C;        // [N][C]
  double* dex = dci + N * C;         // [NM][C] d excl (after the normalisation backward)
  double* lrow = dex + NM * C;       // [NM]
  const double w = wp[0], b = bp[0];
  for (int i = tid; i < N * C; i += kLossThreads) {
    const int j = i / C, cc = i - j * C;
    double s = 0.0;
    for (int k = 0; k < M; ++k) s += e[(static_cast<long long>(j) * M + k) * C + cc];
    S[i] = s;
  }
  __syncthreads();
  for (int j = tid; j < N; j += kLossThreads) {
    double q = 0.0;
    for (int cc = 0; cc < C; ++cc) { const double v = S[j * C + cc] / M; q += v * v; }
    nin[j] = sqrt(q);
  }
  for (int r = tid; r < NM; r += kLossThreads) {
    const int j = r / M;
    double q = 0.0;
    for (int cc = 0; cc < C; ++cc) { const double v = (S[j * C + cc] - e[static_cast<long long>(r) * C + cc]) / (M - 1); q += v * v; }
    nex[r] = sqrt(q);
  }
  __syncthreads();
  for (int i = tid; i < N * C; i += kLossThreads) ci[i] = S[i] / M / nin[i / C];
  for (int i = tid; i < NM * C; i += kLossThreads) {
    const int r = i / C, cc = i - r * C, j = r / M;
    ce[i] = (S[j * C + cc] - e[i]) / (M - 1) / nex[r];
  }
  __syncthreads();
  for (int i = tid; i < NM * N; i += kLossThreads) {
    const int r = i / N, k = i - r * N;
    const double* cv = k == r / M ? ce + static_cast<long long>(r) * C : ci + k * C;
    double q = 0.0;
    for (int cc = 0; cc < C; ++cc) q += e[static_cast<long long>(r) * C + cc] * cv[cc];
    p[i] = q;
    if (sim) sim[i] = static_cast<float>(q * w + b);
  }
  __syncthreads();
  const double inv = 1.0 / NM;
  for (int r = tid; r < NM; r += kLossThreads) {
    const int j = r / M;
    double mx = -1e300;
    for (int k = 0; k < N; ++k) mx = fmax(mx, p[r * N + k] * w + b);
    double se = 0.0;
    for (int k = 0; k < N; ++k) se += exp(p[r * N + k] * w + b - mx);
    lrow[r] = mx + log(se) - (p[r * N + j] * w + b);
    for (int k = 0; k < N; ++k) dsm[r * N + k] = (exp(p[r * N + k] * w + b - mx) / se - (k == j ? 1.0 : 0.0)) * inv;
  }
  __syncthreads();
  double part = 0.0;
  for (int r = tid; r < NM; r += kLossThreads) part += lrow[r];
  const double total = block_sum_tree<kLossThreads>(part, red);
  if (tid == 0) loss[0] = static_cast<float>(total * inv);
  if (!de) return;
  double pw = 0.0, pb = 0.0;
  for (int i = tid; i < NM * N; i += kLossThreads) { pw += dsm[i] * p[i]; pb += dsm[i]; }
  const double gw = block_sum_tree<kLossThreads>(pw, red), gb = block_sum_tree<kLossThreads>(pb, red);
  if (tid == 0) { dw[0] = static_cast<float>(0.01 * gw); db[0] = static_cast<float>(0.01 * gb); }   // do_gradient_ops
  for (int i = tid; i < NM * C; i += kLossThreads) {
    const int r = i / C, cc = i - r * C, j = r / M;
    double q = 0.0;
    for (int k = 0; k < N; ++k) q += dsm[r * N + k] * (k == j ? ce[i] : ci[k * C + cc]);
    ded[i] = w * q;
  }
  for (int i = tid; i < N * C; i += kLossThreads) {
    const int k = i / C, cc = i - k * C;
    double q = 0.0;
    for (int r = 0; r < NM; ++r)
      if (r / M != k) q += dsm[r * N + k] * e[static_cast<long long>(r) * C + cc];
    dci[i] = w * q;
  }
  __syncthreads();
  for (int r = tid; r < NM; r += kLossThreads) {
    // normalisation backward of the exclusive centroid: d = (g - y (y . g)) / |x|, g = w dsm[r, own] e_r
    const int j = r / M;
    const double gsc = w * dsm[r * N + j];
    double yg = 0.0;
    for (int cc = 0; cc < C; ++cc) yg += ce[r * C + cc] * gsc * e[static_cast<long long>(r) * C + cc];
    for (int cc = 0; cc < C; ++cc)
      dex[r * C + cc] = (gsc * e[static_cast<long long>(r) * C + cc] - ce[r * C + cc] * yg) / nex[r] / (M - 1);
  }
  __syncthreads();
  for (int k = tid; k < N; k += kLossThreads) {
    double yg = 0.0;
    for (int cc = 0; cc < C; ++cc) yg += ci[k * C + cc] * dci[k * C + cc];
    for (int cc = 0; cc < C; ++cc) S[k * C + cc] = (dci[k * C + cc] - ci[k * C + cc] * yg) / nin[k] / M;   // S := d incl / M
  }
  __syncthreads();
  for (int i = tid; i < N * C; i += kLossThreads) {          // dci := sum over the speaker's rows of dex
    const int j = i / C, cc = i - j * C;
    double q = 0.0;
    for (int k = 0; k < M; ++k) q += dex[(j * M + k) * C + cc];
    dci[i] = q;
  }
  __syncthreads();
  for (int i = tid; i < NM * C; i += kLossThreads) {
    const int r = i / C, cc = i - r * C, j = r / M;
    de[i] = static_cast<float>(ded[i] + S[j * C + cc] + dci[j * C + cc] - dex[i]);
  }
}

// backward of F.normalize(relu(z)) over rows of n: dz = (z > 0) * (dy - y (y . dy)) / max(|e|, eps), e = relu(z); one warp per row
__global__ void embed_bwd_kernel(const float* __restrict__ e, const float* __restrict__ dy, int rows, int n, float eps,
                                 float* __restrict__ dz) {
  const int row = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* er = e + static_cast<long long>(row) * n;
  const float* gr = dy + static_cast<long long>(row) * n;
  float q = 0.f, eg = 0.f;
  for (int i = lane; i < n; i += 32) { q += er[i] * er[i]; eg += er[i] * gr[i]; }
  for (int o = 16; o > 0; o >>= 1) { q += __shfl_xor_sync(0xffffffffu, q, o); eg += __shfl_xor_sync(0xffffffffu, eg, o); }
  const float nrm = sqrtf(q);
  const float den = fmaxf(nrm, eps);
  const float proj = nrm > eps ? eg / (nrm * nrm) : 0.f;     // y . dy / |e| with y = e / |e|; no projection when clamped
  for (int i = lane; i < n; i += 32) dz[static_cast<long long>(row) * n + i] = er[i] > 0.f ? (gr[i] - er[i] * proj) / den : 0.f;
}

// y[s] = F.normalize(mean of rows offsets[s] .. offsets[s+1]-1 of x, axis=0): embed_utterance over each segment; one block each
__global__ void segment_mean_normalize_kernel(const float* __restrict__ x, const int* __restrict__ offsets, int n, float eps,
                                              float* __restrict__ y) {
  extern __shared__ float acc[];
  __shared__ float red[32];
  const int s = blockIdx.x, a = offsets[s], bnd = offsets[s + 1];
  float q = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    float v = 0.f;
    for (int r = a; r < bnd; ++r) v += x[static_cast<long long>(r) * n + i];
    v /= static_cast<float>(bnd > a ? bnd - a : 1);     // an empty (or reversed) segment yields zeros, not a division by zero
    acc[i] = v;
    q += v * v;
  }
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x / 32] = q;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < blockDim.x / 32 ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) red[0] = v;
  }
  __syncthreads();
  const float den = fmaxf(sqrtf(red[0]), eps);
  for (int i = threadIdx.x; i < n; i += blockDim.x) y[static_cast<long long>(s) * n + i] = acc[i] / den;
}

// grid of a persistent launch: -> CTAs (slices x groups), or 0 when not even one CTA per slice can be co-resident
int schedule(int rows, int slices, int max_ctas, int* groups) {
  const int n_tiles = (rows + kRows - 1) / kRows;
  *groups = std::min(n_tiles, max_ctas / slices);
  return *groups >= 1 ? *groups * slices : 0;
}

template <int H>
int fwd_launch(const float* g_in, const float* b_hh, const void* w_hi, const void* w_lo, int rows, int T, float* h_all, void* h_hi,
               void* h_lo, float* c, int64_t c_step, float* gates, uint32_t* counters, int64_t counters_len, cudaStream_t st) {
  using G = Geo<H>;
  int max_ctas = 0, rc;
  if ((rc = prepare_kernel(lstm_fwd_kernel<H>, kThreads, G::kFwdSmem, &max_ctas))) return rc;
  int groups = 0;
  const int grid = schedule(rows, G::kSlices, max_ctas, &groups);
  if (grid == 0) return fail(PK_ERR_UNSUPPORTED, "pk_lstm_fwd: %d slices cannot be co-resident (%d CTAs fit)", G::kSlices, max_ctas);
  const long long n_counters = static_cast<long long>(T) * ((rows + kRows - 1) / kRows);
  PK_CHECK_ARG(counters_len >= n_counters, "counters must hold t * ceil(rows / %d) = %lld entries", kRows, n_counters);
  FwdArgs<H> p;
  if ((rc = encode_tmap_bf16_planes(&p.tm_w, w_hi, w_lo, H, 4 * H, 1, H, 0, 4 * kSlice))) return rc;
  if ((rc = encode_tmap_bf16_planes(&p.tm_h, h_hi, h_lo, H, rows, T + 1, H, static_cast<uint64_t>(rows) * H, kRows))) return rc;
  p.g_in = g_in; p.b_hh = b_hh; p.h_all = h_all; p.c = c; p.c_step = c_step; p.gates = gates;
  p.h_hi = static_cast<__nv_bfloat16*>(h_hi); p.h_lo = static_cast<__nv_bfloat16*>(h_lo);
  p.counters = reinterpret_cast<unsigned*>(counters);
  p.rows = rows; p.T = T; p.groups = groups;
  PK_CHECK_CUDA(cudaMemsetAsync(counters, 0, n_counters * sizeof(uint32_t), st));
  lstm_fwd_kernel<H><<<grid, kThreads, G::kFwdSmem, st>>>(p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

template <int H>
int bwd_launch(const void* wt_hi, const void* wt_lo, const float* gates, const float* c_all, const float* dh_in, const float* dh_last,
               int rows, int T, float* dc, float* dgates, void* dg_hi, void* dg_lo, uint32_t* counters, int64_t counters_len,
               cudaStream_t st) {
  using G = Geo<H>;
  int max_ctas = 0, rc;
  if ((rc = prepare_kernel(lstm_bwd_kernel<H>, kThreads, G::kBwdSmem, &max_ctas))) return rc;
  int groups = 0;
  const int grid = schedule(rows, G::kSlices, max_ctas, &groups);
  if (grid == 0) return fail(PK_ERR_UNSUPPORTED, "pk_lstm_bwd: %d slices cannot be co-resident (%d CTAs fit)", G::kSlices, max_ctas);
  const long long n_counters = static_cast<long long>(T) * ((rows + kRows - 1) / kRows);
  PK_CHECK_ARG(counters_len >= n_counters, "counters must hold t * ceil(rows / %d) = %lld entries", kRows, n_counters);
  BwdArgs<H> p;
  if ((rc = encode_tmap_bf16_planes(&p.tm_w, wt_hi, wt_lo, 4 * H, H, 1, 4 * H, 0, kSlice))) return rc;
  if ((rc = encode_tmap_bf16_planes(&p.tm_d, dg_hi, dg_lo, 4 * H, rows, T, 4 * H, static_cast<uint64_t>(rows) * 4 * H, kRows))) return rc;
  p.gates = gates; p.c_all = c_all; p.dh_in = dh_in; p.dh_last = dh_last; p.dc = dc; p.dgates = dgates;
  p.dg_hi = static_cast<__nv_bfloat16*>(dg_hi); p.dg_lo = static_cast<__nv_bfloat16*>(dg_lo);
  p.counters = reinterpret_cast<unsigned*>(counters);
  p.rows = rows; p.T = T; p.groups = groups;
  PK_CHECK_CUDA(cudaMemsetAsync(counters, 0, n_counters * sizeof(uint32_t), st));
  lstm_bwd_kernel<H><<<grid, kThreads, G::kBwdSmem, st>>>(p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

}  // namespace lstm
}  // namespace pk

using namespace pk;
using namespace pk::lstm;

extern "C" int pk_lstm_fwd(const float* g_in, const float* b_hh, const void* w_hi, const void* w_lo, int32_t rows, int32_t t,
                           int32_t hidden, float* h_all, void* h_hi, void* h_lo, float* c, int64_t c_step, float* gates,
                           uint32_t* counters, int64_t counters_len, pk_stream_t stream) {
  PK_CHECK_ARG(rows > 0 && t > 0, "rows and t must be positive (got %d, %d)", rows, t);
  PK_CHECK_ARG(g_in && w_hi && w_lo && h_all && h_hi && h_lo && c && counters, "NULL pointer in pk_lstm_fwd");
  PK_CHECK_ARG(aligned16(w_hi) && aligned16(w_lo) && aligned16(h_hi) && aligned16(h_lo), "TMA operands must be 16-byte aligned");
  PK_CHECK_ARG(c_step == 0 || c_step == static_cast<int64_t>(rows) * hidden, "c_step must be 0 or rows * hidden");
  auto st = static_cast<cudaStream_t>(stream);
  if (hidden == 256) return fwd_launch<256>(g_in, b_hh, w_hi, w_lo, rows, t, h_all, h_hi, h_lo, c, c_step, gates, counters, counters_len, st);
  if (hidden == 64) return fwd_launch<64>(g_in, b_hh, w_hi, w_lo, rows, t, h_all, h_hi, h_lo, c, c_step, gates, counters, counters_len, st);
  return fail(PK_ERR_UNSUPPORTED, "pk_lstm_fwd is built for hidden sizes 64 and 256 (got %d)", hidden);
}

extern "C" int pk_lstm_bwd(const void* wt_hi, const void* wt_lo, const float* gates, const float* c_all, const float* dh_in,
                           const float* dh_last, int32_t rows, int32_t t, int32_t hidden, float* dc, float* dgates, void* dg_hi,
                           void* dg_lo, uint32_t* counters, int64_t counters_len, pk_stream_t stream) {
  PK_CHECK_ARG(rows > 0 && t > 0, "rows and t must be positive (got %d, %d)", rows, t);
  PK_CHECK_ARG(wt_hi && wt_lo && gates && c_all && dc && dgates && dg_hi && dg_lo && counters, "NULL pointer in pk_lstm_bwd");
  PK_CHECK_ARG(aligned16(wt_hi) && aligned16(wt_lo) && aligned16(dg_hi) && aligned16(dg_lo), "TMA operands must be 16-byte aligned");
  auto st = static_cast<cudaStream_t>(stream);
  if (hidden == 256) return bwd_launch<256>(wt_hi, wt_lo, gates, c_all, dh_in, dh_last, rows, t, dc, dgates, dg_hi, dg_lo, counters, counters_len, st);
  if (hidden == 64) return bwd_launch<64>(wt_hi, wt_lo, gates, c_all, dh_in, dh_last, rows, t, dc, dgates, dg_hi, dg_lo, counters, counters_len, st);
  return fail(PK_ERR_UNSUPPORTED, "pk_lstm_bwd is built for hidden sizes 64 and 256 (got %d)", hidden);
}

extern "C" int64_t pk_ge2e_loss_scratch(int32_t n, int32_t m, int32_t c) {
  const int64_t nm = static_cast<int64_t>(n) * m;
  return 4 * nm * c + 4 * static_cast<int64_t>(n) * c + n + 2 * nm + 2 * nm * n;
}

extern "C" int pk_ge2e_loss(const float* embeds, int32_t n, int32_t m, int32_t c, const float* w, const float* b, double* scratch,
                            int64_t scratch_len, float* loss, float* sim, float* d_embeds, float* dw, float* db, pk_stream_t stream) {
  PK_CHECK_ARG(n >= 1 && m >= 2 && c >= 1, "pk_ge2e_loss needs n >= 1 speakers, m >= 2 utterances, c >= 1 (got %d, %d, %d)", n, m, c);
  PK_CHECK_ARG(static_cast<int64_t>(n) * m * (n > c ? n : c) < (1ll << 31), "pk_ge2e_loss: batch too large");
  PK_CHECK_ARG(embeds && w && b && scratch && loss, "NULL pointer in pk_ge2e_loss");
  PK_CHECK_ARG((d_embeds == nullptr) == (dw == nullptr) && (dw == nullptr) == (db == nullptr), "d_embeds, dw and db come together");
  PK_CHECK_ARG(scratch_len >= pk_ge2e_loss_scratch(n, m, c), "scratch must hold pk_ge2e_loss_scratch(n, m, c) doubles");
  ge2e_loss_kernel<<<1, kLossThreads, 0, static_cast<cudaStream_t>(stream)>>>(embeds, n, m, c, w, b, scratch, loss, sim, d_embeds, dw, db);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_ge2e_embed_bwd(const float* e, const float* dy, int32_t rows, int32_t n, float eps, float* dz, pk_stream_t stream) {
  PK_CHECK_ARG(rows > 0 && n > 0 && e && dy && dz, "bad arguments to pk_ge2e_embed_bwd");
  embed_bwd_kernel<<<(rows + 7) / 8, 256, 0, static_cast<cudaStream_t>(stream)>>>(e, dy, rows, n, eps, dz);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

extern "C" int pk_segment_mean_normalize(const float* x, const int32_t* offsets, int32_t segments, int32_t n, float eps, float* y,
                                         pk_stream_t stream) {
  PK_CHECK_ARG(segments > 0 && n > 0 && n <= 8192 && x && offsets && y, "bad arguments to pk_segment_mean_normalize");
  segment_mean_normalize_kernel<<<segments, 256, n * sizeof(float), static_cast<cudaStream_t>(stream)>>>(x, offsets, n, eps, y);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}
