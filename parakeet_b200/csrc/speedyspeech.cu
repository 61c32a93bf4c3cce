// pk_ss_residual_block: one SpeedySpeech ResidualBlock.forward (reference speedyspeech.py:21-39) per launch,
//   h_0 = x,  h_i = BN_i(relu(conv_i(h_{i-1}) + b_i))  (i = 1..n, n in {1, 2}),  y = x + h_n,
// on channels-last (batch, t, 128) activations: x as fp32 (the residual) and split-bf16 planes (the GEMM operand); y is written
// the same two ways.  Eval-mode BatchNorm is the per-channel affine h * scale + shift AFTER the ReLU, so it cannot be folded
// into either conv (the next conv zero-pads the BN output).  The taps are undilated with `pad_left` zero rows before the
// sequence and taps - 1 - pad_left after it (Paddle's padding="same", see models/speedyspeech.py `paddle_same_conv`).
//
// One CTA per (128-row tile, utterance); 384 threads:
//   warps 8-11  producer warpgroup: one TMA lane loads the tile's x rows once (both planes, 136 rows including the halo) into
//               region A, then streams the conv weights through a 4-stage ring, one (tap, 64-channel chunk) of 128 x 64
//               split-bf16 per stage (32 KB) - one block's weights (up to 2 x 4 x 64 KB) do not fit on chip next to the tile;
//               it drops to 40 registers so that the consumers can take 232
//   warps 0-7   two consumer warpgroups, 64 rows each.  The A operand comes from REGISTERS (wgmma .rs): each thread loads its
//               m64k16 fragments from region A at row (output row + tap) with plain shared loads, so a tap is a one-row shift
//               of the read address and region A is written once per conv, not once per tap.  Weights are the smem B operand.
//   Two-conv blocks: the first conv produces 128 intermediate rows [t0 - pad_left, t0 - pad_left + 128); after both warpgroups
//   are done reading x, they overwrite region A with the intermediate (zero outside the utterance, which is the second conv's
//   zero padding) and the second conv reads it from there: the intermediate never leaves the SM.  Its output rows
//   [t0, t0 + 128 - (taps - 1)) are the tile's; the last taps - 1 accumulator rows read past the intermediate and are dropped.
//   Split-bf16, 3 wgmma per K-step (hi*hi + lo*hi + hi*lo), fp32 accumulation, as every GEMM of the library.
#include <algorithm>

#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace ss {

constexpr int kC = 128;                                   // channels (every hidden size of the shipped config)
constexpr int kTileRows = 128;                            // rows of the first conv's output per CTA
constexpr int kMaxTaps = 4;
constexpr int kRowsA = 136;                               // tile + up to 3 halo rows, a whole number of 1024-B swizzle atoms
constexpr int kSubBytes = kRowsA * kSwizzleBytes;         // one (64-channel chunk, plane) of region A: 17 KB
constexpr int kABytes = 4 * kSubBytes;                    // 2 chunks x 2 planes
constexpr int kWPlaneBytes = kC * kSwizzleBytes;          // one weight chunk plane: 128 output channels x 64 inputs
constexpr int kStageBytes = 2 * kWPlaneBytes;             // hi + lo: 32 KB
constexpr int kStages = 4;
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kSmemBytes = kABytes + kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
static_assert(kTileRows + kMaxTaps - 1 <= kRowsA, "region A holds the halo");

struct Args {
  int t, n_convs, taps, pad_left, out_rows;
  const int32_t* lens;
  const float* x;
  const float* bias[2];
  const float* scale[2];
  const float* shift[2];
  float* y;
  __nv_bfloat16* y_hi;
  __nv_bfloat16* y_lo;
};

__device__ __forceinline__ void split_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat16 ha, la, hb, lb;
  split_bf16(a, ha, la);
  split_bf16(b, hb, lb);
  hi = pack_bf16x2(ha, hb);
  lo = pack_bf16x2(la, lb);
}

__global__ void __launch_bounds__(kThreads, 1)
ss_residual_block_kernel(const __grid_constant__ CUtensorMap tm_x_hi, const __grid_constant__ CUtensorMap tm_x_lo,
                         const __grid_constant__ CUtensorMap tm_w1_hi, const __grid_constant__ CUtensorMap tm_w1_lo,
                         const __grid_constant__ CUtensorMap tm_w2_hi, const __grid_constant__ CUtensorMap tm_w2_lo, const Args p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;     // region A (1024-B aligned for the 128-B swizzle)
  const uint32_t ring = smem + kABytes;
  const uint32_t full_bar = ring + kStages * kStageBytes;
  const uint32_t empty_bar = full_bar + 8 * kStages;
  const uint32_t x_bar = empty_bar + 8 * kStages;

  const int b = blockIdx.y;
  const int t0 = blockIdx.x * p.out_rows;
  const int len = p.lens != nullptr ? min(__ldg(p.lens + b), p.t) : p.t;
  const long long row0 = static_cast<long long>(b) * p.t;

  if (t0 >= len) {                                   // the whole tile is past the utterance: zero rows, nothing to load
    const int rows = min(p.out_rows, p.t - t0);
    for (int i = threadIdx.x; i < rows * kC; i += blockDim.x) {
      const long long o = (row0 + t0) * kC + i;
      p.y[o] = 0.f;
      p.y_hi[o] = __float2bfloat16_rn(0.f);
      p.y_lo[o] = __float2bfloat16_rn(0.f);
    }
    return;
  }

  const int r0 = t0 - (p.n_convs == 2 ? p.pad_left : 0);    // first row of the first conv's output
  const int chunks = 2 * p.taps;                             // weight chunks per conv: (tap, 64-channel half), tap-major
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == kConsumerThreads) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init_a(full_bar + 8 * s, 1);
      mbar_init_a(empty_bar + 8 * s, kConsumerThreads / 32);     // one elected lane per consumer warp
    }
    mbar_init_a(x_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    // ------------------------------ TMA producer ------------------------------
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      tma_prefetch_desc(&tm_x_hi);
      tma_prefetch_desc(&tm_x_lo);
      mbar_arrive_expect_tx_a(x_bar, kABytes);
      // region A row i = sequence row r0 - pad_left + i; rows outside [0, t) arrive as zeros (the convs' zero padding)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        tma_load_3d_a(smem + (2 * c) * kSubBytes, &tm_x_hi, x_bar, c * 64, r0 - p.pad_left, b);
        tma_load_3d_a(smem + (2 * c + 1) * kSubBytes, &tm_x_lo, x_bar, c * 64, r0 - p.pad_left, b);
      }
      for (int i = 0; i < p.n_convs * chunks; ++i) {
        const int s = i % kStages;
        mbar_wait_a(empty_bar + 8 * s, ((i / kStages) & 1) ^ 1);
        const uint32_t st = ring + s * kStageBytes;
        const uint32_t fb = full_bar + 8 * s;
        mbar_arrive_expect_tx_a(fb, kStageBytes);
        const bool first = i < chunks;
        const int col = (i % chunks) * 64;                       // packed weight column: tap * 128 + half * 64
        tma_load_3d_a(st, first ? &tm_w1_hi : &tm_w2_hi, fb, col, 0, 0);
        tma_load_3d_a(st + kWPlaneBytes, first ? &tm_w1_lo : &tm_w2_lo, fb, col, 0, 0);
      }
    }
    return;
  }

  // ------------------------------ consumers ------------------------------
  setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const int g = lane >> 2;                                   // fragment rows lr and lr + 8
  const int cq = 2 * (lane & 3);                             // fragment columns 8 j + cq + {0, 1}
  const int lr = 64 * wg + 16 * (warp & 3) + g;              // local output row of this thread's first fragment row
  mbar_wait_a(x_bar, 0);

  float acc[64];
  int it = 0;
  for (int conv = 0; conv < p.n_convs; ++conv) {
    for (int j = 0; j < chunks; ++j, ++it) {
      const int s = it % kStages;
      mbar_wait_a(full_bar + 8 * s, (it / kStages) & 1);
      const int tap = j >> 1, half = j & 1;
      const int r = lr + tap;                                // region A row of output row lr at this tap
      const uint32_t a_hi = smem + (2 * half) * kSubBytes + r * kSwizzleBytes + 4 * (lane & 3);
      const uint32_t a_lo = a_hi + kSubBytes;
      const int sw = r & 7;                                  // 128-B swizzle: 16-B chunk q of row r sits at q ^ (r & 7)
      uint32_t fh[4][4], fl[4][4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t o0 = ((2 * k) ^ sw) << 4, o1 = ((2 * k + 1) ^ sw) << 4;
        fh[k][0] = lds_u32(a_hi + o0);
        fh[k][1] = lds_u32(a_hi + 8 * kSwizzleBytes + o0);
        fh[k][2] = lds_u32(a_hi + o1);
        fh[k][3] = lds_u32(a_hi + 8 * kSwizzleBytes + o1);
        fl[k][0] = lds_u32(a_lo + o0);
        fl[k][1] = lds_u32(a_lo + 8 * kSwizzleBytes + o0);
        fl[k][2] = lds_u32(a_lo + o1);
        fl[k][3] = lds_u32(a_lo + 8 * kSwizzleBytes + o1);
      }
      const uint32_t st = ring + s * kStageBytes;
      const uint64_t b_hi = make_smem_desc_sw128(st), b_lo = make_smem_desc_sw128(st + kWPlaneBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        wgmma_rs_n128(acc, fh[k], b_hi + desc_kstep(k), (j | k) != 0);
        wgmma_rs_n128(acc, fl[k], b_hi + desc_kstep(k), 1);
        wgmma_rs_n128(acc, fh[k], b_lo + desc_kstep(k), 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(acc);
      __syncwarp();
      if (lane == 0) mbar_arrive_a(empty_bar + 8 * s);       // this warp is done reading the stage
    }

    // h = BN(relu(acc + bias)), in place
    const float* bias = conv == 0 ? p.bias[0] : p.bias[1];      // constant indices: the parameter block stays out of local memory
    const float* scale = conv == 0 ? p.scale[0] : p.scale[1];
    const float* shift = conv == 0 ? p.shift[0] : p.shift[1];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + cq));
      const float2 sv = __ldg(reinterpret_cast<const float2*>(scale + 8 * j + cq));
      const float2 tv = __ldg(reinterpret_cast<const float2*>(shift + 8 * j + cq));
      acc[4 * j + 0] = fmaf(fmaxf(acc[4 * j + 0] + bv.x, 0.f), sv.x, tv.x);
      acc[4 * j + 1] = fmaf(fmaxf(acc[4 * j + 1] + bv.y, 0.f), sv.y, tv.y);
      acc[4 * j + 2] = fmaf(fmaxf(acc[4 * j + 2] + bv.x, 0.f), sv.x, tv.x);
      acc[4 * j + 3] = fmaf(fmaxf(acc[4 * j + 3] + bv.y, 0.f), sv.y, tv.y);
    }

    if (conv + 1 < p.n_convs) {
      // the intermediate replaces x in region A (row i = sequence row r0 + i); zero outside [0, len)
      named_bar_sync(1, kConsumerThreads);                   // both warpgroups are done reading x
#pragma unroll
      for (int half8 = 0; half8 < 2; ++half8) {
        const int rr = lr + 8 * half8;
        const int grow = r0 + rr;
        const bool live = grow >= 0 && grow < len;
        const uint32_t base = smem + rr * kSwizzleBytes + 4 * (lane & 3);
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          uint32_t hi, lo;
          split_pair(live ? acc[4 * j + 2 * half8] : 0.f, live ? acc[4 * j + 2 * half8 + 1] : 0.f, hi, lo);
          const uint32_t a = base + (2 * (j >> 3)) * kSubBytes + (((j & 7) ^ (rr & 7)) << 4);
          sts_u32(a, hi);
          sts_u32(a + kSubBytes, lo);
        }
      }
      named_bar_sync(1, kConsumerThreads);                   // the intermediate is complete
      continue;
    }

    // y = x + h on the tile's output rows; rows in [len, t) are written as zeros
#pragma unroll
    for (int half8 = 0; half8 < 2; ++half8) {
      const int o = lr + 8 * half8;
      const int t = t0 + o;
      if (o >= p.out_rows || t >= p.t) continue;
      const bool live = t < len;
      const long long off = (row0 + t) * kC + cq;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float2 v = make_float2(0.f, 0.f);
        if (live) {
          const float2 xv = __ldg(reinterpret_cast<const float2*>(p.x + off + 8 * j));
          v = make_float2(xv.x + acc[4 * j + 2 * half8], xv.y + acc[4 * j + 2 * half8 + 1]);
        }
        *reinterpret_cast<float2*>(p.y + off + 8 * j) = v;
        uint32_t hi, lo;
        split_pair(v.x, v.y, hi, lo);
        *reinterpret_cast<uint32_t*>(p.y_hi + off + 8 * j) = hi;
        *reinterpret_cast<uint32_t*>(p.y_lo + off + 8 * j) = lo;
      }
    }
  }
}

}  // namespace ss
}  // namespace pk

extern "C" int pk_ss_residual_block(const pk_ss_residual_block_args* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::ss;
  PK_CHECK_ARG(a != nullptr, "args is NULL");
  if (a->channels != kC)
    return pk::fail(PK_ERR_UNSUPPORTED, "pk_ss_residual_block: channels must be %d (got %d)", kC, a->channels);
  PK_CHECK_ARG(a->batch > 0 && a->t > 0, "batch and t must be > 0");
  PK_CHECK_ARG(a->n_convs == 1 || a->n_convs == 2, "n_convs must be 1 or 2 (got %d)", a->n_convs);
  PK_CHECK_ARG(a->taps >= 1 && a->taps <= kMaxTaps, "taps must be in [1, %d] (got %d)", kMaxTaps, a->taps);
  PK_CHECK_ARG(a->pad_left >= 0 && a->pad_left < a->taps, "pad_left must be in [0, taps) (got %d)", a->pad_left);
  PK_CHECK_ARG(a->x && a->x_hi && a->x_lo && a->y && a->y_hi && a->y_lo, "x / y and their planes must be non-NULL");
  PK_CHECK_ARG(a->w1_hi && a->w1_lo && a->bias1 && a->scale1 && a->shift1, "first conv operands must be non-NULL");
  PK_CHECK_ARG(a->n_convs == 1 || (a->w2_hi && a->w2_lo && a->bias2 && a->scale2 && a->shift2),
               "second conv operands must be non-NULL");
  PK_CHECK_ARG(aligned16(a->x_hi) && aligned16(a->x_lo) && aligned16(a->w1_hi) && aligned16(a->w1_lo) &&
                   (a->n_convs == 1 || (aligned16(a->w2_hi) && aligned16(a->w2_lo))),
               "operand planes must be 16-byte aligned");
  PK_CHECK_ARG(a->x != static_cast<const float*>(a->y), "y must not alias x (neighbouring tiles read x's halo rows)");
  CUtensorMap tx_hi, tx_lo, tw1_hi, tw1_lo, tw2_hi, tw2_lo;
  const uint64_t t = static_cast<uint64_t>(a->t), wcols = static_cast<uint64_t>(a->taps) * kC;
  int rc;
  if ((rc = pk::encode_tmap_bf16_3d(&tx_hi, a->x_hi, kC, t, a->batch, kC, t * kC, kRowsA))) return rc;
  if ((rc = pk::encode_tmap_bf16_3d(&tx_lo, a->x_lo, kC, t, a->batch, kC, t * kC, kRowsA))) return rc;
  if ((rc = pk::encode_tmap_bf16_3d(&tw1_hi, a->w1_hi, wcols, kC, 1, wcols, wcols * kC, kC))) return rc;
  if ((rc = pk::encode_tmap_bf16_3d(&tw1_lo, a->w1_lo, wcols, kC, 1, wcols, wcols * kC, kC))) return rc;
  if (a->n_convs == 2) {
    if ((rc = pk::encode_tmap_bf16_3d(&tw2_hi, a->w2_hi, wcols, kC, 1, wcols, wcols * kC, kC))) return rc;
    if ((rc = pk::encode_tmap_bf16_3d(&tw2_lo, a->w2_lo, wcols, kC, 1, wcols, wcols * kC, kC))) return rc;
  } else {
    tw2_hi = tw1_hi;
    tw2_lo = tw1_lo;
  }
  if ((rc = prepare_kernel(ss_residual_block_kernel, kThreads, kSmemBytes))) return rc;
  Args p;
  p.t = a->t;
  p.n_convs = a->n_convs;
  p.taps = a->taps;
  p.pad_left = a->pad_left;
  p.out_rows = a->n_convs == 2 ? kTileRows - (a->taps - 1) : kTileRows;
  p.lens = a->lens;
  p.x = a->x;
  p.bias[0] = a->bias1; p.scale[0] = a->scale1; p.shift[0] = a->shift1;
  p.bias[1] = a->bias2; p.scale[1] = a->scale2; p.shift[1] = a->shift2;
  p.y = a->y;
  p.y_hi = static_cast<__nv_bfloat16*>(a->y_hi);
  p.y_lo = static_cast<__nv_bfloat16*>(a->y_lo);
  const dim3 grid((a->t + p.out_rows - 1) / p.out_rows, a->batch);
  ss_residual_block_kernel<<<grid, kThreads, kSmemBytes, static_cast<cudaStream_t>(stream)>>>(tx_hi, tx_lo, tw1_hi, tw1_lo, tw2_hi,
                                                                                              tw2_lo, p);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}
