// pk_fused_attention: MultiHeadedAttention.forward_attention of the FFT blocks (reference: parakeet/modules/
// fastspeech2_transformer/attention.py:88-131) as ONE kernel per layer - scores, key-padding mask, softmax and P.V never
// leave the SM (round 1 ran four launches per layer around an fp32 (B*H, T, T) score tensor in HBM).
//
//   S   = Q K^T                       wgmma, split-bf16 operands (3 passes), fp32 in registers           [128 q x 128 keys]
//   P   = exp2((S - m) * scale*log2e) running row max m / row sum l (online softmax), keys >= key_len -> 0 (masked_fill)
//   O   = O * alpha + P V             P (packed bf16x2, hi | lo) stays in registers and is the A operand of the second
//                                     GEMM straight from there; V^T tiles (K-major) come from pk_transpose_heads
//   ctx = O / l                       split planes (B, T, A), heads merged (attention.py:126-129)
//
// Generalised for TransformerTTS's decoder (pk_fused_attention_ex): Q and K may come from different split buffers with their own
// row counts (cross attention: t_q query rows over t_k encoder rows), and `causal` masks keys j > i and skips the key tiles wholly
// above the diagonal.  pk_fused_attention (FastSpeech2's self-attention over one (B, T, 3A) buffer) is the special case Q = K
// buffer, q columns at 0, k columns at A, t_q = t_k, not causal: it runs the same instructions on the same data as before.
//
// One CTA per (utterance, head, 128-query tile); K and V^T tiles of 128 keys stream through one 96 KB buffer, Q (96 KB for
// d_k = 192) stays resident.  Roles: warps 0-7 two consumer warpgroups of 64 query rows each (S = Q K^T with wgmma into
// registers, online softmax in registers, P as the register A operand of P.V, O in registers), warps 8-11 the producer
// warpgroup (one TMA lane).  The attention FLOPs of FastSpeech2 are tiny (T <= ~1 400, 2 heads); the point of the kernel is
// to remove the HBM round trips and the launches, so the K / V phases of a tile are serialised rather than double-buffered.
#include "pk_host.h"
#include "pk_sm90.cuh"

namespace pk {
namespace attn {

constexpr int kTile = 128 * kSwizzleBytes;            // 16 KB: one plane of a 128-row K-chunk
constexpr int kChunkBytes = 2 * kTile;                // hi | lo
constexpr int kMaxDkc = 3;                            // d_k <= 192
constexpr int kBufBytes = kMaxDkc * kChunkBytes;      // 96 KB: Q, and the K / V^T stream buffer
constexpr int kSmem = 2 * kBufBytes + 1024 + 128;
static_assert(kSmem <= 227 * 1024, "shared memory budget");
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;

struct Args {
  int batch, t_q, t_k, heads, dkc, a_dim;   // dkc = d_k / 64, a_dim = heads * d_k (the ctx row width)
  int q_col0, k_col0, causal;           // Q of head h at column q_col0 + h d_k of tm_q, K at k_col0 + h d_k of tm_k
  const int32_t* key_lens;              // keys >= key_lens[b] are masked (NULL: all t_k keys)
  const int32_t* row_lens;              // query rows >= row_lens[b] are written as zero (NULL: all t_q rows)
  float scale_log2e;                    // 1/sqrt(d_k) * log2(e)
  __nv_bfloat16* ctx_hi;
  __nv_bfloat16* ctx_lo;
};

template <int DK>
__device__ __forceinline__ void wgmma_rs_o(float (&d)[DK / 2], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
  if constexpr (DK == 64) wgmma_rs_n64(d, a, b, acc);
  else if constexpr (DK == 128) wgmma_rs_n128(d, a, b, acc);
  else wgmma_rs_n192(d, a, b, acc);
}

template <int DKC>
__global__ void __launch_bounds__(kThreads, 1)
fused_attention_kernel(const __grid_constant__ CUtensorMap tm_q,       // (cols, t_q, B, 2 planes): box 64 x 128 rows x both planes
                       const __grid_constant__ CUtensorMap tm_k,       // (cols, t_k, B, 2 planes): box 64 x 128 rows x both planes
                       const __grid_constant__ CUtensorMap tm_vt,      // (Tp, d_k, B*H, 2 planes): box 64 keys x d_k rows x both planes
                       const Args p) {
  constexpr int dk = DKC * 64;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t qbuf = smem, kvbuf = smem + kBufBytes;
  const uint32_t bars = kvbuf + kBufBytes;
  const uint32_t q_full = bars, kv_full = bars + 8, kv_empty = bars + 16;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * 128;
  const int rows_live = p.row_lens ? min(__ldg(p.row_lens + b), p.t_q) : p.t_q;
  const int klen = p.key_lens ? min(__ldg(p.key_lens + b), p.t_k) : p.t_k;
  int nkv = (q0 < rows_live) ? (klen + 127) >> 7 : 0;                  // no valid query row / no valid key: the tile is zeros
  if (p.causal) nkv = min(nkv, qt + 1);                                // key tiles past the tile's last row are wholly masked
  constexpr uint32_t chunk_bytes = kChunkBytes;
  constexpr uint32_t vchunk = static_cast<uint32_t>(dk) * kSwizzleBytes;   // one plane of a V^T key chunk: d_k rows x 128 B

  if (threadIdx.x == kConsumerThreads) {
    tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_k); tma_prefetch_desc(&tm_vt);
    mbar_init_a(q_full, 1); mbar_init_a(kv_full, 1); mbar_init_a(kv_empty, kConsumerThreads / 32);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    setmaxnreg_dec<40>();
    if (warp == kConsumerThreads / 32 && lane == 0 && nkv > 0) {
      // ------------------------------ TMA producer ------------------------------
      mbar_arrive_expect_tx_a(q_full, DKC * chunk_bytes);
      for (int c = 0; c < DKC; ++c) tma_load_4d_a(qbuf + c * chunk_bytes, &tm_q, q_full, p.q_col0 + h * dk + c * 64, q0, b, 0);
      uint32_t n = 0;                                            // uses of the stream buffer
      for (int j = 0; j < nkv; ++j) {
        mbar_wait_a(kv_empty, (n & 1) ^ 1);
        mbar_arrive_expect_tx_a(kv_full, DKC * chunk_bytes);     // K tile: keys [128 j, +128) x d_k
        for (int c = 0; c < DKC; ++c) tma_load_4d_a(kvbuf + c * chunk_bytes, &tm_k, kv_full, p.k_col0 + h * dk + c * 64, j * 128, b, 0);
        ++n;
        mbar_wait_a(kv_empty, (n & 1) ^ 1);
        mbar_arrive_expect_tx_a(kv_full, 2 * 2 * vchunk);        // V^T tile: d_k rows x keys [128 j, +128) as two 64-key chunks
        for (int kc = 0; kc < 2; ++kc) tma_load_4d_a(kvbuf + kc * 2 * vchunk, &tm_vt, kv_full, j * 128 + kc * 64, 0, b * p.heads + h, 0);
        ++n;
      }
    }
  } else {
    // ------------------ consumers: 64 query rows per warpgroup; this thread holds rows r0 and r0 + 8 ------------------
    setmaxnreg_inc<232>();
    const int wg = warp >> 2;
    const int r0 = wg * 64 + 16 * (warp & 3) + (lane >> 2);   // row inside the tile
    const int cq = 2 * (lane & 3);                            // first of this thread's two columns in each 8-column group
    // key kk is live for this thread's row hh (0: r0, 1: r0 + 8): inside the key length and, when causal, not after the row
    const int row0 = q0 + r0;
    auto live_key = [&](int kk, int hh) { return kk < klen && (!p.causal || kk <= row0 + 8 * hh); };
    float o[dk / 2];
#pragma unroll
    for (int i = 0; i < dk / 2; ++i) o[i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
    if (nkv > 0) mbar_wait_a(q_full, 0);
    uint32_t n = 0;
    for (int j = 0; j < nkv; ++j) {
      const int kv0 = j * 128;
      float s[64];
      mbar_wait_a(kv_full, n & 1); ++n;
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < DKC; ++c) {
        const uint64_t a_hi = make_smem_desc_sw128(qbuf + c * chunk_bytes + wg * 64 * kSwizzleBytes);
        const uint64_t a_lo = make_smem_desc_sw128(qbuf + c * chunk_bytes + kTile + wg * 64 * kSwizzleBytes);
        const uint64_t b_hi = make_smem_desc_sw128(kvbuf + c * chunk_bytes), b_lo = make_smem_desc_sw128(kvbuf + c * chunk_bytes + kTile);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_ss_n128(s, a_hi + desc_kstep(k), b_hi + desc_kstep(k), !(c == 0 && k == 0));
          wgmma_ss_n128(s, a_lo + desc_kstep(k), b_hi + desc_kstep(k), 1);
          wgmma_ss_n128(s, a_hi + desc_kstep(k), b_lo + desc_kstep(k), 1);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      __syncwarp();
      if (lane == 0) mbar_arrive_a(kv_empty);                    // the K tile may be overwritten by V^T
      // online softmax over this tile's keys (row max / sum across the 4 lanes of a quad)
      float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (live_key(kv0 + 8 * jj + cq + (e & 1), e >> 1)) tmax[e >> 1] = fmaxf(tmax[e >> 1], s[4 * jj + e]);
      }
      float alpha[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        tmax[hh] = fmaxf(tmax[hh], __shfl_xor_sync(0xffffffffu, tmax[hh], 1));
        tmax[hh] = fmaxf(tmax[hh], __shfl_xor_sync(0xffffffffu, tmax[hh], 2));
        // finite: tile 0 holds key 0, live for every row; a later causal tile with no live key for a row leaves m (alpha = 1)
        const float m_new = fmaxf(m[hh], tmax[hh]);
        alpha[hh] = ex2_approx((m[hh] - m_new) * p.scale_log2e);   // 0 on the first tile (m = -inf)
        m[hh] = m_new;
      }
#pragma unroll
      for (int i = 0; i < dk / 8; ++i) {
        o[4 * i] *= alpha[0]; o[4 * i + 1] *= alpha[0]; o[4 * i + 2] *= alpha[1]; o[4 * i + 3] *= alpha[1];
      }
      float lsum[2] = {0.f, 0.f};
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float v = live_key(kv0 + 8 * jj + cq + (e & 1), e >> 1) ? ex2_approx((s[4 * jj + e] - m[e >> 1]) * p.scale_log2e) : 0.f;
          s[4 * jj + e] = v;
          lsum[e >> 1] += v;
        }
      }
      l[0] = l[0] * alpha[0] + lsum[0];
      l[1] = l[1] * alpha[1] + lsum[1];
      // O += P V^T-tile: two 64-key chunks, 4 K-steps each; P hi / lo packed from the S fragments
      mbar_wait_a(kv_full, n & 1); ++n;
#pragma unroll
      for (int kc = 0; kc < 2; ++kc) {
        uint32_t ph[4][4], pl[4][4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int kk = 4 * kc + k;                 // keys [16 kk, 16 kk + 16) = S column groups 2 kk, 2 kk + 1
          split2(s[8 * kk + 0], s[8 * kk + 1], ph[k][0], pl[k][0]);
          split2(s[8 * kk + 2], s[8 * kk + 3], ph[k][1], pl[k][1]);
          split2(s[8 * kk + 4], s[8 * kk + 5], ph[k][2], pl[k][2]);
          split2(s[8 * kk + 6], s[8 * kk + 7], ph[k][3], pl[k][3]);
        }
        const uint64_t b_hi = make_smem_desc_sw128(kvbuf + kc * 2 * vchunk), b_lo = make_smem_desc_sw128(kvbuf + kc * 2 * vchunk + vchunk);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_rs_o<dk>(o, ph[k], b_hi + desc_kstep(k), 1);
          wgmma_rs_o<dk>(o, pl[k], b_hi + desc_kstep(k), 1);
          wgmma_rs_o<dk>(o, ph[k], b_lo + desc_kstep(k), 1);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(o);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive_a(kv_empty);
    }
    // epilogue: ctx[b, q0 + r, h d_k + :] = O / l (zeros for rows / tiles without valid queries or keys)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
      l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const int row = q0 + r0 + 8 * hh;
      const bool live = nkv > 0 && row < rows_live;
      const float inv = live ? 1.f / l[hh] : 0.f;
      if (row < p.t_q) {
        const long long off = (static_cast<long long>(b) * p.t_q + row) * p.a_dim + h * dk + cq;
#pragma unroll
        for (int i = 0; i < dk / 8; ++i) {
          uint32_t wh, wl;
          split2(live ? o[4 * i + 2 * hh] * inv : 0.f, live ? o[4 * i + 2 * hh + 1] * inv : 0.f, wh, wl);
          *reinterpret_cast<uint32_t*>(p.ctx_hi + off + 8 * i) = wh;
          *reinterpret_cast<uint32_t*>(p.ctx_lo + off + 8 * i) = wl;
        }
      }
    }
  }
}

}  // namespace attn
}  // namespace pk

extern "C" int pk_fused_attention_ex(const PkAttentionArgs* a, pk_stream_t stream) {
  using namespace pk;
  using namespace pk::attn;
  PK_CHECK_ARG(a != nullptr, "NULL arguments");
  PK_CHECK_ARG(a->q_hi && a->q_lo && a->k_hi && a->k_lo && a->vt_hi && a->vt_lo && a->ctx_hi && a->ctx_lo, "NULL pointer");
  const int dk = a->dk;
  PK_CHECK_ARG(a->batch > 0 && a->t_q > 0 && a->t_k > 0 && a->heads > 0 && dk >= 64 && dk <= 64 * kMaxDkc && (dk % 64) == 0,
               "d_k must be 64, 128 or 192");
  PK_CHECK_ARG(a->tp >= a->t_k && (a->tp % 8) == 0, "the V^T row pitch must cover t_k and be a multiple of 8");
  PK_CHECK_ARG(!a->causal || a->t_q == a->t_k, "causal attention needs t_q == t_k");
  const int a_dim = a->heads * dk;
  PK_CHECK_ARG(a->q_col0 >= 0 && a->k_col0 >= 0 && a->q_col0 + a_dim <= a->q_ld && a->k_col0 + a_dim <= a->k_ld && a->q_ld % 8 == 0 &&
               a->k_ld % 8 == 0, "Q / K head columns must lie inside rows whose pitch is a multiple of 8");
  PK_CHECK_ARG((reinterpret_cast<uintptr_t>(a->ctx_hi) & 31) == 0 && (reinterpret_cast<uintptr_t>(a->ctx_lo) & 31) == 0 && (a_dim % 16) == 0,
               "ctx planes must be 32-byte aligned");
  CUtensorMap tq, tk, tv;
  int rc;
  if ((rc = encode_tmap_bf16_planes(&tq, a->q_hi, a->q_lo, a->q_ld, a->t_q, a->batch, a->q_ld, static_cast<uint64_t>(a->t_q) * a->q_ld, 128)))
    return rc;
  if ((rc = encode_tmap_bf16_planes(&tk, a->k_hi, a->k_lo, a->k_ld, a->t_k, a->batch, a->k_ld, static_cast<uint64_t>(a->t_k) * a->k_ld, 128)))
    return rc;
  if ((rc = encode_tmap_bf16_planes(&tv, a->vt_hi, a->vt_lo, a->tp, dk, static_cast<uint64_t>(a->batch) * a->heads, a->tp,
                                    static_cast<uint64_t>(dk) * a->tp, dk)))
    return rc;
  const int dkc = dk / 64;
  static decltype(&fused_attention_kernel<1>) const kernels[kMaxDkc] = {fused_attention_kernel<1>, fused_attention_kernel<2>,
                                                                        fused_attention_kernel<3>};
  const auto kernel = kernels[dkc - 1];
  if ((rc = prepare_kernel(kernel, kThreads, kSmem))) return rc;
  Args p;
  p.batch = a->batch; p.t_q = a->t_q; p.t_k = a->t_k; p.heads = a->heads; p.dkc = dkc; p.a_dim = a_dim;
  p.q_col0 = a->q_col0; p.k_col0 = a->k_col0; p.causal = a->causal ? 1 : 0;
  p.key_lens = a->key_lens; p.row_lens = a->row_lens;
  p.scale_log2e = a->scale * 1.4426950408889634f;
  p.ctx_hi = static_cast<__nv_bfloat16*>(a->ctx_hi); p.ctx_lo = static_cast<__nv_bfloat16*>(a->ctx_lo);
  dim3 grid((a->t_q + 127) / 128, a->heads, a->batch);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  kernel<<<grid, kThreads, kSmem, st>>>(tq, tk, tv, p);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

// FastSpeech2's self-attention over one (B, T, 3A) qkv buffer
extern "C" int pk_fused_attention(const void* qkv_hi, const void* qkv_lo, const void* vt_hi, const void* vt_lo, int32_t batch, int32_t t,
                                  int32_t heads, int32_t dk, int32_t tp, const int32_t* key_lens, const int32_t* row_lens, float scale,
                                  void* ctx_hi, void* ctx_lo, pk_stream_t stream) {
  PK_CHECK_ARG(heads > 0 && dk > 0, "heads and d_k must be positive");
  PkAttentionArgs a = {};
  a.q_hi = qkv_hi; a.q_lo = qkv_lo; a.k_hi = qkv_hi; a.k_lo = qkv_lo; a.vt_hi = vt_hi; a.vt_lo = vt_lo;
  a.batch = batch; a.t_q = t; a.t_k = t; a.heads = heads; a.dk = dk; a.tp = tp;
  a.q_ld = 3 * heads * dk; a.k_ld = 3 * heads * dk; a.q_col0 = 0; a.k_col0 = heads * dk; a.causal = 0;
  a.key_lens = key_lens; a.row_lens = row_lens; a.scale = scale; a.ctx_hi = ctx_hi; a.ctx_lo = ctx_lo;
  return pk_fused_attention_ex(&a, stream);
}
