/* parakeet_b200 C-ABI: H100 (sm_90a) kernels for the Parakeet TTS hot path.
 *
 * The reference (PaddlePaddle/Parakeet) has no FFI of its own: its hot path is Python calling paddle.nn ops.
 * This header is the boundary a Parakeet maintainer would bind instead of those ops (ctypes stub in
 * INTEGRATION.md).  Every entry point names the reference call site (file:line under /root/reference) it replaces.
 *
 * Rules (SURVEY.md 8b):
 *   - plain C: raw device pointers, sizes, a cudaStream_t passed as void*; no torch / C++ types;
 *   - the caller owns every buffer (inputs, outputs, workspaces); the library owns nothing but its code;
 *   - every function returns 0 (PK_OK) or a negative error code, never throws, never aborts, never falls back to
 *     a CPU path; pk_last_error() returns a thread-local message for the last failing call;
 *   - all work is enqueued on the caller's stream; no internal synchronisation unless documented;
 *   - parakeet_b200/_lib.py builds its ctypes binding from this file: argument structs are `typedef struct ... { } NAME;`,
 *     constants `#define PK_* n` or `enum { PK_* = n }`, and every type is one of those its type map lists.
 *
 * Number format of GEMM operands ("split-bf16"): an fp32 tensor v is carried as two bf16 planes
 * hi = bf16(v), lo = bf16(v - hi).  Producers in this library write both planes; pk_split_f32 converts.
 */
#ifndef PARAKEET_B200_H_
#define PARAKEET_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PK_OK 0
#define PK_ERR_INVALID_ARG (-1)
#define PK_ERR_CUDA (-2)
#define PK_ERR_UNSUPPORTED (-3)

#define PK_ACT_NONE 0
#define PK_ACT_RELU 1
#define PK_ACT_TANH 2

typedef void* pk_stream_t; /* cudaStream_t */

/* Library version (major*10000 + minor*100 + patch). */
int pk_version(void);
/* Thread-local description of the last error returned on this thread ("" if none). */
const char* pk_last_error(void);
/* Number of kernels this library has launched in this process (bench.py's gpu_launches claim). */
int64_t pk_launch_count(void);

/* fp32 -> split-bf16 planes; n elements (any layout, element-wise). */
int pk_split_f32(const float* x, void* hi, void* lo, int64_t n, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Generic channels-last Conv1D / Linear / batched-matmul on wgmma tensor cores.
 *
 *   y[z, t, n] = act( scale * sum_{tap, k} A[za, t + (tap - pad) * dil, a_col + k] * B[zb, n, b_col + tap*Kp + k]
 *                     + bias[n] ) + residual[z, t, n]          ; rows t >= lens[b] are written as 0
 *
 * with z = b * heads + h, za = b * a_bmul + h * a_hmul, a_col = a_col0 + h * a_colh (same for B), Kp = K rounded
 * up to 64.  Rows / channels outside the declared extents read as zero (conv zero padding).
 *
 * Replaces, in the reference: nn.Linear call sites of MultiHeadedAttention (modules/fastspeech2_transformer/
 * attention.py:44-47,74-78,131), the two matmuls (:153-154,126), MultiLayeredConv1d (multi_layer_conv.py:47-77),
 * predictor Conv1D stacks (duration_predictor.py:69-83, variance_predictor.py:59-76), feat_out
 * (models/fastspeech2/fastspeech2.py:271,457) and Postnet convs (modules/tacotron2/decoder.py:128-180).
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct pk_operand {
  const void* hi;         /* bf16 plane */
  const void* lo;         /* bf16 plane, same layout */
  int64_t batch_stride;   /* elements between consecutive "batches" of the plane */
  int32_t ld;             /* elements between consecutive rows (multiple of 8) */
  int32_t rows;           /* rows per batch; rows outside [0, rows) read as zero */
  int32_t cols;           /* channels per row; channels outside [0, cols) read as zero */
  int32_t batches;        /* number of batches in the plane */
  int32_t bmul, hmul;     /* batch index used for (b, h) = b*bmul + h*hmul */
  int32_t col0, colh;     /* first channel used for head h = col0 + h*colh */
} pk_operand;

typedef struct pk_conv_gemm_args {
  pk_operand a;           /* activations: rows = time */
  pk_operand b;           /* weights [n][taps*Kp] (bmul = hmul = 0) or a per-(b,h) matrix [n][K] */
  int32_t batch, heads;   /* grid z = batch * heads */
  int32_t m;              /* output rows per batch (time steps) */
  int32_t n;              /* output channels */
  int32_t k;              /* input channels per tap */
  int32_t taps, dil, pad; /* Conv1D kernel size, dilation, left padding in taps ((taps-1)/2 for "same") */
  float scale;            /* applied to the accumulator before bias */
  const float* bias;      /* [n] or NULL */
  int32_t act;            /* PK_ACT_* */
  const float* residual;  /* fp32, indexed like y_f32, or NULL (added after act) */
  const int32_t* lens;    /* [batch] valid rows per batch or NULL */
  float* y_f32;           /* fp32 output or NULL */
  void* y_hi;             /* split-bf16 output planes or NULL (both or none) */
  void* y_lo;
  int64_t y_batch_stride; /* elements; y offset = b*y_batch_stride + h*y_head_stride + t*y_ld + n */
  int64_t y_head_stride;
  int32_t y_ld;
  int32_t passes;         /* 3 = split-bf16 (fp32-grade), 1 = plain bf16 (hi planes only) */
} pk_conv_gemm_args;

int pk_conv_gemm(const pk_conv_gemm_args* args, pk_stream_t stream);

/* pk_conv_gemm with a fused pair epilogue: the output row has n = 2 * channels columns, column c of the first half is
 * combined with column channels + c of the second half (bias and scale applied to both) and the GEMM result itself is
 * never written.  n <= 256, channels % 32 == 0, heads == 1; act / residual / lens of the base arguments must be unset.
 *   PK_EPI_GATE       z = tanh(a + res_a) * sigmoid(g + res_g) written as split planes y_hi / y_lo (batch, m, y_ld);
 *                     `residual` (fp32, batch stride / row pitch given, 2 * channels columns) may be NULL.  Fuses the gate of
 *                     waveflow.ResidualBlock (models/waveflow.py:277-281) into its dilated-conv GEMM.
 *   PK_EPI_WF_UPDATE  state (batch, m, channels) += a;  skip = skip_init ? g : skip + g;  the new state is also written as
 *                     split planes into buf_hi / buf_lo (batch, m, buf_ld) at column buf_col0 when given.  Fuses
 *                     `res, skip = split(out_proj(z))` (models/waveflow.py:282-294) and ResidualNet.add_input (:386-392). */
enum { PK_EPI_NONE = 0, PK_EPI_GATE = 1, PK_EPI_WF_UPDATE = 2 };
typedef struct pk_gemm_epilogue {
  int32_t mode;                  /* PK_EPI_* */
  int32_t channels;              /* C: n == 2 * C */
  const float* residual;         /* GATE */
  int64_t residual_batch_stride;
  int32_t residual_ld;
  int32_t skip_init;             /* WF_UPDATE */
  float* state;
  float* skip;
  void* buf_hi;
  void* buf_lo;
  int32_t buf_ld, buf_col0;
} pk_gemm_epilogue;
int pk_conv_gemm_ex(const pk_conv_gemm_args* args, const pk_gemm_epilogue* epilogue, pk_stream_t stream);

/* Same contract evaluated with plain fp32 FMAs (one thread per output element).  Debug / cross-check kernel for
 * the tensor-core path at sizes where the CPU oracle is too slow; not used by the models. */
int pk_conv_gemm_simt(const pk_conv_gemm_args* args, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Length regulator: integer repeat-expand, bit-exact row copies.
 *   y[b, cum[b,j] + r, :] = x[b, j, :] for 0 <= r < d[b,j];  rows >= sum_j d[b,j] are 0 up to t_out.
 * out_lens[b] = sum_j max(d[b,j],0)... (durations are clipped >= 0 upstream; negative d is rejected as in the
 * reference's reachable domain).  Replaces LengthRegulator.expand (modules/fastspeech2_predictor/
 * length_regulator.py:46-66): host numpy loop + 0/1-matrix matmul.
 * ------------------------------------------------------------------------------------------------------------ */
/* out_lens[b] = sum_j d[b, j] (int32), device-side; t_in tokens per utterance. */
int pk_length_regulator_lens(const int64_t* dur, int32_t batch, int32_t t_in, int32_t* out_lens, pk_stream_t stream);
/* x: fp32 (batch, t_in, c); y: fp32 (batch, t_out, c), optional split planes y_hi / y_lo (NULL to skip). */
int pk_length_regulate(const float* x, const int64_t* dur, int32_t batch, int32_t t_in, int32_t c, int32_t t_out,
                       float* y, void* y_hi, void* y_lo, pk_stream_t stream);


/* ------------------------------------------------------------------------------------------------------------
 * Parallel WaveGAN generator (reference: parakeet/models/parallel_wavegan/parallel_wavegan.py).
 * Activations are channels-last split-bf16 planes (B, T, C); conditioning c is (B, T, aux).
 * ------------------------------------------------------------------------------------------------------------ */
/* ConvInUpsampleNet.forward (:201-216) = conv_in (Conv1D aux->aux, k = 2*window+1, no padding, no bias) followed by
 * UpsampleNet.forward (:119-138): per scale s, nearest stretch x s (Stretch2D :48-63) then a (1, 2s+1) FIR with zero
 * padding s.  mel: device fp32 (batch, aux, frames + 2*window), channel-first like the reference;
 * conv_in_w: device fp32 [aux][aux][2*window+1]; fir: HOST fp32, the n_stages FIRs concatenated (2*s_k+1 taps each);
 * scales: HOST int32 [n_stages].  Outputs (either or BOTH may be NULL - then only conv_in_ws is produced, which is all the frame-rate path needs): c_f32 (batch, aux, T) channel-first fp32 and
 * c_hi/c_lo (batch, T, aux) channels-last split-bf16, T = frames * prod(scales).  frame_lens (device int32 [batch] or
 * NULL): valid frames per utterance of a ragged batch; each utterance is then upsampled exactly as if alone
 * (zero padding at its own end) and its samples past frame_lens[b]*hop are written as zero.
 * conv_in_ws: device fp32 workspace (batch, frames, aux) that receives the conv_in output (channels-last); aux % 8 == 0.
 * Two launches: conv_in per frame, then the fused stretch/FIR cascade. */
int pk_pwg_upsample(const float* mel, const float* conv_in_w, const float* fir, const int32_t* scales, int32_t n_stages,
                    int32_t batch, int32_t aux, int32_t frames, int32_t window, const int32_t* frame_lens,
                    float* conv_in_ws, float* c_f32, void* c_hi, void* c_lo, pk_stream_t stream);

/* first_conv (:401-402, :464): x[b,t,r] = w[r] * noise[b,t] + bias[r] for 64 residual channels, written as split
 * planes (batch, t, 64); rows t >= lens[b] are written as zero (lens may be NULL). */
int pk_pwg_first_conv(const float* noise, const float* w, const float* bias, const int32_t* lens, int32_t batch, int32_t t,
                      void* x_hi, void* x_lo, pk_stream_t stream);

/* One fused ResidualBlock.forward (:284-315) for residual = skip = 64 channels, gate = 128, kernel 3:
 *   h = conv_k3_dil(x) + b1 + conv1x1_aux(c);  z = tanh(h[:64]) * sigmoid(h[64:]);
 *   skip (+)= conv1x1_skip(z)   [its bias is added once, in pk_pwg_tail];  y = (conv1x1_out(z) + b_out + x) * sqrt(0.5)
 * w1: packed [128][5*64] K-major = taps 0..2 (64 ch each) then the aux weight zero-padded to 128 channels;
 * w2: packed [128][64], rows 0..63 = conv1x1_skip, rows 64..127 = conv1x1_out; bias1 [128]; bias2 = skip bias | out bias.
 * y must not alias x.  Rows t >= lens[b] of y are written as zero and tiles wholly past lens[b] are skipped
 * (their y rows must already be zero). */
typedef struct pk_pwg_layer_args {
  int32_t batch, t, dilation, aux_channels;
  const int32_t* lens;     /* [batch] valid samples or NULL */
  const void* x_hi;        /* input planes (batch, t, 64) */
  const void* x_lo;
  void* y_hi;              /* output planes (batch, t, 64) */
  void* y_lo;
  const void* c_hi;        /* conditioning planes (batch, t, aux_channels) */
  const void* c_lo;
  const void* w1_hi;
  const void* w1_lo;
  const void* w2_hi;
  const void* w2_lo;
  const float* bias1;      /* HOST pointer [128]: conv bias (gate a | gate g); copied into the kernel parameter block */
  const float* bias2;      /* HOST pointer [128]: conv1x1_skip bias (ignored, see pk_pwg_tail) | conv1x1_out bias */
  float* skip;             /* fp32 (batch, t, 64) running sum of skips */
  int32_t skip_init;       /* 1: overwrite (first layer), 0: accumulate */
} pk_pwg_layer_args;
int pk_pwg_residual_layer(const pk_pwg_layer_args* args, pk_stream_t stream);

/* ResidualBlock with FRAME-RATE CONDITIONING (the residual-stack path of the Python model wherever the compact band tables
 * are exact; other upsample scales run pk_pwg_residual_layer).  The upsampling network is linear and per channel, so
 * conv1x1_aux(upsample(m'))[t, n] = sum_j U[t, j] * P[j, n] with P = conv1x1_aux applied to m' = conv_in(mel) at FRAME
 * rate.  Instead of the sample-rate conditioning planes (1.2 GB at cfg 2) the kernel takes
 *   u_hi / u_lo: the COMPACT band table of U as split planes (u_rows, 64) from ONE allocation (lo after hi): a row holds
 *                U[t, j0 + k] in column k < 16 (zeros after), j0 = floor8(((t / 256) * 256) / hop - 2) (the K window of
 *                the 256-sample pair tile of t).  Rows [0, u_period): interior rows by t mod u_period; rows
 *                [u_start_row, +128): the first 128 samples of any utterance; rows [u_end_base + 384 b, +384): the half
 *                tiles of utterance b from 128 * ((len_b - 128) / 128) on (zero at and past len_b).  Built by
 *                parakeet_b200/models/_pwg_frame_cond.py: compact_band_tables (lookup: source_row).
 *   p_hi / p_lo: P as split planes (batch, p_rows, p_ld), one allocation, frames along the last axis (p_frames valid
 *                columns, zeros up to p_ld >= 64); this layer's 128 output channels are rows [p_row0, p_row0 + 128).
 * x / y planes: one allocation each (lo after hi) so that a tile of both planes is ONE 4-D TMA box.
 * w1 / w2 / bias1 / bias2 / skip / lens as in pk_pwg_layer_args (the aux columns of w1 are not read).  hop >= 256.
 *
 * The ends of the stack (at most one of noise / out is set; both NULL: a middle layer):
 *   FIRST LAYER (noise != NULL): x = first_conv(noise) = first_w * noise[b, t] + first_b is computed in place, never read
 *     from memory (x_hi / x_lo must be NULL) - its rows t >= lens[b] are zero as in pk_pwg_first_conv.  first_u / first_v
 *     [3][128] hold W1_tap . first_w and W1_tap . first_b per tap (the conv of x collapses to rank one per tap).
 *   LAST LAYER (out != NULL, skip_init == 0): instead of accumulating into skip, the epilogue applies pk_pwg_tail to
 *     skip + this layer's skip branch and writes out (batch, t) fp32; skip is read, not written.  y is written as usual.
 *     Rows t >= lens[b] of live tiles get 0; the tiles wholly past lens[b] do not write out at all.
 *     tail_w1_hi / lo: last_conv_layers.1 [64 out][64 in] split planes (16-byte aligned); tail_b1 [64], tail_w2 [64],
 *     tail_b2 [1], skip_bias [64] (the sum of all layers' conv1x1_skip biases) are HOST arrays; tail_scale = sqrt(1/layers). */
typedef struct pk_pwg_layer_fc_args {
  int32_t batch, t, dilation, hop;
  const int32_t* lens;
  const void* x_hi;
  const void* x_lo;
  void* y_hi;
  void* y_lo;
  const void* u_hi;
  const void* u_lo;
  int32_t u_rows, u_period, u_start_row, u_end_base;
  int32_t p_rows, p_ld, p_frames, p_row0;
  const void* p_hi;
  const void* p_lo;
  const void* w1_hi;
  const void* w1_lo;
  const void* w2_hi;
  const void* w2_lo;
  const float* bias1;      /* HOST pointers, as in pk_pwg_layer_args */
  const float* bias2;
  float* skip;
  int32_t skip_init;
  const float* noise;      /* first layer: device fp32 (batch, t), or NULL */
  const float* first_w;    /* HOST [64] */
  const float* first_b;    /* HOST [64] */
  const float* first_u;    /* HOST [3][128] */
  const float* first_v;    /* HOST [3][128] */
  float* out;              /* last layer: device fp32 (batch, t), or NULL */
  const void* tail_w1_hi;
  const void* tail_w1_lo;
  const float* tail_b1;    /* HOST [64] */
  const float* tail_w2;    /* HOST [64] */
  const float* tail_b2;    /* HOST [1] */
  const float* skip_bias;  /* HOST [64] */
  float tail_scale;
} pk_pwg_layer_fc_args;
int pk_pwg_residual_layer_fc(const pk_pwg_layer_fc_args* args, pk_stream_t stream);

/* last_conv_layers (:429-440) on the scaled skip sum (:469-471):
 *   out[row] = w2 . relu(W1 relu((skip[row] + skip_bias) * scale) + b1) + b2
 * with skip fp32 (rows, 64), W1 [64 out][64 in], w2 [64]; out fp32 (rows).  skip_bias [64] (or NULL) is the sum of the
 * layers' conv1x1_skip biases: pk_pwg_residual_layer accumulates the skip branch WITHOUT its bias (bias2[0..63] is
 * ignored there) and the constant vector is added once here. */
int pk_pwg_tail(const float* skip, const float* skip_bias, const float* w1, const float* b1, const float* w2, const float* b2,
                float scale, int64_t rows, float* out, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * FastSpeech2 row-wise kernels (reference: parakeet/models/fastspeech2/fastspeech2.py and the files under parakeet/modules).
 * Shapes are (batch, t, channels) channels-last fp32 unless noted.  `lens` (device int32 [batch] or NULL) selects
 * the "independent utterances" mode used for batched inference: rows t >= lens[b] are written as zero so that every
 * utterance sees exactly the zero padding it would see alone; with lens == NULL padded rows are computed like any
 * other row, which is what the reference's batched training forward does.
 * ------------------------------------------------------------------------------------------------------------ */
/* Embedding(padding_idx) + ScaledPositionalEncoding (modules/fastspeech2_transformer/embedding.py:46-62,111-126;
 * encoder.py:103-105): y = (ids ? table[ids] (zeros for padding_idx) : x_in) + alpha[0] * PE. */
int pk_embed_pe(const int64_t* ids, const float* table, int32_t vocab, int32_t padding_idx, const float* x_in,
                const float* alpha, const int32_t* lens, int32_t batch, int32_t t, int32_t d, float* y, pk_stream_t stream);
/* nn.LayerNorm over the last dim (encoder_layer.py:55-56,85,107; encoder.py:143,191; modules/layer_norm.py:47-63).
 * Outputs: y fp32 and/or split planes (either may be NULL). */
int pk_layer_norm(const float* x, const float* gamma, const float* beta, float eps, const int32_t* lens, int32_t batch,
                  int32_t t, int32_t d, float* y, void* y_hi, void* y_lo, pk_stream_t stream);
/* masked_fill(min) -> softmax -> masked_fill(0) of attention.py:107-119 over keys: s fp32 (batch*heads, rows, ld) -> p split
 * planes, same layout.  Query row i of utterance b attends keys j < key_lens[b] (key_lens NULL: all `keys`) and, when
 * causal != 0, j <= i (the TransformerTTS decoder's self-attention mask); the other keys and the padding columns [keys, ld)
 * get probability 0, and a row with no key left is zeros. */
int pk_masked_softmax(const float* s, const int32_t* key_lens, int32_t batch, int32_t heads, int32_t rows, int32_t keys,
                      int32_t ld, int32_t causal, void* p_hi, void* p_lo, pk_stream_t stream);
/* paddle.nn.functional.normalize(x, p=2, axis=1, epsilon) on x viewed as (outer, n, inner), norm over the middle axis: the
 * speaker / tone embedding normalisation of FastSpeech2 (fastspeech2.py:577,581,606,611; axis 1 of a (B, T, D) tone tensor is
 * TIME in the reference's batched forward).  x, y fp32 contiguous; in place allowed. */
int pk_l2_normalize(const float* x, int32_t outer, int32_t n, int32_t inner, float eps, float* y, pk_stream_t stream);
/* Fused scaled-dot-product attention of an FFT block (attention.py:88-131: scores = q k^T / sqrt(d_k), masked_fill(min) ->
 * softmax -> masked_fill(0), p_attn . v, heads merged) in one kernel: scores and probabilities stay in registers.
 *   qkv planes (batch, t, 3 * heads * dk): [q | k | v] of the fused QKV projection, head h in columns h * dk of each third;
 *   vt planes (batch * heads, dk, tp): v transposed per head (pk_transpose_heads), columns >= t zero; both pairs of planes
 *   from one allocation each (lo after hi).  key_lens / row_lens: device int32 [batch] or NULL (keys >= key_lens[b] masked;
 *   query rows >= row_lens[b] written as zero).  ctx planes (batch, t, heads * dk).  dk in {64, 128, 192}. */
int pk_fused_attention(const void* qkv_hi, const void* qkv_lo, const void* vt_hi, const void* vt_lo, int32_t batch, int32_t t,
                       int32_t heads, int32_t dk, int32_t tp, const int32_t* key_lens, const int32_t* row_lens, float scale,
                       void* ctx_hi, void* ctx_lo, pk_stream_t stream);
/* pk_fused_attention_ex: the generalised fused attention.  Q of head h = columns q_col0 + h dk of the split buffer q (batch, t_q,
 * q_ld); K = columns k_col0 + h dk of k (batch, t_k, k_ld); V^T (batch * heads, dk, tp) from pk_transpose_heads, tp >= t_k.
 * ctx (batch, t_q, heads dk) = softmax(scale q k^T, keys >= key_lens[b] masked, with `causal` also keys j > i) v.  Query rows
 * >= row_lens[b] are written as zero (NULL: every row is computed, padded rows included).  causal needs t_q == t_k.  d_k 64 / 128 /
 * 192; q_ld, k_ld multiples of 8. */
typedef struct {
  const void* q_hi; const void* q_lo; const void* k_hi; const void* k_lo; const void* vt_hi; const void* vt_lo;
  int32_t batch, t_q, t_k, heads, dk, tp, q_ld, k_ld, q_col0, k_col0, causal;
  const int32_t* key_lens; const int32_t* row_lens;
  float scale;
  void* ctx_hi; void* ctx_lo;
} PkAttentionArgs;
int pk_fused_attention_ex(const PkAttentionArgs* args, pk_stream_t stream);
/* (batch, t, ld_src)[.., col0 + h*dk + d] -> (batch*heads, dk, ld_dst)[.., d, t] (zero-filled for t in [t, ld_dst)):
 * the value matrix in K-major form for the P.V product (attention.py:126). */
int pk_transpose_heads(const void* src_hi, const void* src_lo, int32_t batch, int32_t t, int32_t ld_src, int32_t col0,
                       int32_t dk, int32_t heads, int32_t ld_dst, void* dst_hi, void* dst_lo, pk_stream_t stream);
/* DurationPredictor.inference post-op (duration_predictor.py:94-101): d = max(round_half_away(exp(x) - offset), 0),
 * padded tokens -> 0.  Outputs fp32 and/or int64 (either may be NULL). */
int pk_duration_post(const float* x, const int32_t* lens, int32_t batch, int32_t t, float offset, float* d_f32, int64_t* d_i64,
                     pk_stream_t stream);
/* LengthRegulator.forward alpha != 1 (length_regulator.py:85-88): out = int64(round_half_away(d * alpha)). */
int pk_duration_scale(const int64_t* d, float alpha, int64_t n, int64_t* out, pk_stream_t stream);
/* masked_fill(x, pad_mask, 0) for predictor outputs (variance_predictor.py:101-103): x (batch, t, inner) in place. */
int pk_mask_rows(float* x, const int32_t* lens, int32_t batch, int32_t t, int32_t inner, pk_stream_t stream);
/* hs + pitch_embed(p) + energy_embed(e) (fastspeech2.py:426-430): Conv1D(1 -> c, k, pad (k-1)/2) on the scalar tracks
 * pitch / energy (batch, t); wp/we are [c][k] (Paddle [c,1,k]), bp/be [c]. */
int pk_variance_embed_add(const float* hs, const float* pitch, const float* energy, const float* wp, const float* bp, int32_t kp,
                          const float* we, const float* be, int32_t ke, const int32_t* lens, int32_t batch, int32_t t, int32_t c,
                          float* y, pk_stream_t stream);
/* ZScore.forward / .inverse over the last dim (modules/normalizer.py:18-33): inverse == 0: (x - mu) / sigma,
 * inverse != 0: x * sigma + mu; n = total elements, c = channels. */
int pk_zscore(const float* x, const float* mu, const float* sigma, int32_t c, int64_t n, int32_t inverse, float* y,
              pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * STFT / mel front-end: batched radix-2 FFT (one CTA per frame, no cuFFT) with fused epilogues.
 * Replaces STFT.forward / .power / .magnitude (parakeet/modules/audio.py:161-215: reflect pad + conv1d with the
 * windowed DFT matrix), MelScale.forward (:218-229), stft() of modules/stft_loss.py:20-67 and the numpy/librosa
 * feature path of data/get_feats.py:47-88 (log-mel) and :196-203 (frame energy).
 *   x (batch, t) fp32; window (n_fft) fp32 = scipy get_window(fftbins=True) centre-padded to n_fft (host builds it);
 *   twiddle (n_fft/2) float2 = (cos, -sin)(2 pi j / n_fft); center != 0: reflect padding n_fft/2, frames = 1 + t/hop.
 * Outputs (any may be NULL): re / im (batch, bins, frames); mag = sqrt(max(re^2+im^2, power_clip)) (power_clip < 0:
 * no clip) in layout 0 (batch, bins, frames) or 1 (batch, frames, bins); mel (batch, frames, n_mels) = mel_w (n_mels,
 * bins) . mag, optionally log10(max(., mel_clip)); energy (batch, frames) = sqrt(max(sum_k |X|^2, energy_clip)).
 * ------------------------------------------------------------------------------------------------------------ */
int pk_stft(const float* x, int32_t batch, int32_t t, const float* window, const void* twiddle, int32_t n_fft, int32_t hop,
            int32_t center, float* re, float* im, float* mag, int32_t mag_layout, float power_clip, const float* mel_w,
            int32_t n_mels, float* mel, int32_t mel_log10, float mel_clip, float* energy, float energy_clip, pk_stream_t stream);

/* Reductions behind SpectralConvergenceLoss / LogSTFTMagnitudeLoss (modules/stft_loss.py:70-118) on two magnitude
 * spectrograms of n elements: out3 = { sum (y-x)^2, sum y^2, sum |log max(y,eps) - log max(x,eps)| } (device fp32[3]). */
int pk_spectral_loss_sums(const float* x_mag, const float* y_mag, int64_t n, float eps, float* out3, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * WaveFlow inference (reference: parakeet/models/waveflow.py).  For configs outside the range of pk_waveflow_flow (below),
 * the per-row residual net of Flow.inverse (:515-556, ResidualBlock.add_input :248-294) runs its GEMMs per layer through
 * pk_conv_gemm_ex on a channels-last row (batch, W, C): the 3-row causal buffer is a (batch, W, 3C) split-bf16 ring
 * (slot = row mod 3) convolved along W with 3 dilated taps and K = 3C; the kernels below are that path's row-wise glue
 * (pk_waveflow_input_proj also writes row 0 for pk_waveflow_flow).
 * ------------------------------------------------------------------------------------------------------------ */
/* One layer of waveflow.UpsampleNet.forward (:103-132): Conv2DTranspose(1,1,(3,2f),stride (1,f),padding (1,f/2)) over
 * (mel, time), trim of the last f columns if trim != 0, leaky_relu(slope).  x (batch, c, t_in) -> y (batch, c,
 * t_in*f - trim*f); w [3][2f] (Paddle [1,1,3,2f]), bias [1]. */
int pk_waveflow_upsample(const float* x, const float* w, const float* bias, int32_t batch, int32_t c, int32_t t_in, int32_t factor,
                         int32_t trim, float slope, float* y, pk_stream_t stream);
/* Flow.input_proj (:437-442, 1x1 conv 1 -> C) on one row: state[b,w,:] = w * x_row[b,w] + bias (fp32 (batch, W, C)) and
 * the same values as split planes into columns [col0, col0 + C) of a (batch, W, ld) ring buffer. */
int pk_waveflow_input_proj(const float* x_row, int64_t x_batch_stride, const float* w, const float* bias, int32_t batch,
                           int32_t width, int32_t c, float* state, void* buf_hi, void* buf_lo, int32_t ld, int32_t col0,
                           pk_stream_t stream);
/* Flow._predict_row_parameters tail + _inverse_transform_row (:496-510): (logs, b) = output_proj(skip) (C -> 2, w [2][C]);
 * x_next[b,w] = (z_row[b,w] - b) * exp(-logs). */
int pk_waveflow_row_out(const float* skip, const float* w, const float* bias, const float* z_row, int64_t z_batch_stride,
                        int32_t batch, int32_t width, int32_t c, float* x_next, int64_t x_batch_stride, pk_stream_t stream);

/* All row steps i = 1 .. n_group-1 of one Flow.inverse (:515-556) in ONE persistent dataflow launch (ConditionalWaveFlow.inverse
 * for 64 and 128 channels, 64 < n_mels <= 128 and 2 to 8 layers per flow).  Per row step, n_layers times
 * ResidualBlock.add_input (:248-285):
 *   a | g = conv2d(3-row ring, dilation (1, 2^l)) + condition_proj(condition row) + bias1;  z = tanh(a) sigmoid(g);
 *   skip | res = out_proj(z) + bias2;  skip accumulator (=|+=) skip;  the next layer's ring slot (i - 1) mod 3 <- row + res,
 * with the newest row (i - 1) as the residual input; then on the completed skip sum (logs, b) = output_proj(skip),
 * x[:, i] = (z[:, i] - b) exp(-logs) (:496-510) and input_proj(x[:, i]) (:437-442) into the first layer's ring slot i mod 3.
 * The caller provides row 0: x[:, 0] = z[:, 0], input_proj(x[:, 0]) in slot 0 of ring 0 (pk_waveflow_input_proj), all other
 * ring contents zero, and `flags` (one uint32 per tile: (n_group - 1) * n_layers * batch * ceil(width / 256)) zeroed.
 * z / x: fp32 (batch, n_group, width).  cond planes (batch, n_group, width, n_mels); cond_rows[i] (HOST) = the condition row
 * used at row step i.  ring / w1 / w2: HOST arrays indexed by layer (w1: 3 * layer + variant, variant = i mod 3) of device
 * split planes, each pair of planes from ONE allocation (lo after hi); bias1 / bias2: HOST arrays indexed by layer of HOST
 * float vectors, copied into the kernel parameter block.  in_w / in_b [channels], out_w [2][channels], out_b [2]: HOST floats.
 * channels == 64: ring planes (batch, width, 192) with slot s in columns [64 s, 64 s + 64); w1 planes (128, 704): row n = gate
 * channel (a: 0..63, g: 64..127); columns [192 tap + 64 s + c] = conv.weight[n, c, kh(s), tap] for the ring slot s holding
 * kernel row kh(s) at this row step, columns [576 + m] = condition_proj.weight[n, m] (zeros from n_mels to 128); w2 planes
 * (128, 64): out_proj.weight with rows reordered to skip (0..63) | res (64..127); bias1 [128] = conv.bias + condition_proj.bias,
 * bias2 [128] = out_proj.bias as skip | res; skip fp32 (batch, width, 64).
 * channels == 128 (examples/waveflow/config.py) runs the same dataflow with the channels as two blocks of 64: ring planes
 * (batch, width, 384) with slot s in columns [128 s, 128 s + 128); w1 planes (256, 1280): rows a0 | g0 | a1 | g1 (64 each: gate
 * channel a_k = conv output 64 k + c, g_k = 128 + 64 k + c), columns [128 (3 tap + s) + c] conv, [1152 + m] condition_proj;
 * w2 planes (256, 128): rows skip0 | res0 | skip1 | res1; bias1 / bias2 [256] in the same row orders; skip (batch, width, 128). */
typedef struct pk_waveflow_flow_args {
  int32_t batch, width, channels, n_mels, n_layers, n_group;
  const int32_t* cond_rows;
  void* const* ring_hi;
  void* const* ring_lo;
  const void* cond_hi;
  const void* cond_lo;
  const void* const* w1_hi;
  const void* const* w1_lo;
  const void* const* w2_hi;
  const void* const* w2_lo;
  const float* const* bias1;
  const float* const* bias2;
  const float* in_w;
  const float* in_b;
  const float* out_w;
  const float* out_b;
  const float* z;
  float* x;
  float* skip;
  uint32_t* flags;
  int64_t flags_len;
} pk_waveflow_flow_args;
int pk_waveflow_flow(const pk_waveflow_flow_args* args, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * WaveFlow density estimation: ConditionalWaveFlow.forward (:759-783) = WaveFlow.forward (:627-672) on the untrimmed encoder
 * output, and WaveFlowLoss (:855-891).  Flow.forward (:465-494) is not autoregressive: every layer runs over all
 * n_group - 1 net rows of all utterances at once.
 * ------------------------------------------------------------------------------------------------------------ */
/* One ResidualBlock.forward (:197-226) over every (utterance, net row r in [0, n_group - 1), column) position, for 64 or 128
 * channels: a | g = conv2d(x, kernel 3x3, dilation (1, dilation), padding causal [2, 0] x same) + condition_proj(condition)
 * + bias1; z = tanh(a) sigmoid(g); skip | res = out_proj(z) + bias2; skip (=|+=) skip; y = x + res.
 * x / y planes (batch * (n_group + 1), width, channels): rows [b (n_group + 1), b (n_group + 1) + 2) stay ZERO (the causal
 * padding), net row r of utterance b is row b (n_group + 1) + 2 + r.  y must be another buffer (neighbouring positions read
 * x), NULL on the last layer; its zero rows are not written.  cond planes (batch, n_group, width, n_mels); cond_rows[h]
 * (HOST [n_group]) = the condition height that height h of this flow reads (the previous flows' permutations, composed):
 * net row r uses height r + 1.  w1 / w2 / bias1 / bias2: the operands of pk_waveflow_flow for ONE layer, row-step variant 0
 * (ring slot s = kernel row s): w1 planes (2 channels, 9 channels + 128), w2 planes (2 channels, channels), biases HOST.
 * skip fp32 (batch, n_group - 1, width, channels).  Every pair of planes comes from ONE allocation (lo after hi). */
typedef struct pk_waveflow_forward_layer_args {
  int32_t batch, width, channels, n_mels, n_group, dilation;
  const int32_t* cond_rows;
  const void* x_hi;
  const void* x_lo;
  const void* cond_hi;
  const void* cond_lo;
  const void* w1_hi;
  const void* w1_lo;
  const void* w2_hi;
  const void* w2_lo;
  const float* bias1;
  const float* bias2;
  void* y_hi;
  void* y_lo;
  float* skip;
  int32_t skip_init;
} pk_waveflow_forward_layer_args;
int pk_waveflow_forward_layer(const pk_waveflow_forward_layer_args* args, pk_stream_t stream);

/* The tail of one Flow.forward plus the height permutation after it (:661-665), and the next flow's input_proj:
 *   (logs, b) = output_proj(skip) (out_w [2][channels], out_b [2], HOST); z[:, 0] = x[:, 0], z[:, h] = x[:, h] exp(logs) + b
 *   (:459-463); x_next[:, i] = z[:, perm[i]] (perm HOST [n_group]); *log_det += sum of logs over all positions, summed in a
 *   fixed order (repeated calls give identical bits); the next flow's input_proj (in_w / in_b HOST [channels]) of x_next rows
 *   0 .. n_group - 2 into the next layer input planes (the x planes of pk_waveflow_forward_layer).
 * skip == NULL: z = x (no output_proj, log_det untouched) - the first flow's input_proj.  x_next, next_hi / next_lo may be
 * NULL (not written).  x / x_next fp32 (batch, n_group, width), distinct.  partials: device fp32 [1024] scratch; counter:
 * device uint32, zero before the first call and left zero by every call. */
typedef struct pk_waveflow_forward_tail_args {
  int32_t batch, width, channels, n_group;
  const float* skip;
  const float* out_w;
  const float* out_b;
  const float* x;
  const int32_t* perm;
  float* x_next;
  const float* in_w;
  const float* in_b;
  void* next_hi;
  void* next_lo;
  float* log_det;
  float* partials;
  uint32_t* counter;
} pk_waveflow_forward_tail_args;
int pk_waveflow_forward_tail(const pk_waveflow_forward_tail_args* args, pk_stream_t stream);
/* WaveFlowLoss.forward: loss[0] = (sq_sum[0] / (2 sigma^2) - log_det[0]) / n + log(2 pi) / 2 + log(sigma), with sq_sum the
 * device double sum of z^2 from pk_sq_sum and n = numel(z). */
int pk_waveflow_nll(const double* sq_sum, const float* log_det, int64_t n, float sigma, float* loss, pk_stream_t stream);

/* FastSpeech2Loss.forward with use_masking=True (models/fastspeech2/fastspeech2.py:701-812; DurationPredictorLoss
 * duration_predictor.py:140-184): out4 = { l1_loss = L1(before, ys) + L1(after, ys) over valid frames,
 * duration_loss = MSE(d_outs, log(ds + 1)), pitch_loss = MSE(p_outs, ps), energy_loss = MSE(e_outs, es) over valid tokens }.
 * before/after/ys (batch, l_max, odim) fp32; d_outs/p_outs/ps/e_outs/es (batch, t_max) fp32; ds int64; workspace12:
 * device fp32[12] scratch (zeroed by the call). */
int pk_fs2_loss(const float* before, const float* after, const float* ys, const int32_t* olens, int32_t l_max, int32_t odim,
                const float* d_outs, const int64_t* ds, const float* p_outs, const float* ps, const float* e_outs,
                const float* es, const int32_t* ilens, int32_t t_max, int32_t batch, float* workspace12, float* out4,
                pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * FastSpeech2 training step (reference: FastSpeech2Updater.update_core, models/fastspeech2/fastspeech2_updater.py:51-99:
 * forward, FastSpeech2Loss, loss.backward(), optimizer.step(); DataParallel gradient averaging is one NCCL all-reduce
 * on the flat gradient buffer, issued by the host through torch.distributed).  GEMM-shaped gradients reuse
 * pk_conv_gemm: dgrad = conv with flipped taps, wgrad / attention gradients = NT matmuls on transposed split planes.
 * ------------------------------------------------------------------------------------------------------------ */
/* dst[z*dst_zstride + c*ld_dst + r] = src[z*src_zstride + (r + shift)*ld_src + c0 + c] for r in [0, r_out), c in [0, cols)
 * (0 where r + shift is outside [0, rows)); split planes.  Builds K-major operands (X^T, dY^T, K^T, dS^T ...). */
int pk_transpose_planes(const void* src_hi, const void* src_lo, int32_t z, int32_t rows, int64_t src_zstride, int32_t ld_src,
                        int32_t c0, int32_t cols, int32_t shift, int32_t r_out, void* dst_hi, void* dst_lo, int64_t dst_zstride,
                        int64_t ld_dst, pk_stream_t stream);
/* LayerNorm backward: dx (+)= d/dx, dgamma += sum dy*xhat, dbeta += sum dy (fp32 [d], accumulated atomically). */
int pk_layer_norm_bwd(const float* x, const float* gamma, const float* dy, float eps, int64_t rows, int32_t d, float* dx,
                      int32_t accumulate, float* dgamma, float* dbeta, pk_stream_t stream);
/* softmax backward: ds = scale * p * (dp' - sum_k p dp') over the first `keys` columns of p, dp, ds (batch * heads, rows, ld),
 * 0 in columns >= keys; dp is not written.  dp' = dp, except that for heads h < guided_heads GuidedMultiHeadAttentionLoss
 * (transformer_tts.py:874-1075) is fused in: for rows i < olens[b] and keys j < ilens[b], dp'[i, j] = dp[i, j] + coef G[i, j]
 * with G = 1 - exp(-(j / ilens[b] - i / olens[b])^2 / (2 sigma^2)) and coef = lambda / (guided_heads * guided_layers *
 * sum_b ilens[b] olens[b]), and partials[(b * guided_heads + h) * rows + i] = sum_j G P (0 for i >= olens[b]).
 * With guided_heads 0, ilens, olens and partials may be NULL. */
int pk_softmax_bwd(const void* p_hi, const void* p_lo, const float* dp, int32_t batch, int32_t heads, int32_t rows, int32_t keys,
                   int32_t ld, float scale, int32_t guided_heads, int32_t guided_layers, const int32_t* ilens, const int32_t* olens,
                   float sigma, float lambda, float* partials, void* ds_hi, void* ds_lo, pk_stream_t stream);
/* out[c] += sum_rows x[row, c] (bias gradients). */
int pk_colsum(const float* x, int64_t rows, int32_t c, float* out, pk_stream_t stream);
/* pk_colsum on split planes (rows, ld): out[c] += sum_rows (x_hi + x_lo)[row, c] for c < cols (bias gradients from the split
 * copy of dY, which - unlike the fp32 dY of a residual stream - nobody updates in place afterwards). */
int pk_colsum_split(const void* x_hi, const void* x_lo, int64_t rows, int32_t cols, int32_t ld, float* out, pk_stream_t stream);
/* out[i] = sum_{s < slices} part[s * n + i] (fp32): the reduction of split-K partial products of a weight gradient; overwrites
 * `out` (unlike pk_colsum, which accumulates). */
int pk_sum_slices(const float* part, int32_t slices, int64_t n, float* out, pk_stream_t stream);
/* BatchNorm1D in training mode on (rows, c) (tacotron2/decoder.py:128-180 under model.train()): batch statistics
 * (biased variance), y = act(gamma * xhat + beta) with act in {PK_ACT_NONE, PK_ACT_TANH}, running statistics updated with
 * Paddle's momentum (running = momentum * running + (1 - momentum) * batch); saves mean / rstd for the backward. */
int pk_batch_norm_train(const float* x, int64_t rows, int32_t c, const float* gamma, const float* beta, float eps, int32_t act,
                        float momentum, float* run_mean, float* run_var, float* sums2c, float* y, void* y_hi, void* y_lo,
                        float* save_mean, float* save_rstd, pk_stream_t stream);
/* backward of the above (including the tanh): dx; afterwards sums2c = { dbeta[c], dgamma[c] }. */
int pk_batch_norm_bwd(const float* x, const float* dy, const float* y_act, const float* mean, const float* rstd, const float* gamma,
                      int32_t act, int64_t rows, int32_t c, float* sums2c, float* dx, pk_stream_t stream);
/* dx = dy * (y > 0), y given by the hi plane of the saved ReLU output; fp32 and/or split output. */
int pk_relu_bwd(const float* dy, const void* y_hi, int64_t n, float* dx, void* dx_hi, void* dx_lo, pk_stream_t stream);
/* y += a * x */
int pk_axpy(float a, const float* x, int64_t n, float* y, pk_stream_t stream);
/* gradients of l1_loss + duration_loss + pitch_loss + energy_loss (pk_fs2_loss) w.r.t. before, after, d_outs, p_outs, e_outs */
int pk_fs2_loss_bwd(const float* before, const float* after, const float* ys, const int32_t* olens, int32_t l_max, int32_t odim,
                    const float* d_outs, const int64_t* ds, const float* p_outs, const float* ps, const float* e_outs,
                    const float* es, const int32_t* ilens, int32_t t_max, int32_t batch, float* g_before, float* g_after,
                    float* g_d, float* g_p, float* g_e, pk_stream_t stream);
/* backward of pk_embed_pe: dtable[ids] += dx (ids may be NULL: positional encoding only), dalpha += sum dx * PE */
int pk_embed_pe_bwd(const int64_t* ids, const float* dx, int32_t vocab, int32_t padding_idx, int32_t batch, int32_t t, int32_t d,
                    float* dtable, float* dalpha, pk_stream_t stream);
/* backward of pk_length_regulate: dx[b, j, :] = sum over the frames of token j of dy[b, frame, :] */
int pk_length_regulate_bwd(const float* dy, const int64_t* dur, int32_t batch, int32_t t_in, int32_t c, int32_t t_out, float* dx,
                           pk_stream_t stream);
/* weight / bias gradients of pitch_embed / energy_embed (Conv1D(1 -> c, k) on a scalar track): dw [c][k], db [c] accumulated */
int pk_scalar_conv_wgrad(const float* dhs, const float* track, int32_t batch, int32_t t, int32_t c, int32_t k, float* dw, float* db,
                         pk_stream_t stream);
/* nn.Dropout in training mode (upscale_in_train): y[i] = keep(i) ? x[i] / (1 - p) : 0, keep(i) = word (i & 3) of
 * Philox4x32-10(counter {i >> 2 low, high, site, step}, key {seed low, high}) >= p * 2^32.  Input fp32 x or split planes
 * (x_hi + x_lo), outputs fp32 and/or split planes; in place allowed.  The backward pass applies the same call to the gradient
 * (same seed / site / step regenerate the mask).  Reference: the Dropout layers of parakeet/modules/fastspeech2_transformer/
 * {embedding.py:79,126, attention.py:124, encoder_layer.py:101,108, multi_layer_conv.py:76}, fastspeech2_predictor/
 * {duration_predictor.py:82, variance_predictor.py:73}, tacotron2/decoder.py:144-180 (Postnet). */
int pk_dropout(const float* x, const void* x_hi, const void* x_lo, int64_t n, float p, uint64_t seed, uint32_t site, uint32_t step,
               const uint32_t* step_dev /* device uint32 added to `step` (NULL: none) - lets a CUDA graph replay draw fresh masks */,
               float* y, void* y_hi, void* y_lo, pk_stream_t stream);
/* paddle.optimizer.Adam step on a flat buffer (training/optimizer.py:17-46) with ClipGradByGlobalNorm folded in: the gradient
 * g * grad_scale * clip_norm / max(sqrt(*sqnorm), clip_norm) (grad_scale 1/world for DataParallel; sqnorm from pk_sq_sum; sqnorm
 * NULL or clip_norm <= 0: no clipping), lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t), p -= lr_t * m / (sqrt(v) + eps *
 * sqrt(1 - beta2^t)). */
int pk_adam(float* params, const float* grads, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
            int32_t step, float grad_scale, const double* sqnorm, float clip_norm, pk_stream_t stream);
/* Speaker conditioning of the multi-speaker training step (fastspeech2.py:148-152 spk_embedding_table = nn.Embedding(num_speakers,
 * D, padding_idx=0); :395-401 and _integrate_with_spk_embed :560-590: F.normalize(p=2, axis=1, epsilon) then the "concat" / "add"
 * projection, whose GEMMs run through pk_conv_gemm).  Speaker ids are int64 on the device and never read on the host; ids equal
 * to padding_idx, or outside [0, num_speakers), embed to zeros and receive no gradient.  No atomics: fixed summation orders. */
/* e[b] = table[ids[b]] / max(||table[ids[b]]||, eps) (batch, d); norms[b] = ||table[ids[b]]|| (0 for padding ids), saved for
 * pk_spk_normalize_bwd. */
int pk_spk_embed_fwd(const float* table, int32_t num_speakers, int32_t d, const int64_t* ids, int32_t batch, int32_t padding_idx,
                     float eps, float* e, float* norms, pk_stream_t stream);
/* out[b, j] = sum over ALL t rows of dx[b, row, col0 + j], j < ncols, dx (batch, t, c) fp32: the gradient of a per-utterance
 * vector broadcast over time.  dhs (or NULL): columns [0, dhs_cols) of dx copied to a contiguous (batch, t, dhs_cols) in the
 * same pass (the hs part of the concat projection's input gradient). */
int pk_spk_time_sum(const float* dx, int32_t batch, int32_t t, int32_t c, int32_t col0, int32_t ncols, float* dhs, int32_t dhs_cols,
                    float* out, pk_stream_t stream);
/* backward of pk_spk_embed_fwd's normalisation: dx = (g - e (e . g)) / ||x|| (g / eps where ||x|| <= eps); rows of padding ids
 * are exact zeros. */
int pk_spk_normalize_bwd(const float* e, const float* norms, const float* g, const int64_t* ids, int32_t batch, int32_t num_speakers,
                         int32_t padding_idx, int32_t d, float eps, float* dx, pk_stream_t stream);
/* dense embedding gradient (Paddle's sparse=False): dtable[r] = sum over b ascending with ids[b] == r of de[b], every row written
 * (absent speakers and padding_idx as zeros), e.g. straight into the table's slice of a flat gradient buffer. */
int pk_spk_table_grad(const float* de, const int64_t* ids, int32_t batch, int32_t num_speakers, int32_t d, int32_t padding_idx,
                      float* dtable, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * Parallel WaveGAN training step (reference: PWGUpdater.update_core, models/parallel_wavegan/parallel_wavegan_updater.py:76-153;
 * generator :445-472, PWGDiscriminator :554-614, MultiResolutionSTFTLoss modules/stft_loss.py:163-219).  Every Conv1D forward /
 * data gradient / weight gradient and the DFTs run through pk_conv_gemm; these are the element-wise pieces in between.
 * Shapes are channels-last (rows = batch * t) fp32 unless noted.
 * ------------------------------------------------------------------------------------------------------------ */
/* z = tanh(h[:, :c]) * sigmoid(h[:, c:])  (ResidualBlock :307-310); h (rows, 2c); outputs fp32 and/or split planes (rows, c). */
int pk_gate_fwd(const float* h, int64_t rows, int32_t c, float* z, void* z_hi, void* z_lo, pk_stream_t stream);
int pk_gate_bwd(const float* h, const float* dz, int64_t rows, int32_t c, float* dh, pk_stream_t stream);
/* nn.LeakyReLU(negative_slope) forward (fp32 and/or split planes out) and backward (x = the pre-activation). */
int pk_leaky_relu(const float* x, int64_t n, float slope, float* y, void* y_hi, void* y_lo, pk_stream_t stream);
int pk_leaky_relu_bwd(const float* x, const float* dy, int64_t n, float slope, float* dx, pk_stream_t stream);
/* nn.utils.weight_norm (dim 0): w[r, :] = g[r] * v[r, :] / ||v[r, :]||; backward: dg, dv from dw.  v (rows, inner). */
int pk_weight_norm_fwd(const float* v, const float* g, int32_t rows, int32_t inner, float* w, float* norm, pk_stream_t stream);
int pk_weight_norm_bwd(const float* v, const float* g, const float* dw, int32_t rows, int32_t inner, float* dg, float* dv, pk_stream_t stream);
/* MSELoss against a constant over x[i * ld + col], i < n: acc[0] += sum (x - target)^2 (device double); dx (or NULL) = coef * (x - target). */
int pk_mse_const(const float* x, int64_t n, int32_t ld, int32_t col, float target, double* acc, float* dx, float coef, pk_stream_t stream);
/* acc[0] += sum x^2 (device double): the global gradient norm of ClipGradByGlobalNorm (pk_adam's sqnorm). */
int pk_sq_sum(const float* x, int64_t n, double* acc, pk_stream_t stream);
/* generator residual / skip update (:311-315, :466-468): so (rows, 128) = [skip | out]; skips (=|+=) skip; xo = (out + x) * sqrt(1/2)
 * as fp32 and split planes; and its backward: dso = [dskips | dxo * sqrt(1/2)], dx_res = dxo * sqrt(1/2). */
int pk_pwg_res_update(const float* so, const float* x, int64_t rows, float* skips, int32_t init, float* xo, void* xo_hi, void* xo_lo,
                      pk_stream_t stream);
int pk_pwg_res_update_bwd(const float* dskips, const float* dxo, int64_t rows, float* dso, float* dx_res, pk_stream_t stream);
/* one upsampling stage (Stretch2D nearest x s + Conv2D FIR of 2s+1 taps, zero pad s; :48-63,119-138) on x (rows, tin) -> (rows, tin*s),
 * and its backward: dx (rows, tin) and/or dfir[2s+1] (device double, accumulated). */
int pk_up_stage_fwd(const float* x, const float* fir, int64_t rows, int32_t tin, int32_t s, float* y, pk_stream_t stream);
int pk_up_stage_bwd(const float* x, const float* dy, const float* fir, int64_t rows, int32_t tin, int32_t s, float* dx, double* dfir,
                    pk_stream_t stream);
/* gradient of weight * (spectral convergence + log STFT magnitude) of ONE resolution (stft_loss.py:20-161) w.r.t. re / im of the
 * generated signal's STFT: x / y re, im (batch, bins, frames) from pk_stft; sums = the device fp32[3] of pk_spectral_loss_sums;
 * g (batch * frames, 2 * bins_p) row-major [re | im] (padding columns are not written: zero them once). */
int pk_stft_loss_grad(const float* xre, const float* xim, const float* yre, const float* yim, int32_t batch, int32_t bins, int32_t frames,
                      int32_t bins_p, const float* sums, float weight, float* g, pk_stream_t stream);
/* adjoint of framing (centre, reflect padding, window): dx[b, reflect(f * hop + k - n_fft / 2)] += frames_grad[b, f, k] * window[k]. */
int pk_frames_overlap_add(const float* frames_grad, const float* window, int32_t batch, int32_t frames, int32_t n_fft, int32_t hop,
                          int32_t t, float* dx, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * SpeedySpeech (reference: parakeet/models/speedyspeech/speedyspeech.py).  Everything but the residual blocks reuses the
 * kernels above (pk_conv_gemm, pk_duration_post, pk_length_regulate, pk_embed_pe, pk_leaky_relu).
 * ------------------------------------------------------------------------------------------------------------ */
/* One ResidualBlock.forward (speedyspeech.py:21-39) in eval mode: h_0 = x, h_i = relu(conv_i(h_{i-1}) + bias_i) * scale_i +
 * shift_i for i = 1..n_convs, y = x + h_n.  scale / shift are the BatchNorm1D affine (gamma / sqrt(var + eps), beta - mean *
 * scale).  The convs are undilated with pad_left zero rows before the sequence and taps - 1 - pad_left after it (Paddle's
 * padding="same").  x fp32 (batch, t, channels) and its split planes; w*_hi / w*_lo the packed weight planes [channels,
 * taps * channels] (ops.pack_weight of the Paddle [out, in, k] weight); bias / scale / shift fp32 [channels].  lens (device
 * int32 [batch], or NULL = t): each utterance is computed as if it were alone - the intermediate is zero outside [0, lens[b])
 * and rows t >= lens[b] of y are written as 0; rows of x at t >= lens[b] must already be 0.  y fp32 and split planes, not
 * aliasing x.  The intermediate of a two-conv block stays in shared memory.  channels must be 128 (PK_ERR_UNSUPPORTED
 * otherwise), taps 1..4, n_convs 1 or 2. */
typedef struct pk_ss_residual_block_args {
  int32_t batch;
  int32_t t;
  int32_t channels;
  int32_t n_convs;
  int32_t taps;
  int32_t pad_left;
  const int32_t* lens;
  const float* x;
  const void* x_hi;
  const void* x_lo;
  const void* w1_hi;
  const void* w1_lo;
  const float* bias1;
  const float* scale1;
  const float* shift1;
  const void* w2_hi;
  const void* w2_lo;
  const float* bias2;
  const float* scale2;
  const float* shift2;
  float* y;
  void* y_hi;
  void* y_lo;
} pk_ss_residual_block_args;
int pk_ss_residual_block(const pk_ss_residual_block_args* args, pk_stream_t stream);

/* SpeedySpeech training step (reference: SpeedySpeechUpdater.update_core, models/speedyspeech/speedyspeech_updater.py:48-85, with
 * the model in train() mode).  The Conv1D / Linear forwards, data gradients and weight gradients run through pk_conv_gemm; these
 * are the train-mode BatchNorm1D of the Conv1D -> ReLU -> BatchNorm1D units (speedyspeech.py:21-39) and the losses.  Every sum is
 * taken over per-block partials in a fixed order (no atomics): repeated calls give identical bits.  c must be 128
 * (PK_ERR_UNSUPPORTED otherwise).  scratch: fp32 workspace of at least 256 * ceil(rows / 128) elements. */
/* BatchNorm1D in training mode on r (rows, c), r = relu(conv(x) + bias) as pk_conv_gemm wrote it: batch mean and biased variance
 * over all rows, y = gamma * (r - mean) * rstd + beta (+ residual, the block input, on the last unit of a ResidualBlock) as fp32
 * and / or split planes; run_mean / run_var (or both NULL) updated as momentum * running + (1 - momentum) * batch (Paddle's
 * convention); save_mean / save_rstd [c] are kept for the backward. */
int pk_ss_bn_train_fwd(const float* r, int64_t rows, int32_t c, const float* gamma, const float* beta, float eps, float momentum,
                       float* run_mean, float* run_var, const float* residual, float* scratch, float* y, void* y_hi, void* y_lo,
                       float* save_mean, float* save_rstd, pk_stream_t stream);
/* Backward of ReLU -> BatchNorm1D in one go: from dy and the saved r / mean / rstd, dbeta = sum dy, dgamma = sum dy * xhat
 * (overwritten), dr = gamma * rstd * (dy - mean(dy) - xhat * mean(dy * xhat)) * [r > 0] - the gradient at the conv's output -
 * as fp32 and / or split planes (the operand of the data and weight gradient GEMMs), and dbias = sum dr (or NULL). */
int pk_ss_bn_relu_bwd(const float* dy, const float* r, const float* mean, const float* rstd, const float* gamma, int64_t rows,
                      int32_t c, float* scratch, float* dgamma, float* dbeta, float* dbias, float* dr, void* dr_hi, void* dr_lo,
                      pk_stream_t stream);
/* The losses of update_core :57-80 and their gradients.  decoded / feats fp32 (batch, l, odim), odim <= 80; num_frames /
 * num_phones device int32 [batch]; pred_durations fp32 and durations int64 (batch, t).
 *   l1       = sum |decoded - feats| * mask / (sum mask * odim)                              (modules/losses.py:60-100)
 *   duration = sum huber(pred, log(max(durations, 1)), delta 1) * token mask / sum token mask (fluid.layers.huber_loss)
 *   ssim     = 1 - mean over all batch * l * odim positions of the SSIM map of (decoded * mask, feats * mask): 11 x 11 Gaussian
 *              window, sigma 1.5, zero padding 5 (modules/ssim.py:21-80), evaluated as two 1-D passes
 * losses[4] = { l1 + ssim + duration, l1, duration, ssim }.  g_decoded (batch, l, odim) and g_durations (batch, t) receive
 * d losses[0] / d decoded and / d pred_durations; both NULL computes the losses only (the evaluator, :110-157).
 * scratch: fp32, at least 2 * batch * ceil(l / 16) elements, plus 3 * batch * l * odim when gradients are requested. */
int pk_ss_loss(const float* decoded, const float* feats, const int32_t* num_frames, int32_t batch, int32_t l, int32_t odim,
               const float* pred_durations, const int64_t* durations, const int32_t* num_phones, int32_t t, float* scratch,
               float* losses, float* g_decoded, float* g_durations, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * WaveFlow training step (reference: examples/waveflow/train.py:95-118 Experiment.train_batch; ConditionalWaveFlow.forward
 * models/waveflow.py:759-783, Flow.forward :465-494, ResidualBlock.forward :209-226, UpsampleNet.forward :103-132,
 * WaveFlowLoss :855-891; loss.backward() and paddle.optimizer.Adam).  The GEMMs run through pk_conv_gemm; these kernels sit
 * between them.  "Net layout": fp32 or split planes (batch * (n_group + 1), width, ld), utterance b's net row j (the flow's
 * height j + 1, j < n_group - 1) at row b * (n_group + 1) + j, its last two rows zero.  "Input layout": the same rows two
 * further down, i.e. two zero rows before each utterance's net rows (the causal height padding of the 3x3 conv).  Flow
 * inputs / outputs x fp32 (batch, n_group, width), sample t = w * n_group + h.  No reduction uses atomics: repeated calls give
 * identical bits.
 * ------------------------------------------------------------------------------------------------------------ */
/* dst[i] = split(idx[i] >= 0 ? src[idx[i]] : 0), i < n: packs GEMM operands from the flat folded weights. */
int pk_waveflow_train_gather_split(const float* src, const int32_t* idx, int64_t n, void* dst_hi, void* dst_lo, pk_stream_t stream);
/* input_proj (Flow._predict_parameters :453, 1x1 Conv2D 1 -> c) of flow input rows 0 .. n_group - 2: h fp32 (net layout, c; pad rows 0) and
 * x_hi / x_lo split planes (input layout, c; only net rows written).  w, bias device fp32 [c]. */
int pk_waveflow_train_input_fwd(const float* x, const float* w, const float* bias, int32_t batch, int32_t n_group, int32_t width, int32_t c,
                                float* h, void* x_hi, void* x_lo, pk_stream_t stream);
/* ResidualBlock.forward (:197-226) after out_proj, and ResidualNet.forward's skip sum (:355-360): out fp32 (net layout, 2c) = (res | skip); h += res; skip = skip_part (skip_init)
 * or skip += skip_part; x_hi / x_lo (input layout, or NULL): the next layer's input planes of h's net rows. */
int pk_waveflow_train_update(const float* out, int32_t batch, int32_t n_group, int32_t width, int32_t c, float* h, float* skip, int32_t skip_init,
                             void* x_hi, void* x_lo, pk_stream_t stream);
/* Flow._predict_parameters / _transform (:455-463) + WaveFlow.forward's permutation (:664): (logs, b) = output_proj(skip) (out_w device [2][c],
 * out_b device [2]); z = x for height 0, x exp(logs) + b above; x_next[:, inv_perm[h]] = z[:, h] (inv_perm device int32
 * [n_group], the inverse of the reference's perm); logs fp32 (batch, n_group - 1, width). */
int pk_waveflow_train_tail_fwd(const float* skip, const float* out_w, const float* out_b, const float* x, const int32_t* inv_perm, int32_t batch,
                               int32_t n_group, int32_t width, int32_t c, float* x_next, float* logs, pk_stream_t stream);
/* Backward of pk_waveflow_train_tail_fwd.  The gradient of x_next is dy, or y_coef * y when dy is NULL (the last flow: y = z
 * and y_coef = 1 / (sigma^2 numel(z)) from WaveFlowLoss); dlogs is added to every logs gradient (-1 / numel(z): the log-det
 * term).  Writes dx (batch, n_group, width) - the direct path only, overwritten - dparams fp32 (net layout, 2) = d(logs, b),
 * dskip fp32 (net layout, c) and the same as split planes at ds[row * ds_ld + ds_col0 + c].  Pad rows are not written. */
int pk_waveflow_forward_tail_bwd(const float* skip, const float* out_w, const float* out_b, const float* x, const int32_t* inv_perm, const float* dy,
                                 const float* y, float y_coef, float dlogs, int32_t batch, int32_t n_group, int32_t width, int32_t c, float* dx,
                                 float* dparams, float* dskip, void* ds_hi, void* ds_lo, int32_t ds_ld, int32_t ds_col0, pk_stream_t stream);
/* Backward of input_proj's data path: dx[b, j, w] += sum_c w[c] dh[(b, j), w, c] for j < n_group - 1 (dh net layout); xcol
 * fp32 (net layout, 1) <- x[b, j, w] on net rows (pad rows not written), the operand of the input_proj weight gradient. */
int pk_waveflow_train_input_bwd(const float* dh, const float* x, const float* w, int32_t batch, int32_t n_group, int32_t width, int32_t c,
                                float* dx, float* xcol, pk_stream_t stream);
/* out[i * os_i + j * os_j] (+)= sum_r a[r * lda + i] * (b ? b[r * ldb + j] : 1), i < ka, j < kb, ka * kb <= 256: bias and small
 * weight gradients in a fixed order (per-block partials in scratch, then their sum). */
int pk_waveflow_train_outer_sum(const float* a, int32_t lda, int32_t ka, const float* b, int32_t ldb, int32_t kb, int64_t rows, float* scratch,
                                int64_t scratch_len, float* out, int64_t os_i, int64_t os_j, int32_t accumulate, pk_stream_t stream);
/* Backward of one untrimmed UpsampleNet stage (:103-132): y = leaky_relu(Conv2DTranspose(x; w [3][2 factor], bias), slope), x
 * (batch, c, t_in), y / dy (batch, c, t_in * factor).  dpre: scratch of y's size; dx (or NULL) (batch, c, t_in); dw [3 * 2 factor]
 * and db [1] overwritten; scratch fp32 for the fixed-order partials. */
int pk_waveflow_upsample_bwd(const float* x, const float* y, const float* dy, const float* w, int32_t batch, int32_t c, int32_t t_in,
                             int32_t factor, float slope, float* dpre, float* dx, float* scratch, int64_t scratch_len, float* dw, float* db,
                             pk_stream_t stream);
/* The condition of one flow in the net layout: row (b, j) = height rows[j + 1] (rows device int32 [n_group], the composed
 * permutation of the flows before it) of cond fp32 (batch, n_mels, t_cond) -> split planes (net layout, n_mels), pad rows 0. */
int pk_waveflow_train_cond_gather(const float* cond, const int32_t* rows, int32_t batch, int32_t n_group, int32_t width, int32_t n_mels,
                                  int32_t t_cond, void* hi, void* lo, pk_stream_t stream);
/* Its adjoint, accumulated: dcond[b, m, w * n_group + rows[j + 1]] += dc[(b, j), w, m] (dc fp32 net layout). */
int pk_waveflow_train_cond_scatter(const float* dc, const int32_t* rows, int32_t batch, int32_t n_group, int32_t width, int32_t n_mels,
                                   int32_t t_cond, float* dcond, pk_stream_t stream);
/* One layer boundary of the residual net's backward (ResidualBlock.forward :197-226 and ResidualNet.forward :339-360,
 * differentiated), the mirror image of pk_waveflow_forward_layer, for channels C = 64 or 128, all net rows of all utterances:
 *   has_gemm1: dx = dx + conv2d^T(dh_in) (the 3x3 conv of layer l, width dilation `dilation`; dh_in rows q + 1, q + 2 below the
 *              last net row are the two zero rows of the net layout, so dh_in needs batch * (n_group + 1) + 2 rows), else dx = 0;
 *              dx fp32 (net layout, C) is read and written in place and also written as split planes into columns [0, C) of a2.
 *   has_gemm2: dz = a2 . W2 (K = 2C, a2 = [dx | dskip] split planes (net layout, 2C) whose columns [C, 2C) hold dskip);
 *              dh_out = gate backward of dz with the pre-gate h fp32 (net layout, 2C) of layer l - 1, as split planes.
 * dh_in / dh_out: split planes with row pitch dh_ld (2C columns each; e.g. column blocks of one (rows, W, n_layers * 2C)
 * allocation).  w1: conv^T planes (C, 18 C), column ((s * 3 + t) * 2C + o) = conv.weight[o, c, 2 - s, 2 - t] of row c;
 * w2: out_proj^T planes (C, 2C) = out_proj.weight[o, c] at (c, o).  Pad rows are not written. */
typedef struct pk_waveflow_backward_layer_args {
  int32_t batch;
  int32_t width;
  int32_t channels;
  int32_t n_group;
  int32_t dilation;
  int32_t has_gemm1;
  int32_t has_gemm2;
  int32_t dh_ld;
  const void* dh_in_hi;
  const void* dh_in_lo;
  const void* w1_hi;
  const void* w1_lo;
  const void* w2_hi;
  const void* w2_lo;
  float* dx;
  void* a2_hi;
  void* a2_lo;
  const float* h;
  void* dh_out_hi;
  void* dh_out_lo;
} pk_waveflow_backward_layer_args;
int pk_waveflow_backward_layer(const pk_waveflow_backward_layer_args* args, pk_stream_t stream);
/* WaveFlowLoss (:855-891) in a fixed order: loss[0] = (sum z^2 / (2 sigma^2) - sum logs) / n + log(2 pi) / 2 + log(sigma). */
int pk_waveflow_train_loss(const float* z, int64_t n, const float* logs, int64_t n_logs, float sigma, float* loss, pk_stream_t stream);

/* ---- GE2E speaker encoder (parakeet/models/lstm_speaker_encoder.py; csrc/lstm.cu) ----
 * One LSTM layer over all t steps as ONE persistent launch (Paddle nn.LSTM, gates i, f, g, o); the per-step GEMM is wgmma in
 * bf16x3 with W_hh resident in shared memory and h_{t-1} read by TMA.  Time-major: row r of step s at s * rows + r.
 * g_in (t, rows, 4H) = x W_ih^T + b_ih (one pk_conv_gemm); b_hh [4H] (or NULL) is added here.
 * w_hi / w_lo: W_hh [4H, H] as split planes (one allocation, lo after hi) with its rows permuted: packed row
 *   32 * 4 * s + 8 * (2 * (u / 4) + g / 2) + 2 * (u % 4) + g % 2  holds  W_hh row g * H + 32 * s + u  (slice s, local unit u < 32,
 *   gate g < 4), so that one thread's accumulator fragment holds the four gates of its units.
 * h_all ((t+1), rows, H) fp32 and h_hi / h_lo its split planes (one allocation): slab 0 holds h0 on entry (both forms), slab s+1
 *   receives h_s.  c: (rows, H) updated in place when c_step == 0, else ((t+1), rows, H) with c0 in slab 0 and c_s in slab s+1
 *   (c_step = rows * H, training).  gates (t, rows, 4H) receives the post-activation gates (or NULL).
 * counters: >= t * ceil(rows / 64) uint32, zeroed on the stream by the call itself.  TMA operands 16-byte aligned.
 * hidden in {64, 256}; any other size returns PK_ERR_UNSUPPORTED, as does a grid that cannot be co-resident. */
int pk_lstm_fwd(const float* g_in, const float* b_hh, const void* w_hi, const void* w_lo, int32_t rows, int32_t t, int32_t hidden,
                float* h_all, void* h_hi, void* h_lo, float* c, int64_t c_step, float* gates, uint32_t* counters,
                int64_t counters_len, pk_stream_t stream);
/* Backward through time of pk_lstm_fwd (training mode's gates and c_all), one persistent launch in reverse time, wgmma bf16x3:
 * dh_s = dh_in[s] (or NULL) + (s == t-1 ? dh_last : 0) (or NULL) + dgates_{s+1} W_hh.  wt_hi / wt_lo: W_hh^T [H, 4H] split planes.
 * dc: (rows, H) scratch.  dgates (t, rows, 4H) fp32 gradients of the pre-activation gates, dg_hi / dg_lo the same as split planes
 * (one allocation; read back by TMA for the next step). */
int pk_lstm_bwd(const void* wt_hi, const void* wt_lo, const float* gates, const float* c_all, const float* dh_in, const float* dh_last,
                int32_t rows, int32_t t, int32_t hidden, float* dc, float* dgates, void* dg_hi, void* dg_lo, uint32_t* counters,
                int64_t counters_len, pk_stream_t stream);
/* doubles of scratch pk_ge2e_loss needs for embeds (n, m, c) */
int64_t pk_ge2e_loss_scratch(int32_t n, int32_t m, int32_t c);
/* LSTMSpeakerEncoder.similarity_matrix + loss on embeds (n, m, c) (m >= 2), one block in double: loss[0] (cross-entropy mean),
 * sim (n*m, n) = (cosine to the inclusive centroids, own speaker: to the exclusive centroid) * w[0] + b[0] (or NULL).
 * With d_embeds / dw / db (all or none): the gradient of the loss, dw and db times 0.01 (do_gradient_ops).  No atomics. */
int pk_ge2e_loss(const float* embeds, int32_t n, int32_t m, int32_t c, const float* w, const float* b, double* scratch,
                 int64_t scratch_len, float* loss, float* sim, float* d_embeds, float* dw, float* db, pk_stream_t stream);
/* backward of F.normalize(relu(z)) (rows, n) given e = relu(z) and dy: dz (z > 0 read as e > 0). */
int pk_ge2e_embed_bwd(const float* e, const float* dy, int32_t rows, int32_t n, float eps, float* dz, pk_stream_t stream);
/* y[s] = F.normalize(mean(x[offsets[s] : offsets[s+1]], 0), axis=0) for s < segments (embed_utterance per utterance), n <= 8192;
 * an empty segment yields zeros */
int pk_segment_mean_normalize(const float* x, const int32_t* offsets, int32_t segments, int32_t n, float eps, float* y,
                              pk_stream_t stream);

/* ---- Tacotron2 (csrc/tacotron2.cu) ----
 * pk_taco2_decode: every step of Tacotron2Decoder.infer (teacher = 0) or of the teacher-forced Tacotron2Decoder.forward
 * (teacher = 1) as one persistent launch, fp32.  Fixed sizes: d_attention_rnn = d_decoder_rnn = 1024, d_prenet 256,
 * d_attention 128; d_enc 512 or 768, batch <= 32, dmr = d_mels * r a multiple of 4, odd loc_k <= 63 (else PK_ERR_UNSUPPORTED,
 * as is a grid of fewer than 32 co-resident CTAs).  Weights are row-major [out, in]:
 *   pre_w1 [256, dmr], pre_w2 [256, 256]; att_w [4096, 256 + d_enc + 1024] = [W_ih | W_hh] of the attention LSTMCell
 *   (gates i, f, g, o), dec_w [4096, 1024 + d_enc + 1024] the same for the decoder LSTMCell, biases [4096] each;
 *   q_w [128, 1024]; loc_w [128, 2, loc_k] = location_layer o location_conv; v_w [128]; proj_w [dmr, 1024 + d_enc], proj_b [dmr];
 *   stop_w [1024 + d_enc], stop_b [1] or both NULL (no stop token).
 * keys (batch, t_enc, d_enc) encoder outputs, pkeys (batch, t_enc, 128) = key_layer(keys); text_lens (int32, teacher only:
 * energies of positions >= text_lens get -1e9); mels (batch, steps, dmr) teacher inputs.  The prenet dropout (ReLU, then
 * p_prenet with pk_dropout's Philox: sites 0 and 1 for the two layers, step = decoder step, element b * 256 + j) is always on.
 * Outputs (batch, steps, dmr) mel_out, (batch, steps, t_enc) align_out, (batch, steps) stop_out; frames[b] (int32) = frames
 * produced.  infer stops on the device, after frame i when (stop token) sigmoid(stop_out[0, i]) > 0.5 (batch must be 1), or
 * (no stop token) argmax(align[0, i]) == t_enc - 1 for an i > first such i + 20, or at i + 1 == steps; rows past the stop are
 * zero.  The call zeroes the workspace (pk_taco2_workspace floats: counters and recurrent state) and the outputs on the stream. */
typedef struct {
  int32_t batch, t_enc, d_enc, dmr, steps, teacher, loc_k;
  float p_prenet;
  uint64_t seed;
  const float* keys; const float* pkeys; const int32_t* text_lens; const float* mels;
  const float* pre_w1; const float* pre_w2;
  const float* att_w; const float* att_b_ih; const float* att_b_hh;
  const float* q_w; const float* loc_w; const float* v_w;
  const float* dec_w; const float* dec_b_ih; const float* dec_b_hh;
  const float* proj_w; const float* proj_b; const float* stop_w; const float* stop_b;
  float* workspace; int64_t workspace_len;
  float* mel_out; float* align_out; float* stop_out; int32_t* frames;
  uint64_t* prof; int64_t prof_len;   /* optional (NULL): per-CTA ns counters, [cta][0..5] time per phase incl. its hand-off,
                                         [cta][6..11] wait from arrival to release; zeroed by the call; pk_taco2_prof_len() entries */
} PkTaco2DecodeArgs;
int64_t pk_taco2_workspace(int32_t batch, int32_t t_enc, int32_t d_enc);
int64_t pk_taco2_prof_len(void);
int pk_taco2_decode(const PkTaco2DecodeArgs* args, pk_stream_t stream);
/* y (batch, t, channels) = table[ids] + (tones ? tone_table[tones], zero for tone 0 (padding_idx) : 0); ids / tones int64 */
int pk_taco2_embed(const int64_t* ids, const float* table, const int64_t* tones, const float* tone_table, int32_t batch, int32_t t,
                   int32_t channels, float* y, pk_stream_t stream);
/* dst (t, batch, channels) = src (batch, t, channels) time-major; with reverse, row s < lens[b] (lens NULL: t) reads src row
 * lens[b] - 1 - s (the backward direction of a bidirectional LSTM over ragged sequences) */
int pk_taco2_time_major(const float* src, const int32_t* lens, int32_t reverse, int32_t batch, int32_t t, int32_t channels, float* dst,
                        pk_stream_t stream);
/* out (batch, t, 2 hidden + gc_dim) = [h_fwd[s] | h_bwd[lens - 1 - s] | gc[b]] for s < lens[b] (NULL: t), zero rows after;
 * h_fwd / h_bwd (t, batch, hidden) time-major */
int pk_taco2_bilstm_merge(const float* h_fwd, const float* h_bwd, const int32_t* lens, const float* gc, int32_t batch, int32_t t,
                          int32_t hidden, int32_t gc_dim, float* out, pk_stream_t stream);
/* Tacotron2Loss.forward, one block in double: out[5] = {loss, mel_loss, post_mel_loss, guided_attn_loss (align != NULL, else 0),
 * stop_loss (stop_logits != NULL, else 0)}; mel / post / target (batch, t, channels), align (batch, t, t_enc), slens / plens int32 */
int pk_taco2_loss(const float* mel, const float* post, const float* target, int32_t batch, int32_t t, int32_t channels, const float* align,
                  int32_t t_enc, const int32_t* slens, const int32_t* plens, float sigma, const float* stop_logits, float* out,
                  pk_stream_t stream);

/* ---- TransformerTTS (csrc/transformer_tts.cu) ---------------------------------------------------------------------------------
 * pk_tts_decode: every step of TransformerTTS.inference's decoder loop (B = 1) in one persistent launch of a co-resident grid.
 * Step t feeds the last of the r frames of step t - 1 (zeros at t = 0) through the prenet (Linear -> ReLU -> dropout p_prenet,
 * Philox site = prenet layer, step = t, element j: pk_dropout's convention), the input Linear and + alpha pe[t], then `layers`
 * pre-LN decoder layers on the new row (self-attention over the cached K / V of rows 0..t, source attention over mem_kv, the
 * position-wise Linear feed-forward), after_norm, prob_out and feat_out.  It stops after step idx = t + 1 once
 * (any sigmoid(prob) >= threshold or idx >= maxlen) and idx >= minlen.  fp32 FFMA, fixed summation order, no atomics.
 *   mem_kv   (t_enc, layers * 2 adim) fp32: [K_0 | V_0 | K_1 | ...] of the source attentions over the encoder output
 *   pre_w    prenet weights [out][in] row-major, layer 0 (prenet_units x odim) then the others; pre_b (prenet_layers, prenet_units)
 *   in_w     (adim, prenet_units), in_b (adim); pe (steps, adim): alpha pe rows of the decoder's ScaledPositionalEncoding
 *   layer_w  layers x pk_tts_layer_floats(adim, units) floats, each: wqkv (3 adim, adim), bqkv, wo_self (adim, adim), bo_self,
 *            wq_src, bq_src, wo_src, bo_src, w1 (units, adim), b1, w2 (adim, units), b2, then gamma / beta of norm1, norm2, norm3
 *   norm     after_norm gamma | beta; out_w (r + r odim, adim) = [prob_out rows | feat_out rows], out_b (r + r odim)
 *   outs     (steps, r odim), probs (steps, r) sigmoid, att_ws (layers, heads, steps, t_enc): zeroed by the call, rows past the
 *            stop stay zero; frames[0] = decoder steps run.  steps >= max(minlen, maxlen) sizes the caches and outputs.
 * Refused with PK_ERR_UNSUPPORTED: head widths other than 64, 128 and 192, units / prenet_units / odim not multiples of 4,
 * r > 16, max(steps, t_enc) past the shared-memory score buffer, fewer co-resident CTAs than heads. */
typedef struct {
  int32_t t_enc, adim, heads, units, odim, r, prenet_layers, prenet_units, layers, steps, minlen, maxlen;
  float threshold, p_prenet;
  uint64_t seed;
  const float* mem_kv; const float* pre_w; const float* pre_b; const float* in_w; const float* in_b; const float* pe;
  const float* layer_w; const float* norm; const float* out_w; const float* out_b;
  float* workspace; int64_t workspace_len;   /* pk_tts_workspace() floats, 16-byte aligned */
  float* outs; float* probs; float* att_ws; int32_t* frames;
} PkTtsDecodeArgs;
int64_t pk_tts_layer_floats(int32_t adim, int32_t units);
int64_t pk_tts_workspace(int32_t adim, int32_t units, int32_t prenet_units, int32_t layers, int32_t steps);
int pk_tts_decode(const PkTtsDecodeArgs* args, pk_stream_t stream);
/* Glue of the teacher-forced forward.  pk_tts_text_eos: xs (batch, t + 1) = text with eos at column lens[b] and zeros after,
 * ilens = lens + 1 (text may be NULL when t = 0).  pk_tts_shift_frames: out (batch, l / r, odim)[b, 0] = 0, [b, i] = ys[b, i r - 1].  pk_tts_prenet_dropout: in
 * place on (batch, l, units), element (b, i, j) kept with Philox site, step i, element b units + j (pk_tts_decode's masks), scaled
 * 1 / (1 - p).  pk_tts_stop_labels: out (batch, width) = 1 where column >= olens[b] - 1 or column == width - 1, else 0. */
int pk_tts_text_eos(const int64_t* text, const int32_t* lens, int32_t batch, int32_t t, int64_t eos, int64_t* xs, int32_t* ilens,
                    pk_stream_t stream);
int pk_tts_shift_frames(const float* ys, int32_t batch, int32_t l, int32_t odim, int32_t r, float* out, pk_stream_t stream);
int pk_tts_prenet_dropout(float* x, int32_t batch, int32_t l, int32_t units, float p, uint64_t seed, int32_t site, pk_stream_t stream);
int pk_tts_stop_labels(const int32_t* olens, int32_t batch, int32_t width, float* out, pk_stream_t stream);

/* ------------------------------------------------------------------------------------------------------------
 * TransformerTTS training step (reference: TransformerTTSUpdater.update_core, models/transformer_tts/
 * transformer_tts_updater.py:73-170).  The attention runs on the materialised path of the FastSpeech2 step (pk_conv_gemm,
 * pk_masked_softmax with its causal mask, pk_dropout, pk_softmax_bwd with the guided source-attention loss fused in); these
 * add the guided loss's value and TransformerTTSLoss.  No atomics.
 * ------------------------------------------------------------------------------------------------------------ */
/* The guided loss from the n partials of pk_softmax_bwd (every guided layer's): lambda * sum / (heads_layers *
 * sum_b min(ilens[b], keys) min(olens[b], rows)) -> losses[4], and added to losses[0]. */
int pk_tts_guided_loss(const float* partials, int64_t n, const int32_t* ilens, const int32_t* olens, int32_t batch, int32_t rows,
                       int32_t keys, int32_t heads_layers, float lambda, float* losses, pk_stream_t stream);
/* TransformerTTSLoss (transformer_tts.py:770-872, use_masking=True) over the frames t < olens[b] of before / after / ys
 * (batch, l_max, odim) and logits / labels (batch, l_max): losses[0..3] = {loss, l1, l2, bce}; l1 = mean|after - ys| +
 * mean|before - ys|, l2 the same with squares, bce = BCEWithLogitsLoss(pos_weight) on the logits, loss = l1 + bce (loss_type 0),
 * l2 + bce (1) or l1 + l2 + bce (2).  workspace: pk_tts_loss_workspace(batch, l_max) floats. */
int64_t pk_tts_loss_workspace(int32_t batch, int32_t l_max);
int pk_tts_loss(const float* before, const float* after, const float* ys, const float* logits, const float* labels, const int32_t* olens,
                int32_t batch, int32_t l_max, int32_t odim, float pos_weight, int32_t loss_type, float* workspace, float* losses,
                pk_stream_t stream);
/* gradients of losses[0] of pk_tts_loss w.r.t. before, after and logits (0 on the padded frames) */
int pk_tts_loss_bwd(const float* before, const float* after, const float* ys, const float* logits, const float* labels,
                    const int32_t* olens, int32_t batch, int32_t l_max, int32_t odim, float pos_weight, int32_t loss_type, float* g_before,
                    float* g_after, float* g_logits, pk_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PARAKEET_B200_H_ */
