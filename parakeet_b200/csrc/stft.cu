// STFT / mel front-end: batched in-shared-memory radix-2 FFT (no cuFFT), one CTA per frame, with fused epilogues
// (real/imag, clipped magnitude, mel filterbank, log10, frame energy).
//   reference: parakeet/modules/audio.py:161-229 (STFT = DFT-matrix conv1d, O(N^2) per frame; MelScale = matmul),
//              parakeet/modules/stft_loss.py:20-67, parakeet/data/get_feats.py:47-88,196-203
#include <algorithm>

#include "pk_host.h"

namespace pk {

struct StftArgs {
  const float* x;        // (B, T)
  const float* window;   // (n_fft) already centre-padded
  const float2* twiddle; // (n_fft/2): (cos, -sin)(2 pi j / n_fft)
  int t, n_fft, log2n, hop, center, frames, bins;
  float* re;             // (B, bins, frames) or NULL
  float* im;
  float* mag;            // magnitude or NULL
  int mag_layout;        // 0: (B, bins, frames)  1: (B, frames, bins)
  float power_clip;      // clip on re^2+im^2 before sqrt (< 0: none)
  const float* mel_w;    // (n_mels, bins) or NULL
  int n_mels;
  float* mel;            // (B, frames, n_mels)
  int mel_log10;         // 1: log10(max(mel, mel_clip))
  float mel_clip;
  float* energy;         // (B, frames) or NULL: sqrt(max(sum_k |X|^2, energy_clip))
  float energy_clip;
};

__global__ void __launch_bounds__(256) stft_kernel(const StftArgs a) {
  extern __shared__ float2 fft_smem[];
  float2* buf = fft_smem;                 // [n_fft]
  float2* tw = fft_smem + a.n_fft;        // [n_fft / 2]
  float* mags = reinterpret_cast<float*>(tw + a.n_fft / 2);   // [bins]
  __shared__ float red[8];
  const int f = blockIdx.x, b = blockIdx.y;
  const int N = a.n_fft;
  const float* xb = a.x + static_cast<long long>(b) * a.t;
  const int start = f * a.hop - (a.center ? N / 2 : 0);
  for (int n = threadIdx.x; n < N; n += blockDim.x) {
    int idx = start + n;
    if (idx < 0) idx = -idx;                          // reflect padding (np.pad mode="reflect")
    if (idx >= a.t) idx = 2 * (a.t - 1) - idx;
    idx = min(max(idx, 0), a.t - 1);
    const float v = __ldg(xb + idx) * __ldg(a.window + n);
    buf[__brev(static_cast<unsigned>(n)) >> (32 - a.log2n)] = make_float2(v, 0.f);
  }
  for (int j = threadIdx.x; j < N / 2; j += blockDim.x) tw[j] = a.twiddle[j];
  __syncthreads();
  for (int s = 1; s <= a.log2n; ++s) {
    const int half = 1 << (s - 1);
    const int tstride = N >> s;
    for (int i = threadIdx.x; i < N / 2; i += blockDim.x) {
      const int pos = i & (half - 1);
      const int ia = ((i >> (s - 1)) << s) + pos;
      const int ib = ia + half;
      const float2 w = tw[pos * tstride];
      const float2 vb = buf[ib], va = buf[ia];
      const float2 tt = make_float2(w.x * vb.x - w.y * vb.y, w.x * vb.y + w.y * vb.x);
      buf[ib] = make_float2(va.x - tt.x, va.y - tt.y);
      buf[ia] = make_float2(va.x + tt.x, va.y + tt.y);
    }
    __syncthreads();
  }
  float esum = 0.f;
  for (int k = threadIdx.x; k < a.bins; k += blockDim.x) {
    const float2 X = buf[k];
    const long long o_bf = (static_cast<long long>(b) * a.bins + k) * a.frames + f;
    if (a.re) a.re[o_bf] = X.x;
    if (a.im) a.im[o_bf] = X.y;
    float pw = X.x * X.x + X.y * X.y;
    esum += pw;
    if (a.power_clip >= 0.f) pw = fmaxf(pw, a.power_clip);
    const float m = sqrtf(pw);
    mags[k] = m;
    if (a.mag) a.mag[a.mag_layout == 0 ? o_bf : (static_cast<long long>(b) * a.frames + f) * a.bins + k] = m;
  }
  if (a.energy) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) esum += __shfl_xor_sync(0xffffffffu, esum, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = esum;
  }
  __syncthreads();
  if (a.energy && threadIdx.x == 0) {
    float s = 0.f;
    for (int w = 0; w < static_cast<int>(blockDim.x) / 32; ++w) s += red[w];
    a.energy[static_cast<long long>(b) * a.frames + f] = sqrtf(fmaxf(s, a.energy_clip));
  }
  if (a.mel_w) {
    // one warp per mel band (dense row; rows are mostly zero - the filters are narrow triangles)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int m = warp; m < a.n_mels; m += blockDim.x / 32) {
      const float* wr = a.mel_w + static_cast<long long>(m) * a.bins;
      float acc = 0.f;
      for (int k = lane; k < a.bins; k += 32) acc = fmaf(__ldg(wr + k), mags[k], acc);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (lane == 0) {
        if (a.mel_log10) acc = log10f(fmaxf(acc, a.mel_clip));
        a.mel[(static_cast<long long>(b) * a.frames + f) * a.n_mels + m] = acc;
      }
    }
  }
}

}  // namespace pk

extern "C" int pk_stft(const float* x, int32_t batch, int32_t t, const float* window, const void* twiddle, int32_t n_fft, int32_t hop,
                       int32_t center, float* re, float* im, float* mag, int32_t mag_layout, float power_clip, const float* mel_w,
                       int32_t n_mels, float* mel, int32_t mel_log10, float mel_clip, float* energy, float energy_clip,
                       pk_stream_t stream) {
  using namespace pk;
  PK_CHECK_ARG(x && window && twiddle, "NULL pointer");
  PK_CHECK_ARG(batch > 0 && t > 0 && hop > 0, "bad sizes");
  PK_CHECK_ARG(n_fft >= 32 && n_fft <= 4096 && (n_fft & (n_fft - 1)) == 0, "n_fft must be a power of two in [32, 4096] (got %d)", n_fft);
  PK_CHECK_ARG(!center || t > n_fft / 2, "reflect padding needs t > n_fft/2");
  PK_CHECK_ARG(center || t >= n_fft, "signal shorter than one frame");
  PK_CHECK_ARG((mel_w == nullptr) == (mel == nullptr), "mel_w and mel must both be set or both NULL");
  PK_CHECK_ARG(re || im || mag || mel || energy, "no output requested");
  StftArgs a;
  a.x = x; a.window = window; a.twiddle = static_cast<const float2*>(twiddle);
  a.t = t; a.n_fft = n_fft; a.hop = hop; a.center = center;
  a.log2n = 0;
  while ((1 << a.log2n) < n_fft) ++a.log2n;
  a.frames = center ? 1 + t / hop : 1 + (t - n_fft) / hop;
  a.bins = n_fft / 2 + 1;
  a.re = re; a.im = im; a.mag = mag; a.mag_layout = mag_layout; a.power_clip = power_clip;
  a.mel_w = mel_w; a.n_mels = n_mels; a.mel = mel; a.mel_log10 = mel_log10; a.mel_clip = mel_clip;
  a.energy = energy; a.energy_clip = energy_clip;
  const size_t smem = sizeof(float2) * (n_fft + n_fft / 2) + sizeof(float) * a.bins;
  if (int rc = prepare_kernel(stft_kernel, 256, smem)) return rc;
  dim3 grid(a.frames, batch);
  stft_kernel<<<grid, 256, smem, static_cast<cudaStream_t>(stream)>>>(a);
  PK_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return PK_OK;
}

namespace pk {
// sums needed by SpectralConvergenceLoss / LogSTFTMagnitudeLoss (stft_loss.py:70-118):
//   out[0] += sum (y-x)^2, out[1] += sum y^2, out[2] += sum |log(max(y,eps)) - log(max(x,eps))|
__global__ void __launch_bounds__(256) spectral_loss_sums_kernel(const float* __restrict__ x, const float* __restrict__ y, long long n,
                                                                 float eps, float* __restrict__ out) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float xv = x[i], yv = y[i];
    s0 += (yv - xv) * (yv - xv);
    s1 += yv * yv;
    s2 += fabsf(logf(fmaxf(yv, eps)) - logf(fmaxf(xv, eps)));
  }
  __shared__ float red[3][8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s0 += __shfl_xor_sync(0xffffffffu, s0, o);
    s1 += __shfl_xor_sync(0xffffffffu, s1, o);
    s2 += __shfl_xor_sync(0xffffffffu, s2, o);
  }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = s0; red[1][threadIdx.x >> 5] = s1; red[2][threadIdx.x >> 5] = s2; }
  __syncthreads();
  if (threadIdx.x < 3) {
    float s = 0.f;
    for (int w = 0; w < 8; ++w) s += red[threadIdx.x][w];
    atomicAdd(out + threadIdx.x, s);
  }
}
}  // namespace pk

extern "C" int pk_spectral_loss_sums(const float* x_mag, const float* y_mag, int64_t n, float eps, float* out3, pk_stream_t stream) {
  PK_CHECK_ARG(x_mag && y_mag && out3 && n > 0, "bad arguments");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PK_CHECK_CUDA(cudaMemsetAsync(out3, 0, 3 * sizeof(float), s));
  const int blocks = static_cast<int>(std::min<long long>((n + 255) / 256, pk::sm_count() * 4LL));
  pk::spectral_loss_sums_kernel<<<blocks, 256, 0, s>>>(x_mag, y_mag, n, eps, out3);
  PK_CHECK_CUDA(cudaGetLastError());
  pk::count_launch();
  return PK_OK;
}
