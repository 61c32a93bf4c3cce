"""STFT / MelScale on H100 (reference parakeet/modules/audio.py:74-229) and the numpy feature extractors of
parakeet/data/get_feats.py (LogMelFBank :20-88, Energy :167-220) - all transforms run in pk_stft (radix-2 FFT kernel).

Window tables (scipy get_window, centre-padded), FFT twiddles and the Slaney mel filterbank (what librosa.filters.mel
returns by default) are built once on the host at construction time, like the reference builds its DFT-matrix weight.
"""
import ctypes as C
import math

import numpy as np
import torch
from scipy import signal

from .. import _lib
from ..layer import Layer
from ..ops import _ptr, _stream


def _hz_to_mel(f):
    f = np.asanyarray(f, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    logstep = np.log(6.4) / 27.0
    return np.where(f >= min_log_hz, min_log_hz / f_sp + np.log(np.maximum(f, 1e-10) / min_log_hz) / logstep, f / f_sp)


def _mel_to_hz(m):
    m = np.asanyarray(m, dtype=np.float64)
    f_sp, min_log_hz = 200.0 / 3, 1000.0
    logstep = np.log(6.4) / 27.0
    return np.where(m >= min_log_hz / f_sp, min_log_hz * np.exp(logstep * (m - min_log_hz / f_sp)), f_sp * m)


def mel_filterbank(sr, n_fft, n_mels=80, fmin=0.0, fmax=None):
    """Slaney-scale, area-normalised triangular filters == librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax)."""
    fmax = sr / 2 if fmax is None else fmax
    freqs = np.linspace(0, sr / 2, 1 + n_fft // 2)
    mel_f = _mel_to_hz(np.linspace(_hz_to_mel(fmin), _hz_to_mel(fmax), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - freqs[None, :]
    w = np.maximum(0, np.minimum(-ramps[:-2] / fdiff[:-1, None], ramps[2:] / fdiff[1:, None]))
    return (w * (2.0 / (mel_f[2:] - mel_f[:-2]))[:, None]).astype(np.float32)


def _window(window, win_length, n_fft):
    w = signal.get_window(window, win_length, fftbins=True)
    if n_fft != win_length:
        lpad = (n_fft - win_length) // 2
        w = np.pad(w, (lpad, n_fft - win_length - lpad))
    return w.astype(np.float32)


def _twiddles(n_fft):
    j = np.arange(n_fft // 2, dtype=np.float64)
    return np.stack([np.cos(2 * np.pi * j / n_fft), -np.sin(2 * np.pi * j / n_fft)], axis=1).astype(np.float32)


class STFT(Layer):
    """reference modules/audio.py:74-215: forward -> (real, imag) (B, bins, frames); power; magnitude."""

    def __init__(self, n_fft, hop_length=None, win_length=None, window="hanning", center=True, pad_mode="reflect", device=None):
        super().__init__(device)
        if pad_mode != "reflect":
            raise NotImplementedError("only reflect padding (the reference supports nothing else either)")
        if win_length is None:
            win_length = n_fft
        if hop_length is None:
            hop_length = int(win_length // 4)
        if window == "hanning":
            window = "hann"
        self.hop_length, self.n_bin, self.n_fft, self.center, self.pad_mode = hop_length, 1 + n_fft // 2, n_fft, center, pad_mode
        self._win = torch.from_numpy(_window(window, win_length, n_fft)).to(self.device)
        self._tw = torch.from_numpy(_twiddles(n_fft)).to(self.device)

    def _run(self, x, re=False, im=False, mag=False, mag_layout=0, power_clip=-1.0, mel_w=None, mel_log10=False, mel_clip=1e-10,
             energy=False, energy_clip=1e-10):
        if not x.is_cuda:
            raise _lib.PkError("STFT needs CUDA tensors (no CPU fallback)")
        x = x.contiguous().float()
        B, T = x.shape
        frames = 1 + T // self.hop_length if self.center else 1 + (T - self.n_fft) // self.hop_length
        dev = x.device
        o = {}
        o["re"] = torch.empty(B, self.n_bin, frames, device=dev) if re else None
        o["im"] = torch.empty(B, self.n_bin, frames, device=dev) if im else None
        o["mag"] = torch.empty((B, self.n_bin, frames) if mag_layout == 0 else (B, frames, self.n_bin), device=dev) if mag else None
        n_mels = mel_w.shape[0] if mel_w is not None else 0
        o["mel"] = torch.empty(B, frames, n_mels, device=dev) if mel_w is not None else None
        o["energy"] = torch.empty(B, frames, device=dev) if energy else None
        _lib.check(_lib.lib().pk_stft(_ptr(x), B, T, _ptr(self._win), _ptr(self._tw), self.n_fft, self.hop_length,
                                      1 if self.center else 0, _ptr(o["re"]), _ptr(o["im"]), _ptr(o["mag"]), mag_layout,
                                      float(power_clip), _ptr(mel_w), n_mels, _ptr(o["mel"]), 1 if mel_log10 else 0,
                                      float(mel_clip), _ptr(o["energy"]), float(energy_clip), _stream()), "pk_stft")
        return o

    def forward(self, x):
        o = self._run(x, re=True, im=True)
        return o["re"], o["im"]

    def magnitude(self, x):
        return self._run(x, mag=True)["mag"]

    def power(self, x):
        m = self._run(x, mag=True)["mag"]
        return m * m


class MelScale(Layer):
    """reference modules/audio.py:218-229: mel = weight (n_mels, bins) @ spec (B, bins, frames)."""

    def __init__(self, sr, n_fft, n_mels, fmin, fmax, device=None):
        super().__init__(device)
        self._register("weight", torch.from_numpy(mel_filterbank(sr, n_fft, n_mels, fmin, fmax)))

    @property
    def weight(self):
        return self._params["weight"]

    def forward(self, spec):
        """(B, bins, frames) -> (B, n_mels, frames) through the tensor-core GEMM (frames as rows)."""
        from .. import ops
        spec_t = spec.transpose(1, 2)                                          # (B, frames, bins)
        pad = (-spec_t.shape[-1]) % 8                                          # TMA row pitch must be a multiple of 16 B
        a = ops.Split.from_f32(torch.nn.functional.pad(spec_t, (0, pad)).contiguous())
        w = ops.pack_weight(self.weight, spec.device)
        y, _ = ops.conv_gemm(a, w, n=self.weight.shape[0], k=self.weight.shape[1])
        return y.transpose(1, 2)


class LogMelFBank:
    """reference data/get_feats.py:20-88 (librosa.stft -> abs -> mel -> clip 1e-10 -> log10), on the GPU."""

    def __init__(self, sr=24000, n_fft=2048, hop_length=300, win_length=None, window="hann", n_mels=80, fmin=80, fmax=7600,
                 eps=1e-10, device=None):
        self.sr, self.n_fft, self.hop_length, self.n_mels = sr, n_fft, hop_length, n_mels
        self.fmin = 0 if fmin is None else fmin
        self.fmax = sr / 2 if fmax is None else fmax
        self._stft = STFT(n_fft, hop_length, win_length, window, device=device)
        self.mel_filter = mel_filterbank(sr, n_fft, n_mels, self.fmin, self.fmax)
        self._mel_w = torch.from_numpy(self.mel_filter).to(self._stft.device)

    def get_log_mel_fbank(self, wav, base="10"):
        x = torch.as_tensor(wav, dtype=torch.float32, device=self._stft.device).reshape(1, -1)
        mel = self._stft._run(x, mel_w=self._mel_w, mel_log10=True, mel_clip=1e-10)["mel"][0]
        return mel if base == "10" else mel * math.log(10.0)


class Energy:
    """reference data/get_feats.py:167-220: sqrt(clip(sum_k |X|^2, 1e-10)) per frame (+ token averaging, :205-220)."""

    def __init__(self, sr=24000, n_fft=2048, hop_length=300, win_length=None, window="hann", center=True, pad_mode="reflect",
                 device=None):
        self._stft = STFT(n_fft, hop_length, win_length, window, center=center, pad_mode=pad_mode, device=device)

    @staticmethod
    def _average_by_duration(energy, d):
        """get_feats.py:205-213 on the device: mean of the frames of each token (0 for zero-length tokens) -> (T, 1)."""
        d = torch.as_tensor(np.asarray(d), dtype=torch.int64, device=energy.device).reshape(-1)
        ends = torch.cumsum(d, 0)
        csum = torch.cat([energy.new_zeros(1, dtype=torch.float64), torch.cumsum(energy.double(), 0)])
        ends_c, starts_c = ends.clamp(max=energy.shape[0]), (ends - d).clamp(max=energy.shape[0])   # numpy slicing clips at the end
        n = (ends_c - starts_c).clamp(min=1)
        avg = (csum[ends_c] - csum[starts_c]) / n
        return torch.where(ends_c > starts_c, avg, torch.zeros_like(avg)).float().reshape(-1, 1)

    def get_energy(self, wav, use_token_averaged_energy=True, duration=None):
        """reference :215-220; without `duration` the frame-level energy (frames,), with it the token average (T, 1)."""
        x = torch.as_tensor(wav, dtype=torch.float32, device=self._stft.device).reshape(1, -1)
        energy = self._stft._run(x, energy=True, energy_clip=1e-10)["energy"][0]
        if use_token_averaged_energy and duration is not None:
            energy = self._average_by_duration(energy, duration)
        return energy
