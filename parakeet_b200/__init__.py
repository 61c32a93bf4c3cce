"""parakeet_b200: H100-native (sm_90a) engine for the Parakeet TTS hot path (FastSpeech2 + Parallel WaveGAN /
WaveFlow + STFT/mel). Host side mirrors parakeet.models.* / parakeet.modules.*; all math runs in
libparakeet_b200.so (hand-written CUDA, C-ABI in include/parakeet_b200.h). No CPU fallback."""
__version__ = "0.1.0"
