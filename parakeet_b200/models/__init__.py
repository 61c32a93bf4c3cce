from .fastspeech2 import FastSpeech2, FastSpeech2Inference, FastSpeech2Loss  # noqa: F401
from .parallel_wavegan import PWGDiscriminator, PWGGenerator, PWGInference  # noqa: F401
from .speedyspeech import SpeedySpeech, SpeedySpeechInference  # noqa: F401
from .waveflow import ConditionalWaveFlow, WaveFlowLoss  # noqa: F401
from .lstm_speaker_encoder import LSTMSpeakerEncoder  # noqa: F401
from .tacotron2 import Tacotron2, Tacotron2Loss  # noqa: F401
from .transformer_tts import TransformerTTS, TransformerTTSInference  # noqa: F401
