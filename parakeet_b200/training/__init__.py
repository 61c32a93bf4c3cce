from .fs2_step import FastSpeech2TrainStep  # noqa: F401
from .flat import FlatAdam, FlatBuffers  # noqa: F401
from .pwg_step import PWGTrainStep  # noqa: F401
from .speedyspeech_step import SpeedySpeechTrainStep  # noqa: F401
from .waveflow_step import WaveFlowTrainStep  # noqa: F401
from .ge2e_step import GE2ETrainStep  # noqa: F401
from .transformer_tts_step import TransformerTTSTrainStep  # noqa: F401
