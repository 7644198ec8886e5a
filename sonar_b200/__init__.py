"""sonar_b200 -- Hopper (sm_90a) engine behind the SONAR ``inference_pipelines`` API.

Only the text-embedding hot path lives here (SURVEY.md §8): host batcher + pipeline mirror
in Python, all arithmetic in ``lib/libsonar_b200.so`` (``include/sonar_b200.h``).
"""

__version__ = "0.1.0"

from .sequence import PaddingMask, SequenceBatch, SonarEncoderOutput  # noqa: F401
from .text_encoder import (  # noqa: F401
    B200TextEncoderModel,
    Pooling,
    SonarTextEncoderConfig,
    VocabularyInfo,
    sonar_text_encoder_config,
)
from .text_decoder import B200TextDecoderModel, SonarTextDecoderConfig, sonar_text_decoder_config  # noqa: F401,E402
from .speech_encoder import B200SpeechEncoderModel, SonarSpeechEncoderConfig, sonar_speech_encoder_config  # noqa: F401,E402
from .laser2 import B200LaserLstmEncoder, Laser2Config, laser2_config  # noqa: F401,E402
from .blaser import B200BlaserModel, BlaserConfig, blaser_config, load_blaser_model  # noqa: F401,E402
