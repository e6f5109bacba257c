"""lhotse_b200 — H100-native (sm_90a) batched Kaldi-style feature extraction behind lhotse's
``FeatureExtractor`` API.  See DESIGN.md for the hot-path scope and INTEGRATION.md for the binding."""
from .plan import EPSILON, LOG_EPSILON, FeaturePlan, build_plan  # noqa: F401
from .extractors import (  # noqa: F401
    B200Fbank,
    B200FbankConfig,
    B200LibrosaFbank,
    B200LibrosaFbankConfig,
    B200LogSpectrogram,
    B200LogSpectrogramConfig,
    B200Mfcc,
    B200MfccConfig,
    B200Spectrogram,
    B200SpectrogramConfig,
    B200WhisperFbank,
    B200WhisperFbankConfig,
    from_reference_config,
    install_as_default,
)
from .families import (  # noqa: F401
    B200KaldifeatFbank,
    B200KaldifeatFbankConfig,
    B200KaldifeatFrameOptions,
    B200KaldifeatMelOptions,
    B200KaldifeatMfcc,
    B200KaldifeatMfccConfig,
    B200TorchaudioFbank,
    B200TorchaudioFbankConfig,
    B200TorchaudioMfcc,
    B200TorchaudioMfccConfig,
    B200TorchaudioSpectrogram,
    B200TorchaudioSpectrogramConfig,
)
from .engine import Engine, B200FeatError, load_library  # noqa: F401

__version__ = "0.1.0"

# LHOTSE_B200_INSTALL_AS_DEFAULT=1: re-point lhotse's own registry names ("kaldi-fbank", "fbank", "whisper-fbank", ...) at the
# B200 classes on import, so that YAML-driven entry points (FeatureExtractor.from_yaml, the `lhotse feat extract` CLI) pick
# them up with nothing but `import lhotse_b200` (e.g. from sitecustomize / a recipe's __init__)
import os as _os

if _os.environ.get("LHOTSE_B200_INSTALL_AS_DEFAULT", "0") not in ("", "0"):
    install_as_default()

