"""H100-native drop-in for the hot path of whisper-timestamped.

Same import name and API surface as the reference package
(/root/reference/whisper_timestamped/__init__.py:1-10): `transcribe`, `transcribe_timestamped`,
`load_model`, `__version__`.  All device work goes through libwts.so (hand-written sm_90a CUDA
behind the C-ABI of include/wts.h); importing this package fails if that library is missing.
"""
from . import _native  # noqa: F401  (fails loudly when libwts.so is absent)
from .model import load_model  # noqa: F401
from .model_zoo import ModelDimensions  # noqa: F401
from .transcribe import transcribe_timestamped  # noqa: F401
from .transcribe import transcribe_timestamped as transcribe  # noqa: F401

__version__ = "1.15.9+h100.r1"
