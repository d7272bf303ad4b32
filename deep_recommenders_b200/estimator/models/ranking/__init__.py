from .deepfm import DeepFM  # noqa: F401
from .wide_and_deep import WDL  # noqa: F401
