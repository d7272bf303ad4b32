"""`deep_recommenders.keras.layers`: BASELINE.json's north_star names this package; the
reference does not have it (SURVEY.md section 0, fact 2).  It is provided here as a re-export
of the hot-path layers so either import path works."""
from .base import Layer, Model, Dense, Sequential, register_keras_serializable  # noqa: F401
from .merge import Multiply, Subtract  # noqa: F401


def __getattr__(name):
    # lazy re-exports (avoid import cycles with keras.models.*)
    if name in ("FM", "FactorizationMachine", "DeepFM"):
        from ..models import ranking
        return getattr(ranking, name)
    if name in ("Cross", "DCN"):
        from ..models.ranking import dcn
        return getattr(dcn, name)
    if name in ("CIN", "XDeepFM"):
        from ..models.ranking import xdeepfm
        return getattr(xdeepfm, name)
    if name in ("ActivationUnit", "Dice", "DIN"):
        from ..models.ranking import din
        return getattr(din, name)
    if name == "DNN":
        from ..models.ranking.deepfm import DNN
        return DNN
    if name in ("Retrieval", "HardNegativeMining", "RemoveAccidentalNegative",
                "SamplingProbabilityCorrection", "TwoTower"):
        from ..models.retrieval import sbcnm
        return getattr(sbcnm, name)
    raise AttributeError(name)
