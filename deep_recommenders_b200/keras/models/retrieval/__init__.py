"""Retrieval models: the two-tower retrieval task and its evaluation half (sbcnm task layers, the brute-force /
streaming top-k indexes and the FactorizedTopK metric), and the GCN layer.  The reference's retrieval/__init__.py:4-5
re-exports FactorizedTopK and GCN, as this one does; its faiss-backed index is outside the hot path (SURVEY.md
section 2)."""
from . import sbcnm  # noqa: F401
from . import factorized_top_k  # noqa: F401
from .factorized_top_k import FactorizedTopK  # noqa: F401
from .gcn import GCN  # noqa: F401
