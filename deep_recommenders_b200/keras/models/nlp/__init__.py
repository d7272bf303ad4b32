"""Same public names as reference keras/models/nlp/__init__.py:4-5."""
from .multi_head_attention import MultiHeadAttention  # noqa: F401
from .transformer import Transformer  # noqa: F401
