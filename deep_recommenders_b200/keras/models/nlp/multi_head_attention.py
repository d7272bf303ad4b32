"""``Embedding``, ``ScaledDotProductAttention`` and ``MultiHeadAttention`` at
``deep_recommenders.keras.models.nlp.multi_head_attention``.

They mirror reference keras/models/nlp/multi_head_attention.py: the constructor arguments and defaults (:11, :38, :95),
the input-list protocol and its assertion messages (:61-66, :123-128), and the arithmetic of :45-58 and :72-84.  The
attention itself, with MultiHeadAttention's head split and merge (:134-147), is one fused CUDA kernel
(``dr_mha_attn_fwd``) that never materialises the ``[heads * batch, Lq, Lk]`` scores.  The three projections have no
bias and there is no output projection, as upstream; they run on ``dr_dense``.

Deviations (DESIGN section 7):
- Dropout applies only in training mode (upstream ``K.dropout`` also runs in ``predict``).
- ``MultiHeadAttention.get_config`` reports the constructor arguments (upstream has none), so ``from_config``
  round-trips.
- ``future=True`` with queries and keys of different lengths raises ``ValueError``.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
from torch import nn

from .... import ops
from ...layers.base import Layer, get_initializer, register_keras_serializable


def _device(x, fallback=None):
    if isinstance(x, torch.Tensor):
        return x.device
    if fallback is not None:
        return torch.device(fallback)
    return torch.device("cuda" if torch.cuda.is_available() else "cpu")


def _float(x, device) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x if x.dtype == torch.float32 else x.float()
    return torch.as_tensor(np.asarray(x, dtype=np.float32), device=device)


def _weight(shape, initializer, device, gen, trainable=True) -> nn.Parameter:
    t = torch.empty(tuple(int(s) for s in shape), dtype=torch.float32, device=device)
    get_initializer(initializer)(t, gen)
    return nn.Parameter(t, requires_grad=trainable)


def _generator(seed: Optional[int]) -> torch.Generator:
    gen = torch.Generator()
    if seed is None:
        gen.seed()
    else:
        gen.manual_seed(int(seed))
    return gen


def _dropout_seed(gen: torch.Generator) -> int:
    """A fresh 64-bit seed of the attention kernel's dropout hash for each training call."""
    return int(torch.randint(0, 1 << 62, (1,), generator=gen).item())


@register_keras_serializable()
class Embedding(Layer):
    """embeddings = table[inputs] * sqrt(model_dim), table [vocab_size, model_dim] glorot-uniform (:9-32)."""

    def __init__(self, vocab_size, model_dim, seed: Optional[int] = None, **kwargs):
        super().__init__(**kwargs)
        self._vocab_size = int(vocab_size)
        self._model_dim = int(model_dim)
        self._seed = seed
        self.embeddings = None

    def build(self, input_shape, device=None):
        gen = None if self._seed is None else torch.Generator().manual_seed(self._seed)
        self.embeddings = _weight((self._vocab_size, self._model_dim), "glorot_uniform", _device(None, device), gen)
        self.built = True

    def forward(self, inputs, **kwargs):
        if not self.built:
            self.build(None, device=_device(inputs))
        return self.call(inputs)

    def call(self, inputs, **kwargs):
        ids = torch.as_tensor(inputs, device=self.embeddings.device)
        if ids.dtype not in (torch.int32, torch.int64):
            ids = ids.to(torch.int32)
        return ops.Gather.apply(self.embeddings, ids, None) * (self._model_dim ** 0.5)

    def compute_output_shape(self, input_shape):
        return tuple(input_shape) + (self._model_dim,)

    def get_config(self):
        return {**super().get_config(), "vocab_size": self._vocab_size, "model_dim": self._model_dim}


def _unpack(inputs, masking: bool):
    if masking:
        assert len(inputs) == 4, "inputs should be set [queries, keys, values, masks]."
        return inputs
    assert len(inputs) == 3, "inputs should be set [queries, keys, values]."
    return (*inputs, None)


def _check_future(future: bool, q_shape, k_shape):
    if future and q_shape[1] != k_shape[1]:
        raise ValueError(f"future masking needs queries and keys of the same length, got {q_shape[1]} and "
                         f"{k_shape[1]}")


def _attend(q, k, v, masks, heads: int, future: bool, rate: float, gen: torch.Generator):
    dev = q.device
    m = None if masks is None else _float(masks, dev).to(dev)
    if m is not None and m.dim() != 2:
        m = m.reshape(m.shape[0], -1)
    seed = _dropout_seed(gen) if rate > 0 else 0
    return ops.MHAttentionFn.apply(q, k, v, m, heads, future, rate, seed)


@register_keras_serializable()
class ScaledDotProductAttention(Layer):
    """softmax(q k^T / sqrt(d) + masks * (-2^32 + 1), future positions replaced by -2^32 + 1) v (:35-89).
    ``masks`` [Bm, Lk] (1 = padding) is tiled over the batch when Bm divides it."""

    def __init__(self, masking=True, future=False, dropout_rate=0., seed: Optional[int] = None, **kwargs):
        super().__init__(**kwargs)
        self._masking = masking
        self._future = future
        self._dropout_rate = dropout_rate
        self._masking_num = -2 ** 32 + 1
        self._gen = _generator(seed)

    def forward(self, inputs, **kwargs):
        self.built = True
        return self.call(inputs, **kwargs)

    def call(self, inputs, **kwargs):
        queries, keys, values, masks = _unpack(inputs, self._masking)
        _check_future(self._future, queries.shape, keys.shape)
        dev = _device(queries)
        q, k, v = _float(queries, dev), _float(keys, dev), _float(values, dev)
        rate = float(self._dropout_rate) if self.training else 0.0
        return _attend(q, k, v, masks, 1, self._future, rate, self._gen)

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        return {**super().get_config(), "masking": self._masking, "future": self._future,
                "dropout_rate": self._dropout_rate}


@register_keras_serializable()
class MultiHeadAttention(Layer):
    """concat_h(attention(queries Wq_h, keys Wk_h, values Wv_h)) with Wq, Wk, Wv [in, n_heads * head_dim], no bias
    and no output projection (:92-152)."""

    def __init__(self, n_heads, head_dim, dropout_rate=.1, masking=True, future=False, trainable=True,
                 seed: Optional[int] = None, **kwargs):
        super().__init__(trainable=trainable, **kwargs)
        self._n_heads = int(n_heads)
        self._head_dim = int(head_dim)
        self._dropout_rate = dropout_rate
        self._masking = masking
        self._future = future
        self._trainable = trainable
        self._seed = seed
        self._gen = _generator(None if seed is None else seed + 7)
        self._weights_queries = self._weights_keys = self._weights_values = None

    def build(self, input_shape, device=None):
        """input_shape: the shapes of [queries, keys, values(, masks)]."""
        dev = _device(None, device)
        gen = None if self._seed is None else torch.Generator().manual_seed(self._seed)
        width = self._n_heads * self._head_dim
        self._weights_queries = _weight((input_shape[0][-1], width), "glorot_uniform", dev, gen, self._trainable)
        self._weights_keys = _weight((input_shape[1][-1], width), "glorot_uniform", dev, gen, self._trainable)
        self._weights_values = _weight((input_shape[2][-1], width), "glorot_uniform", dev, gen, self._trainable)
        self.built = True

    def forward(self, inputs, **kwargs):
        _unpack(inputs, self._masking)
        if not self.built:
            self.build([tuple(x.shape) for x in inputs[:3]], device=_device(inputs[0]))
        return self.call(inputs, **kwargs)

    def call(self, inputs, **kwargs):
        queries, keys, values, masks = _unpack(inputs, self._masking)
        _check_future(self._future, queries.shape, keys.shape)
        dev = self._weights_queries.device
        q = ops.DenseFn.apply(_float(queries, dev), self._weights_queries, None, 0)
        k = ops.DenseFn.apply(_float(keys, dev), self._weights_keys, None, 0)
        v = ops.DenseFn.apply(_float(values, dev), self._weights_values, None, 0)
        rate = float(self._dropout_rate) if self.training else 0.0
        return _attend(q, k, v, masks, self._n_heads, self._future, rate, self._gen)

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        return {**super().get_config(), "n_heads": self._n_heads, "head_dim": self._head_dim,
                "dropout_rate": self._dropout_rate, "masking": self._masking, "future": self._future}
