"""``PositionEncoding``, ``Add``, ``PositionWiseFeedForward``, ``LayerNormalization``, ``Transformer``, ``Noam`` and
``label_smoothing`` at ``deep_recommenders.keras.models.nlp.transformer``.

They mirror reference keras/models/nlp/transformer.py (constructor arguments, defaults and ``get_config`` keys; the
arithmetic of :19-28, :80-85, :109-113, :191-271, :299-324).  The hot paths are CUDA: the attention kernel of
``multi_head_attention``, ``dr_dense`` with the relu epilogue for the feed-forward, ``dr_add_layernorm`` for every
Add & Norm (the residual sum is fused into the normalisation), the tied output projection on ``dr_scores_fwd`` /
``dr_dense`` without a transposed copy of the embedding table, and ``dr_softmax_rows`` over the vocabulary.

Deviation (DESIGN section 7): the dropout on the embeddings, like the attention's, applies only in training mode.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from .... import ops
from ...layers.base import Layer, register_keras_serializable
from .multi_head_attention import MultiHeadAttention, _device, _float, _generator, _weight

_POS_CACHE: dict = {}


def position_encodings(seq_length: int, model_dim: int) -> np.ndarray:
    """The sinusoid table of transformer.py:19-28 in float64: pos / 10000 ** ((i - i % 2) / d), sin on even columns,
    cos on odd ones."""
    pos = np.arange(seq_length, dtype=np.float64)[:, None]
    i = np.arange(model_dim)
    pe = pos / np.power(10000, (i - i % 2) / model_dim)
    pe[:, 0::2] = np.sin(pe[:, 0::2])
    pe[:, 1::2] = np.cos(pe[:, 1::2])
    return pe


@register_keras_serializable()
class PositionEncoding(Layer):
    """[seq_length, model_dim] float32 sinusoids for inputs [batch, seq_length, ...] (:12-31)."""

    def __init__(self, model_dim, **kwargs):
        super().__init__(**kwargs)
        self._model_dim = int(model_dim)

    def forward(self, inputs, **kwargs):
        self.built = True
        return self.call(inputs)

    def call(self, inputs, **kwargs):
        L = int(inputs.shape[1])
        dev = _device(inputs)
        key = (L, self._model_dim, str(dev))
        if key not in _POS_CACHE:
            _POS_CACHE[key] = torch.as_tensor(position_encodings(L, self._model_dim).astype(np.float32), device=dev)
        return _POS_CACHE[key]

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        return {**super().get_config(), "model_dim": self._model_dim}


@register_keras_serializable()
class Add(Layer):
    """input_a + input_b (:34-45)."""

    def forward(self, inputs, **kwargs):
        self.built = True
        return self.call(inputs)

    def call(self, inputs, **kwargs):
        input_a, input_b = inputs
        return input_a + input_b

    def compute_output_shape(self, input_shape):
        return input_shape[0]


@register_keras_serializable()
class PositionWiseFeedForward(Layer):
    """relu(x W_inner + b_inner) W_out + b_out (:48-88); the biases are initialised 'uniform' (U(-0.05, 0.05))."""

    def __init__(self, model_dim, inner_dim, trainable=True, seed: Optional[int] = None, **kwargs):
        super().__init__(trainable=trainable, **kwargs)
        self._model_dim = int(model_dim)
        self._inner_dim = int(inner_dim)
        self._trainable = trainable
        self._seed = seed
        self.weights_inner = self.weights_out = self.bias_inner = self.bias_out = None

    def build(self, input_shape, device=None):
        dev = _device(None, device)
        gen = None if self._seed is None else torch.Generator().manual_seed(self._seed)
        tr = self._trainable
        self.weights_inner = _weight((input_shape[-1], self._inner_dim), "glorot_uniform", dev, gen, tr)
        self.weights_out = _weight((self._inner_dim, self._model_dim), "glorot_uniform", dev, gen, tr)
        self.bias_inner = _uniform((self._inner_dim,), dev, gen, tr)
        self.bias_out = _uniform((self._model_dim,), dev, gen, tr)
        self.built = True

    def forward(self, inputs, **kwargs):
        if not self.built:
            self.build(tuple(inputs.shape), device=_device(inputs))
        return self.call(inputs)

    def call(self, inputs, **kwargs):
        x = _float(inputs, self.weights_inner.device)
        inner = ops.DenseFn.apply(x, self.weights_inner, self.bias_inner, ops.ACT_CODES["relu"])
        return ops.DenseFn.apply(inner, self.weights_out, self.bias_out, 0)

    def compute_output_shape(self, input_shape):
        return self._model_dim

    def get_config(self):
        return {**super().get_config(), "model_dim": self._model_dim, "inner_dim": self._inner_dim}


def _uniform(shape, device, gen, trainable):
    """tf.keras.initializers.get('uniform') == RandomUniform(-0.05, 0.05)."""
    t = torch.empty(shape, dtype=torch.float32).uniform_(-0.05, 0.05, generator=gen)
    return torch.nn.Parameter(t.to(device), requires_grad=trainable)


@register_keras_serializable()
class LayerNormalization(Layer):
    """gamma * (x - mean) / (variance + epsilon) ** 0.5 + beta over the last axis (:91-116).  ``call(inputs,
    residual=None)`` normalises ``inputs + residual`` in the same kernel (the Transformer's Add & Norm)."""

    def __init__(self, epsilon=1e-8, **kwargs):
        super().__init__(**kwargs)
        self._epsilon = epsilon
        self.beta = self.gamma = None

    def build(self, input_shape, device=None):
        dev = _device(None, device)
        C = int(input_shape[-1])
        self.beta = torch.nn.Parameter(torch.zeros(C, dtype=torch.float32, device=dev))
        self.gamma = torch.nn.Parameter(torch.ones(C, dtype=torch.float32, device=dev))
        self.built = True

    def forward(self, inputs, residual=None, **kwargs):
        if not self.built:
            self.build(tuple(inputs.shape), device=_device(inputs))
        return self.call(inputs, residual)

    def call(self, inputs, residual=None, **kwargs):
        dev = self.gamma.device
        return ops.AddLayerNormFn.apply(_float(inputs, dev), None if residual is None else _float(residual, dev),
                                        self.gamma, self.beta, float(self._epsilon))

    def compute_output_shape(self, input_shape):
        return input_shape

    def get_config(self):
        return {**super().get_config(), "epsilon": self._epsilon}


@register_keras_serializable()
class Transformer(Layer):
    """Vaswani et al.'s encoder-decoder (:119-287): ``call(encoder_inputs, decoder_inputs)`` -> softmax over the
    vocabulary [batch, decoder_length, vocab_size].  Token 0 is padding (masked as a key).  The embedding table is
    shared by both inputs and tied to the output projection."""

    def __init__(self, vocab_size, model_dim, n_heads=8, encoder_stack=6, decoder_stack=6, feed_forward_size=2048,
                 dropout_rate=0.1, seed: Optional[int] = None, **kwargs):
        super().__init__(**kwargs)
        self._vocab_size = int(vocab_size)
        self._model_dim = int(model_dim)
        self._n_heads = int(n_heads)
        self._encoder_stack = int(encoder_stack)
        self._decoder_stack = int(decoder_stack)
        self._feed_forward_size = int(feed_forward_size)
        self._dropout_rate = dropout_rate
        self._seed = seed
        self._gen = _generator(None if seed is None else seed + 11)

    def build(self, input_shape, device=None):
        dev = _device(None, device)
        seed = self._seed
        gen = None if seed is None else torch.Generator().manual_seed(seed)
        sub = (lambda k: None) if seed is None else (lambda k: seed + 1000 + k)
        d, h, ff = self._model_dim, self._n_heads, self._feed_forward_size
        n_enc, n_dec = self._encoder_stack, self._decoder_stack
        self.embeddings = _weight((self._vocab_size, d), "glorot_uniform", dev, gen)
        mha = lambda k, future=False: MultiHeadAttention(h, d // h, future=future, seed=sub(k))
        ffn = lambda k: PositionWiseFeedForward(d, ff, seed=sub(k))
        self.EncoderPositionEncoding = PositionEncoding(d)
        self.EncoderMultiHeadAttentions = torch.nn.ModuleList([mha(i) for i in range(n_enc)])
        self.EncoderLayerNorms0 = torch.nn.ModuleList([LayerNormalization() for _ in range(n_enc)])
        self.EncoderPositionWiseFeedForwards = torch.nn.ModuleList([ffn(100 + i) for i in range(n_enc)])
        self.EncoderLayerNorms1 = torch.nn.ModuleList([LayerNormalization() for _ in range(n_enc)])
        self.DecoderPositionEncoding = PositionEncoding(d)
        self.DecoderMultiHeadAttentions0 = torch.nn.ModuleList([mha(200 + i, True) for i in range(n_dec)])
        self.DecoderLayerNorms0 = torch.nn.ModuleList([LayerNormalization() for _ in range(n_dec)])
        self.DecoderMultiHeadAttentions1 = torch.nn.ModuleList([mha(300 + i) for i in range(n_dec)])
        self.DecoderLayerNorms1 = torch.nn.ModuleList([LayerNormalization() for _ in range(n_dec)])
        self.DecoderPositionWiseFeedForwards = torch.nn.ModuleList([ffn(400 + i) for i in range(n_dec)])
        self.DecoderLayerNorms2 = torch.nn.ModuleList([LayerNormalization() for _ in range(n_dec)])
        shape = (None, None, d)
        for m in self.modules():
            if m is not self and isinstance(m, (MultiHeadAttention, PositionWiseFeedForward, LayerNormalization)):
                m.build([shape] * 3 if isinstance(m, MultiHeadAttention) else shape, device=dev)
        self.train(self.training)          # the sub-layers take the mode set before this lazy build
        self.built = True

    def forward(self, encoder_inputs, decoder_inputs, **kwargs):
        if not self.built:
            self.build(None, device=_device(encoder_inputs))
        return self.call(encoder_inputs, decoder_inputs)

    def _ids(self, inputs) -> torch.Tensor:
        ids = torch.as_tensor(inputs, device=self.embeddings.device)
        return ids if ids.dtype == torch.int32 else ids.to(torch.int32)

    def _embed(self, ids, position: PositionEncoding) -> torch.Tensor:
        emb = ops.Gather.apply(self.embeddings, ids, None) * (self._model_dim ** 0.5)
        enc = emb + position(emb)
        if self.training and self._dropout_rate > 0:
            keep = torch.rand(enc.shape, generator=self._gen) >= self._dropout_rate
            enc = enc * (keep.to(enc.device, torch.float32) * (1.0 / (1.0 - self._dropout_rate)))
        return enc

    def encoder(self, inputs):
        ids = self._ids(inputs)
        masks = (ids == 0).to(torch.float32)
        encodings = self._embed(ids, self.EncoderPositionEncoding)
        for i in range(self._encoder_stack):
            attention_out = self.EncoderMultiHeadAttentions[i]([encodings, encodings, encodings, masks])
            attention_out = self.EncoderLayerNorms0[i](attention_out, encodings)
            ff_out = self.EncoderPositionWiseFeedForwards[i](attention_out)
            encodings = self.EncoderLayerNorms1[i](ff_out, attention_out)
        return encodings, masks

    def decoder(self, inputs):
        decoder_inputs, encoder_encodings, encoder_masks = inputs
        ids = self._ids(decoder_inputs)
        decoder_masks = (ids == 0).to(torch.float32)
        encodings = self._embed(ids, self.DecoderPositionEncoding)
        for i in range(self._decoder_stack):
            masked = self.DecoderMultiHeadAttentions0[i]([encodings, encodings, encodings, decoder_masks])
            masked = self.DecoderLayerNorms0[i](masked, encodings)
            attention_out = self.DecoderMultiHeadAttentions1[i](
                [masked, encoder_encodings, encoder_encodings, encoder_masks])
            attention_out = self.DecoderLayerNorms1[i](attention_out, masked)
            ff_out = self.DecoderPositionWiseFeedForwards[i](attention_out)
            encodings = self.DecoderLayerNorms2[i](ff_out, attention_out)
        B, L, d = encodings.shape
        logits = ops.TiedProjectionFn.apply(encodings.reshape(B * L, d), self.embeddings)
        return ops.SoftmaxRowsFn.apply(logits).view(B, L, self._vocab_size)

    def call(self, encoder_inputs, decoder_inputs, **kwargs):
        encoder_encodings, encoder_masks = self.encoder(encoder_inputs)
        return self.decoder([decoder_inputs, encoder_encodings, encoder_masks])

    def compute_output_shape(self, input_shape):
        return input_shape[0][0], input_shape[0][1], self._vocab_size

    def get_config(self):
        config = {
            "vocab_size": self._vocab_size,
            "model_dim": self._model_dim,
            "n_heads": self._n_heads,
            "encoder_stack": self._encoder_stack,
            "decoder_stack": self._decoder_stack,
            "feed_forward_size": self._feed_forward_size,
            "dropout_rate": self._dropout_rate,
        }
        return {**super().get_config(), **config}


class Noam:
    """Learning-rate schedule of Vaswani et al. (:290-317): d^-0.5 * min(step^-0.5, step * warmup^-1.5), set after
    every batch; the rate before the first step is d^-0.5 * warmup^-1.5."""

    def __init__(self, model_dim, step_num=0, warmup_steps=4000, verbose=False):
        self._model_dim = model_dim
        self._step_num = step_num
        self._warmup_steps = warmup_steps
        self.verbose = verbose
        self.model = None

    def on_train_begin(self, logs=None):
        self.model.optimizer.lr = self._model_dim ** -.5 * self._warmup_steps ** -1.5

    def on_batch_end(self, batch, logs=None):
        self._step_num += 1
        self.model.optimizer.lr = self._model_dim ** -.5 * min(self._step_num ** -.5,
                                                               self._step_num * self._warmup_steps ** -1.5)

    def on_epoch_begin(self, epoch, logs=None):
        if self.verbose:
            print(f"epoch {epoch} lr: {self.model.optimizer.lr}")

    def on_epoch_end(self, epoch, logs=None):
        if logs is not None:
            logs["lr"] = self.model.optimizer.lr
        return False


def label_smoothing(inputs, epsilon=0.1):
    """(1 - epsilon) * inputs + epsilon / output_dim (:320-324)."""
    output_dim = inputs.shape[-1]
    return (1 - epsilon) * inputs + (epsilon / output_dim)
