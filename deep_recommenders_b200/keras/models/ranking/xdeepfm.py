"""CIN layer (xDeepFM's Compressed Interaction Network) at
``deep_recommenders.keras.models.ranking.xdeepfm.CIN``, and an ``XDeepFM`` model on it.

``CIN`` mirrors reference keras/models/ranking/xdeepfm.py:8-116 (constructor arguments :12-37, the two
input-type checks of ``build`` :39-48 and the kernel shape ``(1, m*h, feature_map)`` :54-60, the rank check of
``call`` :75-80, ``get_config`` keys :98-116).  The outer product and the width-1 conv1d run as one CUDA kernel
(dr_cin_fwd) whose product operand never reaches global memory; the backward is hand-written (dr_cin_bwd).

Deviation: ``activation=None`` crashes in the reference (``None(conv_out)``); here it is the linear activation.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np
import torch
from torch import nn

from .... import ops
from ....embedding import EmbeddingCollection
from ...layers.base import (Dense, Layer, Model, get_initializer, get_regularizer, register_keras_serializable,
                            regularization_penalty, serialize_initializer)
from .deepfm import DNN


class _TensorShape(list):
    """The shape a single (non-tuple) input hands to ``build``, as Keras hands it a TensorShape."""


def _ndim(x) -> int:
    return x.dim() if isinstance(x, torch.Tensor) else np.ndim(x)


@register_keras_serializable()
class CIN(Layer):
    """ Compressed Interaction Network in xDeepFM """

    def __init__(self,
                 feature_map: Optional[int] = 3,
                 use_bias: bool = False,
                 activation="sigmoid",
                 kernel_init="truncated_normal",
                 kernel_regu=None,
                 bias_init="zeros",
                 bias_regu=None,
                 seed: Optional[int] = None,
                 **kwargs):
        super().__init__(**kwargs)
        self._feature_map = feature_map
        self._use_bias = use_bias
        self._activation = activation
        self._act = ops.act_code(activation)
        self._kernel_init_id = kernel_init
        self._bias_init_id = bias_init
        self._kernel_init = get_initializer(kernel_init)
        self._kernel_regu = get_regularizer(kernel_regu)
        self._bias_init = get_initializer(bias_init)
        self._bias_regu = get_regularizer(bias_regu)
        self._seed = seed
        self.kernel = None
        self.bias = None

    def build(self, input_shape, device=None):
        if not isinstance(input_shape, tuple):
            raise ValueError("`CIN` layer's inputs type should be `tuple`."
                             "Got `CIN` layer's inputs type = `{}`".format(
                                 type(input_shape)))

        if len(input_shape) != 2:
            raise ValueError("`CIN` Layer inputs tuple length should be 2."
                             "Got `length` = {}".format(len(input_shape)))

        x0_shape, x_shape = input_shape
        self._x0_fields = int(x0_shape[1])
        self._x_fields = int(x_shape[1])
        dev = device or ("cuda" if torch.cuda.is_available() else "cpu")
        gen = torch.Generator().manual_seed(self._seed) if self._seed is not None else None
        # initialised as the [m*h, feature_map] matrix it is: the fans of a (1, m*h, H) conv kernel
        k = torch.empty((self._x0_fields * self._x_fields, self._feature_map), dtype=torch.float32, device=dev)
        self._kernel_init(k, gen)
        self.kernel = nn.Parameter(k.view(1, self._x0_fields * self._x_fields, self._feature_map))
        if self._use_bias is True:
            b = torch.empty((self._feature_map,), dtype=torch.float32, device=dev)
            self._bias_init(b, gen)
            self.bias = nn.Parameter(b)
        self.built = True

    def _ensure_built(self, inputs):
        if self.built:
            return
        if isinstance(inputs, tuple):
            shape = tuple(tuple(np.shape(t)) for t in inputs)
            dev = next((t.device for t in inputs if isinstance(t, torch.Tensor)), None)
        else:
            shape, dev = _TensorShape(np.shape(inputs)), None
        self.build(shape, device=dev)

    def forward(self, inputs, **kwargs):
        self._ensure_built(inputs)
        return self.call(inputs, **kwargs)

    def _check(self, inputs):
        x0, x = inputs
        if _ndim(x0) != 3 or _ndim(x) != 3:
            raise ValueError("`x0` and `x` dim should be 3."
                             "Got `x0` dim = {}, `x` dim = {}".format(_ndim(x0), _ndim(x)))
        dev = self.kernel.device

        def as_t(t):
            return t if isinstance(t, torch.Tensor) else torch.as_tensor(np.asarray(t, dtype=np.float32), device=dev)

        same = x is x0
        x0 = as_t(x0)
        return x0, (x0 if same else as_t(x)), same

    def call(self, inputs, **kwargs):
        x0, x, same = self._check(inputs)
        y, _ = ops.CINFn.apply(x0, x, self.kernel, self.bias, self._act, same, False)
        return y

    def call_pooled(self, inputs):
        """(y [B, H, D], sum_d y [B, H]): xDeepFM's sum pooling written by the same kernel."""
        self._ensure_built(inputs)
        x0, x, same = self._check(inputs)
        return ops.CINFn.apply(x0, x, self.kernel, self.bias, self._act, same, True)

    @property
    def losses(self):
        out = []
        if self.kernel is not None and self._kernel_regu is not None:
            out.append(regularization_penalty(self._kernel_regu, self.kernel))
        if self.bias is not None and self._bias_regu is not None:
            out.append(regularization_penalty(self._bias_regu, self.bias))
        return out

    def get_config(self):
        act = self._activation
        config = {
            "feature_map":
                self._feature_map,
            "use_bias":
                self._use_bias,
            "activation":
                "linear" if act is None else (act if isinstance(act, str) else getattr(act, "__name__", str(act))),
            "kernel_init":
                serialize_initializer(self._kernel_init_id),
            "kernel_regu":
                self._kernel_regu,
            "bias_init":
                serialize_initializer(self._bias_init_id),
            "bias_regu":
                self._bias_regu,
        }
        base_config = super().get_config()
        return {**base_config, **config}


class XDeepFM(Model):
    """xDeepFM (Lian et al., KDD 2018, "xDeepFM: Combining Explicit and Implicit Feature Interactions"), this repo's
    definition (the reference has only the ``CIN`` layer):

        linear = bias + sum_s w_s[id_s]                         first-order weights ride in the embedding rows
        x0     = [e_1 .. e_S]  [B, S, D]                        one fused gather (dr_embed_fm_fwd, DR_EMBED_NO_FM)
        x_1    = CIN((x0, x0)),  x_k = CIN((x0, x_{k-1}))       each also sum-pooled over d: p_k [B, H_k]
        deep   = DNN(flatten(x0))
        prob   = sigmoid(Dense(1)([p_1 | .. | p_K | deep]) + linear)
    """

    def __init__(self, rows: Sequence[int], dim: int, cin_layers: Sequence[int] = (128, 128),
                 cin_activation="sigmoid", dnn_units: Sequence[int] = (256, 32), dnn_activation="relu",
                 sparse_lr: Optional[float] = None, seed: Optional[int] = None, device=None, **kwargs):
        super().__init__(**kwargs)
        self.embeddings = EmbeddingCollection(rows, dim, with_linear=True, device=device, seed=seed,
                                              sparse_lr=sparse_lr)
        self.cin = nn.ModuleList([CIN(feature_map=int(h), activation=cin_activation,
                                      seed=None if seed is None else seed + 100 + i)
                                  for i, h in enumerate(cin_layers)])
        self.dnn = DNN(list(dnn_units), activation=dnn_activation, out_units=0,
                       seed=None if seed is None else seed + 200)
        self.head = Dense(1, seed=None if seed is None else seed + 300)
        dev = self.embeddings.weight.device
        S, D = len(list(rows)), int(dim)
        x = (None, S, D)
        for layer in self.cin:
            layer.build(((None, S, D), x), device=dev)
            x = (None, layer._feature_map, D)
        self._cfg = dict(rows=list(rows), dim=dim, cin_layers=[int(h) for h in cin_layers],
                         cin_activation=cin_activation, dnn_units=list(dnn_units), dnn_activation=dnn_activation)
        self.built = True

    def logits(self, ids: torch.Tensor) -> torch.Tensor:
        stack, linear = self.embeddings(ids, want_logit=True, second_order=False)
        x = stack
        pools = []
        for layer in self.cin:
            x, p = layer.call_pooled((stack, x))
            pools.append(p)
        deep = self.dnn(stack.reshape(stack.shape[0], -1))
        return self.head(torch.cat(pools + [deep], dim=1)) + linear.view(-1, 1)

    def call(self, ids, **kwargs):
        return torch.sigmoid(self.logits(ids))

    @property
    def losses(self):
        return [l for layer in self.cin for l in layer.losses]

    def get_config(self):
        return {**super().get_config(), **self._cfg}
