"""GCN layer (reference: keras/models/retrieval/gcn.py:7-67): ``GCN(units, ...)(features, adj)`` is
``Dense(units, activation)(adj @ features)``, plus ``features`` when ``residual``.

``adj`` is a prepared ``ops.CSRAdjacency``, a scipy sparse matrix or a torch sparse tensor (prepared on each call:
prepare it once with ``ops.CSRAdjacency.from_any`` when it is reused), or a dense matrix.

``(A X) W == A (X W)``, so the sparse product runs on the narrower side, ``min(F, units)`` columns:
  - F > units: ``Z = X W`` (Dense GEMM), then one SpMM with the bias and the activation fused (a residual needs
    F == units, so it never takes this order);
  - otherwise (the reference's order, ties included): ``S = A X`` (SpMM), then the Dense GEMM with its epilogue, and
    the row softmax after it when the activation is softmax.
A dense ``adj`` runs both products on the GEMM, in the same order.
"""
from __future__ import annotations

import numpy as np
import torch

from .... import ops
from ...layers.base import Dense, Layer, register_keras_serializable, serialize_initializer

_ACTS = {None: 0, "linear": 0, "relu": 1, "sigmoid": 2, "tanh": 3, "softmax": ops.ACT_SOFTMAX}


def _act_name(activation):
    return getattr(activation, "__name__", activation) if callable(activation) else activation


def _device_tensor(x, device) -> torch.Tensor:
    if isinstance(x, torch.Tensor):
        return x if x.device == device else x.to(device)
    if hasattr(x, "toarray"):
        x = x.toarray()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x, dtype=np.float32))).to(device)


def _is_sparse(adj) -> bool:
    if isinstance(adj, ops.CSRAdjacency):
        return True
    if isinstance(adj, torch.Tensor):
        return adj.layout in (torch.sparse_coo, torch.sparse_csr)
    return hasattr(adj, "tocsr")


@register_keras_serializable()
class GCN(Layer):

    def __init__(self, units: int, residual=False, use_bias=False, activation="relu",
                 kernel_initializer="truncated_normal", kernel_regularizer=None, bias_initializer="zeros",
                 bias_regularizer=None, **kwargs):
        super().__init__(**kwargs)
        name = _act_name(activation)
        if name not in _ACTS:
            raise ValueError(f"GCN: unsupported activation {activation!r}; supported: "
                             f"{sorted(k for k in _ACTS if k)} or None")
        self._units = int(units)
        self._residual = bool(residual)
        self._use_bias = use_bias
        self._activation = name
        self._act = _ACTS[name]
        # the reference's inner Dense; its activation is applied here (it may be the softmax)
        self._kernel = Dense(self._units, activation=None, use_bias=use_bias, kernel_initializer=kernel_initializer,
                             bias_initializer=bias_initializer, kernel_regularizer=kernel_regularizer,
                             bias_regularizer=bias_regularizer)

    def _check_width(self, F: int):
        if self._residual and F != self._units:
            raise ValueError(f"GCN: residual=True adds the features to the output, so units ({self._units}) must equal "
                             f"the feature width ({F})")

    def build(self, input_shape, device=None):
        self._check_width(int(input_shape[-1]))
        self._kernel.build(input_shape, device=device)
        self.built = True

    def forward(self, features, adj, **kwargs):
        dev = features.device if isinstance(features, torch.Tensor) else torch.device("cuda")
        x = _device_tensor(features, dev)
        if not self.built:
            self.build(tuple(x.shape), device=x.device)
        return self.call(x, adj)

    def _epilogue(self, z):
        """act(z @ W + b) on the GEMM, the softmax as a row pass after it."""
        w, b = self._kernel.kernel, self._kernel.bias
        if self._act == ops.ACT_SOFTMAX:
            return ops.SoftmaxRowsFn.apply(ops.DenseFn.apply(z, w, b, 0))
        return ops.DenseFn.apply(z, w, b, self._act)

    def call(self, features, adj, **kwargs):
        x = _device_tensor(features, self._kernel.kernel.device)
        F = x.shape[-1]
        self._check_width(F)
        w, b = self._kernel.kernel, self._kernel.bias
        if _is_sparse(adj):
            a = ops.CSRAdjacency.from_any(adj, x.device)
            if F > self._units:
                z = ops.DenseFn.apply(x, w, None, 0)
                if self._act == ops.ACT_SOFTMAX and self._units > ops.SPMM_SOFTMAX_MAX_F:
                    return ops.SoftmaxRowsFn.apply(ops.SpMMFn.apply(z, b, None, a, 0))
                return ops.SpMMFn.apply(z, b, None, a, self._act)      # residual needs F == units: not this order
            out = self._epilogue(ops.SpMMFn.apply(x, None, None, a, 0))
        else:
            a = _device_tensor(adj, x.device)
            if a.dim() != 2 or a.shape[1] != x.shape[0]:
                raise ValueError(f"GCN: adj must be [N, {x.shape[0]}], got {tuple(a.shape)}")
            if F > self._units:
                z = ops.DenseFn.apply(x, w, None, 0)
                if self._act == ops.ACT_SOFTMAX:
                    return ops.SoftmaxRowsFn.apply(ops.DenseFn.apply(a, z, b, 0))
                return ops.DenseFn.apply(a, z, b, self._act)
            out = self._epilogue(ops.DenseFn.apply(a, x, None, 0))
        return out + x if self._residual else out

    @property
    def kernel(self):
        return self._kernel.kernel

    @property
    def bias(self):
        return self._kernel.bias

    @property
    def losses(self):
        return self._kernel.losses

    def get_config(self):
        cfg = super().get_config()
        cfg.update({
            "units": self._units,
            "residual": self._residual,
            "use_bias": self._use_bias,
            "activation": self._activation,
            "kernel_initializer": serialize_initializer(self._kernel._kernel_initializer),
            "kernel_regularizer": self._kernel._kernel_regularizer,
            "bias_initializer": serialize_initializer(self._kernel._bias_initializer),
            "bias_regularizer": self._kernel._bias_regularizer,
        })
        return cfg
