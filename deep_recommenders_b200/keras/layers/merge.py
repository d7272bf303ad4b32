"""``tf.keras.layers.Subtract`` and ``Multiply``: the interacters the reference's DIN test hands to ``ActivationUnit``
(tests/keras/test_din.py:37).  ``ActivationUnit`` recognises them and runs the fused attention kernel; called on their
own (or inside the unit's composition path) they are the element-wise difference / product of their two inputs."""
from __future__ import annotations

from .base import Layer, register_keras_serializable


def _pair(inputs):
    if not isinstance(inputs, (list, tuple)) or len(inputs) != 2:
        raise ValueError("A merge layer should be called on a list of exactly 2 inputs.")
    return inputs


@register_keras_serializable()
class Subtract(Layer):
    """inputs[0] - inputs[1]"""

    def forward(self, inputs, **kwargs):
        return self.call(inputs)

    def call(self, inputs, **kwargs):
        x, y = _pair(inputs)
        return x - y


@register_keras_serializable()
class Multiply(Layer):
    """inputs[0] * inputs[1]"""

    def forward(self, inputs, **kwargs):
        return self.call(inputs)

    def call(self, inputs, **kwargs):
        x, y = _pair(inputs)
        return x * y
