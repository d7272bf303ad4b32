"""``GroupedTowers``: G independent Dense towers of one shape, run as grouped layers.

The reference builds each tower with its own chain of ``tf.layers.dense`` calls (estimator/models/feature_interaction/
dnn.py:17-29): hidden layers with the activation, the last layer linear.  Here the G towers' layer l is one call:
  * layer 0 of towers that share their input is ONE Dense on the column-concatenated kernel [K, G*N0] (tower g owns
    column block g);
  * every other layer (and layer 0 of towers with separate inputs, given as column blocks of [M, G*K]) is
    ``ops.GroupedDenseFn`` on [G, K, N] weights.
Each tower's kernel is initialised as its own Dense would be: glorot-uniform over (fan_in, fan_out) = (K, N) of that
tower, bias zeros.  The towers do not share weights (the estimator ``dnn()`` helper caches towers by shape, which is
why the multi-task models do not use it).
"""
from __future__ import annotations

import math

import torch
from torch import nn

from .... import ops


def _glorot_blocks(G: int, K: int, N: int, gen) -> torch.Tensor:
    limit = math.sqrt(6.0 / (K + N))
    return torch.empty((G, K, N), dtype=torch.float32).uniform_(-limit, limit, generator=gen)


class GroupedTowers(nn.Module):
    """G towers of ``hidden_units`` on inputs of width ``in_dim``: forward maps [M, in_dim] (``shared_input``) or
    [M, G*in_dim] to [M, G*hidden_units[-1]] (tower g's output is column block g)."""

    def __init__(self, num_towers: int, in_dim: int, hidden_units, activation="relu", shared_input: bool = True,
                 seed=None, device=None):
        super().__init__()
        units = [int(u) for u in hidden_units]
        if num_towers < 1 or in_dim < 1 or not units or min(units) < 1:
            raise ValueError(f"GroupedTowers: bad shape num_towers={num_towers} in_dim={in_dim} units={units}")
        self.num_towers, self.in_dim, self.units = int(num_towers), int(in_dim), units
        self.shared_input = bool(shared_input)
        act = ops.act_code(activation)
        self._acts = [act] * (len(units) - 1) + [0]
        gen = torch.Generator().manual_seed(seed) if seed is not None else None
        dev = torch.device(device) if device is not None else torch.device("cuda")
        G = self.num_towers
        self.kernels = nn.ParameterList()
        self.biases = nn.ParameterList()
        k = self.in_dim
        for layer, n in enumerate(units):
            w = _glorot_blocks(G, k, n, gen)
            if layer == 0 and self.shared_input:
                w = w.permute(1, 0, 2).reshape(k, G * n)          # [K, G*N0]: tower g = column block g
            self.kernels.append(nn.Parameter(w.contiguous().to(dev)))
            self.biases.append(nn.Parameter(torch.zeros((G * n,) if layer == 0 and self.shared_input else (G, n),
                                                        dtype=torch.float32, device=dev)))
            k = n

    @property
    def out_dim(self) -> int:
        return self.units[-1]

    def forward(self, x):
        for layer, (w, b) in enumerate(zip(self.kernels, self.biases)):
            if layer == 0 and self.shared_input:
                x = ops.DenseFn.apply(x, w, b, self._acts[0])
            else:
                x = ops.GroupedDenseFn.apply(x, w, b, self._acts[layer])
        return x

    def dense_views(self):
        """[(kernel [K, N], bias [N])] of every tower's Dense layers in the reference's creation order (tower by tower,
        bottom layer first), as views of the parameters: writing into them sets the weights."""
        out = []
        for g in range(self.num_towers):
            for layer, (w, b) in enumerate(zip(self.kernels, self.biases)):
                n = self.units[layer]
                if layer == 0 and self.shared_input:
                    out.append((w.data[:, g * n:(g + 1) * n], b.data[g * n:(g + 1) * n]))
                else:
                    out.append((w.data[g], b.data[g]))
        return out
