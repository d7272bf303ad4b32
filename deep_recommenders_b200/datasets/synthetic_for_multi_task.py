"""``SyntheticForMultiTask`` (reference datasets/synthetic_for_multi_task.py): the two-task regression data of the
MMoE paper (Ma et al., KDD 2018, section 4.1), two targets whose correlation is set by p.

``synthetic_data`` is plain numpy and draws from the global ``np.random`` state in the reference's order (mu1, mu2,
alpha, beta, examples, then the two label noises), so under the same seed it returns the reference's arrays bit for
bit.  ``input_fn`` keeps the reference's behaviour that every call draws a new dataset (new mu, alpha, beta); it
repeats the examples ``epochs`` times, then cuts batches, keeping the remainder batch, and yields
``(features {"C{i}": [b, 1]}, labels {"labels{i}": [b]})`` as host float32 arrays.
"""
from __future__ import annotations

import numpy as np


def synthetic_data(num_examples, example_dim=100, c=0.3, p=0.8, m=5):
    # two unit-scale orthogonal directions
    u1 = np.random.normal(size=example_dim)
    u1 = (u1 - np.mean(u1)) / (np.std(u1) * np.sqrt(example_dim))
    u2 = np.random.normal(size=example_dim)
    u2 -= u2.dot(u1) * u1
    u2 /= np.linalg.norm(u2)
    # task weights with cosine p between them
    w1 = c * u1
    w2 = c * (p * u1 + np.sqrt(1. - p ** 2) * u2)
    alpha = np.random.normal(size=m)
    beta = np.random.normal(size=m)
    x = np.random.normal(size=(num_examples, example_dim))
    z1 = np.matmul(x, w1)
    z2 = np.matmul(x, w2)
    s1, s2 = 0., 0.
    for i in range(m):
        s1 += np.sin(alpha[i] * z1 + beta[i])
        s2 += np.sin(alpha[i] * z2 + beta[i])
    y1 = z1 + s1 + np.random.normal(size=num_examples, scale=0.01)
    y2 = z2 + s2 + np.random.normal(size=num_examples, scale=0.01)
    return x.astype(np.float32), (y1.astype(np.float32), y2.astype(np.float32))


class _Batches(object):
    """The batches of one ``input_fn`` call, with the ``take`` / ``skip`` of tf.data the reference example uses."""

    def __init__(self, examples, labels, epochs, batch_size, start=0, stop=None):
        self._x, self._y = examples, labels
        self._epochs, self._bs = int(epochs), int(batch_size)
        total = self._x.shape[0] * self._epochs
        n = (total + self._bs - 1) // self._bs
        self._start = min(start, n)
        self._stop = n if stop is None else min(stop, n)

    def __len__(self):
        return max(self._stop - self._start, 0)

    def take(self, count):
        return _Batches(self._x, self._y, self._epochs, self._bs, self._start,
                        self._stop if count < 0 else min(self._stop, self._start + int(count)))

    def skip(self, count):
        return _Batches(self._x, self._y, self._epochs, self._bs, self._start + int(count), self._stop)

    def _rows(self, a, lo, hi):
        n = a.shape[0]
        if lo // n == (hi - 1) // n:
            return a[lo % n:(hi - 1) % n + 1]
        return a[np.arange(lo, hi) % n]                           # a batch across an epoch boundary

    def __iter__(self):
        total = self._x.shape[0] * self._epochs
        for i in range(self._start, self._stop):
            lo, hi = i * self._bs, min((i + 1) * self._bs, total)
            x = self._rows(self._x, lo, hi)
            features = {"C{}".format(j): x[:, j:j + 1] for j in range(x.shape[1])}
            labels = {"labels{}".format(j): self._rows(y, lo, hi) for j, y in enumerate(self._y)}
            yield features, labels


class SyntheticForMultiTask(object):

    def __init__(self, num_examples, example_dim=100, c=0.3, p=0.8, m=5):
        self._num_examples = num_examples
        self._example_dim = example_dim
        self._c = c
        self._p = p
        self._m = m

    def input_fn(self, epochs=1, batch_size=512, buffer_size=512):
        """``buffer_size`` is the reference's prefetch depth; batches here are cut lazily and need none."""
        x, y = synthetic_data(self._num_examples, self._example_dim, c=self._c, p=self._p, m=self._m)
        return _Batches(x, y, epochs, batch_size)
