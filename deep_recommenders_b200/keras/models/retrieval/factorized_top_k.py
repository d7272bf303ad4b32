"""Top-k retrieval indexes and the FactorizedTopK metric at the reference's import path
``deep_recommenders.keras.models.retrieval.factorized_top_k`` (SURVEY.md section 8(f) #3).

Mirrors reference keras/models/retrieval/factorized_top_k.py:
  :26-41    _take_long_axis(arr, indices)
  :44-67    _exclude(scores, identifiers, exclude, k)
  :70-137   TopK (abstract: index / call / query_with_exclusions)
  :139-262  Streaming(k, query_model, handle_incomplete_batches, num_parallel_calls, sorted_order)
  :265-334  BruteForce(k, query_model)
  :464-522  FactorizedTopK(candidates, metrics, k, name)
The arithmetic runs in the CUDA library: scores = Q @ C^T through dr_scores_fwd (wgmma 3xTF32 / FFMA GEMM),
selection through dr_topk_rows (tf.math.top_k order: descending, ties -> lower index), the index shuffles through
dr_take_long_axis / dr_exclude_adjust, the metric through dr_rowwise_dot / dr_column_rank.

`Faiss` (:337-461) wraps a third-party ANN library and is outside the path (SURVEY.md 8f): asking for it raises.
A `tf.data.Dataset` of candidate batches becomes any iterable of CUDA tensors (list, generator factory, DataLoader);
`BruteForce` over more candidates than fit one score matrix scans them in blocks with the same merge `Streaming`
uses, which gives the identical result (the merge keeps earlier = lower-index candidates first on ties).
"""
from __future__ import annotations

import abc
from typing import Iterable, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .... import ops
from ...layers.base import Layer, Model

_SCORE_BLOCK_BYTES = 1 << 30        # BruteForce: at most 1 GiB of materialised scores per block


def _take_long_axis(arr: torch.Tensor, indices: torch.Tensor) -> torch.Tensor:
    """arr [n, m], indices [n, k] -> arr[i, indices[i, j]]."""
    return ops.take_long_axis(arr, indices)


def _top_k(scores: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """tf.math.top_k; k > columns raises the TF message `_wrap_batch_too_small_error` looks for."""
    return ops.topk_rows(scores, int(k))


def _exclude(scores: torch.Tensor, identifiers: torch.Tensor, exclude: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """Drop the candidates whose identifier is in `exclude` (per row) from a top-k result."""
    adjusted = ops.exclude_adjust(scores, identifiers, exclude, 1.0e5)
    k = min(int(k), scores.shape[1])
    _, indices = _top_k(adjusted, k)
    return _take_long_axis(scores, indices), _take_long_axis(identifiers, indices)


def _batches(source) -> Iterable:
    """A re-iterable source of batches: a list / tuple, a zero-argument factory returning an iterator, or any
    object with __iter__ that can be iterated more than once (DataLoader, Dataset-like)."""
    return source() if callable(source) else source


def _as_cuda_f32(x) -> torch.Tensor:
    t = x if isinstance(x, torch.Tensor) else torch.as_tensor(np.asarray(x))
    if not t.is_cuda:
        t = t.cuda(non_blocking=True)
    return t.to(torch.float32).contiguous()


class TopK(Model, abc.ABC):
    """Interface of the retrieval indexes: `index` builds, `call` queries."""

    def __init__(self, k: int, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self._k = k
        self.built = True

    @abc.abstractmethod
    def index(self, candidates, identifiers=None) -> "TopK":
        raise NotImplementedError("Implementers must provide `index` method.")

    @abc.abstractmethod
    def call(self, queries, k: Optional[int] = None, **kwargs) -> Tuple[torch.Tensor, torch.Tensor]:
        raise NotImplementedError()

    def query_with_exclusions(self, queries, exclusions: torch.Tensor, k: Optional[int] = None):
        """Top-k with the per-query `exclusions` [nq, e] identifiers removed (factorized_top_k.py:113-131)."""
        k = k if k is not None else self._k
        adjusted_k = k + exclusions.shape[1]
        scores, identifiers = self(queries=queries, k=adjusted_k)
        return _exclude(scores, identifiers, exclusions, adjusted_k)

    def _reset_tf_function_cache(self):      # no tracing compiler here; kept for interface parity
        pass


def _merge(state, x, k, handle_incomplete, host_ids=False):
    """Reduction step of Streaming.call (:213-230): top-k over [state | x]."""
    (ss, si), (xs, xi) = state, x
    js = xs if ss is None else torch.cat([ss, xs], dim=1)
    ji = xi if si is None else torch.cat([si, xi], dim=1)
    k_ = min(k, js.shape[1]) if handle_incomplete else k
    scores, idx = _top_k(js, k_)
    return scores, _take_long_axis(ji, idx)


class Streaming(TopK):
    """Retrieves top k scoring items and identifiers from a large stream of candidate batches."""

    def __init__(self, k: int = 10, query_model=None, handle_incomplete_batches: bool = True,
                 num_parallel_calls: Optional[int] = None, sorted_order: bool = True, *args, **kwargs):
        super().__init__(k, *args, **kwargs)
        self._query_model = query_model
        self._handle_incomplete_batches = handle_incomplete_batches
        self._num_parallel_calls = num_parallel_calls       # tf.data knob; batches are consumed in order here
        self._sorted_order = sorted_order                   # results are always sorted (allowed by sorted=False)
        self._candidates = None
        self._identifiers = None
        self._counter = 0

    def index(self, candidates, identifiers=None, **kwargs) -> "Streaming":
        self._candidates = candidates
        self._identifiers = identifiers
        return self

    def call(self, queries, k: Optional[int] = None, **kwargs):
        k = k if k is not None else self._k
        if self._candidates is None:
            raise ValueError("The `index` method must be called first to create the retrieval index.")
        if self._query_model is not None:
            queries = self._query_model(queries)
        queries = _as_cuda_f32(queries)
        self._counter = 0
        state = (None, None)
        ident_iter = iter(_batches(self._identifiers)) if self._identifiers is not None else None
        try:
            for batch in _batches(self._candidates):
                cand = _as_cuda_f32(batch)
                n = cand.shape[0]
                if ident_iter is not None:
                    ident = next(ident_iter)
                    ident = ident if isinstance(ident, torch.Tensor) else torch.as_tensor(np.asarray(ident))
                    ident = ident.to(queries.device).reshape(-1)
                else:       # enumerate_rows (:240-245): a running counter numbers the candidates
                    ident = torch.arange(self._counter, self._counter + n, device=queries.device, dtype=torch.int32)
                self._counter += n
                scores = ops.scores(queries, cand)                                   # :199
                k_ = min(k, n) if self._handle_incomplete_batches else k
                s, idx = _top_k(scores, k_)                                         # :206
                state = _merge(state, (s, _take_long_axis(ident, idx)), k, self._handle_incomplete_batches)
        except ValueError as e:
            if "at least k columns" in str(e):     # _wrap_batch_too_small_error (:13-23)
                raise ValueError("Tried to retrieve k={k} top items, but candidate batch too small."
                                 "To resolve this, 1. increase batch-size, 2. set `drop_remainder`=True, "
                                 "3. set `handle_incomplete_batches`=True in constructor.".format(k=k))
            raise
        if state[0] is None:
            dev = queries.device
            return (torch.zeros((queries.shape[0], 0), device=dev), torch.zeros((queries.shape[0], 0), device=dev, dtype=torch.int32))
        return state


class BruteForce(TopK):
    """Exhaustive scoring of every indexed candidate."""

    def __init__(self, k: int = 10, query_model=None, *args, **kwargs):
        super().__init__(k, *args, **kwargs)
        self._query_model = query_model
        self._candidates = None
        self._identifiers = None

    def index(self, candidates, identifiers=None) -> "BruteForce":
        if not isinstance(candidates, (torch.Tensor, np.ndarray)):
            candidates = torch.cat([_as_cuda_f32(b) for b in _batches(candidates)], dim=0)
        candidates = _as_cuda_f32(candidates)
        if candidates.dim() != 2:
            raise ValueError("`candidates` ndim should be 2. Got `ndim` = {}".format(candidates.dim()))
        if identifiers is None:
            identifiers = torch.arange(candidates.shape[0], device=candidates.device, dtype=torch.int32)
        elif not isinstance(identifiers, (torch.Tensor, np.ndarray)):
            identifiers = torch.cat([b if isinstance(b, torch.Tensor) else torch.as_tensor(np.asarray(b))
                                     for b in _batches(identifiers)], dim=0)
        identifiers = identifiers if isinstance(identifiers, torch.Tensor) else torch.as_tensor(identifiers)
        self.register_buffer("candidates", candidates, persistent=True)
        self.register_buffer("identifiers", identifiers.to(candidates.device).reshape(-1), persistent=True)
        self._candidates, self._identifiers = self.candidates, self.identifiers
        self._reset_tf_function_cache()
        return self

    def call(self, queries, k: Optional[int] = None, **kwargs):
        k = k if k is not None else self._k
        if self._candidates is None:
            raise ValueError("The `index` method must be called first to create the retrieval index.")
        if self._query_model is not None:
            queries = self._query_model(queries)
        queries = _as_cuda_f32(queries)
        nq, nc = queries.shape[0], self._candidates.shape[0]
        if k > nc:
            raise ValueError(f"input must have at least k columns. Had {nc}, needed {k}")
        block = max(k, _SCORE_BLOCK_BYTES // (4 * max(nq, 1)))
        if nc <= block:
            scores = ops.scores(queries, self._candidates)               # :330
            scores, indices = _top_k(scores, k)                          # :332
            return scores, _take_long_axis(self._identifiers, indices)   # :334
        state = (None, None)
        for lo in range(0, nc, block):       # same result, bounded memory: block top-k then the streaming merge
            hi = min(nc, lo + block)
            s, idx = _top_k(ops.scores(queries, self._candidates[lo:hi]), min(k, hi - lo))
            state = _merge(state, (s, _take_long_axis(self._identifiers[lo:hi], idx)), k, True)
        return state


class Faiss(TopK):
    """The reference wraps the third-party faiss ANN library here (:337-461); outside this build's path."""

    def __init__(self, *args, **kwargs):
        raise NotImplementedError("Faiss index: third-party ANN library, outside the CUDA hot path (SURVEY.md 8f); "
                                  "use BruteForce or Streaming")

    def index(self, candidates, identifiers=None):   # pragma: no cover
        raise NotImplementedError

    def call(self, queries, k=None, **kwargs):       # pragma: no cover
        raise NotImplementedError


class TopKCategoricalAccuracy:
    """tf.keras.metrics.TopKCategoricalAccuracy(k) restricted to what FactorizedTopK feeds it: the true class is
    column 0 of y_pred (y_true = [1, 0, 0, ...]).  update_state(rank=...) takes the per-row count of predictions
    strictly above the true one (dr_column_rank): in_top_k == rank < k."""

    def __init__(self, k: int = 5, name: Optional[str] = None):
        self.k, self.name = int(k), name or f"top_{k}_categorical_accuracy"
        self.reset_states()

    def reset_states(self) -> None:
        self._hits, self._count = 0.0, 0

    def update_state(self, y_true=None, y_pred=None, rank: Optional[torch.Tensor] = None) -> None:
        if rank is None:
            if y_true is None or y_pred is None:
                raise ValueError("update_state needs (y_true, y_pred) or rank")
            tgt = y_true.argmax(dim=1)
            if not bool((tgt == 0).all()):
                raise NotImplementedError("only y_true = one-hot at column 0 (what FactorizedTopK builds) is supported")
            rank = ops.column_rank(y_pred[:, 0].contiguous(), y_pred[:, 1:].contiguous())
        self._hits += float((rank < self.k).sum().item())
        self._count += int(rank.numel())

    def result(self) -> float:
        return self._hits / self._count if self._count else 0.0


class FactorizedTopK(Layer):
    """Metric for a retrieval model: top-k categorical accuracy of the true candidate among the retrieved ones."""

    def __init__(self, candidates, metrics: Optional[Sequence[TopKCategoricalAccuracy]] = None, k: int = 100,
                 name: str = "factorized_top_k", **kwargs):
        super().__init__(name=name, **kwargs)
        if metrics is None:
            metrics = [TopKCategoricalAccuracy(k=n, name=f"{self.name}/top_{n}_categorical_accuracy")
                       for n in [1, 5, 10, 50, 100]]
        if not isinstance(candidates, TopK):
            candidates = Streaming(k=k).index(candidates)
        self._candidates = candidates
        self._metrics = list(metrics)
        self._k = k
        self.built = True

    @property
    def metrics(self) -> List[TopKCategoricalAccuracy]:
        return self._metrics

    @torch.no_grad()
    def update_state(self, query_embeddings: torch.Tensor, true_candidate_embeddings: torch.Tensor) -> None:
        q = _as_cuda_f32(query_embeddings)
        positive_scores = ops.rowwise_dot(q, _as_cuda_f32(true_candidate_embeddings))       # :487-488
        top_k_predictions, _ = self._candidates(q, k=self._k)                               # :490
        # y_true = [1, 0...], y_pred = [positive | top-k] (:492-499): the metric only needs the rank of column 0
        rank = ops.column_rank(positive_scores, top_k_predictions)
        for metric in self._metrics:
            metric.update_state(rank=rank)

    def reset_states(self) -> None:
        for metric in self.metrics:
            metric.reset_states()

    def result(self) -> List[float]:
        return [metric.result() for metric in self.metrics]

    def call(self, query_embeddings, true_candidate_embeddings):
        self.update_state(query_embeddings, true_candidate_embeddings)
        return self.result()
