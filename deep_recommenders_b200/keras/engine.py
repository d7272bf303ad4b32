"""Keras-style ``compile`` / ``fit`` / ``evaluate`` for the models in this package -- a THIN loop over the CUDA layers
(autograd + torch.optim), so that the reference's Keras example
(/root/reference/examples/train_deepfm_on_movielens_keras.py:38-54: ``model.compile(loss=..., optimizer=Adam(),
metrics=[AUC(), Precision(), Recall()])``, ``model.fit(input_fn, epochs=..., steps_per_epoch=..., validation_data=...,
validation_steps=..., callbacks=[EarlyStopping(patience=3)])``) has every name it uses.  The objects below stand in for
the ``tf.keras.losses / optimizers / metrics / callbacks`` members that script touches; nothing else of Keras is
restated.  The high-throughput path is ``DeepFMTrainStep`` (one CUDA-graph replay per step); this loop is the
drop-in convenience surface.
"""
from __future__ import annotations

import itertools
from typing import Callable, Iterable, List, Optional

import numpy as np
import torch


# ---- tf.keras.losses ----------------------------------------------------------------------------------------------
def binary_crossentropy(y_true: torch.Tensor, y_pred: torch.Tensor) -> torch.Tensor:
    """tf.keras.losses.binary_crossentropy on probabilities (Keras clips to [eps, 1 - eps], eps = 1e-7)."""
    p = y_pred.clamp(1e-7, 1.0 - 1e-7)
    return -(y_true * torch.log(p) + (1.0 - y_true) * torch.log(1.0 - p)).mean(dim=-1)


def mean_squared_error(y_true: torch.Tensor, y_pred: torch.Tensor) -> torch.Tensor:
    """tf.keras.losses.mean_squared_error: mean over the last axis of (y_pred - y_true)^2."""
    return ((y_pred - y_true) ** 2).mean(dim=-1)


def categorical_crossentropy(y_true: torch.Tensor, y_pred: torch.Tensor) -> torch.Tensor:
    """tf.keras.losses.categorical_crossentropy on probabilities: y_pred is renormalised over the last axis, clipped
    to [eps, 1 - eps] (eps = 1e-7), and -sum(y_true * log(y_pred)) is taken over that axis."""
    p = (y_pred / y_pred.sum(dim=-1, keepdim=True)).clamp(1e-7, 1.0 - 1e-7)
    return -(y_true * torch.log(p)).sum(dim=-1)


_LOSSES = {"binary_crossentropy": binary_crossentropy, "mse": mean_squared_error,
           "mean_squared_error": mean_squared_error, "categorical_crossentropy": categorical_crossentropy}


# ---- tf.keras.optimizers ------------------------------------------------------------------------------------------
class Adam:
    """tf.keras.optimizers.Adam defaults (learning_rate 0.001, beta 0.9 / 0.999, epsilon 1e-7)."""

    def __init__(self, learning_rate: float = 0.001, beta_1: float = 0.9, beta_2: float = 0.999, epsilon: float = 1e-7):
        self.kw = dict(lr=learning_rate, betas=(beta_1, beta_2), eps=epsilon)

    def build(self, params):
        return torch.optim.Adam(params, **self.kw)


class SGD:
    def __init__(self, learning_rate: float = 0.01, momentum: float = 0.0):
        self.kw = dict(lr=learning_rate, momentum=momentum)

    def build(self, params):
        return torch.optim.SGD(params, **self.kw)


_OPTIMIZERS = {"adam": Adam, "sgd": SGD}


# ---- tf.keras.metrics ---------------------------------------------------------------------------------------------
class _Confusion:
    """Thresholded confusion counts, accumulated on the device (no host sync per batch)."""

    def __init__(self, thresholds):
        self.thresholds = torch.as_tensor(thresholds, dtype=torch.float32)
        self.reset_state()

    def reset_state(self):
        self.tp = self.fp = self.fn = self.tn = None

    def update_state(self, y_true, y_pred):
        t = self.thresholds.to(y_pred.device)
        pred = y_pred.reshape(1, -1) > t.reshape(-1, 1)
        pos = (y_true.reshape(1, -1) > 0.5)
        add = lambda old, new: new if old is None else old + new
        self.tp = add(self.tp, (pred & pos).sum(1).double())
        self.fp = add(self.fp, (pred & ~pos).sum(1).double())
        self.fn = add(self.fn, (~pred & pos).sum(1).double())
        self.tn = add(self.tn, (~pred & ~pos).sum(1).double())


class AUC(_Confusion):
    """tf.keras.metrics.AUC defaults: ROC, 200 thresholds, trapezoidal ("interpolation") summation."""
    name = "auc"

    def __init__(self, num_thresholds: int = 200):
        eps = 1e-7
        th = [0.0 - eps] + [(i + 1) / (num_thresholds - 1) for i in range(num_thresholds - 2)] + [1.0 + eps]
        super().__init__(th)

    def result(self) -> float:
        if self.tp is None:
            return 0.0
        tpr = (self.tp / (self.tp + self.fn).clamp_min(1e-12)).cpu().numpy()
        fpr = (self.fp / (self.fp + self.tn).clamp_min(1e-12)).cpu().numpy()
        return float(np.sum((fpr[:-1] - fpr[1:]) * (tpr[:-1] + tpr[1:]) / 2.0))


class Precision(_Confusion):
    name = "precision"

    def __init__(self, thresholds: float = 0.5):
        super().__init__([thresholds])

    def result(self) -> float:
        return 0.0 if self.tp is None else float(self.tp[0] / (self.tp[0] + self.fp[0]).clamp_min(1e-12))


class Recall(_Confusion):
    name = "recall"

    def __init__(self, thresholds: float = 0.5):
        super().__init__([thresholds])

    def result(self) -> float:
        return 0.0 if self.tp is None else float(self.tp[0] / (self.tp[0] + self.fn[0]).clamp_min(1e-12))


class WeightedAccuracy:
    """The "acc" of ``compile(weighted_metrics=["acc"])``: sum(w * correct) / sum(w) over the rows seen, where
    correct is argmax agreement under categorical cross-entropy (Keras's categorical accuracy) and agreement of the
    0.5-thresholded prediction otherwise (binary accuracy).  w is the sample weight (1 when none is given)."""

    def __init__(self, name: str = "acc", categorical: bool = True):
        self.name, self.categorical = name, categorical
        self.reset_state()

    def reset_state(self):
        self.hits = self.total = None

    def update_state(self, y_true, y_pred, sample_weight=None):
        if self.categorical:
            correct = (y_pred.argmax(dim=-1) == y_true.argmax(dim=-1)).double()
        else:
            correct = ((y_pred > 0.5) == (y_true > 0.5)).double().reshape(y_pred.shape[0], -1).mean(dim=-1)
        w = correct.new_ones(correct.shape) if sample_weight is None else sample_weight.double().reshape(-1)
        add = lambda old, new: new if old is None else old + new
        self.hits = add(self.hits, (w * correct).sum())
        self.total = add(self.total, w.sum())

    def result(self) -> float:
        return 0.0 if self.total is None or float(self.total) == 0.0 else float(self.hits / self.total)


# ---- tf.keras.callbacks -------------------------------------------------------------------------------------------
class EarlyStopping:
    """tf.keras.callbacks.EarlyStopping(monitor="val_loss", patience=0, min_delta=0): stop when the monitored value
    has not improved for `patience` epochs."""

    def __init__(self, monitor: str = "val_loss", patience: int = 0, min_delta: float = 0.0):
        self.monitor, self.patience, self.min_delta = monitor, int(patience), float(min_delta)
        self.best, self.wait, self.stopped_epoch = None, 0, None

    def on_epoch_end(self, epoch: int, logs: dict) -> bool:
        cur = logs.get(self.monitor)
        if cur is None:
            return False
        if self.best is None or cur < self.best - self.min_delta:
            self.best, self.wait = cur, 0
            return False
        self.wait += 1
        if self.wait >= self.patience:
            self.stopped_epoch = epoch
            return True
        return False


class _OptimizerHandle:
    """``model.optimizer`` as callbacks see it: ``lr`` reads and writes the learning rate of the optimizer spec and,
    once the torch optimizer is built (after the first forward), of each of its parameter groups."""

    def __init__(self, model):
        self._model = model

    @property
    def lr(self) -> float:
        opt = self._model._optimizer
        return float(opt.param_groups[0]["lr"]) if opt is not None else float(self._model._optimizer_spec.kw["lr"])

    @lr.setter
    def lr(self, value: float) -> None:
        self._model._optimizer_spec.kw["lr"] = float(value)
        if self._model._optimizer is not None:
            for group in self._model._optimizer.param_groups:
                group["lr"] = float(value)

    learning_rate = lr


def _hook(cb, name: str):
    return getattr(cb, name, None)


# ---- the loop -----------------------------------------------------------------------------------------------------
def _batches(data) -> Iterable:
    """`data`: an iterable / generator of (features, labels) batches, or a zero-argument callable returning one (the
    reference passes `movielens.training_input_fn`, a tf.data pipeline)."""
    return data() if callable(data) else data


def _labels(y, device) -> torch.Tensor:
    t = y if isinstance(y, torch.Tensor) else torch.as_tensor(np.asarray(y, dtype=np.float32))
    return t.to(device=device, dtype=torch.float32).reshape(t.shape[0], -1)


def _weights(w, device) -> Optional[torch.Tensor]:
    if w is None:
        return None
    t = w if isinstance(w, torch.Tensor) else torch.as_tensor(np.asarray(w, dtype=np.float32))
    return t.to(device=device, dtype=torch.float32).reshape(-1)


def _whole_array_batch(x, y, sample_weight, batch_size):
    """Whole-array input is one full batch (GCN is full-batch): there is nothing to shuffle, and a smaller batch is
    not served."""
    rows = y.shape[0] if hasattr(y, "shape") else len(y)
    if batch_size is not None and batch_size < rows:
        raise NotImplementedError(f"batch_size={batch_size} < {rows} rows: whole-array input runs as one full batch")
    return (x, y, sample_weight)


def _unpack(batch):
    """(features, labels) or (features, labels, sample_weight)."""
    return (batch[0], batch[1], batch[2] if len(batch) > 2 else None)


class TrainingLoopMixin:
    """compile / fit / evaluate for `Model` (keras/layers/base.py)."""

    def compile(self, loss="binary_crossentropy", optimizer="adam", metrics: Optional[List] = None,
                weighted_metrics: Optional[List] = None, **kwargs):
        """weighted_metrics: "acc" / "accuracy" (categorical accuracy under categorical cross-entropy, else binary),
        weighted by the sample weight given to fit / evaluate."""
        self._loss_fn: Callable = _LOSSES[loss] if isinstance(loss, str) else loss
        self._optimizer_spec = _OPTIMIZERS[optimizer]() if isinstance(optimizer, str) else optimizer
        self._optimizer = None
        self._metrics = list(metrics or [])
        self._weighted_metrics = []
        for m in weighted_metrics or []:
            if m not in ("acc", "accuracy"):
                raise ValueError(f"unsupported weighted metric {m!r}; supported: 'acc', 'accuracy'")
            self._weighted_metrics.append(WeightedAccuracy(m, categorical=loss == "categorical_crossentropy"))
        return self

    def _all_metrics(self) -> list:
        return self._metrics + getattr(self, "_weighted_metrics", [])

    def _update_metrics(self, yt, pred, w):
        for m in self._metrics:
            m.update_state(yt, pred)
        for m in getattr(self, "_weighted_metrics", []):
            m.update_state(yt, pred, w)

    @property
    def optimizer(self) -> _OptimizerHandle:
        if not hasattr(self, "_optimizer_spec"):
            raise RuntimeError("call compile() before reading the optimizer")
        return _OptimizerHandle(self)

    def _step_loss(self, x, y, sample_weight=None):
        """Keras's SUM_OVER_BATCH_SIZE: mean over the rows of w * loss (w = 1 without a sample weight)."""
        pred = self(x)
        yt = _labels(y, pred.device)
        w = _weights(sample_weight, pred.device)
        per_row = self._loss_fn(yt, pred)
        loss = per_row.mean() if w is None else (per_row.reshape(-1) * w).sum() / per_row.numel()
        reg = [l for l in getattr(self, "losses", [])] if hasattr(self, "losses") else []
        for r in reg:
            loss = loss + r
        return pred, yt, w, loss

    def evaluate(self, x, y=None, steps: Optional[int] = None, sample_weight=None, batch_size: Optional[int] = None,
                 verbose: int = 0) -> dict:
        """`x`: an iterable (or a callable returning one) of (features, labels[, sample_weight]) batches, of which
        `steps` are read; or, with labels `y`, whole arrays evaluated as one batch with an optional `sample_weight`.
        An int second argument is `steps` (the batch form `evaluate(data, steps)`).  Returns a dict of logs."""
        if not hasattr(self, "_loss_fn"):
            raise RuntimeError("call compile() before evaluate()")
        if isinstance(y, int) and not isinstance(y, bool) and steps is None:
            y, steps = None, y
        data = [_whole_array_batch(x, y, sample_weight, batch_size)] if y is not None else _batches(x)
        metrics = self._all_metrics()
        for m in metrics:
            m.reset_state()
        tot, n = None, 0
        was = self.training
        self.eval()
        with torch.no_grad():
            for batch in itertools.islice(data, steps):
                pred, yt, w, loss = self._step_loss(*_unpack(batch))
                tot = loss.detach().double() if tot is None else tot + loss.detach().double()
                n += 1
                self._update_metrics(yt, pred, w)
        self.train(was)
        logs = {"loss": float(tot / max(n, 1)) if tot is not None else float("nan")}
        logs.update({m.name: m.result() for m in metrics})
        return logs

    def fit(self, x, y=None, epochs: int = 1, steps_per_epoch: Optional[int] = None, validation_data=None,
            validation_steps: Optional[int] = None, callbacks: Optional[List] = None, verbose: int = 0,
            sample_weight=None, batch_size: Optional[int] = None, shuffle: bool = True):
        """`x`: iterable (or callable returning one) of (features, labels) batches that is consumed ACROSS epochs, as
        the reference's repeated tf.data pipeline is; `steps_per_epoch` batches make one epoch.  With labels `y`, `x`
        and `y` are whole arrays trained as one full batch per step, weighted by `sample_weight` when it is given;
        `batch_size` below the number of rows raises NotImplementedError, and `shuffle` has no effect on a single
        full batch.  With `batch_size` given (Keras's whole-array form) and no `steps_per_epoch`, an epoch is one pass
        over the arrays: one step.  `validation_data` is then `(x, y)` or `(x, y, sample_weight)`; without `y` it is a batch iterable
        (or callable) read for `validation_steps` batches.  Returns a dict of per-epoch logs (`history`)."""
        if not hasattr(self, "_loss_fn"):
            raise RuntimeError("call compile() before fit()")
        if y is not None:
            if batch_size is not None and steps_per_epoch is None:
                steps_per_epoch = 1
            x = [_whole_array_batch(x, y, sample_weight, batch_size)] * (steps_per_epoch or 1) * epochs
            if validation_data is not None:
                vx, vy, vw = _unpack(validation_data)
                validation_data = [_whole_array_batch(vx, vy, vw, None)]
                validation_steps = 1
        stream = iter(_batches(x))
        history: dict = {}
        callbacks = list(callbacks or [])
        for cb in callbacks:                         # Keras callbacks reach the model through `self.model`
            if _hook(cb, "on_train_begin") or _hook(cb, "on_batch_end"):
                cb.model = self
        for cb in callbacks:
            if _hook(cb, "on_train_begin"):
                cb.on_train_begin({})
        for epoch in range(epochs):
            for m in self._all_metrics():
                m.reset_state()
            tot, n = None, 0
            for batch in itertools.islice(stream, steps_per_epoch):
                pred, yt, w, loss = self._step_loss(*_unpack(batch))
                if self._optimizer is None:        # parameters of lazily built layers exist after the first forward
                    self._optimizer = self._optimizer_spec.build([p for p in self.parameters() if p.requires_grad])
                self._optimizer.zero_grad(set_to_none=True)
                loss.backward()
                self._optimizer.step()
                tot = loss.detach().double() if tot is None else tot + loss.detach().double()
                for cb in callbacks:
                    if _hook(cb, "on_batch_end"):
                        cb.on_batch_end(n, {})
                n += 1
                self._update_metrics(yt, pred.detach(), w)
            if n == 0:
                break                                # input exhausted
            logs = {"loss": float(tot / n)}
            logs.update({m.name: m.result() for m in self._all_metrics()})
            if validation_data is not None:
                logs.update({"val_" + k: v for k, v in self.evaluate(validation_data, steps=validation_steps).items()})
            for k, v in logs.items():
                history.setdefault(k, []).append(v)
            if verbose:
                print(f"epoch {epoch + 1}/{epochs} " + " ".join(f"{k}={v:.4f}" for k, v in logs.items()), flush=True)
            if any(cb.on_epoch_end(epoch, logs) for cb in callbacks):
                break
        self.history = history
        return history
