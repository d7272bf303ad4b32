"""Feature-column *specs* in the argument positions the reference passes tf.feature_column
objects (examples/train_deepfm_on_movielens_keras.py:10-35).  TensorFlow is not available
here, so a column is a small immutable description; the lookup arithmetic lives in the CUDA
gather kernel (deep_recommenders_b200/csrc/embed_fm.cu).

Id pipeline semantics restated from TensorFlow's documented behaviour (SURVEY.md 8a row E):
  * hash_bucket:     id = FarmHash Fingerprint64(str(value)) mod hash_bucket_size
                     (deep_recommenders_b200/hashing.py).  Integer inputs that are already
                     ids in [0, N) can bypass hashing with `categorical_column_with_identity`.
  * vocabulary_list: id = index in the list, out-of-vocabulary -> -1 -> zero embedding and
                     all-zero indicator row (default num_oov_buckets=0, default_value=-1).
  * identity:        id = value, out of range -> treated as OOV (-1).
  * embedding_column: dimension D, combiner "mean", initializer truncated-normal(0, 1/sqrt(D)).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional, Sequence, Tuple


@dataclass
class RaggedFeature:
    """A multi-valued feature for one batch (what tf.io.VarLenFeature / a SparseTensor carries, e.g. "Genres",
    datasets/movielens.py): flat raw `values` (list / numpy / torch) and `row_splits` [B+1]; example b owns
    values[row_splits[b]:row_splits[b+1]].  Embedding columns mean-combine it, indicator columns count it."""
    values: object
    row_splits: object

    @property
    def batch_size(self) -> int:
        return len(self.row_splits) - 1


@dataclass
class PackedStrings:
    """n byte strings as ONE uint8 buffer + int64 offsets [n+1] (numpy, host): what the native TFRecord parser emits
    for a string feature and what the C-ABI hash / vocabulary entries consume -- no per-value Python objects."""
    data: object
    offsets: object

    def __len__(self) -> int:
        return len(self.offsets) - 1

    def tolist(self):
        d, o = bytes(memoryview(self.data)), self.offsets
        return [d[int(o[i]):int(o[i + 1])] for i in range(len(self))]


@dataclass(frozen=True)
class CategoricalColumn:
    key: str
    kind: str                      # "hash" | "vocab" | "identity"
    num_buckets: int
    vocabulary_list: Tuple = field(default=())
    dtype: str = "string"

    @property
    def name(self) -> str:
        return self.key


def categorical_column_with_hash_bucket(key: str, hash_bucket_size: int, dtype: str = "string") -> CategoricalColumn:
    if hash_bucket_size is None or hash_bucket_size < 1:
        raise ValueError(f"hash_bucket_size must be at least 1. hash_bucket_size: {hash_bucket_size}, key: {key}")
    return CategoricalColumn(key, "hash", int(hash_bucket_size), (), dtype)


def categorical_column_with_vocabulary_list(key: str, vocabulary_list: Sequence, dtype=None) -> CategoricalColumn:
    if vocabulary_list is None or len(vocabulary_list) < 1:
        raise ValueError(f"vocabulary_list {vocabulary_list} must be non-empty, column_name: {key}")
    if len(set(vocabulary_list)) != len(vocabulary_list):
        raise ValueError(f"Duplicate keys in vocabulary_list: {vocabulary_list}, column_name: {key}")
    return CategoricalColumn(key, "vocab", len(vocabulary_list), tuple(vocabulary_list),
                             dtype or ("string" if isinstance(vocabulary_list[0], str) else "int64"))


def categorical_column_with_identity(key: str, num_buckets: int) -> CategoricalColumn:
    if num_buckets < 1:
        raise ValueError(f"num_buckets {num_buckets} < 1, column_name {key}")
    return CategoricalColumn(key, "identity", int(num_buckets), (), "int64")


@dataclass(frozen=True)
class IndicatorColumn:
    categorical_column: CategoricalColumn

    @property
    def name(self) -> str:
        return f"{self.categorical_column.key}_indicator"


@dataclass(frozen=True)
class EmbeddingColumn:
    categorical_column: CategoricalColumn
    dimension: int
    combiner: str = "mean"
    initializer_stddev: Optional[float] = None   # None -> 1/sqrt(dimension) (TF default)

    @property
    def name(self) -> str:
        return f"{self.categorical_column.key}_embedding"


def indicator_column(categorical_column: CategoricalColumn) -> IndicatorColumn:
    return IndicatorColumn(categorical_column)


@dataclass(frozen=True)
class NumericColumn:
    """tf.feature_column.numeric_column: the feature's values, reshaped to [batch, prod(shape)] and cast to float32."""
    key: str
    shape: Tuple = (1,)
    dtype: str = "float32"

    @property
    def name(self) -> str:
        return self.key

    @property
    def width(self) -> int:
        w = 1
        for s in self.shape:
            w *= int(s)
        return w


def numeric_column(key: str, shape=(1,), dtype: str = "float32") -> NumericColumn:
    shape = (int(shape),) if isinstance(shape, int) else tuple(int(s) for s in shape)
    if not shape or any(s < 1 for s in shape):
        raise ValueError(f"shape dimensions must be greater than 0. shape: {shape}, key: {key}")
    if dtype not in ("float32", "float64", "float16", "int32", "int64"):
        raise ValueError(f"dtype must be convertible to float. dtype: {dtype}, key: {key}")
    return NumericColumn(key, shape, dtype)


def input_layer(features, feature_columns, device=None):
    """tf.feature_column.input_layer for numeric columns: the columns concatenated in order of their names (as
    TensorFlow sorts them, so C10 comes before C2) into one float32 [batch, sum of widths] CUDA tensor.  Host
    features are concatenated on the host and copied to the device once per batch."""
    import numpy as np
    import torch

    cols = list(feature_columns) if isinstance(feature_columns, (list, tuple)) else [feature_columns]
    if not cols:
        raise ValueError("feature_columns must not be empty")
    for c in cols:
        if not isinstance(c, NumericColumn):
            raise NotImplementedError(f"input_layer serves numeric columns only; got {type(c).__name__} "
                                      f"{getattr(c, 'name', c)!r} (categorical columns go through the embedding "
                                      "models' own lookup)")
    cols = sorted(cols, key=lambda c: c.name)
    parts = []
    for c in cols:
        if c.key not in features:
            raise KeyError(f"feature {c.key!r} of numeric_column {c.name!r} is missing from the features")
        v = features[c.key]
        n = v.shape[0]
        if int(np.prod(v.shape[1:], dtype=np.int64)) != c.width:
            raise ValueError(f"feature {c.key!r} has shape {tuple(v.shape)}, numeric_column expects "
                             f"[batch, {', '.join(map(str, c.shape))}]")
        parts.append(v.reshape(n, c.width))
    dev = torch.device(device) if device is not None else torch.device("cuda")
    if all(isinstance(p, torch.Tensor) and p.is_cuda for p in parts):
        return torch.cat([p.to(torch.float32) for p in parts], dim=1)
    host = np.concatenate([p.detach().cpu().numpy() if isinstance(p, torch.Tensor) else np.asarray(p)
                           for p in parts], axis=1).astype(np.float32, copy=False)
    return torch.from_numpy(np.ascontiguousarray(host)).to(dev)


def embedding_column(categorical_column: CategoricalColumn, dimension: int, combiner: str = "mean",
                     initializer_stddev: Optional[float] = None) -> EmbeddingColumn:
    if dimension is None or dimension < 1:
        raise ValueError(f"Invalid dimension {dimension}.")
    if combiner not in ("mean", "sqrtn", "sum"):
        raise ValueError(f"Invalid combiner {combiner}.")
    return EmbeddingColumn(categorical_column, int(dimension), combiner, initializer_stddev)


DEFAULT_CROSS_HASH_KEY = 0xDECAFCAFFE    # TensorFlow's sparse_cross_hashed default hash_key


@dataclass(frozen=True)
class CrossedColumn:
    """tf.feature_column.crossed_column over raw features: id = FingerprintCat64 chain over the keys' values, mod
    hash_bucket_size (csrc/cross.cuh).  Strings enter through Fingerprint64 of their bytes, int64 values raw; a
    single-valued key drops empty strings and -1 (a RaggedFeature keeps every value, as TensorFlow keeps a
    SparseTensor's); multi-valued keys cross every combination."""
    keys: Tuple[str, ...]
    hash_bucket_size: int
    hash_key: int = DEFAULT_CROSS_HASH_KEY

    @property
    def key(self) -> str:
        return self.name

    @property
    def name(self) -> str:
        return "_X_".join(sorted(self.keys))

    @property
    def num_buckets(self) -> int:
        return self.hash_bucket_size


def crossed_column(keys, hash_bucket_size: int, hash_key: Optional[int] = None) -> CrossedColumn:
    if len(keys) < 2:
        raise ValueError(f"keys must be a list with length > 1. Given: {keys}")
    if hash_bucket_size is None or hash_bucket_size < 1:
        raise ValueError(f"hash_bucket_size must be > 1. hash_bucket_size: {hash_bucket_size}")
    for k in keys:
        if not isinstance(k, str):
            raise NotImplementedError(f"crossed_column serves raw feature names as keys; got {type(k).__name__} "
                                      f"{getattr(k, 'name', k)!r}")
    return CrossedColumn(tuple(keys), int(hash_bucket_size),
                         DEFAULT_CROSS_HASH_KEY if hash_key is None else int(hash_key))


def linear_model(features, feature_columns, table):
    """tf.feature_column.linear_model over indicator columns of categorical or crossed columns: [B, 1] =
    bias + sum over the columns of the weights of the example's ids (multi-valued features count every value).
    It owns nothing: `table` (embedding.LinearTable with one slot per column, in this order) holds the weights."""
    from .hashing import wide_ids
    cols = list(feature_columns) if isinstance(feature_columns, (list, tuple)) else [feature_columns]
    for c in cols:
        if not isinstance(c, IndicatorColumn):
            raise NotImplementedError(f"linear_model serves indicator columns only; got {type(c).__name__} "
                                      f"{getattr(c, 'name', c)!r}")
    if len(cols) != table.num_slots or any(int(c.categorical_column.num_buckets) != r
                                           for c, r in zip(cols, table.rows_list)):
        raise ValueError("the table's columns do not match feature_columns")
    ids, bags = wide_ids([c.categorical_column for c in cols], features, table.state.device)
    return table(ids, bags).unsqueeze(1)
