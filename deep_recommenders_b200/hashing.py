"""Host side of the id pipeline (SURVEY.md section 8(f) #2): raw feature value -> int64 id.

`categorical_column_with_hash_bucket` in TensorFlow is ``string_to_hash_bucket_fast(str(value), N)`` =
FarmHash ``Fingerprint64`` of the UTF-8 bytes, modulo N; `categorical_column_with_vocabulary_list` is the
position in the list with out-of-vocabulary -> -1.  The arithmetic lives in the C-ABI library
(deep_recommenders_b200/csrc/farmhash.cuh, idpipe.cu):

  * features that are already CUDA integer tensors are hashed / looked up on the device
    (`dr_hash_bucket_i64`, `dr_vocab_lookup_i64`) and never leave it;
  * features that arrive as host strings (TFRecord parse, python lists) go through the host twins
    (`dr_hash_bucket_bytes_host`: same source compiled for the CPU, as TensorFlow's own hash op is a CPU op),
    packed as one byte buffer + offsets, then one H2D copy of the ids.

There is no pure-Python path here; the independent Python restatement used to pin the hash lives in
oracle/farmhash_py.py (test infrastructure).
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Sequence

import numpy as np
import torch

from . import _lib
from .feature_column import CategoricalColumn, PackedStrings, RaggedFeature


def _to_bytes(v) -> bytes:
    if isinstance(v, bytes):
        return v
    if isinstance(v, str):
        return v.encode("utf-8")
    if isinstance(v, (np.bytes_,)):
        return bytes(v)
    if isinstance(v, (int, np.integer)):
        return str(int(v)).encode()      # TF: as_string(int) before hashing
    return str(v).encode("utf-8")


def fingerprint64(s: bytes) -> int:
    """farmhash::Fingerprint64 of a byte string (native host twin)."""
    lib = _lib.load()
    buf = (C.c_uint8 * max(1, len(s))).from_buffer_copy(s if s else b"\0")
    return int(lib.dr_fingerprint64_host(C.cast(buf, C.c_void_p), len(s)))


def pack_strings(values: Iterable):
    """python values -> (uint8 buffer, int64 offsets [n+1]) in the layout the C-ABI hash entries take."""
    if isinstance(values, PackedStrings):
        data = np.ascontiguousarray(values.data, dtype=np.uint8)
        return (data if data.size else np.zeros(1, dtype=np.uint8)), np.ascontiguousarray(values.offsets, dtype=np.int64)
    parts = [_to_bytes(v) for v in values]
    offsets = np.zeros(len(parts) + 1, dtype=np.int64)
    if parts:
        np.cumsum([len(p) for p in parts], out=offsets[1:])
    data = np.frombuffer(b"".join(parts), dtype=np.uint8) if offsets[-1] else np.zeros(1, dtype=np.uint8)
    return data, offsets


def hash_bucket(values: Iterable, num_buckets: int) -> np.ndarray:
    """tf.strings.to_hash_bucket_fast(values, num_buckets) for host values -> int64 ids (numpy)."""
    lib = _lib.load()
    if isinstance(values, np.ndarray) and values.dtype.kind in "iu":
        v = np.ascontiguousarray(values, dtype=np.int64).reshape(-1)
        out = np.empty_like(v)
        _lib.check(lib.dr_hash_bucket_i64_host(v.ctypes.data, v.size, int(num_buckets), out.ctypes.data),
                   "dr_hash_bucket_i64_host")
        return out
    data, offsets = pack_strings(values)
    n = offsets.size - 1
    out = np.empty(n, dtype=np.int64)
    _lib.check(lib.dr_hash_bucket_bytes_host(data.ctypes.data, offsets.ctypes.data, n, int(num_buckets),
                                             out.ctypes.data), "dr_hash_bucket_bytes_host")
    return out


def vocabulary_ids(col: CategoricalColumn, values: Sequence) -> np.ndarray:
    """categorical_column_with_vocabulary_list on host values: index in the list, OOV -> -1."""
    if col.dtype == "string":
        lib = _lib.load()
        data, offsets = pack_strings(values)
        vdata, voffsets = pack_strings(col.vocabulary_list)
        out = np.empty(offsets.size - 1, dtype=np.int64)
        _lib.check(lib.dr_vocab_lookup_bytes_host(data.ctypes.data, offsets.ctypes.data, out.size, vdata.ctypes.data,
                                                  voffsets.ctypes.data, voffsets.size - 1, -1, out.ctypes.data),
                   "dr_vocab_lookup_bytes_host")
        return out
    table = {int(k): i for i, k in enumerate(col.vocabulary_list)}
    return np.asarray([table.get(int(v), -1) for v in values], dtype=np.int64)


def _vocab_device_tables(col: CategoricalColumn, device):
    cache = _vocab_device_tables.cache
    key = (col, str(device))
    if key not in cache:
        keys = np.asarray([int(k) for k in col.vocabulary_list], dtype=np.int64)
        order = np.argsort(keys, kind="stable")
        cache[key] = (torch.from_numpy(keys[order]).to(device), torch.from_numpy(order.astype(np.int64)).to(device))
    return cache[key]


_vocab_device_tables.cache = {}


def flat_ids(col: CategoricalColumn, values, device) -> torch.Tensor:
    """Raw values of one categorical column (any shape, flattened) -> int64 ids on `device`.

    CUDA integer tensors stay on the device; everything else is converted on the host and copied once.
    Out-of-vocabulary / out-of-range values become -1 (TF default), which the gather kernels turn into a zero row.
    """
    from . import ops
    if isinstance(values, torch.Tensor) and values.is_cuda and values.dtype in (torch.int64, torch.int32):
        v = values.reshape(-1).to(torch.int64)
        if col.kind == "identity":
            return torch.where((v >= 0) & (v < col.num_buckets), v, torch.full_like(v, -1))
        if col.kind == "hash":
            return ops.hash_bucket_i64(v, col.num_buckets)
        if col.dtype != "string":
            keys, index = _vocab_device_tables(col, v.device)
            return ops.vocab_lookup_i64(v, keys, index, -1)
        raise TypeError(f"column {col.key!r} has a string vocabulary but received an integer tensor")
    if isinstance(values, PackedStrings):
        if col.kind == "hash":
            ids = hash_bucket(values, col.num_buckets)
        elif col.kind == "vocab" and col.dtype == "string":
            ids = vocabulary_ids(col, values)
        else:
            raise TypeError(f"column {col.key!r} ({col.kind}, dtype {col.dtype}) received packed strings")
        return torch.from_numpy(ids).to(device)
    arr = values.detach().cpu().numpy() if isinstance(values, torch.Tensor) else np.asarray(values)
    arr = arr.reshape(-1)
    if col.kind == "hash":
        ids = hash_bucket(arr if arr.dtype.kind in "iu" else arr.tolist(), col.num_buckets)
    elif col.kind == "vocab":
        ids = vocabulary_ids(col, arr.tolist())
    else:
        ids = arr.astype(np.int64)
        ids = np.where((ids >= 0) & (ids < col.num_buckets), ids, -1)
    return torch.from_numpy(np.ascontiguousarray(ids)).to(device)


def column_ids(col: CategoricalColumn, value, device) -> torch.Tensor:
    """Single-valued categorical column -> int64 ids [B] on `device` (accepts [B] or [B, 1])."""
    if isinstance(value, PackedStrings):
        return flat_ids(col, value, device)
    shape = tuple(value.shape) if hasattr(value, "shape") else np.asarray(value).shape
    if len(shape) == 2 and shape[1] == 1:
        shape = shape[:1]
    if len(shape) != 1:
        raise ValueError(f"column {col.key!r}: expected one value per example ([B] or [B, 1]), got shape {shape}; "
                         "pass multi-valued features as a RaggedIds")
    return flat_ids(col, value, device)


def ids_and_bags(keys: Sequence[str], cats: dict, inputs, device):
    """Feature dict -> (ids [B, S] int64 on `device`, {slot: (flat ids, row_splits)} or None).

    Slot order is `keys`.  Single-valued features fill their column of `ids`; a RaggedFeature (multi-valued
    slot) goes to the bag dict and leaves a zero column that the mixed gather ignores.
    """
    cols, bags, B = [], {}, None
    for s, k in enumerate(keys):
        if k not in inputs:
            raise KeyError(f"feature {k!r} missing from inputs")
        v = inputs[k]
        if isinstance(v, RaggedFeature):
            rs = v.row_splits
            splits = (rs if isinstance(rs, torch.Tensor) else torch.from_numpy(np.asarray(rs, dtype=np.int64)))
            splits = splits.to(device=device, dtype=torch.int64)
            bags[s] = (flat_ids(cats[k], v.values, device), splits)
            cols.append(None)
            B = splits.numel() - 1 if B is None else B
        else:
            cols.append(column_ids(cats[k], v, device))
            B = cols[-1].shape[0]
    cols = [c if c is not None else torch.zeros((B,), dtype=torch.int64, device=device) for c in cols]
    return torch.stack(cols, dim=1), (bags or None)


def _cross_key_host(v):
    """One key's raw feature -> (values, byte offsets or None, row_splits or None) as numpy arrays."""
    splits = None
    if isinstance(v, RaggedFeature):
        rs = v.row_splits
        splits = np.ascontiguousarray(rs.detach().cpu().numpy() if isinstance(rs, torch.Tensor) else rs,
                                      dtype=np.int64)
        v = v.values
    if isinstance(v, PackedStrings):
        data, offsets = pack_strings(v)
        return data, offsets, splits
    arr = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
    if splits is None:
        if arr.ndim == 2 and arr.shape[1] == 1:
            arr = arr[:, 0]
        if arr.ndim != 1:
            raise ValueError(f"crossed_column: expected one value per example ([B] or [B, 1]), got shape {arr.shape}; "
                             "pass multi-valued features as a RaggedFeature")
    arr = arr.reshape(-1)
    if arr.dtype.kind in "iu":
        return np.ascontiguousarray(arr, dtype=np.int64), None, splits
    data, offsets = pack_strings(arr.tolist())
    return data, offsets, splits


def cross_ids(col, features, device):
    """crossed_column ids of a batch: [B] int64 (-1 = no cross) when every key is single-valued, else
    (flat ids, row_splits [B+1]), on `device`.  When some key is a CUDA tensor the crossing runs on the device
    (host strings are copied there as bytes + offsets); otherwise it runs in the host twin and the ids are copied."""
    from . import ops
    for k in col.keys:
        if k not in features:
            raise KeyError(f"feature {k!r} of crossed_column {col.name!r} is missing from the features")
    raw = [features[k] for k in col.keys]
    on_device = any(isinstance(v.values if isinstance(v, RaggedFeature) else v, torch.Tensor)
                    and (v.values if isinstance(v, RaggedFeature) else v).is_cuda for v in raw)
    if on_device:
        vals, offs, spl = [], [], []
        for v in raw:
            rs = v.row_splits if isinstance(v, RaggedFeature) else None
            x = v.values if isinstance(v, RaggedFeature) else v
            if isinstance(x, torch.Tensor) and x.is_cuda and x.dtype in (torch.int64, torch.int32):
                vals.append(x.reshape(-1).to(torch.int64).contiguous())
                offs.append(None)
            else:
                data, o, _ = _cross_key_host(x if rs is None else RaggedFeature(x, rs))
                vals.append(torch.from_numpy(data.copy()).to(device))
                offs.append(None if o is None else torch.from_numpy(o).to(device))
            if rs is not None:
                rs = rs if isinstance(rs, torch.Tensor) else torch.from_numpy(np.asarray(rs, dtype=np.int64))
                rs = rs.to(device=device, dtype=torch.int64).contiguous()
            spl.append(rs)
        B = next((s.numel() - 1 for s in spl if s is not None), None)
        B = (vals[0].numel() if offs[0] is None else offs[0].numel() - 1) if B is None else B
        return ops.cross_hash(vals, offs, spl, B, col.hash_bucket_size, col.hash_key)
    keys = [_cross_key_host(v) for v in raw]
    B = next((len(s) - 1 for _, _, s in keys if s is not None), None)
    B = (keys[0][1].size - 1 if keys[0][1] is not None else keys[0][0].size) if B is None else B
    ids, splits = cross_hash_host(keys, B, col.hash_bucket_size, col.hash_key)
    if splits is None:
        return torch.from_numpy(ids).to(device)
    return torch.from_numpy(ids).to(device), torch.from_numpy(splits).to(device)


def cross_hash_host(keys, B: int, num_buckets: int, hash_key: int):
    """dr_cross_hash_host on numpy keys [(values, byte offsets or None, row_splits or None)] -> (ids, None) when
    every key is single-valued (ids [B], -1 = no cross), else (flat ids, row_splits [B+1])."""
    lib = _lib.load()
    K = len(keys)
    for vals, offs, spl in keys:
        n = (offs.size - 1) if offs is not None else vals.size
        if (spl is None and n != B) or (spl is not None and (spl.size != B + 1 or spl[-1] > n)):
            raise ValueError(f"crossed_column: a key has {n} values, which does not fit a batch of {B}")
    vp = (C.c_void_p * K)(*[k[0].ctypes.data for k in keys])
    op = (C.c_void_p * K)(*[None if k[1] is None else k[1].ctypes.data for k in keys])
    sp = (C.c_void_p * K)(*[None if k[2] is None else k[2].ctypes.data for k in keys])
    hk = int(hash_key) & 0xFFFFFFFFFFFFFFFF
    if all(k[2] is None for k in keys):
        out = np.empty(B, dtype=np.int64)
        _lib.check(lib.dr_cross_hash_host(K, vp, op, sp, B, hk, int(num_buckets), None, out.ctypes.data),
                   "dr_cross_hash_host")
        return out, None
    splits = np.empty(B + 1, dtype=np.int64)
    _lib.check(lib.dr_cross_hash_host(K, vp, op, sp, B, hk, int(num_buckets), splits.ctypes.data, None),
               "dr_cross_hash_host")
    np.cumsum(splits, out=splits)
    out = np.empty(max(int(splits[-1]), 1), dtype=np.int64)
    _lib.check(lib.dr_cross_hash_host(K, vp, op, sp, B, hk, int(num_buckets), splits.ctypes.data, out.ctypes.data),
               "dr_cross_hash_host")
    return out[:int(splits[-1])], splits


def wide_ids(columns, inputs, device):
    """Categorical / crossed columns -> (ids [B, S] int64 on `device`, {slot: (flat ids, row_splits)} or None), the
    layout LinearTable takes: single-valued columns fill their column of ids, multi-valued ones go to the bags."""
    from .feature_column import CrossedColumn
    cols, bags, B = [], {}, None
    for s, c in enumerate(columns):
        if isinstance(c, CrossedColumn):
            r = cross_ids(c, inputs, device)
        elif isinstance(c, CategoricalColumn):
            ids, b = ids_and_bags([c.key], {c.key: c}, inputs, device)
            r = ids[:, 0] if b is None else b[0]
        else:
            raise NotImplementedError(f"column {getattr(c, 'name', c)!r}: linear_model serves categorical and "
                                      "crossed columns")
        if isinstance(r, tuple):
            bags[s] = r
            cols.append(None)
            B = r[1].numel() - 1
        else:
            cols.append(r)
            B = r.shape[0]
    cols = [c if c is not None else torch.full((B,), -1, dtype=torch.int64, device=device) for c in cols]
    return torch.stack(cols, dim=1), (bags or None)
