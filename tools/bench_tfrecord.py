"""Host-side throughput of the native TFRecord / tf.train.Example reader (csrc/tfrecord.cu) on MovieLens-shaped
records (datasets/movielens.py:54-62 schema), against parsing the same records with the protobuf library's Python
API.  CPU only.  Prints one JSON line."""
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from deep_recommenders_b200.datasets import TFRecordFile, TFRecordWriter  # noqa: E402
from deep_recommenders_b200.datasets.movielens import MovieLens, _serialize_example  # noqa: E402
from deep_recommenders_b200.hashing import hash_bucket  # noqa: E402


def main():
    n = int(os.environ.get("N", 200_000))
    rng = np.random.default_rng(0)
    genres = [b"Action", b"Comedy", b"Drama", b"Sci-Fi", b"Children's"]
    path = os.path.join(tempfile.mkdtemp(prefix="dr_tfr_"), "m.tfrecords")
    t0 = time.perf_counter()
    with TFRecordWriter(path) as w:
        for i in range(n):
            w.write(_serialize_example({
                "UserID": str(int(rng.integers(1, 6041))).encode(), "MovieID": str(int(rng.integers(1, 3953))).encode(),
                "Gender": b"FM"[i % 2:i % 2 + 1], "Zip-code": b"%05d" % (i % 99999), "Title": b"Movie %d (1999)" % (i % 3952),
                "Age": 25, "Occupation": i % 21, "Rating": 1 + i % 5, "Timestamp": 978300000 + i,
                "Genres": [genres[j] for j in range(1 + i % 3)]}))
    t_write = time.perf_counter() - t0
    size = os.path.getsize(path)
    t0 = time.perf_counter()
    f = TFRecordFile(path)                                   # mmap + index + both CRC-32C checks
    t_index = time.perf_counter() - t0
    t0 = time.perf_counter()
    B, nb = 1024, 0
    for lo in range(0, n, B):
        ex = f.parse(lo, lo + B, MovieLens._SPEC)
        nb += 1
    t_parse = time.perf_counter() - t0
    t0 = time.perf_counter()
    for lo in range(0, n, B):
        ex = f.parse(lo, lo + B, {"UserID": ("string", True), "MovieID": ("string", True)})
        hash_bucket(ex["UserID"], 6040)
        hash_bucket(ex["MovieID"], 3952)
    t_ids = time.perf_counter() - t0
    lib = f._lib
    big = {}
    for threads in (1, 2, 4, 8):                          # one call over all records (batch 65536-style parsing)
        lib.dr_set_host_threads(threads)
        t0 = time.perf_counter()
        f.parse(0, n, MovieLens._SPEC)
        big[str(threads)] = round(n / (time.perf_counter() - t0))
    lib.dr_set_host_threads(1)
    out = dict(records=n, file_mb=round(size / 1e6, 1), write_s=round(t_write, 2),
               index_crc_s=round(t_index, 3), index_gb_per_s=round(size / t_index / 1e9, 2),
               parse_all_10_features_s=round(t_parse, 3), parse_records_per_s=round(n / t_parse),
               parse_two_ids_and_farmhash_s=round(t_ids, 3), ids_records_per_s=round(n / t_ids),
               batch_1024_threads=1, one_call_records_per_s_by_threads=big, host_cpus=os.cpu_count())
    try:        # context: the protobuf library's Python API on the same records (one Example at a time)
        sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
        from test_cpu_datasets import _example_classes
        Example = _example_classes()
        m = min(n, 20000)
        t0 = time.perf_counter()
        for i in range(m):
            e = Example.FromString(f.record(i))
            _ = e.features.feature["UserID"].bytes_list.value[0], e.features.feature["Age"].int64_list.value[0]
        out["protobuf_python_records_per_s"] = round(m / (time.perf_counter() - t0))
    except Exception as e:      # pragma: no cover
        out["protobuf_python_records_per_s"] = f"unavailable: {e}"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
