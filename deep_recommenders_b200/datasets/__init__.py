"""Input formats of the hot path (SURVEY.md section 8(f) #4): TFRecord files of tf.train.Example protos and the
MovieLens dataset classes of the reference (datasets/movielens.py), on the native parser of the C-ABI library, the
synthetic multi-task data of datasets/synthetic_for_multi_task.py, and the Cora citation graph of datasets/cora.py."""
from .tfrecord import TFRecordFile, TFRecordWriter, serialize_example  # noqa: F401
from .movielens import MovieLens, MovielensRanking, serialize_tfrecords  # noqa: F401
from .synthetic_for_multi_task import SyntheticForMultiTask  # noqa: F401


def __getattr__(name):
    # Cora needs scipy: import it on first use, so importing the package does not
    if name in ("Cora", "write_synthetic_cora"):
        import importlib
        return getattr(importlib.import_module(__name__ + ".cora"), name)
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
