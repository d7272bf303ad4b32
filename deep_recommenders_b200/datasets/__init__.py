"""Input formats of the hot path (SURVEY.md section 8(f) #4): TFRecord files of tf.train.Example protos and the
MovieLens dataset classes of the reference (datasets/movielens.py), on the native parser of the C-ABI library, and the
synthetic multi-task data of datasets/synthetic_for_multi_task.py."""
from .tfrecord import TFRecordFile, TFRecordWriter, serialize_example  # noqa: F401
from .movielens import MovieLens, MovielensRanking, serialize_tfrecords  # noqa: F401
from .synthetic_for_multi_task import SyntheticForMultiTask  # noqa: F401
