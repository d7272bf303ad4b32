"""deep_recommenders_b200 -- CUDA-native (H100, sm_90a) implementation of the data-parallel hot path of
LongmaoTeamTf/deep_recommenders: embedding lookup -> FM / DeepFM / DCN Cross, and the two-tower
in-batch softmax, forward and backward, behind the reference's Keras-layer API.

Layout:
  csrc/         hand-written CUDA kernels + the C-ABI (include/deeprec_b200.h)
  _lib.py       ctypes binding (no fallback: raises if the .so is missing)
  ops.py        torch.autograd.Function wrappers (PyTorch = memory/streams/autograd plumbing)
  keras/, estimator/   same-named classes at the reference's import paths
The top-level `deep_recommenders` package in this repo is an import alias of this one so the
reference's import lines work unchanged.
"""
__version__ = "0.1.0"


def __getattr__(name):
    # the whole-step trainers, resolved on first use (importing the package stays free of torch)
    if name == "DCNTrainStep":
        from .dcn_training import DCNTrainStep
        return DCNTrainStep
    raise AttributeError(f"module {__name__!r} has no attribute {name!r}")
