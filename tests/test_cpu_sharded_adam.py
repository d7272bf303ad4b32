"""CPU-side checks of optimizer="adam_rows_tf" on the row-sharded DeepFM step: the dr_shard_adam_* entries are exported
and reject bad arguments before any CUDA call; the Adam moments re-shard through checkpoint.save_rows / load_rows like
the weights; the SGD config is unchanged and a checkpoint of one optimizer does not load into a trainer of the other."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

DR_EINVAL, DR_EALIGN = -1, -2
P = 1 << 12            # a 16-B aligned non-null address: never dereferenced, the checks fail first


def test_shard_adam_symbols_exported():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    names = ("dr_shard_adam_mark", "dr_shard_adam_prepare", "dr_shard_adam_apply")
    for n in names:
        assert n in _lib.header_symbols() and n in _lib._SIGS and hasattr(lib, n)


def test_shard_adam_entries_reject_bad_arguments_without_gpu():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    mark = lambda n=8, world=2, ids=P, idb=8, touch=P, step=P: lib.dr_shard_adam_mark(ids, idb, n, 2, P, P, world,
                                                                                     touch, step, None)
    assert mark(world=0) == DR_EINVAL
    assert mark(world=65) == DR_EINVAL and b"world=65" in lib.dr_last_error()
    assert mark(ids=None) == DR_EINVAL
    assert mark(touch=None) == DR_EINVAL
    assert mark(step=None) == DR_EINVAL
    assert mark(idb=2) == DR_EINVAL
    assert mark(n=-1) == DR_EINVAL
    prep = lambda D=16, rs=32, lin_off=0, flags=1, touch=P, state=P, hist=0, hp=None, local=10, b2=0.999, shard=P: \
        lib.dr_shard_adam_prepare(touch, local, P, P, D, rs, lin_off, flags, shard, state, P, hp, hist, 0.01, 0.9, b2,
                                  1e-7, None)
    assert prep(local=-1) == DR_EINVAL and b"local_rows=-1" in lib.dr_last_error()
    assert prep(local=1 << 31) == DR_EINVAL
    assert prep(D=6) == DR_EINVAL and b"D=6" in lib.dr_last_error()
    assert prep(D=132) == DR_EINVAL
    assert prep(D=0) == DR_EINVAL
    assert prep(rs=16) == DR_EINVAL                          # no room for the in-row first-order weight
    assert prep(lin_off=320) == DR_EINVAL                    # a trailing array AND an in-row weight
    assert prep(flags=0, lin_off=100) == DR_EINVAL           # the trailing array overlaps the rows
    assert prep(touch=None) == DR_EINVAL
    assert prep(state=None) == DR_EINVAL
    assert prep(hist=16) == DR_EINVAL                        # a ring length without a ring
    assert prep(b2=1.0) == DR_EINVAL and b"dr_shard_adam_prepare" in lib.dr_last_error()
    assert prep(shard=P + 4) == DR_EALIGN
    assert prep(state=P + 8) == DR_EALIGN
    app = lambda D=16, grad=P, lr_t=P, b1=0.9, eps=1e-7: lib.dr_shard_adam_apply(P, P, 10, D, 32, 0, 1, P, grad, P, P,
                                                                                  lr_t, b1, 0.999, eps, None)
    assert app(D=130) == DR_EINVAL
    assert app(grad=None) == DR_EINVAL
    assert app(lr_t=None) == DR_EINVAL
    assert app(b1=1.0) == DR_EINVAL
    assert app(eps=-1.0) == DR_EINVAL and b"dr_shard_adam_apply" in lib.dr_last_error()
    assert app(grad=P + 4) == DR_EALIGN


@pytest.mark.parametrize("new_world", [2, 5])
def test_moments_reshard_like_the_weights(tmp_path, new_world):
    """m / v saved by 3 ranks in the weights' shape ([local, vdim] with the in-row first-order moment, or a trailing
    [local] array) come back on any other world size with the rows each new rank owns."""
    from deep_recommenders_b200 import checkpoint, shard_plan
    total, V, W = 23, 32, 3
    rng = np.random.default_rng(new_world)
    glob = {k: torch.from_numpy(rng.standard_normal((total, V)).astype(np.float32)) for k in ("weight", "m", "v")}
    glob.update({k: torch.from_numpy(rng.standard_normal(total).astype(np.float32)) for k in ("m_lin", "v_lin")})
    prefix = str(tmp_path / "ck")
    for r in range(W):
        checkpoint.save_rows(prefix, r, W, total, {k: t[r::W] for k, t in glob.items()}, save_id=7)
    checkpoint.save_meta(prefix, {"optimizer": "adam_rows_tf"}, {"adam_step": torch.tensor([5])}, world=W, save_id=7)
    for r in range(new_world):
        got = checkpoint.load_rows(prefix, r, new_world)
        assert set(got) == set(glob)
        for k, t in glob.items():
            assert got[k].shape[0] == shard_plan.local_rows(total, r, new_world)
            assert torch.equal(got[k], t[r::new_world]), (k, r)


def _stub(optimizer, exchange="p2p"):
    """A trainer object with just what get_config / load read before they touch a GPU."""
    from deep_recommenders_b200.sharded import ShardedDeepFMTrainStep
    t = ShardedDeepFMTrainStep.__new__(ShardedDeepFMTrainStep)
    t.emb = SimpleNamespace(rows_list=[5, 7], vdim=32, lin_in_row=True)
    t.D, t.B, t.lr, t.exchange, t.optimizer = 16, 64, 0.01, exchange, optimizer
    t.layers = [SimpleNamespace(units=32), SimpleNamespace(units=8), SimpleNamespace(units=1)]
    return t


def test_sgd_config_unchanged_and_adam_config_names_the_optimizer():
    sgd = _stub("sgd").get_config()
    assert sgd == {"class": "ShardedDeepFMTrainStep", "rows": [5, 7], "dim": 16, "dnn_units": [32, 8],
                   "batch_size": 64, "lr": 0.01, "exchange": "p2p", "row_width": 32, "lin_in_row": True}
    adam = _stub("adam_rows_tf").get_config()
    assert adam == dict(sgd, optimizer="adam_rows_tf")


@pytest.mark.parametrize("saved,loader", [("sgd", "adam_rows_tf"), ("adam_rows_tf", "sgd")])
def test_loading_across_optimizers_raises(tmp_path, saved, loader):
    from deep_recommenders_b200 import checkpoint
    prefix = str(tmp_path / "ck")
    checkpoint.save_meta(prefix, _stub(saved).get_config(), {"flat": torch.zeros(4)}, world=1, save_id=1)
    with pytest.raises(ValueError, match="optimizer"):
        _stub(loader).load(prefix)

