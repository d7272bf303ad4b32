"""Host-side checks of optimizers.KerasAdam and dr_adam_step_multi, without a GPU: the export, the entry's rejections
(before any launch), the oracle's difference from torch.optim.Adam, compile() with the spec, and what build_for_model
puts in the dense group and on the row-sparse optimizers."""
import ctypes as C

import numpy as np
import pytest
import torch

from keras_adam_oracle import keras_adam

DR_EINVAL = -1
P = 1 << 12            # a 16-B aligned non-null address: never dereferenced, the checks fail first


def _lib():
    from deep_recommenders_b200 import _lib as L
    return L


def _multi(lib, ns, ptr=P, b1=0.9, b2=0.999, eps=1e-7, null_at=None, arrays=True, k=None):
    k = len(ns) if k is None else k
    arr = lambda: (C.c_void_p * max(len(ns), 1))(*[None if i == null_at else ptr for i in range(len(ns))])
    n = (C.c_int64 * max(len(ns), 1))(*ns)
    if not arrays:
        return lib.dr_adam_step_multi(k, None, None, None, None, None, 0.01, b1, b2, eps, None, None)
    return lib.dr_adam_step_multi(k, arr(), arr(), arr(), arr(), n, 0.01, b1, b2, eps, None, None)


def test_symbol_exported():
    L = _lib()
    assert "dr_adam_step_multi" in L.header_symbols() and "dr_adam_step_multi" in L._SIGS
    assert hasattr(L.load(), "dr_adam_step_multi")


def test_multi_rejects_before_any_launch():
    L = _lib()
    lib = L.load()
    before = L.launch_count()

    def rejects(rc, *needles):
        assert rc == DR_EINVAL, rc
        for s in needles:
            assert s.encode() in lib.dr_last_error(), lib.dr_last_error()

    rejects(_multi(lib, [4], k=-1), "dr_adam_step_multi", "n_tensors=-1")
    rejects(_multi(lib, [4], arrays=False), "null pointer array")
    rejects(_multi(lib, [8, 4, -3, 4]), "n[2]=-3")
    rejects(_multi(lib, [8, 4, 4], null_at=1), "null pointer in tensor 1")
    rejects(_multi(lib, [4], b1=1.0), "out of range")
    rejects(_multi(lib, [4], b2=-0.1), "out of range")
    rejects(_multi(lib, [4], eps=-1e-9), "out of range")
    # a bad tensor after 70 good ones (more than one launch holds) still stops the call before the first launch
    rejects(_multi(lib, [4] * 70 + [-1]), "n[70]=-1")
    # nothing to do: no tensors, or only empty ones (whose pointers may be NULL)
    assert _multi(lib, [], arrays=False, k=0) == 0
    assert _multi(lib, [0, 0, 0], ptr=None) == 0
    assert L.launch_count() == before


def test_oracle_is_tf_adam_not_torch_adam():
    """At a large eps the restatement differs from torch.optim.Adam by far more than rounding; at a tiny one it agrees."""
    rng = np.random.default_rng(0)
    p0 = rng.standard_normal(64)
    grads = [rng.standard_normal(64) * 1e-2 for _ in range(6)]
    lrs = [0.01, 0.01, 0.01, 0.005, 0.005, 0.005]
    for eps, differs in ((1e-3, True), (1e-12, False)):
        want, _, _ = keras_adam(p0, grads, lrs, 0.9, 0.999, eps)
        p = torch.tensor(p0, dtype=torch.float64, requires_grad=True)
        opt = torch.optim.Adam([p], lr=lrs[0], betas=(0.9, 0.999), eps=eps)
        for g, lr in zip(grads, lrs):
            opt.param_groups[0]["lr"] = lr
            p.grad = torch.tensor(g, dtype=torch.float64)
            opt.step()
        gap = np.abs(p.detach().numpy() - want).max()
        assert (gap > 1e-4) if differs else (gap < 1e-7), (eps, gap)


def _fm(**kw):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import FactorizationMachine
    cats = [fc.categorical_column_with_identity(k, n) for k, n in (("a", 5), ("b", 7))]
    return FactorizationMachine([fc.indicator_column(c) for c in cats], [fc.embedding_column(c, 8) for c in cats],
                                seed=0, device="cpu", **kw)


def test_compile_stores_the_spec_and_rejects_amsgrad():
    from deep_recommenders_b200.optimizers import KerasAdam
    with pytest.raises(NotImplementedError, match="amsgrad"):
        KerasAdam(amsgrad=True)
    with pytest.raises(ValueError, match="tables"):
        KerasAdam(tables="sparse")
    spec = KerasAdam()
    model = _fm()
    model.compile(loss="binary_crossentropy", optimizer=spec)
    assert model._optimizer_spec is spec and model._optimizer is None
    assert model.optimizer.lr == pytest.approx(0.001)
    model.optimizer.lr = 0.02
    assert spec.kw["lr"] == 0.02 and spec.param_groups[0]["lr"] == 0.02


def test_build_groups_and_rejections():
    from deep_recommenders_b200.optimizers import KerasAdam, RowSparseAdam
    model = _fm()
    coll = model.embeddings
    opt = KerasAdam(0.01).build_for_model(model)
    assert [ro.collection for ro in opt.row_optimizers] == [coll] and coll.row_optimizer is opt.row_optimizers[0]
    assert opt.clock.lr_hist is not None and opt.clock.lr == 0.01
    dense = [p for p, _, _ in opt.dense]
    assert dense == [coll.bias]
    dm = _fm()
    dense_opt = KerasAdam(tables="dense").build_for_model(dm)
    assert not dense_opt.row_optimizers and dm.embeddings.row_optimizer is None
    assert {id(p) for p, _, _ in dense_opt.dense} == {id(dm.embeddings.weight), id(dm.embeddings.bias)}
    for p, m, v in dense_opt.dense:             # every variable's moments start 16-B aligned in the flat arenas
        assert m.shape == p.shape and v.shape == p.shape and m.data_ptr() % 16 == 0 and v.data_ptr() % 16 == 0
    with pytest.raises(ValueError, match="sparse_lr"):
        KerasAdam().build_for_model(_fm(sparse_lr=0.1))
    mine = _fm()
    RowSparseAdam(mine.embeddings, 0.001, epsilon=1e-7)
    with pytest.raises(ValueError, match="already has a RowSparseAdam"):
        KerasAdam().build_for_model(mine)
