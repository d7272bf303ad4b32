"""Host-side checks of optimizers.RowSparseAdam and its kernels' entries, without a GPU: the conflict with fused SGD, the
guards of step() and of the clock, the model accessors, and dr_embed_adam_catch_up / dr_embed_adam_rows_tf rejecting
bad arguments before any CUDA call."""
import pytest

DR_EINVAL, DR_EALIGN = -1, -2
P = 1 << 12            # a 16-B aligned non-null address: never dereferenced, the checks fail first


def _collection(**kw):
    from deep_recommenders_b200.embedding import EmbeddingCollection
    return EmbeddingCollection([5, 7], 8, device="cpu", **kw)


def test_symbols_exported():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    for n in ("dr_embed_adam_catch_up", "dr_embed_adam_rows_tf"):
        assert n in _lib.header_symbols() and n in _lib._SIGS and hasattr(lib, n)


def test_sparse_lr_conflict_raises():
    from deep_recommenders_b200.optimizers import RowSparseAdam
    with pytest.raises(ValueError, match="sparse_lr"):
        RowSparseAdam(_collection(sparse_lr=0.1), 0.01)


def test_step_without_backward_raises():
    from deep_recommenders_b200.optimizers import RowSparseAdam
    coll = _collection()
    opt = RowSparseAdam(coll, 0.01)
    assert coll.row_optimizer is opt
    assert (opt.lr, opt.beta1, opt.beta2, opt.eps) == (0.01, 0.9, 0.999, 1e-8)     # TF1 AdamOptimizer's defaults
    assert opt.clock.lr_hist is not None and opt.clock.lr_hist.numel() == 1 << 16
    with pytest.raises(RuntimeError, match="no backward"):
        opt.step()
    with pytest.raises(ValueError, match="already"):
        RowSparseAdam(coll, 0.01)


def test_clock_must_match_and_keep_a_ring():
    from deep_recommenders_b200 import ops
    from deep_recommenders_b200.optimizers import RowSparseAdam
    with pytest.raises(ValueError, match="history"):
        RowSparseAdam(_collection(), 0.01, clock=ops.AdamClock(0.01, 0.9, 0.999, 1e-8, device="cpu"))
    with pytest.raises(ValueError, match="eps"):
        RowSparseAdam(_collection(), 0.01, clock=ops.AdamClock(0.01, 0.9, 0.999, 1e-7, device="cpu", history=16))
    coll = _collection()
    clock = ops.AdamClock(0.01, 0.9, 0.999, 1e-8, device="cpu", history=16)
    assert RowSparseAdam(coll, 0.01, clock=clock).clock is clock


def test_models_expose_their_collection_and_dense_variables():
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders.estimator.models.feature_interaction import FM
    from deep_recommenders.estimator.models.ranking import DeepFM, WDL
    cats = [fc.categorical_column_with_identity(k, n) for k, n in (("a", 5), ("b", 7))]
    cols = [fc.indicator_column(c) for c in cats], [fc.embedding_column(c, dimension=8) for c in cats]
    fm = FM(*cols, device="cpu")
    assert fm.embedding_collection() is fm.collection
    assert [id(p) for p in fm.dense_variables()] == [id(fm.collection.bias)]
    dfm = DeepFM(*cols, [4], device="cpu")
    dv = dfm.dense_variables()
    arena = {id(p) for p in dfm.embedding_collection().parameters()} - {id(dfm.embedding_collection().bias)}
    assert len(dv) == 1 + 4 and not arena & {id(p) for p in dv}        # bias, two kernels, two biases
    assert {id(p) for p in dfm.parameters()} == arena | {id(p) for p in dv}
    wdl = WDL(*cols, [4], device="cpu")
    assert wdl.embedding_collection() is wdl.embeddings
    assert {id(p) for p in wdl.deep_variables()} == {id(wdl.embeddings.weight)} | {id(p) for p in wdl.dense_variables()}


def test_unsupported_dimension():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    assert lib.dr_embed_adam_state_stride(6) == -1
    catch = lambda D: lib.dr_embed_adam_catch_up(P, 8, 4, 2, D, P, P, 0, 0, 0, P, None, P, P, None, 0, 0.01, 0.9,
                                                 0.999, 1e-8, None)
    rows = lambda D: lib.dr_embed_adam_rows_tf(P, 8, 4, 2, 2, None, P, P, P, 2 * D, D, None, 0, 0, D, 0, 0, 0, P, None,
                                               P, P, P, None, 0, 0.01, 0.9, 0.999, 1e-8, None)
    for D in (0, 6, 132):
        assert catch(D) == DR_EINVAL and f"D={D}".encode() in lib.dr_last_error()
        assert rows(D) == DR_EINVAL


def _rows_call(lib, n=8, B=4, S=2, splits=None, g=P, g_ld=16, g_slot=8, gl=None, gl_ld=0, gl_slot=0, D=8, rs=0,
               flags=0, lp=None, ids=P, state=P, step=P, lr_t=P, hist=None, hist_len=0, b1=0.9):
    return lib.dr_embed_adam_rows_tf(ids, 8, n, B, S, splits, P, P, g, g_ld, g_slot, gl, gl_ld, gl_slot, D, rs, 0, flags,
                                     P, lp, state, step, lr_t, hist, hist_len, 0.01, b1, 0.999, 1e-8, None)


def test_rows_tf_rejects_bad_arguments():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    assert _rows_call(lib, g_ld=6) == DR_EINVAL and b"gradient strides" in lib.dr_last_error()   # not a multiple of 4
    assert _rows_call(lib, g_slot=4) == DR_EINVAL            # slot rows overlap (g_slot < D)
    assert _rows_call(lib, g_ld=4, g_slot=0) == DR_EINVAL    # example rows overlap (g_ld < D)
    assert _rows_call(lib, gl=P, gl_ld=-1, flags=1, rs=32) == DR_EINVAL
    assert _rows_call(lib, rs=6) == DR_EINVAL and b"bad strides" in lib.dr_last_error()
    assert _rows_call(lib, rs=8, flags=1, gl=P, gl_ld=2, gl_slot=1) == DR_EINVAL     # no room for the in-row weight
    assert _rows_call(lib, flags=2) == DR_EINVAL
    assert _rows_call(lib, n=7) == DR_EINVAL                 # n != B * S
    assert _rows_call(lib, splits=P) == DR_EINVAL            # bags need S = 1
    assert _rows_call(lib, gl=P, gl_ld=2, gl_slot=1) == DR_EINVAL and b"come together" in lib.dr_last_error()
    assert _rows_call(lib, rs=32, flags=1) == DR_EINVAL      # an in-row weight without its gradient
    assert _rows_call(lib, rs=32, flags=1, lp=P, gl=P, gl_ld=2, gl_slot=1) == DR_EINVAL
    assert _rows_call(lib, hist_len=16) == DR_EINVAL         # a ring length without a ring
    assert _rows_call(lib, b1=1.0) == DR_EINVAL and b"dr_embed_adam_rows_tf" in lib.dr_last_error()
    assert _rows_call(lib, n=-1) == DR_EINVAL
    assert _rows_call(lib, ids=None) == DR_EINVAL
    assert _rows_call(lib, state=None) == DR_EINVAL
    assert _rows_call(lib, step=None) == DR_EINVAL
    assert _rows_call(lib, lr_t=None) == DR_EINVAL
    assert _rows_call(lib, g=P + 4) == DR_EALIGN
    assert _rows_call(lib, state=P + 8) == DR_EALIGN
    assert _rows_call(lib, n=0, B=0, ids=None) == 0           # nothing to do: no launch, no pointer needed


def test_catch_up_rejects_bad_arguments():
    from deep_recommenders_b200 import _lib
    lib = _lib.load()
    call = lambda n=8, S=2, rs=0, flags=0, lp=None, ids=P, state=P, hist=None, hist_len=0, idb=8, b1=0.9: \
        lib.dr_embed_adam_catch_up(ids, idb, n, S, 8, P, P, rs, 0, flags, P, lp, state, P, hist, hist_len, 0.01, b1,
                                   0.999, 1e-8, None)
    assert call(n=7) == DR_EINVAL                            # not whole examples of S slots
    assert call(S=0) == DR_EINVAL
    assert call(flags=2) == DR_EINVAL and b"flags=2" in lib.dr_last_error()
    assert call(b1=1.0) == DR_EINVAL and b"dr_embed_adam_catch_up" in lib.dr_last_error()
    assert call(rs=6) == DR_EINVAL and b"bad strides" in lib.dr_last_error()
    assert call(rs=8, flags=1) == DR_EINVAL
    assert call(rs=32, flags=1, lp=P) == DR_EINVAL
    assert call(idb=2) == DR_EINVAL
    assert call(hist_len=4) == DR_EINVAL
    assert call(ids=None) == DR_EINVAL
    assert call(state=P + 4) == DR_EALIGN
    assert call(n=0, ids=None) == 0
