"""optimizers.KerasAdam and dr_adam_step_multi on the GPU.

  * The kernel: about 300 tensors (more than one launch holds), sizes 0, 1, 3, 4, 5, 4097, 2^20 + 3 and random small
    ones, some views at float offsets that are not multiples of 4; bitwise equal to dr_adam_step on each tensor, with
    lr_t from the host and from the clock, and sentinel guards around every buffer unchanged.
  * The models, each trained through fit() for 12 steps (3 epochs of 4, an evaluation between epochs, a learning-rate
    write through model.optimizer.lr after step 6): FactorizationMachine with a bag slot, Keras DeepFM, DCN, xDeepFM,
    DIN with context slots, the Transformer example's classifier (Adam(beta_2=0.98, epsilon=1e-9), Noam rates) and
    GCN on the Cora fixture.  The batches carry duplicate ids, pruned ids and rows that sit out 1, 3 and 11 steps.
    Every step, every dense variable that has a gradient is held per element to the float64 oracle (tests/adam_oracle.py
    `moments` and `functor` from the kernel's own inputs, lr_t to the per-step schedule) and every other one keeps its
    bits; for FactorizationMachine and DeepFM the table rows are held to it too (the replay of skipped steps at the
    schedule's rates, then the step).  The collections' models also train with tables="dense" on the same seed: per-step
    losses, evaluation logs and the final state_dict() agree within the atomic-order tolerance of
    test_gpu_layer_adam_rows.py.
  * TF's formula: one variable at epsilon=1e-3 matches it and misses torch.optim.Adam.
  * Rebuilds and rejections: a recompile restarts at step 1 from flushed tables; a RowSparseAdam the user attached and a
    sparse_lr model raise ValueError.
"""
import importlib.util
import math
import pathlib

import numpy as np
import pytest
import torch

from adam_oracle import U, Entry, check_bound, functor, lr_t, moments
from keras_adam_oracle import keras_adam, replay_sched
from test_gpu_layer_adam_rows import ROWS, _batch, _columns, _grads64, _host

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
HERE = pathlib.Path(__file__).resolve().parent
SENTINEL_BITS = 0x5EBADBAD


def _lib():
    from deep_recommenders_b200 import _lib as L
    return L


# ---- 1. the kernel ----------------------------------------------------------------------------------------------------
def _tensors(sizes, offsets, seed, G=8):
    """Per tensor four sentinel-framed buffers and the views (p, g, m, v) at the given float offsets."""
    rng = np.random.default_rng(seed)
    sentinel = float(np.frombuffer(np.uint32(SENTINEL_BITS).tobytes(), F32)[0])
    bufs, views = [], []
    for n, offs in zip(sizes, offsets):
        b4, v4 = [], []
        for k, off in enumerate(offs):
            buf = torch.full((n + off + 2 * G,), sentinel, device="cuda")
            x = rng.standard_normal(n).astype(F32)
            if k == 2:
                x *= 0.1
            if k == 3:
                x = np.abs(x) * 1e-2
            buf[G + off:G + off + n] = torch.from_numpy(x).cuda()
            b4.append(buf)
            v4.append(buf[G + off:G + off + n])
        bufs.append(b4)
        views.append(v4)
    return bufs, views


@pytest.mark.parametrize("lr_from", ["host", "clock"])
def test_multi_equals_per_tensor_adam_step(lr_from):
    from deep_recommenders_b200 import ops
    L = _lib()
    lib = L.load()
    rng = np.random.default_rng(7)
    sizes = [0, 1, 3, 4, 5, 4097, (1 << 20) + 3] + [int(s) for s in rng.integers(0, 3000, 293)]
    offsets = [tuple(int(o) for o in rng.integers(0, 4, 4)) if i % 3 == 1 else (0, 0, 0, 0) for i in range(len(sizes))]
    offsets[4] = (1, 1, 1, 1)                                         # misaligned, size 5: scalar throughout
    b1, b2, eps, host_lr = 0.9, 0.98, 1e-9, 0.0123
    clock = ops.AdamClock(0.01, b1, b2, eps, device="cuda")
    clock.advance()
    clock.advance()
    lr_dev = clock.lr_t.data_ptr() if lr_from == "clock" else None
    ref_bufs, ref = _tensors(sizes, offsets, 1)
    got_bufs, got = _tensors(sizes, offsets, 1)
    st = ops._stream()
    for (p, g, m, v), n in zip(ref, sizes):
        assert lib.dr_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), n, host_lr, b1, b2, eps, 0,
                                lr_dev, st) == 0
    import ctypes as C
    k = len(sizes)
    arr = lambda j: (C.c_void_p * k)(*[t[j].data_ptr() for t in got])
    ns = (C.c_int64 * k)(*sizes)
    before = L.launch_count()
    assert lib.dr_adam_step_multi(k, arr(0), arr(1), arr(2), arr(3), ns, host_lr, b1, b2, eps, lr_dev, st) == 0
    assert L.launch_count() - before == math.ceil(sum(1 for n in sizes if n) / 64)
    torch.cuda.synchronize()
    for i, (rb, gb) in enumerate(zip(ref_bufs, got_bufs)):
        for j in range(4):
            a, b = rb[j].cpu().numpy().view(np.uint32), gb[j].cpu().numpy().view(np.uint32)
            assert np.array_equal(a, b), f"tensor {i} (n={sizes[i]}, offsets {offsets[i]}) array {'pgmv'[j]}"
            n, off = sizes[i], offsets[i][j]
            assert (b[:8 + off] == SENTINEL_BITS).all() and (b[8 + off + n:] == SENTINEL_BITS).all(), (i, j)
    # the ops wrapper is the same launch
    p, g, m, v = (torch.randn(1000, device="cuda") for _ in range(4))
    v = v.abs()
    want = [t.clone() for t in (p, g, m, v)]
    ops.adam_step_(want[0], want[1], want[2], want[3], 0.0, b1, b2, eps, zero_grad=False, lr_t_dev=clock.lr_t)
    ops.adam_step_multi_([p], [g], [m], [v], clock)
    for x, y in zip((p, g, m, v), want):
        assert torch.equal(x, y)


# ---- 2. the models ------------------------------------------------------------------------------------------------
T_STEPS, EPOCHS, LR_WRITE_AFTER, LR_NEW = 12, 3, 6, 0.004


def _spec_class():
    from deep_recommenders_b200.optimizers import KerasAdam

    class Probe(KerasAdam):
        """KerasAdam that holds every step to the float64 oracle."""

        def __init__(self, *a, check_tables=False, **kw):
            super().__init__(*a, **kw)
            self.check_tables, self.t, self.lrs, self.last = check_tables, 0, [], {}

        def build_for_model(self, model):
            out = super().build_for_model(model)
            self.t, self.lrs, self.last = 0, [], {}
            return out

        def step(self):
            self.t += 1
            t = self.t
            self.lrs.append(float(self.kw["lr"]))
            b1, b2, eps = self.beta_1, self.beta_2, self.epsilon
            live, idle = [], []
            for p, m, v in self.dense:
                if p.grad is None:
                    idle.append((p, p.detach().clone()))
                else:
                    live.append((p, m, v, *(x.detach().double().cpu().numpy() for x in (p, p.grad, m, v))))
            rows = []
            for ro in (self.row_optimizers if self.check_tables else []):
                coll = ro.collection
                s0 = _host(coll, ro)
                prev = self.last.get(id(ro))
                if prev is not None:            # rows read since the last step were replayed to step t - 1
                    moved = prev["stamp"] != s0["stamp"]
                    assert (s0["stamp"][moved] == t - 1).all()
                    rp, rm, rv, bp, bm, bv = replay_sched(prev["p"][moved], prev["m"][moved], prev["v"][moved],
                                                          prev["stamp"][moved], t - 1, self.lrs, b1, b2, eps)
                    check_bound(f"replay to {t - 1} p", s0["p"][moved], rp, bp)
                    check_bound(f"replay to {t - 1} m", s0["m"][moved], rm, bm)
                    check_bound(f"replay to {t - 1} v", s0["v"][moved], rv, bv)
                    assert np.array_equal(s0["w"][~moved], prev["w"][~moved])
                rows.append((ro, s0, *(_grads64(ro, coll) if ro.has_pending else (None, None))))
            super().step()
            got_lr = float(self.clock.lr_t)
            want_lr = float(lr_t(t, self.lrs[-1], b1, b2))
            assert abs(got_lr - want_lr) <= 4 * U * want_lr, (t, got_lr, want_lr)
            for p, m, v, p0, g, m0, v0 in live:
                m1, bm1, v1, bv1 = moments(m0, v0, Entry(g, 0.0, 0.0), 0.0, b1, b2)
                mk, vk = m.double().cpu().numpy(), v.double().cpu().numpy()
                check_bound(f"step {t} m {tuple(p.shape)}", mk, m1, bm1)
                check_bound(f"step {t} v {tuple(p.shape)}", vk, v1, bv1)
                p1, bp1 = functor(p0, mk, vk, got_lr, eps)
                check_bound(f"step {t} p {tuple(p.shape)}", p.detach().double().cpu().numpy(), p1, bp1)
            for p, before in idle:
                assert torch.equal(p.detach(), before), "a variable without a gradient moved"
            for ro, s0, entry, hits in rows:
                s1 = _host(ro.collection, ro)
                if hits is None:
                    assert np.array_equal(s1["st"], s0["st"]) and np.array_equal(s1["w"], s0["w"])
                else:
                    hit = hits > 0
                    e = Entry(entry.ref[hit], 0.0, entry.slack[hit])
                    m1, bm1, v1, bv1 = moments(s0["m"][hit], s0["v"][hit], e, 0.0, b1, b2)
                    check_bound(f"step {t} table m", s1["m"][hit], m1, bm1)
                    check_bound(f"step {t} table v", s1["v"][hit], v1, bv1)
                    p1, bp1 = functor(s0["p"][hit], s1["m"][hit], s1["v"][hit], got_lr, eps)
                    check_bound(f"step {t} table p", s1["p"][hit], p1, bp1)
                    assert (s1["stamp"][hit] == t).all()
                    assert np.array_equal(s1["w"][~hit], s0["w"][~hit])
                    assert np.array_equal(s1["st"][~hit], s0["st"][~hit])
                self.last[id(ro)] = s1

    return Probe


class _LrWrite:
    """model.optimizer.lr = LR_NEW after step LR_WRITE_AFTER (it applies from the next step on)."""

    def __init__(self):
        self.n = 0

    def on_batch_end(self, batch, logs=None):
        self.n += 1
        if self.n == LR_WRITE_AFTER:
            self.model.optimizer.lr = LR_NEW

    def on_epoch_end(self, epoch, logs):
        return False


def _recording(loss_name, out):
    from deep_recommenders_b200.keras import engine as K
    fn = K._LOSSES[loss_name]

    def loss(yt, yp):
        per_row = fn(yt, yp)
        out.append(float(per_row.mean().detach()))
        return per_row
    return loss


def _skip_ids(t):
    """[BATCH, 2] ids over tables of ROWS a, b rows: column a carries the skip pattern of test_gpu_layer_adam_rows."""
    feats, y = _batch(t, False)
    return torch.from_numpy(np.stack([feats["a"], feats["b"]], 1)).cuda(), y


def _ranking(kind):
    """(model factory, train batches, validation batches, loss, check tables)."""
    if kind in ("fm_bags", "deepfm"):
        from deep_recommenders.keras.models.ranking import DeepFM, FactorizationMachine
        bags = kind == "fm_bags"
        D = 32 if bags else 8

        def make():
            cols = _columns(D, bags)
            if bags:
                return FactorizationMachine(*cols, seed=3, device="cuda")
            return DeepFM(*cols, dnn_units_size=[16, 8], seed=3, device="cuda")
        train = lambda: [_batch(t, bags) for t in range(1, T_STEPS + 1)]
        val = lambda e: [_batch(100 + e, bags)]
        return make, train, val, True
    rows = [ROWS["a"], ROWS["b"]]
    if kind == "dcn":
        from deep_recommenders.keras.layers import DCN
        make = lambda: DCN(rows, 8, num_cross=2, dnn_units=[16, 8], seed=3, device="cuda")
    elif kind == "xdeepfm":
        from deep_recommenders.keras.layers import XDeepFM
        make = lambda: XDeepFM(rows, 8, cin_layers=(8, 8), dnn_units=(16, 8), seed=3, device="cuda")
    else:
        from deep_recommenders.keras.layers import DIN
        make = lambda: DIN(item_rows=30, dim=8, context_rows=rows, att_units=8, dnn_units=(16, 8),
                           dnn_activation="dice", seed=3, device="cuda")
    if kind != "din":
        return make, lambda: [_skip_ids(t) for t in range(1, T_STEPS + 1)], lambda e: [_skip_ids(100 + e)], False

    def din_batch(t):
        ids, y = _skip_ids(t)
        rng = np.random.default_rng(500 + t)
        item = torch.from_numpy(rng.integers(-1, 31, ids.shape[0])).cuda()
        hist = torch.from_numpy(rng.integers(-1, 31, (ids.shape[0], 5))).cuda()
        return (ids, item, hist), y
    return make, lambda: [din_batch(t) for t in range(1, T_STEPS + 1)], lambda e: [din_batch(100 + e)], False


def _fit(make, train, val, spec):
    torch.manual_seed(0)
    model = make()
    losses = []
    model.compile(loss=_recording("binary_crossentropy", losses), optimizer=spec)
    vals = iter(range(EPOCHS))
    hist = model.fit(train(), epochs=EPOCHS, steps_per_epoch=T_STEPS // EPOCHS,
                     validation_data=lambda: val(next(vals)), validation_steps=1, callbacks=[_LrWrite()])
    assert spec.t == T_STEPS
    return model, losses, hist


@pytest.mark.parametrize("kind", ["fm_bags", "deepfm", "dcn", "xdeepfm", "din"])
def test_ranking_models_rows_equal_dense_and_the_oracle(kind):
    make, train, val, check_tables = _ranking(kind)
    Probe = _spec_class()
    rows_spec = Probe(0.01, check_tables=check_tables)
    dense_spec = Probe(0.01, tables="dense")
    rows_model, rows_losses, rows_hist = _fit(make, train, val, rows_spec)
    dense_model, dense_losses, dense_hist = _fit(make, train, val, dense_spec)
    assert rows_spec.row_optimizers and not dense_spec.row_optimizers
    assert rows_spec.lrs == dense_spec.lrs == [0.01] * LR_WRITE_AFTER + [LR_NEW] * (T_STEPS - LR_WRITE_AFTER)
    assert len(rows_losses) == T_STEPS + EPOCHS                        # every training step and every evaluation
    np.testing.assert_allclose(rows_losses, dense_losses, rtol=1e-4, atol=1e-5)
    for k in dense_hist:
        np.testing.assert_allclose(rows_hist[k], dense_hist[k], rtol=1e-4, atol=1e-5, err_msg=k)
    want, got = dense_model.state_dict(), rows_model.state_dict()       # the rows run's tables are flushed first
    assert got.keys() == want.keys()
    for k in want:
        torch.testing.assert_close(got[k], want[k], rtol=1e-4, atol=1e-5, msg=k)


def _transformer():
    spec = importlib.util.spec_from_file_location("ex_transformer",
                                                  HERE.parent / "examples" / "train_transformer_on_synthetic_keras.py")
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    return ex


def test_transformer_and_gcn_dense_variables_follow_the_oracle():
    from deep_recommenders.keras.models.nlp.transformer import Noam
    Probe = _spec_class()
    ex = _transformer()
    torch.manual_seed(0)
    model = ex.TransformerClassifier(60, 12, seed=0)
    spec = Probe(beta_1=0.9, beta_2=0.98, epsilon=1e-9)
    model.compile(optimizer=spec, loss="categorical_crossentropy")
    model.fit(ex.synthetic_batches(60, 12, 16, 0), epochs=EPOCHS, steps_per_epoch=T_STEPS // EPOCHS,
              validation_data=lambda: ex.synthetic_batches(60, 12, 16, 1), validation_steps=1,
              callbacks=[Noam(model_dim=8, warmup_steps=4)])
    assert spec.t == T_STEPS and len(set(spec.lrs)) > T_STEPS // 2    # Noam writes a new rate every step
    assert len(spec.dense) == len([p for p in model.parameters() if p.requires_grad])

    from deep_recommenders.datasets import Cora
    from deep_recommenders_b200 import ops
    from deep_recommenders.keras.models.retrieval import GCN
    from deep_recommenders.keras.layers import Model
    np.random.seed(0)
    cora = Cora(str(HERE / "golden" / "cora_small"))
    ids, features, labels = cora.load_content()
    g = ops.CSRAdjacency.from_any(cora.spectral_graph(cora.build_graph(ids)))
    cora.sample_train_nodes(labels)
    (ytr, wtr), (yva, wva), _ = cora.split_labels(labels, num_valid_nodes=50)
    feats = torch.from_numpy(np.asarray(features.todense(), dtype=np.float32)).cuda()

    class Net(Model):
        def __init__(self):
            super().__init__()
            self.gcn1, self.gcn2 = GCN(16), GCN(cora.num_classes, activation="softmax")
            self.built = True

        def call(self, inputs, **kwargs):
            adj, x = inputs
            return self.gcn2(self.gcn1(x, adj), adj)

    torch.manual_seed(0)
    net = Net()
    spec = Probe(0.01)
    net.compile(optimizer=spec, loss="categorical_crossentropy", weighted_metrics=["acc"])
    net.fit([g, feats], ytr, sample_weight=wtr, validation_data=([g, feats], yva, wva), batch_size=feats.shape[0],
            epochs=T_STEPS, shuffle=False, callbacks=[_LrWrite()])
    assert spec.t == T_STEPS and spec.lrs[-1] == LR_NEW


def test_tf_formula_not_torch_at_large_epsilon():
    """One variable, epsilon = 1e-3: KerasAdam lands on TF's update and misses torch.optim.Adam's."""
    from deep_recommenders.keras.layers import Model
    from deep_recommenders_b200.optimizers import KerasAdam
    grads = [np.full(4, 1e-2 * (t + 1), F64) for t in range(5)]

    class One(Model):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.ones(4, device="cuda"))
            self.built = True

        def call(self, inputs, **kwargs):     # d loss / d w at step t is grads[t]: loss = mean(per-row w . x)
            return (self.w * inputs).sum(1, keepdim=True)

    def run(opt):
        m = One()
        m.compile(loss=lambda yt, yp: yp.sum(1), optimizer=opt)
        data = [(torch.from_numpy(g.astype(F32)).cuda()[None], np.zeros((1, 1), F32)) for g in grads]
        m.fit(data, epochs=1, steps_per_epoch=len(grads))
        return m.w.detach().double().cpu().numpy()

    from deep_recommenders_b200.keras import engine as K
    tf_like, torch_like = run(KerasAdam(0.01, epsilon=1e-3)), run(K.Adam(0.01, epsilon=1e-3))
    want, _, _ = keras_adam(np.ones(4), [g.astype(F32) for g in grads], [0.01] * 5, F64(F32(0.9)), F64(F32(0.999)),
                            F64(F32(1e-3)))
    np.testing.assert_allclose(tf_like, want, rtol=0, atol=1e-6)
    assert np.abs(torch_like - want).max() > 1e-4


# ---- 3. rebuilds and rejections -------------------------------------------------------------------------------------
def test_recompile_restarts_from_flushed_tables_and_rejections():
    from deep_recommenders.keras.models.ranking import FactorizationMachine
    from deep_recommenders_b200.optimizers import KerasAdam, RowSparseAdam
    model = FactorizationMachine(*_columns(8, False), seed=3, device="cuda")
    first = KerasAdam(0.01)
    model.compile(loss="binary_crossentropy", optimizer=first)
    model.fit([_batch(t, False) for t in range(1, 6)], epochs=1, steps_per_epoch=5)
    old = model.embeddings.row_optimizer
    assert int(first.clock.step) == 5
    flushed = model.embeddings.state_dict()["weight"].clone()          # every row brought to step 5
    second = KerasAdam(0.01)
    model.compile(loss="binary_crossentropy", optimizer=second)
    model.fit([_batch(1, False)], epochs=1, steps_per_epoch=1)
    new = model.embeddings.row_optimizer
    assert new is not old and new is second.row_optimizers[0] and int(second.clock.step) == 1
    st = new.state[:, 3 * 8 + 4].view(torch.int32)
    assert set(st.unique().tolist()) <= {0, 1}                         # fresh slots: nothing older than step 1
    touched = st == 1
    assert torch.equal(model.embeddings.weight.detach()[~touched], flushed[~touched])
    # a torch optimizer compiled afterwards gets the tables back
    model.compile(loss="binary_crossentropy", optimizer="adam")
    model.fit([_batch(2, False)], epochs=1, steps_per_epoch=1)
    assert model.embeddings.row_optimizer is None and model.embeddings.weight.grad is not None

    mine = FactorizationMachine(*_columns(8, False), seed=3, device="cuda")
    RowSparseAdam(mine.embeddings, 0.001, epsilon=1e-7)
    mine.compile(loss="binary_crossentropy", optimizer=KerasAdam())
    with pytest.raises(ValueError, match="already has a RowSparseAdam"):
        mine.fit([_batch(1, False)], epochs=1, steps_per_epoch=1)
    sgd = FactorizationMachine(*_columns(8, False), seed=3, device="cuda", sparse_lr=0.05)
    sgd.compile(loss="binary_crossentropy", optimizer=KerasAdam())
    with pytest.raises(ValueError, match="sparse_lr"):
        sgd.fit([_batch(1, False)], epochs=1, steps_per_epoch=1)
