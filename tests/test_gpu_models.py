"""Row M (model assembly) on the GPU: the reference's model-level tests ported
(tests/keras/test_fm.py:67-107, tests/keras/test_deepfm.py:16-56: two hash-bucket(100) columns,
dim 16, train, predict, save / load round trip with get_config equality and assertAllEqual on the
predictions), plus parity of the whole DeepFM forward against the oracle."""
import os
import tempfile

import numpy as np
import pytest
import torch

from oracle import reference_np as R

pytestmark = pytest.mark.gpu


def build_columns():
    from deep_recommenders_b200 import feature_column as fc
    user_id = fc.categorical_column_with_hash_bucket("user_id", 100)
    movie_id = fc.categorical_column_with_hash_bucket("movie_id", 100)
    base = [user_id, movie_id]
    return [fc.indicator_column(c) for c in base], [fc.embedding_column(c, dimension=16) for c in base]


def collection_arrays(coll):
    tables = [coll.table(s).detach().cpu().numpy() for s in range(coll.num_slots)]
    lins = [coll.linear_of(s).detach().cpu().numpy() for s in range(coll.num_slots)]
    return tables, lins, float(coll.bias)


def test_deepfm_forward_matches_oracle():
    from deep_recommenders.keras.models.ranking import DeepFM
    from deep_recommenders_b200 import feature_column as fc
    cols = [fc.categorical_column_with_identity(f"c{i}", 50 + i) for i in range(6)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, 16) for c in cols],
                   dnn_units_size=[64, 32], seed=3, device="cuda")
    with torch.no_grad():
        model.embeddings.lin_view().normal_(0, 0.1)
        model.embeddings.bias.fill_(0.1)
    rng = np.random.default_rng(0)
    ids = np.stack([rng.integers(-1, 50 + i, 300) for i in range(6)], axis=1).astype(np.int64)
    inputs = {f"c{i}": torch.from_numpy(ids[:, i]).cuda() for i in range(6)}
    prob = model(inputs)
    assert prob.shape == (300, 1)
    tables, lins, bias = collection_arrays(model.embeddings)
    ws = [l.kernel.detach().cpu().numpy() for l in model._dnn.layers]
    bs = [l.bias.detach().cpu().numpy() for l in model._dnn.layers]
    ref_prob, ref_logits, _, _ = R.deepfm_forward(tables, lins, bias, ws, bs, ids, "relu", np.float64)
    assert np.allclose(prob.detach().cpu().numpy(), ref_prob, rtol=1e-5, atol=1e-6)
    assert np.allclose(model.logits(inputs).detach().cpu().numpy(), ref_logits, rtol=1e-5, atol=2e-5)
    assert set(model.get_config()) >= {"dnn_units_size", "dnn_activation"}


@pytest.mark.parametrize("which", ["fm", "deepfm"])
def test_ref_model_train_predict_save_load(which):
    from deep_recommenders.keras.models.ranking import DeepFM, FactorizationMachine
    ind, emb = build_columns()
    mk = (lambda: FactorizationMachine(ind, emb, seed=1, device="cuda")) if which == "fm" else \
         (lambda: DeepFM(ind, emb, dnn_units_size=[10, 5], seed=1, device="cuda"))
    model = mk()
    feats = {"user_id": np.asarray([["1"]] * 1000), "movie_id": np.asarray([["2"]] * 1000)}
    labels = torch.zeros(1000, 1, device="cuda")                 # np.random.randint(0, 1) is always 0
    model(feats)                                                 # build lazily-created layers
    opt = torch.optim.Adam(model.parameters())
    first = None
    for _ in range(20):
        opt.zero_grad()
        p = model(feats)
        loss = torch.nn.functional.binary_cross_entropy(p, labels)
        loss.backward()
        opt.step()
        first = first if first is not None else float(loss)
    assert float(loss) < first
    test_data = {"user_id": np.asarray([["1"], ["2"]]), "movie_id": np.asarray([["1"], ["2"]])}
    pred = model.predict(test_data)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.pt")
        model.save(path)
        blob = torch.load(path, weights_only=False)
        loaded = mk()
        loaded(test_data)
        loaded.load_state_dict(blob["state"])
        loaded_pred = loaded.predict(test_data)
    assert model.get_config() == loaded.get_config()
    assert torch.equal(pred, loaded_pred)                         # assertAllEqual


def test_estimator_twins():
    from deep_recommenders.estimator.models.feature_interaction import FM, dnn
    from deep_recommenders.estimator.models.ranking.deepfm import DeepFM
    ind, emb = build_columns()
    feats = {"user_id": np.asarray(["7", "8", "9"]), "movie_id": np.asarray(["1", "2", "3"])}
    fm = FM(ind, emb, seed=0, device="cuda")
    out = fm(feats)
    assert out.shape == (3, 1) and len(fm.embeddings) == 2 and fm.embeddings[0].shape == (3, 16)
    y = dnn(torch.randn(5, 8, device="cuda"), [4, 2], name="t")
    assert y.shape == (5, 2)
    with pytest.raises(TypeError):
        dnn(torch.randn(5, 8, device="cuda"), [4, 2], batch_normalization=True)
    p = DeepFM(ind, emb, [8, 4], seed=0, device="cuda")(feats)
    assert p.shape == (3, 1) and float(p.min()) > 0 and float(p.max()) < 1


def test_dcn_and_two_tower_train_step():
    from deep_recommenders.keras.layers import DCN, TwoTower
    model = DCN([100] * 6, 8, num_cross=2, dnn_units=[32, 16], seed=0, device="cuda")
    ids = torch.randint(0, 100, (64, 6), device="cuda")
    y = torch.randint(0, 2, (64, 1), device="cuda").float()
    z = model.logits(ids)
    params = list(model.parameters())
    opt = torch.optim.SGD(params, lr=0.1)
    l0 = None
    for _ in range(30):
        opt.zero_grad()
        loss = torch.nn.functional.binary_cross_entropy_with_logits(model.logits(ids), y)
        loss.backward()
        opt.step()
        l0 = l0 if l0 is not None else float(loss)
    assert float(loss) < l0
    tt = TwoTower(500, 800, dim=32, temperature=0.5, seed=0, device="cuda")
    u = torch.randint(0, 500, (128,), device="cuda")
    i = torch.randint(0, 800, (128,), device="cuda")
    opt = torch.optim.SGD(tt.parameters(), lr=0.05)
    l0 = None
    for _ in range(20):
        opt.zero_grad()
        loss = tt(u, i, remove_accidental_hits=True)
        loss.backward()
        opt.step()
        l0 = l0 if l0 is not None else float(loss)
    assert float(loss) < l0


def test_c1_movielens_shaped_fm_matches_oracle():
    """BASELINE config C1 (examples/train_fm_on_movielens_estimator.py:10-35 columns, D=16, B=1024):
    hash-bucket ids via FarmHash Fingerprint64, vocabulary ids with OOV -> -1, the always-OOV genre slot."""
    import importlib.util
    import pathlib
    from deep_recommenders_b200.hashing import hash_bucket
    spec = importlib.util.spec_from_file_location(
        "c1_example", pathlib.Path(__file__).resolve().parent.parent / "examples" / "train_fm_on_movielens_synthetic.py")
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    from deep_recommenders.estimator.models.feature_interaction import FM
    ind, emb = ex.build_columns()
    model = FM(ind, emb, seed=1, device="cuda")
    coll = model.collection
    with torch.no_grad():
        coll.lin_view().normal_(0, 0.1)
        coll.bias.fill_(-0.2)
    rng = np.random.default_rng(0)
    feats, labels = ex.synthetic_batch(rng, 1024)
    logits = model(feats)
    assert logits.shape == (1024, 1) and len(model.embeddings) == 6
    ids = np.stack([
        hash_bucket(feats["user_id"].tolist(), ex.NUM_USERS),
        np.asarray([ex.GENDER_VOCAB.index(v) for v in feats["user_gender"]]),
        np.asarray([ex.AGE_VOCAB.index(int(v)) for v in feats["user_age"]]),
        np.asarray([ex.OCCUPATION_VOCAB.index(int(v)) for v in feats["user_occupation"]]),
        hash_bucket(feats["movie_id"].tolist(), ex.NUM_MOVIES),
        np.full(1024, -1),                                   # genres are never in the gender vocabulary
    ], axis=1).astype(np.int64)
    tables, lins, bias = collection_arrays(coll)
    ref, stack = R.fm_logit(tables, lins, bias, ids, np.float64)
    assert float(np.abs(stack[:, 5]).max()) == 0.0
    assert np.allclose(logits.detach().cpu().numpy(), ref, rtol=1e-5, atol=2e-5)
    assert torch.equal(model.embeddings[5], torch.zeros_like(model.embeddings[5]))
    opt = torch.optim.Adam(model.parameters(), lr=0.01)
    y = torch.from_numpy(labels).cuda()
    first = None
    for _ in range(15):
        loss = torch.nn.functional.binary_cross_entropy_with_logits(model(feats), y)
        opt.zero_grad()
        loss.backward()
        opt.step()
        first = first if first is not None else float(loss)
    assert float(loss) < first


def test_keras_compile_fit_evaluate_like_reference_example():
    """/root/reference/examples/train_deepfm_on_movielens_keras.py:38-54: compile(loss, Adam, [AUC, Precision, Recall]) +
    fit(input_fn, epochs, steps_per_epoch, validation_data, validation_steps, [EarlyStopping(patience=3)])."""
    import importlib.util
    import pathlib
    from deep_recommenders_b200.keras import engine as K
    from deep_recommenders.keras.models.ranking import DeepFM
    spec = importlib.util.spec_from_file_location(
        "ex_keras", pathlib.Path(__file__).resolve().parents[1] / "examples" / "train_deepfm_on_movielens_keras.py")
    ex = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ex)
    ind, emb = ex.build_columns()
    model = DeepFM(ind, emb, dnn_units_size=[32, 8], seed=0, device="cuda")
    model.compile(loss=K.binary_crossentropy, optimizer=K.Adam(learning_rate=0.01), metrics=[K.AUC(), K.Precision(), K.Recall()])
    hist = model.fit(ex.synthetic_input_fn(1, 512), epochs=4, steps_per_epoch=25, validation_data=ex.synthetic_input_fn(2, 512),
                     validation_steps=4, callbacks=[K.EarlyStopping(patience=3)])
    assert len(hist["loss"]) == 4 and hist["loss"][-1] < hist["loss"][0]
    assert set(hist) >= {"loss", "auc", "precision", "recall", "val_loss", "val_auc"}
    assert hist["val_auc"][-1] > 0.55                      # the synthetic labels depend on the ids: better than chance
    # metric arithmetic against numpy on one batch
    y = np.asarray([0, 0, 1, 1, 1, 0], np.float32)
    p = np.asarray([0.1, 0.6, 0.8, 0.4, 0.9, 0.2], np.float32)
    m = [K.AUC(), K.Precision(), K.Recall()]
    for x in m:
        x.update_state(torch.from_numpy(y).cuda(), torch.from_numpy(p).cuda())
    assert abs(m[1].result() - 2 / 3) < 1e-6 and abs(m[2].result() - 2 / 3) < 1e-6
    assert abs(m[0].result() - 8 / 9) < 0.02               # exact ROC AUC of this batch = 8/9 (200-threshold trapezoid)
    # EarlyStopping: stops after `patience` epochs without improvement
    es = K.EarlyStopping(patience=2)
    assert [es.on_epoch_end(i, {"val_loss": v}) for i, v in enumerate([1.0, 0.9, 0.95, 0.97])] == [False, False, False, True]


@pytest.mark.gpu
@pytest.mark.parametrize("chunks", [2, 3])
@pytest.mark.parametrize("use_graph", [False, True])
def test_train_step_fwd_chunks_equal_whole_batch(chunks, use_graph):
    """fwd_chunks > 1 runs the gather and the first tower GEMM as alternating launches over slices of the batch; examples
    are independent in both kernels, so every activation, the loss and the updated parameters equal the unsliced step
    (bit for bit in the forward; the parameter update differs only by atomic summation order)."""
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    rows, B, D = [500, 7, 300, 41], 1000, 16       # B not a multiple of 128: the last slice is ragged
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]

    def make(n):
        model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                       dnn_units_size=[64, 32], seed=7, device="cuda", sparse_lr=0.05)
        with torch.no_grad():
            model.embeddings.lin_view().normal_(0, 0.1, generator=torch.Generator(device="cuda").manual_seed(3))
        tr = DeepFMTrainStep(model, batch_size=B, lr=0.05, use_graph=use_graph, fwd_chunks=n)
        return model, (tr.capture() if use_graph else tr)

    (m1, t1), (m2, t2) = make(1), make(chunks)
    rng = np.random.default_rng(5)
    for k in range(3):
        ids = torch.from_numpy(np.stack([rng.integers(-1, r, size=B) for r in rows], axis=1).astype(np.int64)).cuda()
        lab = torch.from_numpy(rng.integers(0, 2, size=B).astype(np.float32)).cuda()
        l1, l2 = float(t1.step(ids, lab).item()), float(t2.step(ids, lab).item())
        assert abs(l1 - l2) <= 5e-6 * abs(l1)        # float atomics: summation order differs run to run
        if k == 0:      # same parameters going in: the sliced forward is bit-identical (later steps start from parameters
            torch.cuda.synchronize()          # that differ by the atomic summation order of the previous update)
            assert torch.equal(t1.stack, t2.stack) and torch.equal(t1.fm_logit, t2.fm_logit)
            assert torch.equal(t1.acts[0], t2.acts[0])
    assert torch.allclose(t1.stack, t2.stack, rtol=1e-5, atol=1e-7)
    assert torch.allclose(t1.acts[0], t2.acts[0], rtol=1e-5, atol=1e-6)
    assert torch.allclose(m1.embeddings.weight, m2.embeddings.weight, rtol=1e-5, atol=1e-7)
    for a, b in zip(t1.w + t1.b, t2.w + t2.b):          # (the flat buffer has uninitialised 16-B padding between them)
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7)


def _small_deepfm_trainer(B=1000, use_graph=True, rows=(500, 7, 300, 41), dnn=(64, 32), **kw):
    from deep_recommenders_b200 import feature_column as fc
    from deep_recommenders_b200.keras.models.ranking import DeepFM
    from deep_recommenders_b200.training import DeepFMTrainStep
    rows, D = list(rows), 16
    cols = [fc.categorical_column_with_identity(f"c{i}", r) for i, r in enumerate(rows)]
    model = DeepFM([fc.indicator_column(c) for c in cols], [fc.embedding_column(c, D) for c in cols],
                   dnn_units_size=list(dnn), seed=7, device="cuda", sparse_lr=0.05)
    with torch.no_grad():
        model.embeddings.lin_view().normal_(0, 0.1, generator=torch.Generator(device="cuda").manual_seed(3))
    tr = DeepFMTrainStep(model, batch_size=B, lr=0.05, use_graph=use_graph, **kw)
    return rows, model, (tr.capture() if use_graph else tr)


def test_fit_host_returns_every_steps_loss_like_blocking_calls():
    """fit_host (pipelined: H2D of the next batch and the D2H loss read off the critical path) must produce exactly the
    losses of the same batches fed one blocking train_step_host call at a time."""
    rows, m1, t1 = _small_deepfm_trainer()
    _, m2, t2 = _small_deepfm_trainer()
    rng = np.random.default_rng(9)
    B = t1.B
    batches = []
    for _ in range(7):
        ids = torch.from_numpy(np.stack([rng.integers(-1, r, size=B) for r in rows], axis=1).astype(np.int64)).pin_memory()
        lab = torch.from_numpy(rng.integers(0, 2, size=B).astype(np.float32)).pin_memory()
        batches.append((ids, lab))
    ref = [t1.train_step_host(*batches[k], *(batches[k + 1] if k + 1 < len(batches) else (None, None))) for k in range(7)]
    t1._staged = None
    got = t2.fit_host(batches[:3]) + t2.fit_host(batches[3:])        # two calls: the second one restages its first batch
    assert len(got) == 7
    for a, b in zip(ref, got):
        assert abs(a - b) <= 5e-6 * abs(a), (ref, got)      # float atomics: summation order differs run to run
    assert t2.fit_host([]) == []


@pytest.mark.parametrize("use_graph", [False, True])
def test_train_step_dw_first_with_shared_sm_gemm_equals_default(use_graph):
    """dw_first + knob tc_dw_share: the layer-0 weight-gradient GEMM (co-residency build: capped registers, one staging
    slab) is enqueued before the embedding update and shares the SMs with it -- scheduling only, same arithmetic."""
    from deep_recommenders_b200 import _lib
    shape = dict(rows=(500, 7, 300, 41, 90, 1000, 3, 64), dnn=(256, 32), B=3000)     # layer-0 dW: [128 x 3000] x [3000 x 256]
    rows, m1, t1 = _small_deepfm_trainer(use_graph=use_graph, **shape)
    _lib.tune("tc_dw_share", 1)
    try:
        _, m2, t2 = _small_deepfm_trainer(use_graph=use_graph, dw_first=True, **shape)
        rng = np.random.default_rng(5)
        B = t1.B
        for _ in range(3):
            ids = torch.from_numpy(np.stack([rng.integers(-1, r, size=B) for r in rows], axis=1).astype(np.int64)).cuda()
            lab = torch.from_numpy(rng.integers(0, 2, size=B).astype(np.float32)).cuda()
            l1 = float(t1.step(ids, lab).item())
            l2 = float(t2.step(ids, lab).item())
            assert abs(l1 - l2) <= 5e-6 * abs(l1)        # float atomics: summation order differs run to run
        torch.cuda.synchronize()
    finally:
        _lib.tune("tc_dw_share", 0)
    assert float((t1.gw[0] - t2.gw[0]).abs().max()) <= 1e-5 * float(t1.gw[0].abs().max())   # split-K partial sums meet in another order
    assert torch.allclose(m1.embeddings.weight, m2.embeddings.weight, rtol=1e-5, atol=1e-7)
    for a, b in zip(t1.w + t1.b, t2.w + t2.b):          # (the flat buffer has uninitialised 16-B padding between them)
        assert torch.allclose(a, b, rtol=1e-5, atol=1e-7)


def test_bench_dump_outputs_is_reproducible(tmp_path):
    """`bench.py --dump-outputs DIR` writes the last timed step's outputs as float32 arrays, and two runs with the same
    arguments see the same inputs: their dumps agree up to the summation order of the atomics."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dumps = []
    for run in ("a", "b"):
        d = tmp_path / run
        r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", "3", "--warmup", "3",
                            "--no-cpu-baseline", "--dump-outputs", str(d)], capture_output=True, text=True, timeout=900,
                           cwd=str(tmp_path))
        assert r.returncode == 0, r.stderr[-2000:]
        import json
        assert json.loads(r.stdout.strip().splitlines()[-1])["steps"] == 3
        dumps.append({f[:-4]: np.load(d / f) for f in sorted(os.listdir(d))})
    a, b = dumps
    assert set(a) == set(b) == {"loss", "prob", "tower", "embedding_rows_sample"}
    assert a["loss"].shape == (1,) and a["prob"].shape == (65536,)
    total = 0
    for name in a:
        assert a[name].dtype == np.float32 and np.isfinite(a[name]).all(), name
        assert np.abs(a[name] - b[name]).max() <= 1e-5 * np.abs(a[name]).max() + 1e-7, name
        total += a[name].nbytes
    assert total <= 64 << 20
    assert np.abs(a["embedding_rows_sample"]).max() > 0 and 0.0 <= a["prob"].min() and a["prob"].max() <= 1.0
